// device_lc.cuh -- lane change on the device ("laneChange": true): SimpleLaneChange::makeSignal (lanechange.cpp:151-184),
// Engine::scheduleLaneChange / insertShadow (engine.cpp:792-820, lanechange.cpp:71-102), yieldSpeed (:186-206) and the
// partner coupling of Engine::vehicleControl (engine.cpp:195-244).
//
// STATUS: part of the library.  On the GPU (H100) it is bit-equal, every field of every vehicle including shadows, every step,
// to the restatement -- which is pinned against oracle/_ref/refdump_lcorder, the reference with its per-worker vehicle
// sets ordered by priority instead of by heap address (tests/test_gpu_parity.py::test_lane_change_vs_restatement,
// tools/lc_gpu_check.py; compute-sanitizer racecheck clean) -- and statistically equal to the unmodified reference.
//
// The algorithm is the "device form" that tests/test_cpu.py::test_lane_change_device_form_is_equivalent
// proves equal to the reference-ordered restatement (DESIGN.md section 10), in its simplest shape:
//   * everything that does not depend on processing order stays in the parallel kernels;
//   * the two order-dependent parts -- Engine::scheduleLaneChange (engine.cpp:792-809) and the tail of
//     Engine::vehicleControl for the few vehicles involved in a lane change (engine.cpp:195-244) -- run
//     per ROAD (one thread serves one road's candidates in the global order; roads are independent),
//     CITYFLOW_B200_LC_SERIAL=1 selects the one-thread-for-everything form.
// Included by device_sim.cu after its helpers (min2, noCollisionSpeed, Tail, View ...).
#pragma once

namespace cfb {

// ---- segments -------------------------------------------------------------------------------
// Lane::initSegments roadnet.cpp:863-875: the segment cursor only moves down while the list is walked
// front to back, so segmentIndex(p) = min(natural segment of p, segmentIndex(p - 1)).
__device__ void lcInitSegments(const View &V, const LcView &C, int lane) {
    const int base = V.off[lane], n = V.count[lane];
    const int sb = C.segBeg[lane], ns = C.segBeg[lane + 1] - sb;
    int run = ns - 1;
    for (int k = 0; k < n; ++k) {
        const double dis = V.kin[base + k].x;
        int nat = ns - 1;
        while (nat > 0 && !(dis >= C.segStart[sb + nat])) --nat;
        if (nat < run) run = nat;
        C.segIdx[base + k] = run;
    }
}
// Lane::getVehicleAfterDistance roadnet.cpp:889-898 -- the segment lists are the lane's list filtered by
// segment index (checked on the CPU: no shadow insertion ever left a segment list in another order)
__device__ int lcVehicleAfter(const View &V, const LcView &C, int lane, double dis, int seg) {
    const int base = V.off[lane], n = V.count[lane];
    const int ns = C.segBeg[lane + 1] - C.segBeg[lane];
    for (int i = seg; i < ns; ++i)
        for (int k = n - 1; k >= 0; --k)
            if (C.segIdx[base + k] == i && V.kin[base + k].x >= dis) return base + k;
    return -1;
}
// Lane::getVehicleBeforeDistance roadnet.cpp:877-887
__device__ int lcVehicleBefore(const View &V, const LcView &C, int lane, double dis, int seg) {
    const int base = V.off[lane], n = V.count[lane];
    for (int i = seg; i >= 0; --i)
        for (int k = 0; k < n; ++k)
            if (C.segIdx[base + k] == i && V.kin[base + k].x < dis) return base + k;
    return -1;
}

// ---- routing helpers ------------------------------------------------------------------------
// position of the vehicle's current road in its route: plans list lane, link, lane, link, ...
__device__ __forceinline__ int lcRoadPos(const View &V, const LcView &C, int plan, int planIdx) {
    return C.planRoadPos[plan] + ((planIdx - V.planBeg[plan]) >> 1);
}
// plan a vehicle of `plan`'s route would follow from lane `lane` (same road as its current lane)
__device__ __forceinline__ int lcLanePlan(const LcView &C, int plan, int roadPos, int lane) {
    const int route = C.planRoute[plan];
    return C.lanePlanId[C.lanePlanBeg[C.lanePlanRoad[route] + roadPos] + C.laneIdx[lane]];
}
// router.onLastRoad() || router.getNextDrivable(lane) != nullptr  (lanechange.cpp:168, :176)
__device__ __forceinline__ bool lcLaneContinues(const View &V, const LcView &C, int plan, int roadPos, int lane, bool onLastRoad) {
    if (onLastRoad) return true;
    const int np = lcLanePlan(C, plan, roadPos, lane);
    return V.planData[V.planBeg[np] + 1] >= 0;
}

// ---- SimpleLaneChange::makeSignal lanechange.cpp:152-187 -----------------------------------------
// Reads only state committed before the phase: one thread per running vehicle.
__device__ void lcMakeSignal(const View &V, const LcView &C, int p, int d, int epoch) {
    const int4 idv = V.ids[p];
    LcSlot &L = C.slot[idv.x];
    if (L.type == 2) return;                                   // shadows do not plan (engine.cpp:379)
    bool candidate = false;
    if (L.changing) {
        candidate = true;                                      // makeSignal returns at once, planChange() holds
    } else if (!((epoch - 1) * V.dt - L.lastChange < 3)) {     // coolingTime (lanechange.h:46); currentTime = step * interval
        L.sendEpoch = epoch;
        L.sendTarget = -1;
        L.sendDir = 0;
        if (d < V.nLanes) {
            const double2 kk = V.kin[p];
            const DTmpl &T = V.tmpl[idv.y];
            const double len = V.drvLength[d];
            bool go = !(len - kk.x < 30);
            const double curEst = L.gap;
            double outerEst = 0;
            const double expectedGap = 2 * T.len + 4 * V.dt * T.maxSpeed;
            if (go && (L.gap > expectedGap || L.gap < 1.5 * T.len)) go = false;
            if (go) {
                const int planIdx = V.nav[p].x;
                const int roadPos = lcRoadPos(V, C, L.plan, planIdx);
                // Router::onLastRoad (router.cpp:131-138) compares the road with route.back(): true on EVERY visit of that
                // road, e.g. on the first road of a route that returns to it
                const bool onLast = C.laneRoad[d] == C.routeLastRoad[C.planRoute[L.plan]];
                const int seg = C.segIdx[p];
                if (C.laneIdx[d] < C.laneRoadN[d] - 1) {
                    const int outer = d + 1;
                    if (lcLaneContinues(V, C, L.plan, roadPos, outer, onLast)) {
                        const int lp = lcVehicleAfter(V, C, outer, kk.x, seg);   // estimateGap lanechange.cpp:220-225
                        outerEst = lp < 0 ? V.drvLength[outer] - kk.x : V.kin[lp].x - kk.x - V.tmpl[V.ids[lp].y].len;
                        if (outerEst > curEst + T.len) L.sendTarget = outer;
                    }
                }
                if (C.laneIdx[d] > 0) {
                    const int inner = d - 1;
                    if (lcLaneContinues(V, C, L.plan, roadPos, inner, onLast)) {
                        const int lp = lcVehicleAfter(V, C, inner, kk.x, seg);
                        const double innerEst = lp < 0 ? V.drvLength[inner] - kk.x : V.kin[lp].x - kk.x - V.tmpl[V.ids[lp].y].len;
                        if (innerEst > curEst + T.len && innerEst > outerEst) L.sendTarget = inner;
                    }
                }
            }
            // LaneChange::getDirection lanechange.cpp:104-113
            if (L.sendTarget >= 0) L.sendDir = L.sendTarget == d + 1 ? 1 : (L.sendTarget == d - 1 ? -1 : 0);
        }
        candidate = L.sendTarget >= 0 && L.sendTarget != d;
    }
    if (candidate) {
        const int i = atomicAdd(&C.ctrl->nCand, 1);
        if (i < LC_MAX_CAND) C.cand[i] = idv.x; else atomicOr(&C.ctrl->error, 1);
    }
}

// ---- ordering ---------------------------------------------------------------------------------
__device__ __forceinline__ int lcPriorityOf(const View &V, int slot) { return V.ids[V.pos[slot]].z; }

// slots[0..n) ascending by priority (vehiclePool order).  One thread; n is a few hundred at most.
__device__ void lcSortByPriority(const View &V, int *slots, int n) {
    for (int i = 1; i < n; ++i) {   // insertion sort: the atomics that filled the list left it nearly in list order
        const int s = slots[i];
        const int ps = lcPriorityOf(V, s);
        int j = i - 1;
        while (j >= 0 && lcPriorityOf(V, slots[j]) > ps) { slots[j + 1] = slots[j]; --j; }
        slots[j + 1] = s;
    }
}
// The permutation libstdc++'s std::sort applies to n indistinguishable elements (engine.cpp:793, all
// urgencies are 1): lc_order.h, replayed in place.  `stack` needs 2 * 32 ints.
__device__ void lcAllEqualSortPermute(int *a, int n) {
    int stackF[40], stackL[40];
    int sp = 0;
    if (n > 0) { stackF[0] = 0; stackL[0] = n; sp = 1; }
    while (sp > 0) {
        --sp;
        int first = stackF[sp], last = stackL[sp];
        while (last - first > 16) {
            const int mid = first + (last - first) / 2;
            int t = a[first]; a[first] = a[mid]; a[mid] = t;
            int f = first + 1, l = last;
            for (;;) {
                --l;
                if (!(f < l)) break;
                t = a[f]; a[f] = a[l]; a[l] = t;
                ++f;
            }
            stackF[sp] = f; stackL[sp] = last; ++sp;
            last = f;
        }
    }
}

// ---- scheduling (Engine::scheduleLaneChange engine.cpp:792-809), one thread --------------------------
__device__ __forceinline__ double lcMinBrake(const View &V, int p) {   // Vehicle::getMinBrakeDistance vehicle.h:239
    const double s = V.kin[p].y;
    return 0.5 * s * s / V.tmpl[V.ids[p].y].maxNegAcc;
}
// SimpleLaneChange::safeGapBefore lanechange.cpp:212-214
__device__ __forceinline__ double lcSafeGapBefore(const View &V, const LcSlot &L, int epoch) {
    if (L.tgtEpoch != epoch || L.tgtFollower < 0) return 0;
    return lcMinBrake(V, V.pos[L.tgtFollower]);
}
// Vehicle::receiveSignal vehicle.cpp:391-402
__device__ void lcReceiveSignal(const View &V, const LcView &C, int me, int sender, int epoch) {
    LcSlot &M = C.slot[me];
    if (M.changing) return;
    const bool hasRecv = lcRecvValid(M, epoch);
    const int curPriority = hasRecv ? lcPriorityOf(V, M.recvSrc) : -1;
    const int newPriority = lcPriorityOf(V, sender);
    const bool hasSend = M.sendEpoch == epoch;
    if ((!hasRecv || curPriority < newPriority) && (!hasSend || lcPriorityOf(V, me) < newPriority)) {
        M.recvSrc = sender;
        M.recvEpoch = epoch;
    }
}
// LaneChange::updateLeaderAndFollower lanechange.cpp:27-62
__device__ void lcUpdateLeaderAndFollower(const View &V, const LcView &C, int slot, int epoch) {
    LcSlot &L = C.slot[slot];
    const int p = V.pos[slot];
    const int cur = C.posDrv[p], target = L.sendTarget;
    const double dis = V.kin[p].x;
    const int seg = C.segIdx[p];
    L.tgtEpoch = epoch;
    L.tgtLeader = L.tgtFollower = -1;
    L.leaderGap = L.followerGap = 1.7976931348623157e308;
    const int lp = lcVehicleAfter(V, C, target, dis, seg);
    if (lp < 0) {
        const double rest = V.drvLength[cur] - dis;
        L.leaderGap = rest;
        double gap = 1.7976931348623157e308;
        for (int q = V.laneOutBeg[target]; q < V.laneOutBeg[target + 1]; ++q) {
            const Tail t = V.tail[V.nLanes + V.laneOutLinks[q]];
            if (t.pos >= 0 && t.dis + rest < gap) {
                gap = t.dis + rest;
                if (gap < t.len) {
                    L.tgtLeader = V.ids[t.pos].x;
                    L.leaderGap = rest - (t.len - gap);
                }
            }
        }
    } else {
        L.tgtLeader = V.ids[lp].x;
        L.leaderGap = V.kin[lp].x - dis - V.tmpl[V.ids[lp].y].len;
    }
    const int fp = lcVehicleBefore(V, C, target, dis, seg);
    if (fp >= 0) {
        L.tgtFollower = V.ids[fp].x;
        L.followerGap = dis - V.kin[fp].x - V.tmpl[V.ids[p].y].len;
    }
}
// Engine::insertShadow engine.cpp:811-819 + LaneChange::insertShadow lanechange.cpp:73-102.
// The shadow becomes a vehicle of its own in the target lane's bucket, right before targetFollower
// (or at the end); the records behind it move back by one position.
// Returns the shadow's slot (-1: no room).  Safe to run for different ROADS at the same time: it touches the
// target lane's bucket, per-slot records of vehicles on that road, and shared counters through atomics.
__device__ int lcInsertShadow(const View &V, const LcView &C, int slot, int epoch) {
    LcSlot &L = C.slot[slot];
    const int target = L.sendTarget;
    const int base = V.off[target], n = V.count[target];
    if (n >= V.off[target + 1] - base) { atomicOr(&V.ctrl->error, ERR_BUCKET_OVERFLOW); return -1; }
    const int u = atomicAdd(&C.ctrl->spareUsed, 1);
    if (u >= C.nSpare) { atomicOr(&C.ctrl->error, 2); return -1; }
    const int sh = C.spare[u];
    const int pv = V.pos[slot];
    int at = n;                                                    // list position (0-based) of the shadow
    if (L.tgtFollower >= 0) {
        const int fp = V.pos[L.tgtFollower];
        if (fp >= base && fp < base + n) at = fp - base;            // targetFollower->getListIterator()
    }
    for (int k = n; k > at; --k) {                                  // shift [at, n) back by one
        const int dst = base + k, src = base + k - 1;
        V.kin[dst] = V.kin[src];
        V.ids[dst] = V.ids[src];
        V.nav[dst] = V.nav[src];
        V.gap[dst] = V.gap[src];
        V.cust[dst] = V.cust[src];
        C.segIdx[dst] = C.segIdx[src];
        V.pos[V.ids[dst].x] = dst;
    }
    const int q = base + at;
    const int4 pid = V.ids[V.pos[slot]];                            // (the parent may have moved if target == its own lane: it cannot)
    const int4 pnv = V.nav[V.pos[slot]];
    // the shadow follows the parent's route from the target lane (Router copy + update, router.cpp:11-14, :78-94)
    const int roadPos = lcRoadPos(V, C, L.plan, pnv.x);
    const int np = lcLanePlan(C, L.plan, roadPos, target);
    const int npIdx = V.planBeg[np];
    V.kin[q] = V.kin[pv];
    V.ids[q] = make_int4(sh, pid.y, LC_PRIO_PENDING, V.planData[npIdx + 1]);
    V.nav[q] = make_int4(npIdx, pnv.y, -1, pnv.w);                  // blocker = nullptr (lanechange.cpp:88)
    V.gap[q] = L.gap;
    V.cust[q] = V.cust[pv];                                         // Buffer is copied member-wise (vehicle.cpp:29)
    C.segIdx[q] = C.segIdx[pv];                                     // laneChangeInfo.segmentIndex copied: the PARENT's index
    V.pos[sh] = q;
    V.blk[sh] = -1;
    V.count[target] = n + 1;
    {   // Drivable::getLastVehicle of the target lane
        const int lastp = base + n;
        Tail t;
        const double2 kq = V.kin[lastp];
        t.dis = kq.x; t.speed = kq.y; t.len = V.tmpl[V.ids[lastp].y].len; t.pos = lastp; t.prev = V.nav[lastp].y;
        V.tail[target] = t;
    }
    LcSlot &S = C.slot[sh];
    lcResetSlot(S, np);
    S.gap = L.gap;
    // The two immediate updates of LaneChange::insertShadow (lanechange.cpp:98-100).  The full leader pass that
    // follows (engine.cpp:573) recomputes leaders, but a vehicle keeps its last gap VALUE when that pass finds
    // no leader for it, and a later candidate of this same scheduling pass may copy that value into its own
    // shadow (the follower updated here can be the next parent) -- so both are applied as the reference does.
    {   // shadow->updateLeaderAndGap(targetLeader), vehicle.cpp:157-196
        const int tlp = L.tgtLeader >= 0 ? V.pos[L.tgtLeader] : -1;
        if (tlp >= 0 && C.posDrv[tlp] == target) {
            S.gap = V.kin[tlp].x - V.tmpl[V.ids[tlp].y].len - V.kin[q].x;
            V.gap[q] = S.gap;
        } else {
            int ld = -1;
            double g = 0;
            headSearch(V, target, V.kin[q].x, V.ids[q].w, V.nav[q].x, V.tmpl[V.ids[q].y], -1, ld, g);
            if (ld >= 0) { S.gap = g; V.gap[q] = g; }
        }
    }
    if (L.tgtFollower >= 0) {   // targetFollower->updateLeaderAndGap(shadow): same lane by construction
        const int fp = V.pos[L.tgtFollower];
        if (C.posDrv[fp] == target) {
            const double g = V.kin[q].x - V.tmpl[V.ids[q].y].len - V.kin[fp].x;
            C.slot[L.tgtFollower].gap = g;
            V.gap[fp] = g;
        }
    }
    S.type = 2; S.partner = slot;                                   // setParent
    L.type = 1; L.partner = sh;                                     // setShadow
    L.changing = 1;
    L.waiting = 0;
    // the new vehicle takes part in the rest of this step
    const int cpar = V.par;
    const int vi = atomicAdd(&V.ctrl->nVeh[cpar], 1);
    if (vi < V.vehCap) V.vehList[cpar][vi] = make_int2(base + n, target);   // the position that became occupied
    if (n == 0) V.actList[cpar][atomicAdd(&V.ctrl->nAct[cpar], 1)] = target;
    atomicAdd(&V.ctrl->active, 1);                                  // activeVehicleCount++ (engine.cpp:818)
    return sh;
}

// one candidate of Engine::scheduleLaneChange's loop (engine.cpp:795-807); returns the shadow's slot or -1
__device__ int lcScheduleOne(const View &V, const LcView &C, int slot, int epoch) {
    LcSlot &L = C.slot[slot];
    lcUpdateLeaderAndFollower(V, C, slot, epoch);
    if (L.tgtLeader >= 0) lcReceiveSignal(V, C, L.tgtLeader, slot, epoch);      // SimpleLaneChange::sendSignal
    if (L.tgtFollower >= 0) lcReceiveSignal(V, C, L.tgtFollower, slot, epoch);
    const int p = V.pos[slot];
    const int d = C.posDrv[p];
    if (lcPlanChange(L, d, epoch) && lcSendValid(L, epoch) && !lcRecvValid(L, epoch) && !L.changing) {
        const bool gapValid = L.leaderGap >= lcMinBrake(V, p) && L.followerGap >= lcSafeGapBefore(V, L, epoch);
        if (gapValid && d < V.nLanes) return lcInsertShadow(V, C, slot, epoch);
    }
    return -1;
}
// the whole loop in one thread, in the reference's order (kept for the host probe and as a debugging fallback)
__device__ void lcSchedule(const View &V, const LcView &C, int epoch) {
    int n = min(C.ctrl->nCand, LC_MAX_CAND);
    lcSortByPriority(V, C.cand, n);          // threadVehiclePool order (priority-ordered reference, oracle/lc_order_patch.sh)
    lcAllEqualSortPermute(C.cand, n);        // std::sort by urgency, all equal
    int k = 0;
    for (int i = 0; i < n; ++i) {
        const int sh = lcScheduleOne(V, C, C.cand[i], epoch);
        if (sh >= 0) C.shadowLog[k++] = make_int2(C.cand[i], sh);
    }
    C.ctrl->nShadows = k;
}

// ---- control tail (Engine::vehicleControl engine.cpp:188-251 for the involved vehicles), one thread -----
// LaneChange::clearSignal lanechange.cpp:129-139
__device__ __forceinline__ void lcClearSignal(LcSlot &L, int epoch) {
    L.tgtEpoch = -1;
    L.lastDir = lcSendValid(L, epoch) ? L.sendDir : 0;
    if (L.changing) return;
    L.sendEpoch = -1;
    L.recvEpoch = -1;
}
// SimpleLaneChange::yieldSpeed lanechange.cpp:189-210 + the rest of Vehicle::getNextSpeed vehicle.cpp:323-333
__device__ double lcTailSpeed(const View &V, const LcView &C, int slot, int epoch) {
    LcSlot &L = C.slot[slot];
    const int p = V.pos[slot];
    const int d = C.posDrv[p];
    const double2 kk = V.kin[p];
    const int4 idv = V.ids[p];
    const DTmpl &T = V.tmpl[idv.y];
    double s = L.head;
    if (lcPlanChange(L, d, epoch)) L.waiting += V.dt;
    double y = 100;
    if (lcRecvValid(L, epoch)) {
        const int src = L.recvSrc;
        const LcSlot &S = C.slot[src];
        const bool tgt = S.tgtEpoch == epoch;
        if (tgt && S.tgtLeader == slot) {
            y = 100;
        } else {
            const int sp = V.pos[src];
            const double gap = S.followerGap - lcSafeGapBefore(V, S, epoch);
            y = noCollisionSpeed(V.kin[sp].y, V.tmpl[V.ids[sp].y].maxNegAcc, kk.y, T.maxNegAcc, gap, V.dt, 0);
            if (y < 0) y = 100;
        }
    }
    s = min2(s, y);
    if (d < V.nLanes && idv.w == -2)      // !onValidLane(): PLAN_DEAD
        s = min2(s, noCollisionSpeed(0, 1, kk.y, T.maxNegAcc, V.drvLength[d] - kk.x, V.dt, T.minGap));
    s = max2(s, kk.y - T.maxNegAcc * V.dt);
    return s;
}

// Stage a vehicle that enters another drivable (Engine::pushBuffer, engine.cpp:247-249); same staging as
// the parallel path of k_control, without the warp aggregation (one thread).
__device__ void lcStageMover(const View &V, int d, const int4 idv, const int4 nv, double nd, double v, int newDrv,
                             int newBlocker, int hops, int epoch) {
    const int m = atomicAdd(&V.ctrl->moverCount, 1);
    if (m >= V.moverCap) { atomicOr(&V.ctrl->error, ERR_MOVER_OVERFLOW); return; }
    V.mkin[m] = make_double2(nd, v);
    V.mids[m] = make_int4(idv.x, idv.y, idv.z, V.planData[nv.x + 1 + hops]);
    V.mnav[m] = make_int4(nv.x + hops, d, newBlocker, newDrv >= V.nLanes ? epoch - 1 : INT_MAX);
    const int e = atomicAdd(&V.entCnt[newDrv], 1);
    if (e >= ENT_CAP) atomicOr(&V.ctrl->error, ERR_ENTRANT_OVERFLOW);
    else V.ent[newDrv * ENT_CAP + e] = m;
    if (e == 0 && V.count[newDrv] == 0) V.extraList[atomicAdd(&V.ctrl->nExtra, 1)] = newDrv;
}

// LaneChange::finishChanging lanechange.cpp:115-127 (+ Vehicle::finishChanging vehicle.cpp:378-381: setEnd)
__device__ void lcFinishChanging(const LcView &C, int slot, int epoch, double now) {
    LcSlot &L = C.slot[slot];
    L.changing = 0;
    L.finished = 1;
    L.lastChange = now;
    const int ps = L.partner;
    LcSlot &P = C.slot[ps];
    P.type = 0;            // the shadow becomes the vehicle (and takes over the name: host bookkeeping)
    P.offset = 0;
    P.partner = -1;
    L.partner = -1;
    lcClearSignal(L, epoch);
}
// Vehicle::abortLaneChange vehicle.cpp:413-417 + LaneChange::abortChanging lanechange.cpp:141-148
__device__ void lcAbort(const LcView &C, int slot, int epoch) {
    LcSlot &L = C.slot[slot];
    const int ps = L.partner;
    LcSlot &P = C.slot[ps];
    P.changing = 0;
    P.type = 0;
    P.offset = 0;
    P.partner = -1;
    P.sendEpoch = epoch;   // the parent's signal object lives until its own clearSignal at the end of the step
    lcClearSignal(L, epoch);
}

// Engine::vehicleControl (engine.cpp:188-251) for ONE vehicle involved in a lane change, given its head
__device__ void lcControlOne(const View &V, const LcView &C, int slot, int epoch) {
    const double dt = V.dt;
    const double now = (epoch - 1) * dt;
    {
        LcSlot &L = C.slot[slot];
        const int p = V.pos[slot];
        const int d = C.posDrv[p];
        const double2 kk = V.kin[p];
        const int4 idv = V.ids[p];
        const int4 nv = V.nav[p];
        const DTmpl &T = V.tmpl[idv.y];
        const double dis = kk.x, speed = kk.y;
        double v = L.speedEpoch == epoch ? L.bufSpeed : lcTailSpeed(V, C, slot, epoch);
        {   // engine.cpp:195-205: a vehicle and its shadow move as one
            const int ps = L.partner;
            if (ps >= 0 && C.slot[ps].speedEpoch != epoch) {
                const double partnerSpeed = lcTailSpeed(V, C, ps, epoch);
                v = min2(v, partnerSpeed);
                C.slot[ps].bufSpeed = v;
                C.slot[ps].speedEpoch = epoch;
            }
        }
        double deltaDis;
        if (v < 0) {
            deltaDis = 0.5 * speed * speed / T.maxNegAcc;
            v = 0;
        } else {
            deltaDis = (speed + v) * dt / 2;
        }
        L.bufSpeed = v;
        L.speedEpoch = epoch;
        // Vehicle::setDeltaDistance vehicle.cpp:49-68
        double nd = deltaDis + dis;
        int cur = d, hops = 0, newDrv = -1;
        double curLen = V.drvLength[d];
        while (cur >= 0 && nd > curLen) {
            nd -= curLen;
            const int nx = V.planData[nv.x + 1 + hops];
            ++hops;
            if (nx < 0) {
                if (nx != PLAN_LOOKAHEAD_END) atomicOr(&V.ctrl->error, ERR_ROUTE_DEAD_END);
                newDrv = -2;
                cur = -1;
            } else {
                cur = nx;
                newDrv = nx;
                curLen = V.drvLength[nx];
            }
        }
        // engine.cpp:224-244
        bool end = newDrv == -2;
        if (L.type == 2 && newDrv >= 0) { lcAbort(C, slot, epoch); end = true; }
        if (L.changing) {
            const int dir = lcSendValid(L, epoch) ? L.sendDir : 0;
            const double curWidth = d < V.nLanes ? C.laneWidth[d] : 0.0;
            const double maxOffset = (C.laneWidth[L.sendTarget] + curWidth) / 2;     // vehicle.h:347-350
            double newOffset = fabs(L.offset + max2(0.2 * v, 1) * dt * dir);
            newOffset = min2(newOffset, maxOffset);
            L.offset = newOffset * dir;
            if (newOffset >= maxOffset) { lcFinishChanging(C, slot, epoch, now); end = true; }
        }
        V.nkin[p] = make_double2(nd, v);
        V.nbuf[p] = make_int2(end ? -2 : newDrv, L.headBlocker);
        if (!end && newDrv >= 0) lcStageMover(V, d, idv, nv, nd, v, newDrv, L.headBlocker, hops, epoch);
    }
}
// all involved vehicles in one thread, ascending priority = the order one worker walks its vehicles in
// (kept for the host probe and as a debugging fallback)
__device__ void lcControlTail(const View &V, const LcView &C, int epoch) {
    const int n = min(C.ctrl->nInvolved, LC_MAX_CAND);
    lcSortByPriority(V, C.involved, n);
    for (int i = 0; i < n; ++i) lcControlOne(V, C, C.involved[i], epoch);
}
// Engine::threadUpdateAction -> clearSignal (engine.cpp:424) for the involved vehicles (the plain ones took
// their lastDir in k_control; their epoch-stamped signals expire by themselves)
__device__ void lcClearInvolved(const LcView &C, int epoch) {
    const int n = min(C.ctrl->nInvolved, LC_MAX_CAND);
    for (int i = 0; i < n; ++i) lcClearSignal(C.slot[C.involved[i]], epoch);
}

#ifndef CFB_LC_HOST_PROBE   // (tests/lc_device_probe.cpp compiles the functions above for the host)
// ---- kernels ----------------------------------------------------------------------------------
// segment index of every vehicle on an occupied lane (warp per list entry would be overkill: <= ~40 per lane)
__global__ void __launch_bounds__(256) k_lc_segments(View V, LcView C) {
    const int cpar = V.par;
    const int nAct = V.ctrl->nAct[cpar];
    for (int w = blockIdx.x * blockDim.x + threadIdx.x; w < nAct; w += gridDim.x * blockDim.x) {
        const int d = V.actList[cpar][w];
        if (d < V.nLanes) lcInitSegments(V, C, d);
    }
}
// Engine::handleWaiting gives a vehicle admitted to an EMPTY lane its leader at once (engine.cpp:512); the
// default pipeline defers that search to k_notify, but makeSignal reads the gap before.
__global__ void __launch_bounds__(256) k_lc_admitted(View V, LcView C) {
    const int cpar = V.par;
    const int nAct = V.ctrl->nAct[cpar];
    for (int w = blockIdx.x * blockDim.x + threadIdx.x; w < nAct; w += gridDim.x * blockDim.x) {
        const int d = V.actList[cpar][w];
        if (d >= V.nLanes || !(V.inserted[d] & 2) || V.count[d] == 0) continue;
        const int base = V.off[d];
        const int4 idv = V.ids[base];
        int ld = -1;
        double g = 0;
        headSearch(V, d, 0.0, idv.w, V.nav[base].x, V.tmpl[idv.y], d, ld, g);
        V.leader[base] = ld;
        if (ld >= 0) { V.gap[base] = g; C.slot[idv.x].gap = g; }
    }
}
__global__ void __launch_bounds__(256) k_lc_signal(View V, LcView C) {
    const int cpar = V.par;
    const int nVeh = min(V.ctrl->nVeh[cpar], V.vehCap);
    const int epoch = V.ctrl->step + 1;
    for (int it = blockIdx.x * blockDim.x + threadIdx.x; it < nVeh; it += gridDim.x * blockDim.x) {
        const int2 vd = V.vehList[cpar][it];
        lcMakeSignal(V, C, vd.x, vd.y & ~HEAD_BIT, epoch);
    }
}
__global__ void k_lc_schedule(View V, LcView C) {
    if (blockIdx.x == 0 && threadIdx.x == 0) lcSchedule(V, C, V.ctrl->step + 1);
}
// the host drew the shadows' priorities (vehicle.cpp:33, in schedule order): give them to the records
__global__ void k_lc_priorities(View V, LcView C, const int *prio, int n) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) V.ids[V.pos[C.shadowLog[i].y]].z = prio[i];
}
// Engine::updateLeaderAndGap between scheduling and notifyCross (engine.cpp:573): every occupied drivable
__global__ void __launch_bounds__(256) k_lc_leader(View V, LcView C) {
    const int cpar = V.par;
    const int nAct = V.ctrl->nAct[cpar];
    for (int w = blockIdx.x * blockDim.x + threadIdx.x; w < nAct; w += gridDim.x * blockDim.x) {
        const int d = V.actList[cpar][w];
        const int base = V.off[d], n = V.count[d];
        for (int k = 0; k < n; ++k) {
            const int p = base + k;
            const int4 idv = V.ids[p];
            if (k > 0) {
                const double g = V.kin[p - 1].x - V.tmpl[V.ids[p - 1].y].len - V.kin[p].x;
                V.leader[p] = p - 1;
                V.gap[p] = g;
                C.slot[idv.x].gap = g;
            } else {
                int ld = -1;
                double g = 0;
                headSearch(V, d, V.kin[p].x, idv.w, V.nav[p].x, V.tmpl[idv.y], -1, ld, g);
                V.leader[p] = ld;
                if (ld >= 0) { V.gap[p] = g; C.slot[idv.x].gap = g; }
            }
        }
    }
}
__global__ void k_lc_control_tail(View V, LcView C) {
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        lcControlTail(V, C, V.ctrl->step + 1);
        lcClearInvolved(C, V.ctrl->step + 1);
    }
}
// ---- the same two phases, spread over the roads ---------------------------------------------------------
// Candidates (and involved vehicles) of different roads never interact (DESIGN.md section 10, checked on the
// CPU), so each road walks ITS entries in the global order while the roads run side by side.  Three small
// kernels per phase: order (one block), roads (one thread per entry; the first entry of a road serves the
// whole road), log / clear (one thread).
// k_lc_order: global order of `list[0..n)` = ascending priority (rank sort, priorities are unique) and, for
// the candidates, libstdc++'s all-equal-keys permutation on top; then the group of every entry.
__device__ void lcOrderBlock(const View &V, const LcView &C, int *list, int n, bool candidates, int epoch) {
    int *key = C.scratchA, *sorted = C.scratchB, *group = C.scratchC, *created = C.scratchD;
    for (int i = threadIdx.x; i < n; i += blockDim.x) key[i] = lcPriorityOf(V, list[i]);
    __syncthreads();
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        int r = 0;
        const int k = key[i];
        for (int j = 0; j < n; ++j) r += key[j] < k;
        sorted[r] = list[i];
    }
    __syncthreads();
    for (int i = threadIdx.x; i < n; i += blockDim.x) list[i] = sorted[i];
    __syncthreads();
    if (candidates && threadIdx.x == 0) lcAllEqualSortPermute(list, n);   // std::sort by urgency, all equal (engine.cpp:793)
    __syncthreads();
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        const int slot = list[i];
        const int d = C.posDrv[V.pos[slot]];
        int g;
        if (d < V.nLanes) g = C.laneRoad[d];
        else {   // on a laneLink: only the road its signal source is on can matter to it
            const LcSlot &X = C.slot[slot];
            g = lcRecvValid(X, epoch) ? C.laneRoad[C.posDrv[V.pos[X.recvSrc]]] : -1 - i;
        }
        group[i] = g;
        created[i] = -1;
    }
}
__global__ void __launch_bounds__(256) k_lc_order(View V, LcView C) {
    if (blockIdx.x == 0) lcOrderBlock(V, C, C.cand, min(C.ctrl->nCand, LC_MAX_CAND), true, V.ctrl->step + 1);
}
__global__ void __launch_bounds__(128) k_lc_schedule_roads(View V, LcView C) {
    const int n = min(C.ctrl->nCand, LC_MAX_CAND), epoch = V.ctrl->step + 1;
    const int *group = C.scratchC;
    int *created = C.scratchD;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const int g = group[i];
        bool first = true;
        for (int j = 0; j < i && first; ++j) first = group[j] != g;
        if (!first) continue;
        for (int j = i; j < n; ++j)
            if (group[j] == g) created[j] = lcScheduleOne(V, C, C.cand[j], epoch);
    }
}
// shadows in the global schedule order = the order their priorities are drawn in (vehicle.cpp:33)
__global__ void k_lc_log(View V, LcView C) {
    if (blockIdx.x != 0 || threadIdx.x != 0) return;
    const int n = min(C.ctrl->nCand, LC_MAX_CAND);
    int k = 0;
    for (int i = 0; i < n; ++i)
        if (C.scratchD[i] >= 0) C.shadowLog[k++] = make_int2(C.cand[i], C.scratchD[i]);
    C.ctrl->nShadows = k;
}
__global__ void __launch_bounds__(256) k_lc_tail_order(View V, LcView C) {
    if (blockIdx.x == 0) lcOrderBlock(V, C, C.involved, min(C.ctrl->nInvolved, LC_MAX_CAND), false, V.ctrl->step + 1);
}
__global__ void __launch_bounds__(128) k_lc_tail_roads(View V, LcView C) {
    const int n = min(C.ctrl->nInvolved, LC_MAX_CAND), epoch = V.ctrl->step + 1;
    const int *group = C.scratchC;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const int g = group[i];
        bool first = true;
        for (int j = 0; j < i && first; ++j) first = group[j] != g;
        if (!first) continue;
        for (int j = i; j < n; ++j)
            if (group[j] == g) lcControlOne(V, C, C.involved[j], epoch);
    }
}
__global__ void k_lc_tail_clear(View V, LcView C) {
    if (blockIdx.x == 0 && threadIdx.x == 0) lcClearInvolved(C, V.ctrl->step + 1);
}

// per-step reset of the small counters (before k_lc_signal)
__global__ void k_lc_begin(LcView C) {
    C.ctrl->nCand = 0; C.ctrl->nInvolved = 0; C.ctrl->nShadows = 0; C.ctrl->spareUsed = 0;
}

#endif  // CFB_LC_HOST_PROBE

}  // namespace cfb
