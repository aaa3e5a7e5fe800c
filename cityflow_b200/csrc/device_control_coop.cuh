// device_control_coop.cuh -- k_control with the crosses evaluated by the whole warp.  EXPERIMENT, compiled only
// with -DCFB_CONTROL_COOP; never timed (written when no GPU was left).  Logic verified on the emulated device.
//
// Why: k_control lasts as long as its slowest thread, and the slowest threads are the few vehicles that walk
// four or five flagged crosses one after the other (a per-thread cycle count showed 3x the mean for them), while most lanes of their warp -- the vehicles further back on the same lane -- have nothing to do
// during that loop.  Here every flagged cross at or beyond a vehicle is a work item in shared memory, the 32
// lanes evaluate the warp's items side by side (Cross::canPass has no side effect), and each vehicle then takes
// the first failing cross of its own list in link order.  Same arithmetic, same results; the grid-stride loop is
// made warp-uniform for the shuffles.  Generated from phase_control's text; keep the two in step.
#pragma once

namespace cfb {

__device__ __forceinline__ void phase_control_coop(const View &V, const int bid, const int nblk) {
#ifndef CFB_COOP_ITEMS
#define CFB_COOP_ITEMS 64
#endif
    constexpr int ITEMS = CFB_COOP_ITEMS, WARPS = 8;   // items per round and warp (tests shrink it to exercise the rounds); blockDim.x <= 256
    __shared__ int sItemP[WARPS][ITEMS], sItemQ[WARPS][ITEMS], sRes[WARPS][ITEMS];
    __shared__ double sItemStart[WARPS][ITEMS];
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    const int cpar = V.par;
    const int nVeh = min(V.ctrl->nVeh[cpar], V.vehCap);
    const double dt = V.dt;
    const int epoch = V.ctrl->step + 1;
    for (int it0 = bid * blockDim.x + threadIdx.x - lane; it0 < nVeh; it0 += nblk * blockDim.x) {   // trip count uniform per warp
        const int it = it0 + lane;
        const bool valid = it < nVeh;
        const long long tStart = clock64();
        const int2 vd = V.vehList[cpar][valid ? it : 0];
        const int p = vd.x, d = vd.y & ~HEAD_BIT;
        // ---- load phase: everything the branches below may need is requested up front with
        // clamped (always valid) indices, so the dependent-load depth is 3 levels, not one
        // round trip per branch ----
        const double2 kk = V.kin[p];
        const int4 idv = V.ids[p];
        const int4 nv = V.nav[p];
        const int lp = V.leader[p];
        const double g = V.gap[p];
        const double dLen = V.drvLength[d], dMax = V.drvMaxSpeed[d];
        const bool onLink = d >= V.nLanes;
        const double dis = kk.x, speed = kk.y;
        const int lpc = lp >= 0 ? lp : p;
        const double leaderSpeed = V.kin[lpc].y;
        const int leaderTmpl = V.ids[lpc].y;
        const int llc = idv.w >= V.nLanes ? idv.w - V.nLanes : (onLink ? d - V.nLanes : 0);  // the laneLink of interest
        const int4 li = V.linkInfo[llc];          // {roadLink, endLane, crossBeg, turn | type << 8}
        const unsigned mask0 = V.foeMask[llc * V.maskWords];
        const DTmpl &T = V.tmpl[idv.y];
        const DTmpl &LT = V.tmpl[leaderTmpl];
        const unsigned char linkGreen = V.rlAvail[li.x];
        const Tail endTail = V.tail[li.y];
        const int planBase = nv.x + 1;
        double custom = 0;
        bool hasCustom = false;
        if (valid && V.ctrl->nCustom > 0) {  // uniform; zero cost when set_vehicle_speed is not in use
            custom = V.cust[p];
            hasCustom = custom == custom;
            if (hasCustom) {  // consumed this step (Vehicle::update clears it, vehicle.cpp:120-122)
                V.cust[p] = __longlong_as_double(-1LL);
                atomicSub(&V.ctrl->nCustom, 1);
            }
        }

        double v = T.maxSpeed;
        v = min2(v, speed + T.maxPosAcc * dt);
        v = min2(v, dMax);
        // ---- car following ----
        {
            double cf;
            if (lp < 0) {
                cf = hasCustom ? custom : T.maxSpeed;
            } else if (hasCustom) {
                cf = min2(custom, noCollisionSpeed(leaderSpeed, LT.maxNegAcc, speed, T.maxNegAcc, g, dt, 0));
            } else {
                cf = noCollisionSpeed(leaderSpeed, LT.maxNegAcc, speed, T.maxNegAcc, g, dt, 0);
                double assumeDecel = 0;
                if (speed > leaderSpeed) assumeDecel = speed - leaderSpeed;
                cf = min2(cf, noCollisionSpeed(leaderSpeed, LT.usualNegAcc, speed, T.usualNegAcc, g, dt, T.minGap));
                cf = min2(cf, (g + (leaderSpeed + assumeDecel / 2) * dt - speed * dt / 2) / (T.headwayTime + dt / 2));
            }
            v = min2(v, cf);
        }
        const long long tCf = clock64(); (void) tCf;
        // ---- intersection logic, up to the crosses ----
        int newBlocker = -1;
        const int nd0 = idv.w;
        const bool related = valid && (onLink || (nd0 >= V.nLanes && dLen - dis <= T.approachDist));
        double s = T.maxSpeed;
        int ll = -1;
        bool done = false;
        double toStart = 0;
        if (related) {
            if (nd0 >= V.nLanes) {
                ll = nd0 - V.nLanes;
                bool blocked = !linkGreen;
                if (!blocked) {  // Lane::canEnter roadnet.cpp:437-445
                    if (endTail.pos >= 0) blocked = !(endTail.dis > endTail.len + T.len || endTail.speed >= 2);
                }
                if (blocked) {
                    if (0.5 * speed * speed / T.maxNegAcc > dLen - dis) {
                        // cannot stop before the line any more
                    } else {
                        s = min2(s, stopBeforeSpeed(T, speed, dLen - dis, dt));
                        done = true;
                    }
                }
                if (!done && (li.w & 1)) s = min2(s, T.turnSpeed);
            }
            if (!done) {
                if (ll < 0 && onLink) ll = d - V.nLanes;
                toStart = onLink ? dis : -(dLen - dis);
            }
        }
        // ---- the crosses: every flagged cross at or beyond the vehicle is one work item; the WARP evaluates the
        // items of all its vehicles side by side (Cross::canPass has no side effect), then every vehicle takes the
        // first failing cross of its own list in link order -- what the sequential loop stops at (vehicle.cpp:362-373)
        const bool wantsCrosses = related && !done;
        int cnt = 0;
        if (wantsCrosses) {
            const int cb = li.z;
            for (int wd = 0; wd < V.maskWords; ++wd) {
                unsigned bits = wd == 0 ? mask0 : V.foeMask[ll * V.maskWords + wd];
                while (bits) {
                    const int b = __ffs(bits) - 1;
                    bits &= bits - 1;
                    const int q = cb + wd * 32 + b;
                    if (V.lcDist[q] < toStart) continue;
                    if (V.notify[V.lcIdx[q] ^ 1].epoch != epoch) continue;
                    ++cnt;
                }
            }
        }
        int off = cnt;   // inclusive scan over the warp
        for (int o = 1; o < 32; o <<= 1) {
            const int up = __shfl_up_sync(0xffffffffu, off, o);
            if (lane >= o) off += up;
        }
        const int total = __shfl_sync(0xffffffffu, off, 31);
        off -= cnt;
        int failJ = INT_MAX, failQ = -1, failFoe = -1;
        for (int base = 0; base < total; base += ITEMS) {
            if (wantsCrosses && off < base + ITEMS && off + cnt > base) {   // my items that fall into this chunk
                const int cb = li.z;
                int j = 0;
                for (int wd = 0; wd < V.maskWords; ++wd) {
                    unsigned bits = wd == 0 ? mask0 : V.foeMask[ll * V.maskWords + wd];
                    while (bits) {
                        const int b = __ffs(bits) - 1;
                        bits &= bits - 1;
                        const int q = cb + wd * 32 + b;
                        if (V.lcDist[q] < toStart) continue;
                        if (V.notify[V.lcIdx[q] ^ 1].epoch != epoch) continue;
                        const int k = off + j - base;
                        if (k >= 0 && k < ITEMS) { sItemP[wib][k] = p; sItemQ[wib][k] = q; sItemStart[wib][k] = toStart; }
                        ++j;
                    }
                }
            }
            __syncwarp();
            const int here = min(ITEMS, total - base);
            for (int k = lane; k < here; k += 32) {
                const int p2 = sItemP[wib][k], q2 = sItemQ[wib][k];
                const int4 id2 = V.ids[p2];
                const int cs = V.lcIdx[q2];
                const Notify f = V.notify[cs ^ 1];
                int foeSlot = -1;
                const bool pass = canPass(V, f, V.linkInfo[V.csLink[cs]].w, V.tmpl[id2.y], V.kin[p2].y, V.nav[p2].w, id2.z, sItemStart[wib][k], V.lcDist[q2], foeSlot);
                sRes[wib][k] = pass ? -1 : foeSlot;
            }
            __syncwarp();
            if (wantsCrosses)
                for (int j = max(0, base - off); j < cnt && off + j < base + ITEMS; ++j) {
                    const int k = off + j - base;
                    if (sRes[wib][k] >= 0 && j < failJ) { failJ = j; failQ = sItemQ[wib][k]; failFoe = sRes[wib][k]; }
                }
            __syncwarp();
        }
        if (!valid) continue;
        if (related) {
            if (failQ >= 0) {
                s = min2(s, stopBeforeSpeed(T, speed, V.lcDist[failQ] - toStart - T.yieldDistance, dt));
                newBlocker = failFoe;
            }
            v = min2(v, s);
        }
        if (V.lcOn) {   // vehicle.cpp:323-329 / engine.cpp:195-244, see device_lc.cuh
            LcSlot &L = V.lc.slot[idv.x];
            if (L.partner >= 0 || lcRecvValid(L, epoch) || L.type != 0 || L.changing) {
                // involved in a lane change: the rest depends on the order vehicles are processed in
                L.head = v;
                L.headBlocker = newBlocker;
                const int k = atomicAdd(&V.lc.ctrl->nInvolved, 1);
                if (k < LC_MAX_CAND) V.lc.involved[k] = idv.x; else atomicOr(&V.lc.ctrl->error, 1);
                continue;
            }
            if (lcPlanChange(L, d, epoch)) L.waiting += dt;                 // yieldSpeed's side effect (lanechange.cpp:190)
            v = min2(v, 100.0);                                             // no signal received: yieldSpeed() == 100
            if (!onLink && nd0 == PLAN_DEAD)
                v = min2(v, noCollisionSpeed(0, 1, speed, T.maxNegAcc, dLen - dis, dt, T.minGap));
            // Engine::threadUpdateAction -> clearSignal (engine.cpp:424) happens after EVERY vehicle's control:
            // a receiver finished later (k_lc_control_tail) still reads this vehicle's target leader /
            // follower, so only lastDir is taken here; the epoch-stamped signals expire by themselves
            L.lastDir = lcSendValid(L, epoch) ? L.sendDir : 0;
        }
        // vehicle.cpp:323-329 runs with laneChange=false too (the `if` there tests the LaneChange OBJECT):
        // yieldSpeed() is 100 without signals, and a vehicle whose lane cannot continue its route stops
        // at the end of the lane.  Found by the fuzz tests (DESIGN.md section 6); NOT compiled in by
        // default until it has been validated on a GPU (tools/gpu_fuzz_check.py).
        v = min2(v, 100.0);
        if (!onLink && nd0 == PLAN_DEAD)
            v = min2(v, noCollisionSpeed(0, 1, speed, T.maxNegAcc, dLen - dis, dt, T.minGap));
        v = max2(v, speed - T.maxNegAcc * dt);
        // ---- Engine::vehicleControl ----
        double deltaDis;
        if (v < 0) {
            deltaDis = 0.5 * speed * speed / T.maxNegAcc;
            v = 0;
        } else {
            deltaDis = (speed + v) * dt / 2;
        }
        // ---- setDeltaDistance: walk over the planned drivables ----
        double nd = deltaDis + dis;
        int cur = d, hops = 0, newDrv = -1;
        double curLen = dLen;
        while (cur >= 0 && nd > curLen) {
            nd -= curLen;
            int nx = V.planData[planBase + hops];
            ++hops;
            if (nx < 0) {
                if (nx != PLAN_LOOKAHEAD_END) atomicOr(&V.ctrl->error, ERR_ROUTE_DEAD_END);
                newDrv = -2;  // ran off the last road: end
                cur = -1;
            } else {
                cur = nx;
                newDrv = nx;
                curLen = V.drvLength[nx];
            }
        }
        V.nkin[p] = make_double2(nd, v);
        V.nbuf[p] = make_int2(newDrv, newBlocker);
#ifdef CFB_DEBUG_COUNTERS
        V.dbgCyc[p] = (unsigned) (clock64() - tStart);
        V.dbgPath[p] = 0;
#endif
        (void) tStart;
        if (newDrv >= 0) {  // Engine::pushBuffer (engine.cpp:247-249)
            int m;
            {  // one atomic per warp for the movers of this warp
                auto g = cg::coalesced_threads();
                int b = 0;
                if (g.thread_rank() == 0) b = atomicAdd(&V.ctrl->moverCount, (int) g.size());
                m = g.shfl(b, 0) + (int) g.thread_rank();
            }
            if (m >= V.moverCap) {
                atomicOr(&V.ctrl->error, ERR_MOVER_OVERFLOW);
            } else {
                V.mkin[m] = make_double2(nd, v);
                V.mids[m] = make_int4(idv.x, idv.y, idv.z, V.planData[planBase + hops]);  // next drivable after the new one
                // enterLaneLinkTime: step for links, INT_MAX for lanes (engine.cpp:486-490)
                V.mnav[m] = make_int4(nv.x + hops, d, newBlocker, newDrv >= V.nLanes ? epoch - 1 : INT_MAX);
                const int e = atomicAdd(&V.entCnt[newDrv], 1);
                if (e >= ENT_CAP) atomicOr(&V.ctrl->error, ERR_ENTRANT_OVERFLOW);
                else V.ent[newDrv * ENT_CAP + e] = m;
                // an empty target is on no work list yet: queue it for k_move
                if (V.owned && V.owned[newDrv] != 1) {
                    V.pos[idv.x] = -1;   // the record travels to the owner of the lane (k_pack_movers)
                } else if (e == 0 && V.count[newDrv] == 0) {
                    V.extraList[atomicAdd(&V.ctrl->nExtra, 1)] = newDrv;
                }
            }
        }
    }
}

}  // namespace cfb
