// device_control.cuh -- Cross::canPass and the control phase (k_control's body).  Part of device_sim.cu
// (included there); a header only so that tests/lc_device_probe.cpp can run the phase on the host, one
// vehicle after the other, against the restatement.
#pragma once

namespace cfb {

// ------------------------------------------------------------------------------------------
// Cross::canPass roadnet.cpp:603-676, split at the line between what depends on the foe alone and what depends on
// the asking vehicle.  foeTerms() is the foe half: called by k_notify for every cross side it notifies (`n.dist`,
// `n.pos` set; `foeLinkW` = linkInfo.w of the notified vehicle's laneLink: turn | type << 8).  Same FP64
// expressions as the reference, evaluated on the same committed state (nothing between k_notify and k_control
// changes a vehicle, a blocker or delStep).
// Chosen over the asker doing everything (k_control shorter by more than k_notify grows, at 1.3e5 vehicles) and over a
// lighter record (k_notify only gathers the foe's fields, the asker computes the reach steps and walks the blocker
// chain), on the GPU the engine was first built for; the split has not been re-measured on the H100.
__device__ __forceinline__ void foeTerms(const View &V, Notify &n, int foeLinkW) {
    const int fp = n.pos;
    const int4 fid = V.ids[fp];
    const DTmpl &FT = V.tmpl[fid.y];
    const double foeSpeed = V.kin[fp].y, d2 = n.dist;
    n.slot = fid.x;
    n.prio = fid.z;
    n.enterLL = V.nav[fp].w;          // a size_t compared as double in the reference (vehicle.h:262)
    int fl = (foeLinkW >> 8) << 8;
    if (canYield(FT, foeSpeed, d2)) fl |= NF_CAN_YIELD;
    if (d2 + FT.len < 0) fl |= NF_PASSED;
    n.steps = d2 > 0 ? reachSteps(foeSpeed, d2, (foeLinkW & 1) ? FT.turnSpeed : FT.maxSpeed, FT.usualPosAcc, V.dt) : 0;
    // deadlock detection over the committed blocker chain (Floyd), roadnet.cpp:662-674.  A reference to a vehicle
    // that left the network in the previous step counts as null (Engine::threadUpdateAction drops it,
    // engine.cpp:419-421): evaluated lazily here.
    const int prevStep = V.ctrl->step - 1;
    auto blockerOf = [&](int s) -> int {
        int b = V.blk[s];
        if (b >= 0 && V.delStep[b] == prevStep) b = -1;
        return b;
    };
    int fast = fid.x, slow = fid.x;
    while (fast >= 0) {
        int fb = blockerOf(fast);
        if (fb < 0) break;
        slow = blockerOf(slow);
        fast = blockerOf(fb);
        if (slow == fast) {
            fl |= NF_CYCLE;
            break;
        }
    }
    n.flags = fl;
    n.pad0 = n.pad1 = n.pad2 = 0;
}

// The asking half.  `myLinkW` = linkInfo.w of the asking vehicle's laneLink; `f` = the other side's record.
__device__ __forceinline__ bool canPass(const View &V, const Notify &f, int myLinkW, const DTmpl &T, double mySpeed, int myEnterLL,
                                        int myPriority, double distanceToLaneLinkStart, double distOnLane, int &foeSlot) {
    foeSlot = f.slot;
    const int t1 = myLinkW >> 8, t2 = f.flags >> 8;
    const double d1 = distOnLane - distanceToLaneLinkStart, d2 = f.dist;
    if (!canYield(T, mySpeed, d1)) return true;
    int yield = 0;
    if (!(f.flags & NF_CAN_YIELD)) yield = 1;
    if (yield == 0) {
        if (t1 > t2) {
            yield = -1;
        } else {
            if (d2 > 0) {
                const int foeSteps = f.steps;
                const int mySteps = reachSteps(mySpeed, d1, (myLinkW & 1) ? T.turnSpeed : T.maxSpeed, T.usualPosAcc, V.dt);
                if (foeSteps > mySteps) yield = -1;
                else if (t1 < t2) yield = 1;
                else if (foeSteps < mySteps) yield = 1;
                else {
                    const int foeEnter = f.enterLL;
                    if (myEnterLL == foeEnter) {
                        if (d1 == d2) yield = myPriority > f.prio ? -1 : 1;
                        else yield = d1 < d2 ? -1 : 1;
                    } else {
                        yield = myEnterLL < foeEnter ? -1 : 1;
                    }
                }
            } else {
                yield = (f.flags & NF_PASSED) ? -1 : 1;
            }
        }
    }
    if (yield == 1 && (f.flags & NF_CYCLE)) yield = -1;
    return yield == -1;
}

}  // namespace cfb
#include "device_lc.cuh"
namespace cfb {

// k_control: one thread per running vehicle (grid-stride over the position list).
// Vehicle::getNextSpeed vehicle.cpp:308-335, getCarFollowSpeed :212-238, getIntersectionRelatedSpeed
// :337-376, Engine::vehicleControl engine.cpp:188-251, Vehicle::setDeltaDistance vehicle.cpp:49-68.
__device__ __forceinline__ void phase_control(const View &V, const int bid, const int nblk) {
    const int cpar = V.par;
    const int nVeh = min(V.ctrl->nVeh[cpar], V.vehCap);
    const double dt = V.dt;
    const int epoch = V.ctrl->step + 1;
    for (int it = bid * blockDim.x + threadIdx.x; it < nVeh; it += nblk * blockDim.x) {
        const long long tStart = clock64();
        const int2 vd = V.vehList[cpar][it];
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
        if (V.ctrl->nCustom > 0) {  // uniform; zero cost when set_vehicle_speed is not in use
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
        unsigned pathBits = (lp >= 0 ? 1u : 0u); (void) pathBits;
        // ---- intersection logic ----
        int newBlocker = -1;
        const int nd0 = idv.w;
        if (onLink || (nd0 >= V.nLanes && dLen - dis <= T.approachDist)) {
            pathBits |= 2u;
            double s = T.maxSpeed;
            int ll = -1;
            bool done = false;
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
                const double toStart = onLink ? dis : -(dLen - dis);
                // crosses of the link in ascending distance; only those with a notified foe matter
                // (a cross without foe passes, roadnet.cpp:613), and k_notify marked exactly those
                const int cb = li.z;
                bool stop = false;
                for (int wd = 0; wd < V.maskWords && !stop; ++wd) {
                    unsigned bits = wd == 0 ? mask0 : V.foeMask[ll * V.maskWords + wd];
                    while (bits) {
                        const int b = __ffs(bits) - 1;
                        bits &= bits - 1;
                        const int q = cb + wd * 32 + b;
                        const double dOn = V.lcDist[q];
                        if (dOn < toStart) continue;
                        const int cs = V.lcIdx[q];
                        const Notify f = V.notify[cs ^ 1];
                        if (f.epoch != epoch) continue;
                        pathBits |= 4u;
                        int foeSlot;
                        if (!canPass(V, f, li.w, T, speed, nv.w, idv.z, toStart, dOn, foeSlot)) {
                            s = min2(s, stopBeforeSpeed(T, speed, dOn - toStart - T.yieldDistance, dt));
                            newBlocker = foeSlot;
                            stop = true;
                            break;
                        }
                    }
                }
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
        V.dbgPath[p] = pathBits | ((unsigned) (tCf - tStart) >> 6 << 8);
#endif
        (void) tStart;
        if (newDrv >= 0) pathBits |= 8u;
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
