// device_phases_b.cuh -- bodies of k_move and k_leader.  Part of device_sim.cu (included there); a header so
// that tests/lc_device_probe.cpp can run the phases on the host with an emulated warp.
#pragma once

namespace cfb {

// ------------------------------------------------------------------------------------------
// k_move: warp per drivable that is occupied or receives entrants.  Survivors are compacted in
// place with a ballot/popc scan (stable, so list order is preserved); the few entrants are
// rank-sorted by (new distance desc, priority asc) -- the reference's global std::sort on distance
// (engine.cpp:480) restricted to one target -- and appended.  Commits Buffer -> state
// (Vehicle::update, vehicle.cpp:107-143) and emits the next step's work lists.
__device__ __forceinline__ void phase_move(const View &V, const int bid, const int nblk) {
    const int lane = threadIdx.x & 31;
    const int warp = (bid * blockDim.x + threadIdx.x) >> 5;
    const int nWarps = (nblk * blockDim.x) >> 5;
    const int cpar = V.par, npar = cpar ^ 1;
    const int nAct = V.ctrl->nAct[cpar];
    const int nTot = nAct + V.ctrl->nExtra;
    __shared__ int sTot[8];
    __shared__ int sBaseVeh, sBaseAct;
    const int wib = threadIdx.x >> 5, wpb = blockDim.x >> 5;
    (void) warp; (void) nWarps;
    for (int w0 = bid * wpb; w0 < nTot; w0 += nblk * wpb) {  // trip count uniform per block
        const int w = w0 + wib;
        int total = 0, d = -1, base = 0;
        if (w < nTot) {
        d = w < nAct ? V.actList[cpar][w] : V.extraList[w - nAct];
        const int n = V.count[d];
        int m = V.entCnt[d];
        base = V.off[d];
        const int cap = V.off[d + 1] - base;
        int nsurv = 0;
        // Leader / gap of every vehicle that is not the head of the list (Vehicle::updateLeaderAndGap, vehicle.cpp:158-160:
        // leader = list predecessor, gap = leader.dis - leader.len - dis on the committed values) is settled right here:
        // the warp that compacts the bucket holds every survivor's new distance in registers, the predecessor's arrive by
        // shuffle, and `carry` hands the last committed vehicle over to the next chunk / to the entrants.  Only list heads
        // (cross-drivable search) are left to k_leader.
        double carryDis = 0, carryLen = 0;
        for (int c0 = 0; c0 < n; c0 += 32) {
            const int k = c0 + lane;
            const bool valid = k < n;
            double2 nk = make_double2(0, 0);
            int2 nb = make_int2(0, 0);
            int4 idv = make_int4(0, 0, 0, 0), nv = make_int4(0, 0, 0, 0);
            if (valid) {
                const int p = base + k;
                nk = V.nkin[p];
                nb = V.nbuf[p];
                idv = V.ids[p];
                nv = V.nav[p];
            }
            const bool keep = valid && nb.x == -1;
            const unsigned mask = __ballot_sync(0xffffffffu, keep);
            const unsigned below = mask & ((1u << lane) - 1);
            const int dst = nsurv + __popc(below);
            const double myLen = keep ? V.tmpl[idv.y].len : 0.0;
            const int predLane = below ? 31 - __clz(below) : 0;    // nearest survivor in front of me inside this chunk
            double pd = __shfl_sync(0xffffffffu, nk.x, predLane);
            double pl = __shfl_sync(0xffffffffu, myLen, predLane);
            if (!below) { pd = carryDis; pl = carryLen; }
            __syncwarp();
            if (keep) {
                const int q = base + dst;
                V.kin[q] = nk;                                     // dis, speed
                if (nb.y != nv.z) blkSet(V, idv.x, nb.y);
                nv.z = nb.y;                                       // blocker := buffer.blocker or null
                V.nav[q] = nv;
                if (dst != k) {
                    V.ids[q] = idv;
                    V.pos[idv.x] = q;
                }
                if (dst > 0) {
                    V.leader[q] = q - 1;
                    V.gap[q] = pd - pl - nk.x;
                    if (V.lcOn) V.lc.slot[idv.x].gap = pd - pl - nk.x;
                }
            } else if (valid && nb.x == -2) {                      // finished (engine.cpp:296-310)
                V.pos[idv.x] = -1;
                blkSet(V, idv.x, -2);
                const int f = atomicAdd(&V.ctrl->finCount, 1);
                // a vehicle replaced by its shadow is not a "finished vehicle" (engine.cpp:297-301): flagged for the host
                const int finTag = (V.lcOn && V.lc.slot[idv.x].finished) ? (idv.x | 0x40000000) : idv.x;
                if (f < V.finCap) V.finSlots[f] = make_int2(finTag, V.ctrl->step); else atomicOr(&V.ctrl->error, ERR_FINISHED_OVERFLOW);
                atomicSub(&V.ctrl->active, 1);
            }
            if (mask) {
                const int last = 31 - __clz(mask);
                carryDis = __shfl_sync(0xffffffffu, nk.x, last);
                carryLen = __shfl_sync(0xffffffffu, myLen, last);
            }
            nsurv += __popc(mask);
        }
        if (m > 0) {
            if (m > ENT_CAP) m = ENT_CAP;
            if (nsurv + m > cap) {
                if (lane == 0) atomicOr(&V.ctrl->error, ERR_BUCKET_OVERFLOW);
                m = max(0, cap - nsurv);
            }
            int mi = -1;
            double myDis = 0, myLen = 0;
            int myPrio = 0;
            if (lane < m) {
                mi = V.ent[d * ENT_CAP + lane];
                myDis = V.mkin[mi].x;
                const int4 mid = V.mids[mi];
                myPrio = mid.z;
                myLen = V.tmpl[mid.y].len;
            }
            int rank = 0;
            for (int j = 0; j < m; ++j) {
                const double od = __shfl_sync(0xffffffffu, myDis, j);
                const int op = __shfl_sync(0xffffffffu, myPrio, j);
                if (lane < m && j != lane && (od > myDis || (od == myDis && op < myPrio))) ++rank;
                // each same-distance pair once; the rank above orders it by priority (tests/edgenet.py merge_ties)
                if (lane < m && j < lane && od == myDis) atomicAdd(&V.ctrl->ties, 1);
            }
            double pd = carryDis, pl = carryLen;                   // list predecessor of the first entrant: the last survivor
            for (int j = 0; j < m; ++j) {
                const double od = __shfl_sync(0xffffffffu, myDis, j);
                const double ol = __shfl_sync(0xffffffffu, myLen, j);
                const int orank = __shfl_sync(0xffffffffu, rank, j);
                if (lane < m && orank == rank - 1) { pd = od; pl = ol; }
            }
            if (lane < m) {
                const int q = base + nsurv + rank;
                const int4 idv = V.mids[mi];
                V.kin[q] = V.mkin[mi];
                V.ids[q] = idv;
                const int4 mnv = V.mnav[mi];
                V.nav[q] = mnv;
                blkSet(V, idv.x, mnv.z);
                V.pos[idv.x] = q;
                if (nsurv + rank > 0) {
                    V.leader[q] = q - 1;
                    V.gap[q] = pd - pl - myDis;
                    if (V.lcOn) V.lc.slot[idv.x].gap = pd - pl - myDis;
                }
            }
            if (lane == 0) V.entCnt[d] = 0;
        }
        total = nsurv + m;
        __syncwarp();  // the committed records written above are read back by lane 0
        if (lane == 0) {
            V.count[d] = total;
            Tail t;
            t.dis = 0; t.len = 0; t.speed = 0; t.pos = -1; t.prev = -1;
            if (total > 0) {  // re-read the committed last vehicle (written by this warp just above)
                const int q = base + total - 1;
                const double2 kq = V.kin[q];
                t.dis = kq.x; t.speed = kq.y; t.len = V.tmpl[V.ids[q].y].len; t.pos = q; t.prev = V.nav[q].y;
            }
            V.tail[d] = t;
        }
        }  // w < nTot
        // next step's work lists: one pair of atomics per block, offsets by a scan over its warps
        if (lane == 0) sTot[wib] = total;
        __syncthreads();
        if (threadIdx.x == 0) {
            int sv = 0, sa = 0;
            for (int k = 0; k < wpb; ++k) { sv += sTot[k]; sa += sTot[k] > 0; }
            sBaseVeh = sv ? atomicAdd(&V.ctrl->nVeh[npar], sv) : 0;
            sBaseAct = sa ? atomicAdd(&V.ctrl->nAct[npar], sa) : 0;
        }
        __syncthreads();
        if (total > 0) {
            int offV = sBaseVeh, offA = sBaseAct;
            for (int k = 0; k < wib; ++k) { offV += sTot[k]; offA += sTot[k] > 0; }
            if (lane == 0) V.actList[npar][offA] = d;
            for (int k = lane; k < total; k += 32)
                if (offV + k < V.vehCap) V.vehList[npar][offV + k] = make_int2(base + k, k == 0 ? (d | HEAD_BIT) : d);
        }
        __syncthreads();
    }
}

// ------------------------------------------------------------------------------------------
// k_leader: thread per occupied drivable (the list k_move just wrote): the cross-drivable leader search of the list
// HEAD (vehicle.cpp:162-195).  Everybody else's leader / gap was settled by k_move while it had the bucket in
// registers.  In the leading threads: the traffic lights (TrafficLight::passTime, trafficlight.cpp:29-37) and the
// step counter.
__device__ __forceinline__ void phase_leader(const View &V, const int bid, const int nblk) {
    const int gtid = bid * blockDim.x + threadIdx.x;
    const int lane = threadIdx.x & 31;
    const int warp = gtid >> 5;
    const int nWarps = (nblk * blockDim.x) >> 5;
    const int npar = V.par ^ 1;
    const int nAct = V.ctrl->nAct[npar];
    if (gtid == 0) {  // nothing in this kernel reads these (list parity is the host-provided V.par)
        V.ctrl->step += 1;                                             // Engine::step (engine.cpp:593)
        V.ctrl->epoch += 1;
        V.ctrl->vehicleSteps += (unsigned long long) (long long) V.ctrl->active;   // may be negative on one rank of a sharded run  // all finishes of this step are in
        if (V.hostMirror) {   // the step's result, stored straight into host memory: get_vehicle_count() needs no copy
            volatile int *m = V.hostMirror;
            m[1] = V.ctrl->active;
            m[2] = V.ctrl->error;
            m[3] = V.ctrl->ties;
            __threadfence_system();
            m[0] = V.ctrl->epoch;
        }
    }
    if (!V.rl) {
        for (int in = gtid; in < V.nInter; in += nblk * blockDim.x) {
            if (V.interVirtual[in]) continue;
            double rem = V.remain[in] - V.dt;
            int cur = V.curPhase[in];
            const int pb = V.interPhaseBeg[in], nph = V.interPhaseBeg[in + 1] - pb;
            while (rem <= 0.0) {
                cur = (cur + 1) % nph;
                rem += V.phaseTime[pb + cur];
            }
            V.remain[in] = rem;
            V.curPhase[in] = cur;
        }
    }
    const int stride = nblk * blockDim.x;
    (void) lane; (void) warp; (void) nWarps;
    // list heads: dense pass, one thread per occupied drivable (their cross-drivable search is a
    // chain of dependent loads; keeping it out of the streaming pass above avoids one slow lane
    // per warp)
    for (int w = gtid; w < nAct; w += stride) {
        const int d = V.actList[npar][w];
        const int p = V.off[d];
        const int4 idv = V.ids[p];
        int ld = -1;
        double g = 0;
        headSearch(V, d, V.kin[p].x, idv.w, V.nav[p].x, V.tmpl[idv.y], -1, ld, g);
        V.leader[p] = ld;
        if (ld >= 0) V.gap[p] = g;
        if (V.lcOn && ld >= 0) V.lc.slot[idv.x].gap = g;
    }
}

}  // namespace cfb
