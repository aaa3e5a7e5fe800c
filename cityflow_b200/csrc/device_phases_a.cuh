// device_phases_a.cuh -- bodies of k_ingest and k_notify (+ blocker commit, cross-drivable leader search).
// Part of device_sim.cu (included there); a header so that tests/lc_device_probe.cpp can run the phases on
// the host with an emulated warp.
#pragma once

namespace cfb {

// Commit a vehicle's blocker (slot-indexed copy used by chain walks); in sharded mode the change is
// also queued for the other ranks.  val == -2: the vehicle left the network this step.
__device__ __forceinline__ void blkSet(const View &V, int slot, int val) {
    if (val == -2) {
        V.blk[slot] = -1;
        V.delStep[slot] = V.ctrl->step;
    } else {
        V.blk[slot] = val;
    }
    if (V.blkUpd) {
        const int i = atomicAdd(&V.ctrl->nBlkUpd, 1);
        if (i < V.blkUpdCap) V.blkUpd[1 + i] = make_int2(slot, val); else atomicOr(&V.ctrl->error, ERR_MOVER_OVERFLOW);
    }
}

__device__ __forceinline__ int planAt(const View &V, int plan, int idx) { return V.planData[V.planBeg[plan] + idx]; }
__device__ __forceinline__ void foeTerms(const View &V, Notify &n, int foeLinkW);   // device_control.cuh

// Cross-drivable leader search for the head of a list (Vehicle::updateLeaderAndGap, else-branch,
// vehicle.cpp:162-195).  Candidates are read from the per-drivable tail records.  `myLane >= 0`
// enables the handleWaiting ordering rule: lanes later in roadnet order have not been served yet
// when the reference inserts into `myLane` (engine.cpp:503), so their admission is ignored.
__device__ void headSearch(const View &V, int d, double dis, int nextDrv, int planIdx, const DTmpl &T, int myLane,
                           int &outLeader, double &outGap) {
    int leader = -1;
    double gap = 0;
    double x = V.drvLength[d] - dis;
    int nd = nextDrv;
    for (int i = 0;; ++i) {
        if (i > 0) nd = V.planData[planIdx + 1 + i];
        if (nd < 0) break;
        if (nd >= V.nLanes) {
            const int sl = V.llStartLane[nd - V.nLanes];
            for (int q = V.laneOutBeg[sl]; q < V.laneOutBeg[sl + 1]; ++q) {
                const Tail t = V.tail[V.nLanes + V.laneOutLinks[q]];
                if (t.pos >= 0) {
                    double candGap = x + t.dis - t.len;
                    if (leader < 0 || candGap < gap) {
                        leader = t.pos;
                        gap = candGap;
                    }
                }
            }
            if (leader >= 0) break;
        } else {
            Tail t = V.tail[nd];
            if (myLane >= 0 && nd > myLane && (V.inserted[nd] & 1)) {  // undo the later lane's admission
                const int c = V.count[nd] - 1;
                if (c > 0) {
                    const int tp = V.off[nd] + c - 1;
                    t.pos = tp;
                    t.dis = V.kin[tp].x;
                    t.len = V.tmpl[V.ids[tp].y].len;
                } else {
                    t.pos = -1;
                }
            }
            if (t.pos >= 0) {
                leader = t.pos;
                gap = x + t.dis - t.len;
                break;
            }
        }
        x += V.drvLength[nd];
        if (x > T.approachDist) break;  // same expression as the look-ahead bound, vehicle.cpp:190-191
    }
    outLeader = leader;
    if (leader >= 0) outGap = gap;
}

// ------------------------------------------------------------------------------------------
// k_ingest: thread i serves lane i (queue append + admission) and roadLink i (light mask).
// Flow::nextStep / planRoute stay on the host (serial mt19937 order); their result arrives as
// lane-sorted SpawnRec's whose lane keys are staged in shared memory for the per-lane lookup.
// handleWaiting: engine.cpp:502-516, Lane::available roadnet.cpp:428-435.
__device__ __forceinline__ void phase_ingest(const View &V, const int bid, const int nblk) {
    __shared__ int sLane[SPAWN_SMEM];
    const int gtid0 = bid * blockDim.x + threadIdx.x;
    int i = gtid0;
    const int nSpawn = V.spawn[-1].slot;
    const int cpar = V.par;
    const bool staged = nSpawn <= SPAWN_SMEM;
    if (staged)
        for (int k = threadIdx.x; k < nSpawn; k += blockDim.x) sLane[k] = V.spawn[k].lane;
    __syncthreads();
    const int nRLmine = V.ingRL ? V.nIngRL : V.nRL;
    for (int x = i; x < nRLmine; x += nblk * blockDim.x) {
        const int r = V.ingRL ? V.ingRL[x] : x;
        int in = V.rlInter[r];
        int ph = V.interPhaseBeg[in] + V.curPhase[in];
        V.rlAvail[r] = V.phaseAvail[V.phaseAvailBeg[ph] + (r - V.interRLBeg[in])];
    }
    if (V.ingLinks) {
        for (int x = i; x < V.nIngLinks * V.maskWords; x += nblk * blockDim.x)
            V.foeMask[V.ingLinks[x / V.maskWords] * V.maskWords + x % V.maskWords] = 0u;
    } else {
        for (int k = i; k < V.nLinks * V.maskWords; k += nblk * blockDim.x) V.foeMask[k] = 0u;
    }
    if (i == 0) {  // lists of the other parity are rebuilt by this step's k_move
        V.ctrl->moverCount = 0;
        V.ctrl->nVeh[cpar ^ 1] = 0;
        V.ctrl->nAct[cpar ^ 1] = 0;
        V.ctrl->nExtra = 0;
    }
    const int nLanesMine = V.ingLanes ? V.nIngLanes : V.nLanes;
    for (int x = gtid0; x < nLanesMine; x += nblk * blockDim.x) {
    i = V.ingLanes ? V.ingLanes[x] : x;
    // Sharded: a lane this rank FEEDS is admitted into here as well, on the ghost copy, with the same
    // inputs as on its owner (spawn records and queue are replicated, the ghost tail is exact after
    // the previous step's exchange) -- so the owner need not report the admission.
    const int own = V.owned ? V.owned[i] : 1;
    if (own == 0) continue;
    if (nSpawn > 0) {
        int lo = 0, hi = nSpawn;  // lower bound of lane i
        while (lo < hi) {
            int mid = (lo + hi) >> 1;
            int key = staged ? sLane[mid] : V.spawn[mid].lane;
            if (key < i) lo = mid + 1; else hi = mid;
        }
        if (lo < nSpawn && (staged ? sLane[lo] : V.spawn[lo].lane) == i) {
            int tail = V.waitTail[i];
            for (int r = lo; r < nSpawn && (staged ? sLane[r] : V.spawn[r].lane) == i; ++r) {
                SpawnRec s = V.spawn[r];
                V.slotInfo[s.slot] = make_int4(s.tmpl, s.priority, s.plan, 0);
                V.waitNext[s.slot] = -1;
                if (tail < 0) V.waitHead[i] = s.slot; else V.waitNext[tail] = s.slot;
                tail = s.slot;
            }
            V.waitTail[i] = tail;
        }
    }
    unsigned char ins = 0;
    const int h = V.waitHead[i];
    if (h >= 0) {
        const int n = V.count[i], base = V.off[i];
        const int4 info = V.slotInfo[h];
        const DTmpl &T = V.tmpl[info.x];
        bool avail = true;
        const Tail tl = V.tail[i];
        if (n > 0) avail = tl.dis > tl.len + T.minGap;
        if (avail) {
            if (n >= V.off[i + 1] - base) {
                atomicOr(&V.ctrl->error, ERR_BUCKET_OVERFLOW);
            } else {
                const int p = base + n;
                V.kin[p] = make_double2(0.0, T.speed0);
                const int planIdx = V.planBeg[info.z];
                V.ids[p] = make_int4(h, info.x, info.y, V.planData[planIdx + 1]);
                V.nav[p] = make_int4(planIdx, -1, -1, INT_MAX);
                Tail nt;
                nt.dis = 0.0; nt.len = T.len; nt.speed = T.speed0; nt.pos = p; nt.prev = -1;
                V.tail[i] = nt;
                if (V.lcOn) lcResetSlot(V.lc.slot[h], info.z);
                if (n > 0) {
                    V.leader[p] = p - 1;
                    V.gap[p] = tl.dis - tl.len - 0.0;
                    if (V.lcOn) V.lc.slot[h].gap = tl.dis - tl.len - 0.0;
                    ins = 1;
                } else {
                    V.leader[p] = -1;
                    ins = 3;  // admitted to an empty lane: leader search runs in k_notify
                    if (own == 1) V.actList[cpar][atomicAdd(&V.ctrl->nAct[cpar], 1)] = i;
                }
                if (V.ctrl->nCustom > 0) {
                    const double cs = V.slotCust[h];
                    if (cs == cs) { V.cust[p] = cs; V.slotCust[h] = __longlong_as_double(-1LL); }
                }
                V.count[i] = n + 1;
                V.blk[h] = -1;
                if (own == 1) {
                    V.pos[h] = p;
                    atomicAdd(&V.ctrl->active, 1);
                    const int vi = atomicAdd(&V.ctrl->nVeh[cpar], 1);
                    if (vi < V.vehCap) V.vehList[cpar][vi] = make_int2(p, n == 0 ? (i | HEAD_BIT) : i);
                }
                int nx = V.waitNext[h];
                V.waitHead[i] = nx;
                if (nx < 0) V.waitTail[i] = -1;
            }
        }
    }
    V.inserted[i] = ins;
    }  // lanes
}

// ------------------------------------------------------------------------------------------
// Cross::notify for one laneLink, executed by a 16-lane tile (half a warp): one lane per cross.
// Engine::threadNotifyCross (engine.cpp:317-372) walks the link's crosses from the far end with
// one cursor shared by three sources in order -- (1) the end lane's last vehicle if it came out
// of this link, (2) the vehicles on the link front to back, (3) the start lane's first vehicle
// if it heads for this link and the link is green.  Every source keeps taking crosses while a
// condition that is monotone along the link holds, so the owner of a cross is simply the first
// source whose condition (same FP64 expression as the reference) holds for it.  Notify slots are
// epoch-stamped instead of cleared (Cross::clearNotify would sweep every cross every step).
//
// Both tiles of the warp call this together, each with its own link (`ll < 0`: none).  Every loop
// around a shuffle runs to the larger trip count of the two tiles and predicates its work, so all 32
// lanes meet at every warp primitive.
__device__ void notifyLink(const View &V, const int ll, const int tl, const int epoch) {
    int cb = 0, nc = 0, c2 = 0, base2 = 0;
    int tp = -1, hp = -1;   // the owners sources 1 and 3 offer (-1: the source is absent)
    double tdis = 0, vehDistance1 = 0, vehDistance3 = 0;
    if (ll >= 0) {
        cb = V.llCrossBeg[ll];
        nc = V.llCrossBeg[ll + 1] - cb;
    }
    const int linkDrv = V.nLanes + ll;
    if (nc > 0) {
        // source 1
        const Tail t = V.tail[V.llEndLane[ll]];
        if (t.pos >= 0 && t.prev == linkDrv) {
            tp = t.pos;
            tdis = t.dis;
            vehDistance1 = tdis - t.len;
        }
        // source 3
        const int sl = V.llStartLane[ll];
        if (V.count[sl] > 0) {
            const int h = V.off[sl];
            if (V.ids[h].w == linkDrv && V.rlAvail[V.llRoadLink[ll]]) {
                hp = h;
                vehDistance3 = V.drvLength[sl] - V.kin[h].x;
            }
        }
        c2 = V.count[linkDrv];
        base2 = V.off[linkDrv];
        if (tp < 0 && hp < 0 && c2 == 0) nc = 0;   // nothing to notify
    }
    if (nc == 0) c2 = 0;
    const int tb = threadIdx.x & 16;   // the tile's first lane: shuffles read inside the caller's tile
    const int ncMax = max(nc, __shfl_xor_sync(0xffffffffu, nc, 16));
    const int c2Max = max(c2, __shfl_xor_sync(0xffffffffu, c2, 16));
    const double L = nc > 0 ? V.drvLength[linkDrv] : 0.0;
    const int linkW = nc > 0 ? V.linkInfo[ll].w : 0;
    for (int k0 = 0; k0 < ncMax; k0 += 16) {
        const int k = k0 + tl;
        const bool valid = k < nc;
        const double dk = valid ? V.lcDist[cb + k] : 0.0;
        int owner = -1;
        double ndist = 0;
        if (valid && tp >= 0) {
            const double crossDistance = L - dk;
            if (crossDistance + vehDistance1 < 0) {
                owner = tp;
                ndist = -(tdis + crossDistance);
            }
        }
        for (int j0 = 0; j0 < c2Max; j0 += 16) {  // vehicles on the link, front to back
            double vj = 0, lj = 0;
            if (j0 + tl < c2) {
                vj = V.kin[base2 + j0 + tl].x;
                lj = V.tmpl[V.ids[base2 + j0 + tl].y].len;
            }
            const int m = min(16, c2Max - j0);
            for (int j = 0; j < m; ++j) {
                const double v = __shfl_sync(0xffffffffu, vj, tb + j);
                const double l = __shfl_sync(0xffffffffu, lj, tb + j);
                if (valid && owner < 0 && j0 + j < c2) {
                    bool take = true;
                    if (v > dk) take = (v - dk - l <= 0);
                    if (take) {
                        owner = base2 + j0 + j;
                        ndist = dk - v;
                    }
                }
            }
        }
        if (valid && owner < 0 && hp >= 0) {
            owner = hp;
            ndist = vehDistance3 + dk;
        }
        if (valid && owner >= 0) {
            Notify n;
            n.dist = ndist;
            n.pos = owner;
            n.epoch = epoch;
            foeTerms(V, n, linkW);
            V.notify[V.lcIdx[cb + k]] = n;
            // tell the crossing link which of ITS crosses now has a foe (k_control visits only those)
            const int peer = V.lcPeer[cb + k];
            const int foeLink = V.csLink[V.lcIdx[cb + k] ^ 1];
            const int bit = peer - V.llCrossBeg[foeLink];
            atomicOr(&V.foeMask[foeLink * V.maskWords + (bit >> 5)], 1u << (bit & 31));
        }
    }
}

// k_notify: two occupied drivables per warp, one per 16-lane tile.  A link handles itself; a lane
// triggers the (empty) links its tail vehicle came out of / its head vehicle heads for, so no empty
// link is swept.  Also runs the leader search of a vehicle admitted to an empty lane this step.
// Most laneLinks have at most 20 crosses and hold a few vehicles, so half a warp per link leaves
// fewer lanes idle, and a resident wave of tiles covers the whole list in about one pass.
__device__ __forceinline__ void phase_notify(const View &V, const int bid, const int nblk) {
    const int lane = threadIdx.x & 31, tile = lane >> 4, tl = lane & 15;
    const int warp = (bid * blockDim.x + threadIdx.x) >> 5;
    const int nWarps = (nblk * blockDim.x) >> 5;
    const int cpar = V.par;
    const int nAct = V.ctrl->nAct[cpar];
    const int epoch = V.ctrl->step + 1;
    for (int w0 = 2 * warp; w0 < nAct; w0 += 2 * nWarps) {  // trip count uniform per warp
        const int w = w0 + tile;
        int la = -1, lb = -1;   // the links this tile notifies
        if (w < nAct) {
            const int d = V.actList[cpar][w];
            if (d >= V.nLanes) {
                la = d - V.nLanes;
            } else if (V.count[d] > 0) {
                const int c = V.count[d], base = V.off[d];
                // with lane change the search already ran before the signals (k_lc_admitted) and the full leader
                // pass after scheduling (k_lc_leader) has the final word
                if ((V.inserted[d] & 2) && tl == 0 && !V.lcOn) {
                    const int4 idv = V.ids[base];
                    int ld = -1;
                    double g = 0;
                    headSearch(V, d, 0.0, idv.w, V.nav[base].x, V.tmpl[idv.y], d, ld, g);
                    V.leader[base] = ld;
                    if (ld >= 0) V.gap[base] = g;
                    if (V.lcOn && ld >= 0) V.lc.slot[idv.x].gap = g;
                }
                // the link the tail came out of, if it is empty now (otherwise it is on the list itself)
                const int prev = V.nav[base + c - 1].y;
                if (prev >= V.nLanes && V.count[prev] == 0 && (!V.owned || V.owned[prev] == 1)) la = prev - V.nLanes;
                // the link the head is about to take, if empty
                const int nx = V.ids[base].w;
                if (nx >= V.nLanes && V.count[nx] == 0 && nx - V.nLanes != la) lb = nx - V.nLanes;
                if (la < 0) { la = lb; lb = -1; }
            }
        }
        notifyLink(V, la, tl, epoch);
        if (__ballot_sync(0xffffffffu, lb >= 0)) notifyLink(V, lb, tl, epoch);
    }
    for (int w0 = 2 * warp; w0 < V.nBoundOut; w0 += 2 * nWarps) {  // sharded: source 1 may sit on a lane another rank owns
        const int w = w0 + tile;
        int l = -1;
        if (w < V.nBoundOut) {
            const Tail t = V.tail[V.boundOut[w]];
            if (t.pos >= 0 && t.prev >= V.nLanes && V.owned[t.prev] == 1 && V.count[t.prev] == 0) l = t.prev - V.nLanes;
        }
        notifyLink(V, l, tl, epoch);
    }
}

}  // namespace cfb
