// device_vehobs.cuh -- per-vehicle observations and actions for a consumer on the same GPU: the table of every running
// vehicle (DeviceSim::observeVehicles), what lies ahead of each row (DeviceSim::observeVehicleContext) and the batched
// custom speed (DeviceSim::setCustomSpeedsFromDevice).  Kernel
// bodies only, written as (View, block, grid) functions, so that the emulated device (tests/device_sim_emu.cpp) runs the
// same code as device_sim.cu.  Nothing here is part of a step.
#pragma once

namespace cfb {

// The observation table, drivable-major: the rows of drivable d are [drvBegin[d], drvBegin[d + 1]), in list order (front
// first, Drivable::getVehicles).  Rows at and beyond *count are padding with slot -1.
struct VehObsTable {
    int *slot, *priority, *drivable;
    double *distance, *speed;
    unsigned char *shadow;     // 1: a lane-change shadow (LcSlot.type == 2, Vehicle::isReal() == false)
    int *drvBegin;             // nDrv + 1 entries
    int *count;                // = drvBegin[nDrv]
    int *tileSum;              // vehicles per tile of VOBS_TILE drivables (written by the first launch)
    int *prevCount;            // *count before this refresh: rows [count, prevCount) are set back to padding
};
constexpr int VOBS_TILE = 256;   // drivables per tile = threads per block on the GPU (a 32-lane block on the emulated warp)

// Exclusive prefix sum of x over the block; *total = the block's sum.  blockDim.x: a multiple of 32, at most VOBS_TILE.
__device__ __forceinline__ int vobsBlockScan(int x, int *total) {
    __shared__ int sWarp[VOBS_TILE / 32];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = blockDim.x >> 5;
    int incl = x;
    for (int o = 1; o < 32; o <<= 1) {
        const int y = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += y;
    }
    if (lane == 31) sWarp[w] = incl;
    __syncthreads();
    int before = 0, all = 0;
    for (int k = 0; k < nw; ++k) {
        const int s = sWarp[k];
        if (k < w) before += s;
        all += s;
    }
    __syncthreads();   // (sWarp is reused by the next scan)
    *total = all;
    return before + incl - x;
}

// First launch: the vehicle count of every tile of drivables.  Block 0 keeps the row count of the previous refresh.
__device__ __forceinline__ void vobsTileSums(const View &V, const VehObsTable &T, int b) {
    const int d = b * blockDim.x + threadIdx.x;
    int all = 0;
    vobsBlockScan(d < V.nDrv ? V.count[d] : 0, &all);
    if (threadIdx.x == 0) {
        T.tileSum[b] = all;
        if (b == 0) *T.prevCount = *T.count;
    }
}

// Second launch: the tile's row offsets (the tiles before it + a block scan), then one warp per drivable copies the
// bucket in list order; finally the rows the previous refresh filled beyond the new count become padding again.
__device__ __forceinline__ void vobsFill(const View &V, const VehObsTable &T, int b, int nb) {
    __shared__ int sBeg[VOBS_TILE], sCnt[VOBS_TILE];
    __shared__ int sOff, sAll;
    if (threadIdx.x < 32) {
        int before = 0, all = 0;
        for (int k = threadIdx.x; k < nb; k += 32) {
            const int s = T.tileSum[k];
            all += s;
            if (k < b) before += s;
        }
        for (int o = 16; o; o >>= 1) {
            before += __shfl_xor_sync(0xffffffffu, before, o);
            all += __shfl_xor_sync(0xffffffffu, all, o);
        }
        if (threadIdx.x == 0) { sOff = before; sAll = all; }
    }
    __syncthreads();
    const int d = b * blockDim.x + threadIdx.x;
    const int c = d < V.nDrv ? V.count[d] : 0;
    int tile = 0;
    const int beg = sOff + vobsBlockScan(c, &tile);
    sBeg[threadIdx.x] = beg;
    sCnt[threadIdx.x] = c;
    if (d < V.nDrv) T.drvBegin[d] = beg;
    const int total = sAll;
    if (b == nb - 1 && threadIdx.x == 0) {
        T.drvBegin[V.nDrv] = total;
        *T.count = total;
    }
    __syncthreads();
    const int lane = threadIdx.x & 31, nw = blockDim.x >> 5;
    for (int k = threadIdx.x >> 5; k < (int) blockDim.x; k += nw) {
        const int dd = b * blockDim.x + k;
        if (dd >= V.nDrv) break;
        const int n = sCnt[k], r0 = sBeg[k], base = V.off[dd];
        for (int j = lane; j < n; j += 32) {
            const int p = base + j, r = r0 + j;
            const int4 id = V.ids[p];
            const double2 kk = V.kin[p];
            T.slot[r] = id.x;
            T.priority[r] = id.z;
            T.drivable[r] = dd;
            T.distance[r] = kk.x;
            T.speed[r] = kk.y;
            T.shadow[r] = (V.lcOn && V.lc.slot[id.x].type == 2) ? 1 : 0;
        }
    }
    const int prev = *T.prevCount;
    for (int r = total + b * blockDim.x + threadIdx.x; r < prev; r += nb * blockDim.x) T.slot[r] = -1;
}

// What lies ahead of every row of a VehObsTable, filled right after the table in the same refresh
// (DeviceSim::observeVehicleContext).  Capacity rows each; rows at and beyond *T.count hold the padding values
// leader -1, gap +inf, nextDrivable -1, signal -1.
struct VehCtxTable {
    int *leader;               // row of Vehicle::getLeader (View::leader), -1 none
    double *gap;               // ControllerInfo::gap to it, +inf without a leader
    int *nextDrivable;         // Router::getNextDrivable: ids[p].w (PLAN_END / PLAN_DEAD where there is none)
    signed char *signal;       // a lane row heading for a laneLink: RoadLink::isAvailable of its roadLink (0 / 1); else -1
    int *mark;                 // two entries: rows filled by the previous context refresh, read from mark[par] ...
    int par;                   // ... and this refresh's row count written to mark[par ^ 1]
};

// One thread per row, grid-stride.  Row r of drivable d is position off[d] + (r - drvBegin[d]).  A leader one position
// ahead on the same drivable is the row before; any other leader (the next lane, or an overlapping laneLink from the
// same start lane, vehicle.cpp:157-190) is found by a binary search of View::off for its drivable.  The rows the
// previous context refresh filled beyond the new count become padding again: that mark is kept here, apart from the
// table's prevCount, which a refresh without the context also moves.
__device__ __forceinline__ void vctxFill(const View &V, const VehObsTable &T, const VehCtxTable &C, int b, int nb) {
    const int n = *T.count, mark = C.mark[C.par];
    if (b == 0 && threadIdx.x == 0) C.mark[C.par ^ 1] = n;
    const int end = n > mark ? n : mark;
    for (int r = b * blockDim.x + threadIdx.x; r < end; r += nb * blockDim.x) {
        if (r >= n) {
            C.leader[r] = -1;
            C.gap[r] = (double) INFINITY;
            C.nextDrivable[r] = -1;
            C.signal[r] = -1;
            continue;
        }
        const int d = T.drivable[r], k = r - T.drvBegin[d], p = V.off[d] + k;
        const int lp = V.leader[p];
        int lr = -1;
        double g = (double) INFINITY;
        if (lp >= 0) {
            if (k > 0 && lp == p - 1) {
                lr = r - 1;
            } else {
                int lo = 0, hi = V.nDrv - 1;   // the last drivable whose bucket starts at or before lp
                while (lo < hi) {
                    const int mid = (lo + hi + 1) >> 1;
                    if (V.off[mid] <= lp) lo = mid; else hi = mid - 1;
                }
                lr = T.drvBegin[lo] + (lp - V.off[lo]);
            }
            g = V.lcOn ? V.lc.slot[V.ids[p].x].gap : V.gap[p];
        }
        const int nd = V.ids[p].w;
        signed char sig = -1;
        if (d < V.nLanes && nd >= V.nLanes) sig = (signed char) roadLinkAvailable(V, V.llRoadLink[nd - V.nLanes]);
        C.leader[r] = lr;
        C.gap[r] = g;
        C.nextDrivable[r] = nd;
        C.signal[r] = sig;
    }
}

// Vehicle::setCustomSpeed (vehicle.h:128) for every entry i with slot[i] >= 0, one thread per entry.  (slot, priority)
// must still name the same running vehicle -- a vehicle that left has pos -1, a slot handed to a later vehicle holds
// another priority -- else ERR_VEHICLE_STALE.  A slot given twice in one call raises ERR_VEHICLE_DUPLICATE (parallel
// writes would keep one of the two values by timing): `stamp` holds, per slot, the last call that named it.  A cell
// that held no request yet (NaN) counts one more outstanding request, as DeviceSim::setCustomSpeed counts it.
__device__ __forceinline__ void vspeedApply(const View &V, const int *slot, const int *priority, const double *speed, int n,
                                            int *stamp, int slotCap, int call, int b, int nb) {
    for (int i = b * blockDim.x + threadIdx.x; i < n; i += nb * blockDim.x) {
        const int s = slot[i];
        if (s < 0) continue;
        const int p = s < slotCap ? V.pos[s] : -1;
        if (p < 0 || V.ids[p].x != s || V.ids[p].z != priority[i]) {
            atomicOr(&V.ctrl->error, ERR_VEHICLE_STALE);
            continue;
        }
        if (atomicExch(&stamp[s], call) == call) {
            atomicOr(&V.ctrl->error, ERR_VEHICLE_DUPLICATE);
            continue;
        }
        const unsigned long long old = atomicExch(reinterpret_cast<unsigned long long *>(V.cust + p),
                                                  (unsigned long long) __double_as_longlong(speed[i]));
        const double was = __longlong_as_double((long long) old);
        if (was != was) atomicAdd(&V.ctrl->nCustom, 1);
    }
}

}  // namespace cfb
