// device_tlobs.cuh -- per-intersection and per-movement observations for a signal controller on the same GPU
// (DeviceSim::observeIntersections): each light's phase, and the queues and pressure of every roadLink ("movement").
// Kernel body only, written as a (View, block, grid) function, so that the emulated device (tests/device_sim_emu.cpp)
// runs the same code as device_sim.cu.  Nothing here is part of a step.
#pragma once

namespace cfb {

// The static tables (intObsLayout, device_layout.cuh) and the output columns.  A movement is a roadLink r (global
// index, intersections in file order, then the intersection's "roadLinks" in order); in_lanes(r) / out_lanes(r) are
// the distinct start / end lanes of its laneLinks, in_lanes(i) / out_lanes(i) their union over intersection i.
struct IntObsTable {
    int nTl;                            // non-virtual intersections
    int maxPhases;                      // row length of phasePressure
    const int *tl;                      // [nTl] their indices
    const int *inBeg, *inLane;          // per intersection: in_lanes(i) = inLane[inBeg[i] .. inBeg[i + 1])
    const int *outBeg, *outLane;        //                   out_lanes(i)
    const int *rlInBeg, *rlInLane;      // per roadLink:     in_lanes(r)
    const int *rlOutBeg, *rlOutLane;    //                   out_lanes(r)
    const int *rlLinkBeg;               //                   its laneLinks [rlLinkBeg[r], rlLinkBeg[r + 1])
    int *phase;                         // [nInter]
    double *remaining;                  // [nInter]
    int *pressure, *queue;              // [nInter]
    int *mvIn, *mvInWaiting, *mvOut, *mvInside, *mvPressure;   // [nRL]
    int *phasePressure;                 // [nInter * maxPhases]; entries past an intersection's phase count stay INT_MIN
    int *laneWait;                      // [nLanes] scratch: waiting vehicles of every lane that ends at a light
};
constexpr int TOBS_WARPS = 4;   // warps per block on the GPU (the emulated block is one warp)

// One warp per non-virtual intersection (grid-stride over them).  Every lane ends at one intersection, so each bucket
// is scanned once: its waiting vehicles by a ballot per 32 positions.  Then the lanes of the warp take the
// intersection's roadLinks, and after them its phases, 32 at a time; __syncwarp orders the warp's own stores of
// laneWait and mvPressure before the loops that read them.  Every loop that holds a warp primitive has a bound that
// is the same for the whole warp.
__device__ __forceinline__ void tobsFill(const View &V, const IntObsTable &T, int b, int nb) {
    const int lane = threadIdx.x & 31, wpb = blockDim.x >> 5;
    for (int t = b * wpb + (threadIdx.x >> 5); t < T.nTl; t += nb * wpb) {
        const int i = T.tl[t];
        int inCount = 0, queue = 0;
        for (int q = T.inBeg[i]; q < T.inBeg[i + 1]; ++q) {
            const int l = T.inLane[q], n = V.count[l], base = V.off[l];
            int w = 0;
            for (int k0 = 0; k0 < n; k0 += 32) {
                const int k = k0 + lane;
                w += __popc(__ballot_sync(0xffffffffu, k < n && isWaiting(V.kin[base + k].y)));
            }
            if (lane == 0) T.laneWait[l] = w;
            inCount += n;
            queue += w;
        }
        int outCount = 0;
        for (int q = T.outBeg[i] + lane; q < T.outBeg[i + 1]; q += 32) outCount += V.count[T.outLane[q]];
        for (int o = 16; o; o >>= 1) outCount += __shfl_xor_sync(0xffffffffu, outCount, o);
        __syncwarp();
        const int r0 = V.interRLBeg[i], r1 = V.interRLBeg[i + 1];
        for (int r = r0 + lane; r < r1; r += 32) {
            int in = 0, inW = 0, out = 0, inside = 0;
            for (int q = T.rlInBeg[r]; q < T.rlInBeg[r + 1]; ++q) {
                const int l = T.rlInLane[q];
                in += V.count[l];
                inW += T.laneWait[l];
            }
            for (int q = T.rlOutBeg[r]; q < T.rlOutBeg[r + 1]; ++q) out += V.count[T.rlOutLane[q]];
            for (int ll = T.rlLinkBeg[r]; ll < T.rlLinkBeg[r + 1]; ++ll) inside += V.count[V.nLanes + ll];
            T.mvIn[r] = in;
            T.mvInWaiting[r] = inW;
            T.mvOut[r] = out;
            T.mvInside[r] = inside;
            T.mvPressure[r] = in - out;
        }
        __syncwarp();
        const int pb = V.interPhaseBeg[i], nph = V.interPhaseBeg[i + 1] - pb;
        for (int k = lane; k < nph; k += 32) {
            const unsigned char *avail = V.phaseAvail + V.phaseAvailBeg[pb + k];
            int s = 0;
            for (int r = r0; r < r1; ++r)
                if (avail[r - r0]) s += T.mvPressure[r];
            T.phasePressure[(size_t) i * T.maxPhases + k] = s;
        }
        if (lane == 0) {
            T.phase[i] = V.curPhase[i];
            T.remaining[i] = V.remain[i];
            T.pressure[i] = inCount - outCount;
            T.queue[i] = queue;
        }
    }
}

}  // namespace cfb
