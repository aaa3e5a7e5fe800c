// H100 (sm_90a) step engine: device-resident vehicle state + the kernel sequence that replaces
// the reference's barrier-delimited thread phases (Engine::nextStep, engine.cpp:566-594).
//
// Data layout (see DESIGN.md §3).  Vehicles do not live in a slot-indexed pool; they live in
// *lane buckets*: every drivable (lane or laneLink) owns a fixed-capacity, contiguous range of
// "positions" [off[d], off[d+1]) in a set of structure-of-arrays, and the vehicles on it occupy
// the first count[d] positions in the reference's list order (front -> back, FIFO with
// mid-list removal).  A vehicle's list predecessor -- its leader -- is therefore the previous
// position, every per-vehicle phase reads and writes its fields with unit stride inside a
// warp, and the reference's std::list erase / std::sort+append (engine.cpp:282-315, :477-494)
// becomes a warp-scan compaction plus a per-bucket rank sort of the few entrants.
//
//   kin[p]   double2 {dis, speed}            gap[p] double      leader[p] int (position, -1)
//   ids[p]   int4 {slot, tmpl, priority, nextDrivable}      (next drivable on the plan, cached)
//   nav[p]   int4 {planIdx, prevDrivable, blocker(slot), enterLaneLinkTime}   (planIdx: absolute index into planData)
//   tail[d]  {dis, len, speed, position, prevDrivable} of the last vehicle of every drivable (position -1 = empty):
//            the one record other drivables' vehicles look at (leader search, Lane::canEnter, notify source 1)
//
// Work lists.  At ~1e5 vehicles only ~8 k of the 43 k drivables of the 30x30 grid are occupied,
// so no kernel sweeps the topology: k_move leaves behind the list of occupied drivables and the
// list of occupied positions (double-buffered on step parity), k_ingest appends what it admits,
// and every phase is a grid-stride loop over one of those lists with a fixed, SM-count-sized
// grid (CUDA-graph friendly, no host knowledge of the population needed).
//
// Kernel sequence per step (all FP64, -fmad=false so every operation rounds exactly like the
// reference's SSE2 build; expression shapes follow vehicle.cpp verbatim):
//   k_ingest   P0-P2  waiting-queue append, Lane::available admission, light -> roadLink mask
//   k_notify   P3     Cross::notify, half a warp (16-lane tile) per occupied drivable, one lane per cross
//   k_control  P4     getNextSpeed / vehicleControl / setDeltaDistance, thread per vehicle
//   k_move     P5-P6  16-lane tile per drivable: bucket compaction (ballot scan), entrant rank-sort + append, commit,
//                     finished ring, next step's work lists
//   k_leader   P7-P8  leader/gap rebuild (warp shuffle), cross-drivable head search, blocker drop,
//                     TrafficLight::passTime
#include <cuda_runtime.h>
#include <cooperative_groups.h>

#include <algorithm>
#include <chrono>
#include <climits>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <stdexcept>
#include <string>
#include <vector>

#include "device_sim.h"
#include "partition.h"
#include "shard.h"

namespace cfb {
namespace cg = cooperative_groups;

#define CFB_CUDA(x)                                                                                  \
    do {                                                                                             \
        cudaError_t e_ = (x);                                                                        \
        if (e_ != cudaSuccess)                                                                       \
            throw std::runtime_error(std::string("cityflow_b200 CUDA error: ") + cudaGetErrorString(e_) + \
                                     " at " + __FILE__ + ":" + std::to_string(__LINE__));           \
    } while (0)

}  // namespace cfb
#include "device_view.cuh"
#include "device_image.cuh"
#include "device_layout.cuh"
#include "device_phases_a.cuh"
namespace cfb {
static_assert(DeviceSim::LC_MAX_CANDIDATES == LC_MAX_CAND, "the host lends one spare slot per schedulable candidate");
// Programmatic dependent launch: the five step kernels are chained with programmatic stream serialisation, so the next
// kernel's launch, block scheduling and prologue overlap the tail of the previous one (each kernel is latency-bound and
// drains unevenly).  `griddepcontrol.wait` returns once the whole previous grid has completed and its memory operations
// are visible -- the data dependence between the phases is unchanged -- and `launch_dependents` right behind it lets the
// kernel after this one be scheduled as early as possible.  Both are no-ops in a launch without the attribute.
__device__ __forceinline__ void pdlEnter() {
    asm volatile("griddepcontrol.wait;" ::: "memory");
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
}
__global__ void __launch_bounds__(256) k_ingest(View V) { pdlEnter(); phase_ingest(V, blockIdx.x, gridDim.x); }
__global__ void __launch_bounds__(256) k_notify(View V) { pdlEnter(); phase_notify(V, blockIdx.x, gridDim.x); }

}  // namespace cfb
#include "device_control.cuh"
namespace cfb {

__global__ void __launch_bounds__(256, 4) k_control(View V) { pdlEnter(); phase_control(V, blockIdx.x, gridDim.x); }

}  // namespace cfb
#include "device_phases_b.cuh"
namespace cfb {
__global__ void __launch_bounds__(256) k_move(View V) { pdlEnter(); phase_move(V, blockIdx.x, gridDim.x); }
__global__ void __launch_bounds__(256) k_leader(View V) { pdlEnter(); phase_leader(V, blockIdx.x, gridDim.x); }

// ------------------------------------------------------------------------------------------
// k_step: the whole step as ONE cooperative kernel -- the five phases separated by grid-wide
// barriers instead of kernel boundaries (each boundary costs a launch + drain + ramp of several
// microseconds, comparable to the phases themselves at ~1e5 vehicles).  One resident wave of
// 256-thread blocks; every phase is a grid-stride loop over its work list.
__global__ void __launch_bounds__(256, 4) k_step(View V) {
    cg::grid_group grid = cg::this_grid();
    phase_ingest(V, blockIdx.x, gridDim.x);
    grid.sync();
    phase_notify(V, blockIdx.x, gridDim.x);
    grid.sync();
    phase_control(V, blockIdx.x, gridDim.x);
    grid.sync();
    phase_move(V, blockIdx.x, gridDim.x);
    grid.sync();
    phase_leader(V, blockIdx.x, gridDim.x);
}

// ------------------------------------------------------------------------------------------
// Sharded mode: the seam records and both of their transports (device_shard.cuh).
}  // namespace cfb
#include "device_shard.cuh"
namespace cfb {

__global__ void k_mask_counts(View V, int *out) {  // out[0] = vehicles this rank accounts for, out[1+l] = owned lane counts
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i == 0) out[0] = V.ctrl->active;
    if (i < V.nLanes) out[1 + i] = (!V.owned || V.owned[i] == 1) ? V.count[i] : 0;
}
__global__ void k_mask_waiting(View V, const int *waiting, int *out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < V.nLanes) out[i] = (!V.owned || V.owned[i] == 1) ? waiting[i] : 0;
}

// ------------------------------------------------------------------------------------------
// Observation kernels
__global__ void __launch_bounds__(256) k_lane_waiting(View V, int *out) {  // engine.cpp:636-648
    const int d = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (d >= V.nLanes) return;
    const int n = V.count[d], base = V.off[d];
    int c = 0;
    for (int k = lane; k < n; k += 32) c += isWaiting(V.kin[base + k].y);
    for (int o = 16; o; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
    if (lane == 0) out[d] = c;
}

__global__ void k_set_phases(View V, const int *src) {  // TrafficLight::setPhase trafficlight.cpp:39-41, all lights at once
    const int in = blockIdx.x * blockDim.x + threadIdx.x;
    if (in >= V.nInter || V.interVirtual[in]) return;
    const int p = src[in], nph = V.interPhaseBeg[in + 1] - V.interPhaseBeg[in];
    if (p >= 0 && p < nph) V.curPhase[in] = p;
    else atomicOr(&V.ctrl->error, ERR_PHASE_RANGE);
}

// Per-lane observation vector for consumers on the same GPU (RL policies): list length
// (engine.cpp:628-634), vehicles slower than 0.1 m/s (:636-648) and the sum of speeds, one warp per lane.
__global__ void __launch_bounds__(256) k_lane_obs(View V, int *cnt, int *wait, double *speedSum) {
    const int d = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (d >= V.nLanes) return;
    const int n = V.count[d], base = V.off[d];
    int c = 0;
    double s = 0.0;
    for (int k = lane; k < n; k += 32) {
        const double v = V.kin[base + k].y;
        c += isWaiting(v);
        s += v;
    }
    for (int o = 16; o; o >>= 1) {
        c += __shfl_xor_sync(0xffffffffu, c, o);
        s += __shfl_xor_sync(0xffffffffu, s, o);
    }
    if (lane == 0) {
        cnt[d] = n;
        wait[d] = c;
        speedSum[d] = s;
    }
}

__global__ void __launch_bounds__(256) k_gather_running(View V, SpeedRec *out, int *cursor, int cap) {
    const int d = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (d >= V.nDrv) return;
    const int n = V.count[d], base = V.off[d];
    if (n == 0) return;
    int start = 0;
    if (lane == 0) start = atomicAdd(cursor, n);
    start = __shfl_sync(0xffffffffu, start, 0);
    for (int k = lane; k < n; k += 32) {
        if (start + k < cap) {
            SpeedRec r;
            r.slot = V.ids[base + k].x;
            r.drivable = d;
            const double2 kk = V.kin[base + k];
            r.speed = kk.y;
            r.dis = kk.x;
            out[start + k] = r;
        }
    }
}

}  // namespace cfb
#include "device_vehobs.cuh"
namespace cfb {
// The per-vehicle table (device_vehobs.cuh): tile sums, then offsets + bucket copies.  And the batched custom speed.
__global__ void __launch_bounds__(VOBS_TILE) k_vobs_sums(View V, VehObsTable T) { vobsTileSums(V, T, blockIdx.x); }
__global__ void __launch_bounds__(VOBS_TILE) k_vobs_fill(View V, VehObsTable T) { vobsFill(V, T, blockIdx.x, gridDim.x); }
// What lies ahead of every row (leader, gap, next drivable, light), one thread per row after the two above.
__global__ void __launch_bounds__(256) k_vctx(View V, VehObsTable T, VehCtxTable C) { vctxFill(V, T, C, blockIdx.x, gridDim.x); }
__global__ void __launch_bounds__(256) k_vspeed(View V, const int *slot, const int *priority, const double *speed, int n,
                                                int *stamp, int slotCap, int call) {
    vspeedApply(V, slot, priority, speed, n, stamp, slotCap, call, blockIdx.x, gridDim.x);
}

}  // namespace cfb
#include "device_tlobs.cuh"
namespace cfb {
// The intersection observations (device_tlobs.cuh): one warp per signalised intersection.
__global__ void __launch_bounds__(TOBS_WARPS * 32) k_tobs(View V, IntObsTable T) { tobsFill(V, T, blockIdx.x, gridDim.x); }

__global__ void k_lane_slots(View V, int *out, const int *laneBeg) {
    const int d = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (d >= V.nLanes) return;
    const int n = V.count[d], base = V.off[d], o = laneBeg[d];
    for (int k = lane; k < n; k += 32) out[o + k] = V.ids[base + k].x;
}

// ------------------------------------------------------------------------------------------
// Host side
template <class T>
struct DevBuf {
    T *p = nullptr;
    size_t n = 0;
    void alloc(size_t count) {
        release();
        n = count;
        if (count) CFB_CUDA(cudaMalloc(&p, count * sizeof(T)));
    }
    void upload(const std::vector<T> &v) {
        alloc(v.size());
        if (!v.empty()) CFB_CUDA(cudaMemcpy(p, v.data(), v.size() * sizeof(T), cudaMemcpyHostToDevice));
    }
    void fill(int byte) {
        if (n) CFB_CUDA(cudaMemset(p, byte, n * sizeof(T)));
    }
    void release() {
        if (p) cudaFree(p);
        p = nullptr;
        n = 0;
    }
    ~DevBuf() { release(); }
};

// The engine's stream is non-blocking, so it is NOT ordered against the legacy default stream that
// plain cudaMemcpy / cudaMemset run on (and those may return before the device side is done:
// memsets, device-to-device copies, staged pageable uploads).  Every function that writes device
// state that way ends with this barrier, before anything can be enqueued on the engine's stream.
static void legacySync() { CFB_CUDA(cudaStreamSynchronize(cudaStreamLegacy)); }
static void applyFills(const std::vector<Fill> &fills) {
    for (const Fill &f : fills) if (f.bytes) CFB_CUDA(cudaMemset(f.p, f.byte, f.bytes));
}

// A step kernel, optionally with programmatic stream serialisation (see pdlEnter()).
template <class... A>
static void launchPdl(void (*k)(A...), int grid, int block, cudaStream_t s, bool pdl, A... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(grid);
    cfg.blockDim = dim3(block);
    cfg.dynamicSmemBytes = 0;
    cfg.stream = s;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = at;
    cfg.numAttrs = pdl ? 1 : 0;
    CFB_CUDA(cudaLaunchKernelEx(&cfg, k, args...));
}

// A step replayed as ONE CUDA graph per list parity.  Re-launching an executable graph whose previous launch has not
// finished makes the driver wait on the host (observed: ~1 ms per step), so each parity has a small ring of instances of
// the same graph: the host may run 2 * GRING steps ahead of the device before a step falls back to plain launches.
struct GraphRing {
    static constexpr int GRING = 4;
    cudaGraph_t tmpl[2] = {nullptr, nullptr};   // the captured step, per parity
    cudaGraphExec_t exec[2][GRING] = {};
    cudaEvent_t done[2][GRING] = {};
    static int slot(long long steps) { return (int) ((steps >> 1) % GRING); }   // the instance of the step after `steps`
    bool instantiate(int par, int r) { return cudaGraphInstantiate(&exec[par][r], tmpl[par], 0) == cudaSuccess; }
    // the instance's last launch has not finished
    bool busy(int par, int r) const { return done[par][r] && cudaEventQuery(done[par][r]) != cudaSuccess; }
    void launch(int par, int r, cudaStream_t s) {
        if (!done[par][r]) CFB_CUDA(cudaEventCreateWithFlags(&done[par][r], cudaEventDisableTiming));
        CFB_CUDA(cudaGraphLaunch(exec[par][r], s));
        CFB_CUDA(cudaEventRecord(done[par][r], s));
    }
    void drop(cudaStream_t s) {
        for (int k = 0; k < 2; ++k) {
            for (int r = 0; r < GRING; ++r)
                if (exec[k][r]) { cudaStreamSynchronize(s); cudaGraphExecDestroy(exec[k][r]); exec[k][r] = nullptr; }
            if (tmpl[k]) { cudaGraphDestroy(tmpl[k]); tmpl[k] = nullptr; }
        }
    }
    void release(cudaStream_t s) {
        drop(s);
        for (auto &row : done)
            for (cudaEvent_t &e : row) if (e) cudaEventDestroy(e);
    }
};

struct DeviceSim::Impl {
    DeviceSimOptions opt;
    View V{};
    cudaStream_t stream = nullptr;
    int P = 0;
    DeviceLayout L;                   // host copy of the static tables (device_layout.cuh)
    // static
    DevBuf<double> drvLength, drvMaxSpeed, lcDist, phaseTime;
    DevBuf<int> off, laneOutBeg, laneOutLinks, llStartLane, llEndLane, llRoadLink, llCrossBeg, lcIdx, csLink,
        interPhaseBeg, interRLBeg, phaseAvailBeg, rlInter, planBeg, planData;
    DevBuf<unsigned char> phaseAvail, interVirtual;
    DevBuf<DTmpl> tmpl;
    // dynamic
    DevBuf<double2> kin, nkin, mkin;
    DevBuf<double> gap, remain, cust, slotCust;
    DevBuf<int> leader, count, pos, waitHead, waitTail, waitNext, curPhase, entCnt, ent, scratchI;
    DevBuf<int2> finSlots, vehList0, vehList1;
    DevBuf<int> act0, act1, extra, lcPeer, blk, delStep, boundOut, boundIn;
    DevBuf<unsigned char> owned;
    DevBuf<int> ingBuf;
    DevBuf<TailMsg> tailSend, tailRecv;
    DevBuf<MoverMsg> moverSend, moverRecv;
    DevBuf<int2> blkUpd, blkAll;
    std::vector<int> outBeg, inBeg;
    std::vector<unsigned char> ownedHost;
    int shardRank = 0, shardWorld = 1;
    GraphRing shardGraphs;       // the whole sharded step (kernels + NCCL groups)
    bool shardGraphOk = true;
    DevBuf<int> shardScratch;
    DevBuf<unsigned char> finGather;
    // peer-memory transport (device_shard.cuh)
    DevBuf<unsigned char> arena;
    DevBuf<ShardPeer> peers;
    DevBuf<int> p2pInts;              // nbr | outPeer | outDst | inPeer | inDst | ticket[2]
    ShardP2P S{};
    bool p2p = false;
    bool shardSplit = false;          // CITYFLOW_B200_SHARD_SPLIT=1: separate send / receive kernels (also used for the per-phase timing)
    bool arenaShared = false;         // mapped by other PROCESSES (as opposed to the in-process loop-back group)
    std::vector<std::vector<int>> bsize;   // bsize[a][b] = lanes rank a feeds and rank b owns
    static constexpr int SHARD_SLOT_CAP = 1 << 22;   // slot-indexed arrays are fixed once peers have mapped delStep
    struct ArenaLayout { size_t flags, delStep, blkIn, moverIn, tailIn, total; };
    static ArenaLayout arenaLayout(int world, int nIn, int nOut) {
        auto up = [](size_t x) { return (x + 255) & ~(size_t) 255; };
        ArenaLayout L;
        L.flags = 0;
        L.delStep = up((size_t) SHARD_FLAG_KINDS * world * sizeof(int));
        L.blkIn = L.delStep + up((size_t) SHARD_SLOT_CAP * sizeof(int));
        L.moverIn = L.blkIn + up((size_t) 2 * world * (1 + BLK_IN_CAP) * sizeof(int2));
        L.tailIn = L.moverIn + up((size_t) 2 * std::max(nIn, 1) * sizeof(MoverMsg));
        L.total = L.tailIn + up((size_t) 2 * std::max(nOut, 1) * sizeof(TailMsg));
        return L;
    }
    int nInOf(int q) const { int n = 0; for (int p = 0; p < shardWorld; ++p) n += bsize[p][q]; return n; }
    int nOutOf(int q) const { int n = 0; for (int p = 0; p < shardWorld; ++p) n += bsize[q][p]; return n; }
    DevBuf<Tail> tail;
    DevBuf<unsigned> dbgCyc, dbgPath;
    DevBuf<int4> linkInfo;
    DevBuf<unsigned> foeMask;
    DevBuf<int4> ids, nav, slotInfo, mids, mnav;
    DevBuf<int2> nbuf;
    DevBuf<unsigned char> inserted, rlAvail;
    DevBuf<Notify> notify;
    DevBuf<Ctrl> ctrl;
    DevBuf<SpawnRec> spawn;
    DevBuf<SpeedRec> speedOut;
    int spawnCap = 0;
    // pinned staging
    static constexpr int RING = 64;
    SpawnRec *hSpawn[RING] = {};
    int hSpawnCap[RING] = {};
    cudaEvent_t spawnDone[RING] = {};
    int ringIdx = 0;
    std::vector<int> hPhase;            // authoritative phases in rlTrafficLight mode (set_tl_phase)
    int *hPhaseRing[RING] = {};         // pinned staging, one per ring slot
    bool phaseDirty = false;
    Ctrl *hCtrl = nullptr;  // pinned readback
    volatile int *hMirror = nullptr;   // pinned + mapped: {epoch, active, error, ties}, written by k_leader (device_phases_b.cuh)
    long long epochHost = 0;           // steps enqueued since the engine was created (what hMirror[0] will reach)
    int *hInts = nullptr;   // pinned readback (lanes)
    size_t hIntsCap = 0;
    // timing
    bool timing = false;
    cudaEvent_t ev[6] = {};
    DevBuf<int> obsI;                  // observeOnDevice(): [count | waiting] per lane
    DevBuf<double> obsD;               //                    speed sum per lane
    cudaEvent_t obsReady = nullptr, obsConsumed = nullptr;
    cudaEvent_t actReady = nullptr, actTaken = nullptr;   // setPhasesFromDevice()
    bool hPhaseStale = false;          // the device copy is newer than hPhase (phases were set on the device)
    DevBuf<int> vobsI;                 // observeVehicles(): slot | priority | drivable (capacity rows each), drivable begin,
                                       //   count, previous count, tile sums
    DevBuf<double> vobsD;              //                    distance | speed
    DevBuf<unsigned char> vobsShadow;
    VehObsTable vobs{};
    int vobsTiles = 0;
    cudaEvent_t vobsReady = nullptr, vobsConsumed = nullptr;
    DevBuf<int> vctxI;                 // observeVehicleContext(): leader | next drivable (capacity rows each), mark (2)
    DevBuf<double> vctxGap;
    DevBuf<signed char> vctxSignal;
    VehCtxTable vctx{};
    DevBuf<int> speedStamp;            // setCustomSpeedsFromDevice(): per slot, the last call that named it
    int speedCall = 0;
    cudaEvent_t speedReady = nullptr, speedTaken = nullptr;
    DevBuf<int> tobsStatic;            // observeIntersections(): the kernel's tables (IntObsLayout::ints)
    DevBuf<int> tobsI;                 //   phase | pressure | queue | 5 movement columns | phase pressure | lane scratch |
                                       //   movement begin | movement intersection | phase count
    DevBuf<double> tobsD;              //   phase remaining
    DevBuf<unsigned char> tobsMv;      //   phase movements
    IntObsTable tobs{};
    DeviceIntersectionObs tobsOut{};
    int *hPhaseFlush[RING] = {};       //   pinned staging of the setPhase calls a refresh sends up, one per ring slot ...
    cudaEvent_t phaseFlushDone[RING] = {};   // ... free again once its copy has run
    int phaseFlushIdx = 0;
    cudaEvent_t tobsReady = nullptr, tobsConsumed = nullptr;
    std::vector<cudaEvent_t> stepEv;   // timed-step brackets (bench)
    size_t stepEvUsed = 0;
    DevBuf<unsigned char> flushBuf;
    KernelTimes times;
    cudaEvent_t shardEv[SHARD_PHASES + 1] = {};
    double shardMs[SHARD_PHASES] = {};
    long long shardTimedSteps = 0;

    DevBuf<LcSlot> lcSlot;
    DevBuf<int> lcLaneRoad, lcRouteLastRoad, lcScratch;
    bool lcSerial = false;            // CITYFLOW_B200_LC_SERIAL=1: scheduling / control tail in one thread each (debugging)
    DevBuf<int> lcSegIdx, lcPosDrv, lcSegBeg, lcLaneIdx, lcLaneRoadN, lcPlanRoute, lcPlanRoadPos, lcLanePlanRoad,
        lcLanePlanBeg, lcLanePlanId, lcCand, lcInvolved, lcSpare, lcPrio;
    DevBuf<double> lcSegStart, lcLaneWidth;
    DevBuf<int2> lcShadowLog;
    DevBuf<LcCtrl> lcCtrl;
    LcCtrl *hLcCtrl = nullptr;        // pinned readback
    int lcSpareCap = 0;
    int slotCap = 0;
    int numSMs = 132;   // H100 SXM; read from the device at construction
    int gridNotify = 0, gridMove = 0, gridLeader = 0, gridControl = 0;
    bool mirrorStale = false;   // something other than a step changed active / error (reset, restore, a setter): read the device
    bool usePdl = true;   // CITYFLOW_B200_NO_PDL=1: plain stream order between the step kernels
    bool useGraph = true, useCoop = false;   // cooperative k_step measured slower (DESIGN.md §4)
    GraphRing graphs;        // the five kernels of a single-GPU step
    int gridStep = 0;
    int lastForm[4] = {};   // {graph, pdl, coop, mirror} of the last step() (launchForm)

    // The graphs bake in the View's pointers: every change of a device buffer or table drops them (rebuilt on use).
    void invalidateGraphs() {
        graphs.drop(stream);
        shardGraphs.drop(stream);
    }
    // Grids of the list-driven step kernels: one resident wave each (occupancy x #SM blocks, grid-stride loops inside).
    void ensureGrids() {
        if (gridNotify) return;
        int b = 0;
        CFB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&b, k_notify, 256, 0)); gridNotify = std::max(b, 1) * numSMs;
        CFB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&b, k_move, 256, 0)); gridMove = std::max(b, 1) * numSMs;
        CFB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&b, k_leader, 256, 0)); gridLeader = std::max(b, 1) * numSMs;
        CFB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&b, k_control, 256, 0)); gridControl = std::max(b, 1) * numSMs;
    }
    // The five step kernels, each with its one launch description.  k_ingest covers its lane / roadLink lists (a rank of a
    // sharded run: only those it ingests into) and follows a copy, never a kernel, so it is never chained by PDL; `pdl`
    // chains the others behind the kernel before them (see pdlEnter()).
    enum StepKernel { INGEST, NOTIFY, CONTROL, MOVE, LEADER };
    void launchStep(StepKernel k, bool pdl) {
        static void (*const kernel[5])(View) = {k_ingest, k_notify, k_control, k_move, k_leader};
        ensureGrids();
        const int TPB = 256;
        const int ingest = (V.ingLanes ? std::max(std::max(V.nIngLanes, V.nIngRL), V.nIngLinks * V.maskWords / 4)
                                       : std::max(V.nLanes, V.nRL)) + TPB - 1;
        const int grid[5] = {std::max(ingest / TPB, 1), gridNotify, gridControl, gridMove, gridLeader};
        launchPdl(kernel[k], grid[k], TPB, stream, pdl && k != INGEST, V);
    }
    bool pdl() const { return usePdl && !timing; }   // (events between the kernels would serialise them anyway)

    // ---- the sharded step (DeviceSim::shardStep / shardSegment) ----
    void shardTimeMark(int k) {
        if (!shardEv[k]) CFB_CUDA(cudaEventCreate(&shardEv[k]));
        CFB_CUDA(cudaEventRecord(shardEv[k], stream));
    }
    void shardTimeCollect() {   // after mark SHARD_PHASES: accumulates the phase durations
        CFB_CUDA(cudaEventSynchronize(shardEv[SHARD_PHASES]));
        for (int k = 0; k < SHARD_PHASES; ++k) {
            float ms = 0;
            cudaEventElapsedTime(&ms, shardEv[k], shardEv[k + 1]);
            shardMs[k] += ms;
        }
        shardTimedSteps += 1;
    }
    // The seam kernels of the peer-memory form: a warp per boundary lane for the movers, 16 blocks for the tails.
    static int moverGrid(int lanes) { return std::max(1, std::min(64, (lanes * 32 + 127) / 128)); }
    static constexpr int TAIL_GRID = 16;
    void launchSeam(void (*k)(View, ShardP2P), int grid) { launchPdl(k, grid, 128, stream, pdl(), V, S); }
    // Segment k of the step, the work between two seam exchanges (see DeviceSim::shardSegment), over peer memory when
    // connected, else through the staging buffers.  `marks`: record the phase events of kernel timing (peer memory).
    void shardSegment(int k, bool marks, long long &launches) {
        auto mark = [&](int e) { if (marks) shardTimeMark(e); };
        if (k == 0) {
            mark(0);
            launchStep(INGEST, false);
            mark(1);
            launchStep(NOTIFY, pdl());
            launchStep(CONTROL, pdl());
            mark(2);
            if (p2p) launchSeam(k_send_movers, moverGrid(V.nBoundOut));   // X1
            else if (V.nBoundOut) k_pack_movers<<<(V.nBoundOut * 32 + 127) / 128, 128, 0, stream>>>(V, moverSend.p);
            launches += 4;
        } else if (k == 1) {
            mark(3);
            if (p2p) launchSeam(k_recv_movers, moverGrid(V.nBoundIn));
            else if (V.nBoundIn) k_unpack_movers<<<(V.nBoundIn * 32 + 127) / 128, 128, 0, stream>>>(V, moverRecv.p);
            mark(4);
            launchStep(MOVE, pdl());
            mark(5);
            if (p2p) {
                launchSeam(k_send_tails, TAIL_GRID);   // X2
            } else {
                if (V.nBoundIn) k_pack_tails<<<(V.nBoundIn + 127) / 128, 128, 0, stream>>>(V, tailSend.p);
                k_seal_blk<<<1, 1, 0, stream>>>(V);
            }
            launches += p2p ? 3 : 4;
        } else {
            mark(6);
            if (p2p) {
                launchSeam(k_recv_tails, TAIL_GRID);
            } else {
                if (V.nBoundOut) k_unpack_tails<<<(V.nBoundOut + 127) / 128, 128, 0, stream>>>(V, tailRecv.p);
                k_apply_blk<<<dim3(32, shardWorld), 256, 0, stream>>>(V, blkAll.p, shardRank, 1 + V.blkUpdCap);
            }
            mark(7);
            launchStep(LEADER, pdl());
            mark(8);
            if (marks) shardTimeCollect();
            launches += p2p ? 2 : 3;
        }
    }
    // The kernels of one sharded step.  Peer memory: by default 7 kernels (ingest, notify, control, exchange movers, move,
    // exchange tails, leader), nothing but kernels on the stream; split into separate send / receive kernels with
    // CITYFLOW_B200_SHARD_SPLIT=1 or kernel timing, which records the eight phases.  Staged: the three segments with
    // t's two exchanges in between.
    void shardKernels(ShardTransport *t, long long &launches) {
        if (p2p && !shardSplit && !timing) {
            launchStep(INGEST, false);
            launchStep(NOTIFY, pdl());
            launchStep(CONTROL, pdl());
            launchSeam(k_xchg_movers, moverGrid(std::max(V.nBoundOut, V.nBoundIn)));   // X1
            launchStep(MOVE, pdl());
            launchSeam(k_xchg_tails, TAIL_GRID);   // X2
            launchStep(LEADER, pdl());
            launches += 7;
        } else if (p2p) {
            for (int k = 0; k < 3; ++k) shardSegment(k, timing, launches);
        } else {
            shardSegment(0, false, launches);
            t->exchange(stream, moverSend.p, outBeg, moverRecv.p, inBeg, sizeof(MoverMsg));   // X1
            shardSegment(1, false, launches);
            t->exchangeAndGather(stream, tailSend.p, inBeg, tailRecv.p, outBeg, sizeof(TailMsg),
                                 blkUpd.p, blkAll.p, (size_t) (1 + V.blkUpdCap) * sizeof(int2));   // X2
            shardSegment(2, false, launches);
        }
    }
    // The sharded step of `steps` is captured into a CUDA graph per list parity and replayed: one launch call per step
    // instead of ~17.  The first steps run uncaptured so that NCCL can set up its connections; any capture failure
    // switches the engine back to plain launches for good.  Returns 0 plain, 1 replayed (nothing left to enqueue),
    // 2 capturing (enqueue the kernels, then shardGraphEnd).
    int shardGraphBegin(long long steps) {
        const int par = V.par, r = GraphRing::slot(steps);
        if (!shardGraphOk || steps < 8 || timing) return 0;
        GraphRing &G = shardGraphs;
        if (G.exec[par][r] || G.tmpl[par]) {
            if (!G.exec[par][r] && !G.instantiate(par, r)) { cudaGetLastError(); G.exec[par][r] = nullptr; return 0; }
            else if (G.busy(par, r)) { cudaGetLastError(); return 0; }   // this instance is still running: just enqueue
            G.launch(par, r, stream);
            return 1;
        }
        if (cudaStreamBeginCapture(stream, cudaStreamCaptureModeRelaxed) != cudaSuccess) {
            cudaGetLastError();
            shardGraphOk = false;
            return 0;
        }
        return 2;
    }
    bool shardGraphEnd(int state, long long steps) {   // false: capture failed, nothing ran -> repeat the step plainly
        if (state != 2) return true;
        const int par = V.par, r = GraphRing::slot(steps);
        GraphRing &G = shardGraphs;
        cudaGraph_t g = nullptr;
        cudaError_t e = cudaStreamEndCapture(stream, &g);
        if (e == cudaSuccess && g) e = cudaGraphInstantiate(&G.exec[par][r], g, 0);
        if (e != cudaSuccess || !G.exec[par][r]) {
            if (g) cudaGraphDestroy(g);
            cudaGetLastError();
            G.exec[par][r] = nullptr;
            shardGraphOk = false;
            return false;
        }
        G.tmpl[par] = g;
        G.launch(par, r, stream);
        return true;
    }
    void ensureHostInts(size_t n) {
        if (n <= hIntsCap) return;
        if (hInts) cudaFreeHost(hInts);
        CFB_CUDA(cudaMallocHost(&hInts, n * sizeof(int)));
        hIntsCap = n;
    }
};

DeviceSim::DeviceSim(const RoadNet &net, const std::vector<VehicleTemplate> &templates, const Routing &routing,
                     const DeviceSimOptions &opt)
    : impl_(new Impl()) {
    Impl &I = *impl_;
    I.opt = opt;
    int ndev = 0;
    cudaError_t e = cudaGetDeviceCount(&ndev);
    if (e != cudaSuccess || ndev == 0) {
        delete impl_;
        impl_ = nullptr;
        throw std::runtime_error(std::string("cityflow_b200: no CUDA device available (") +
                                 (e != cudaSuccess ? cudaGetErrorString(e) : "device count 0") +
                                 "); this engine has no CPU fallback");
    }
    CFB_CUDA(cudaSetDevice(opt.device));
    CFB_CUDA(cudaStreamCreateWithFlags(&I.stream, cudaStreamNonBlocking));
    CFB_CUDA(cudaDeviceGetAttribute(&I.numSMs, cudaDevAttrMultiProcessorCount, opt.device));
    if (const char *g = getenv("CITYFLOW_B200_NO_GRAPH")) I.useGraph = !(g[0] == '1');
    if (const char *g = getenv("CITYFLOW_B200_COOP")) I.useCoop = (g[0] == '1');
    if (const char *g = getenv("CITYFLOW_B200_NO_PDL")) I.usePdl = !(g[0] == '1');
    {
        int coop = 0;
        cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, opt.device);
        if (!coop) I.useCoop = false;
    }
    View &V = I.V;
    V.dt = opt.interval;
    V.rl = opt.rlTrafficLight ? 1 : 0;

    // ---- static tables ----
    I.L = deviceLayout(net, V, cfb::bucketSpacing(templates));
    const DeviceLayout &L = I.L;
    const int nL = V.nLanes, nK = V.nLinks, nD = V.nDrv;
    I.P = L.P;
    I.drvLength.upload(L.drvLength); I.drvMaxSpeed.upload(L.drvMaxSpeed); I.off.upload(L.off);
    I.laneOutBeg.upload(L.laneOutBeg); I.laneOutLinks.upload(L.laneOutLinks);
    I.llStartLane.upload(L.llStartLane); I.llEndLane.upload(L.llEndLane); I.llRoadLink.upload(L.llRoadLink);
    I.linkInfo.upload(L.linkInfo);
    I.llCrossBeg.upload(L.llCrossBeg); I.lcIdx.upload(L.lcIdx); I.lcDist.upload(L.lcDist); I.lcPeer.upload(L.lcPeer); I.csLink.upload(L.csLink);
    I.interPhaseBeg.upload(L.interPhaseBeg); I.interRLBeg.upload(L.interRLBeg);
    I.phaseAvailBeg.upload(L.phaseAvailBeg); I.rlInter.upload(L.rlInter);
    I.phaseTime.upload(L.phaseTime); I.phaseAvail.upload(L.phaseAvail); I.interVirtual.upload(L.interVirtual);

    V.drvLength = I.drvLength.p; V.drvMaxSpeed = I.drvMaxSpeed.p; V.off = I.off.p;
    V.laneOutBeg = I.laneOutBeg.p; V.laneOutLinks = I.laneOutLinks.p;
    V.llStartLane = I.llStartLane.p; V.llEndLane = I.llEndLane.p; V.llRoadLink = I.llRoadLink.p; V.linkInfo = I.linkInfo.p;
    V.llCrossBeg = I.llCrossBeg.p; V.lcIdx = I.lcIdx.p; V.lcDist = I.lcDist.p; V.lcPeer = I.lcPeer.p; V.csLink = I.csLink.p;
    V.interPhaseBeg = I.interPhaseBeg.p; V.interRLBeg = I.interRLBeg.p; V.phaseAvailBeg = I.phaseAvailBeg.p;
    V.rlInter = I.rlInter.p; V.phaseTime = I.phaseTime.p; V.phaseAvail = I.phaseAvail.p; V.interVirtual = I.interVirtual.p;

    uploadTemplates(templates);
    uploadPlans(routing);

    // ---- dynamic state ----
    const size_t P = (size_t) I.P;
    I.kin.alloc(P); I.nkin.alloc(P); I.gap.alloc(P); I.leader.alloc(P); I.ids.alloc(P); I.nav.alloc(P); I.nbuf.alloc(P);
    I.count.alloc(nD); I.entCnt.alloc(nD); I.ent.alloc((size_t) nD * ENT_CAP);
    I.waitHead.alloc(std::max(nL, 1)); I.waitTail.alloc(std::max(nL, 1)); I.inserted.alloc(std::max(nL, 1));
    I.notify.alloc(std::max(2 * net.nCross(), 1));
    I.curPhase.alloc(net.nInter()); I.remain.alloc(net.nInter()); I.rlAvail.alloc(std::max(net.nRoadLinks(), 1));
    I.mkin.alloc(V.moverCap); I.mids.alloc(V.moverCap); I.mnav.alloc(V.moverCap);
    I.cust.alloc(P); V.cust = I.cust.p;
    I.tail.alloc(nD); I.foeMask.alloc((size_t) std::max(nK, 1) * V.maskWords);
    V.tail = I.tail.p; V.foeMask = I.foeMask.p;
#ifdef CFB_DEBUG_COUNTERS
    I.dbgCyc.alloc(P); I.dbgPath.alloc(P); I.dbgCyc.fill(0); I.dbgPath.fill(0);
    V.dbgCyc = I.dbgCyc.p; V.dbgPath = I.dbgPath.p;
#endif
    I.vehList0.alloc(P); I.vehList1.alloc(P); I.act0.alloc(nD); I.act1.alloc(nD); I.extra.alloc(nD);
    V.vehList[0] = I.vehList0.p; V.vehList[1] = I.vehList1.p; V.actList[0] = I.act0.p; V.actList[1] = I.act1.p;
    V.extraList = I.extra.p;
    I.finSlots.alloc(V.finCap);
    I.ctrl.alloc(1);
    CFB_CUDA(cudaMallocHost(&I.hCtrl, sizeof(Ctrl)));
    {
        int *hm = nullptr, *dm = nullptr;
        CFB_CUDA(cudaHostAlloc(&hm, 64, cudaHostAllocMapped));
        memset(hm, 0, 64);
        CFB_CUDA(cudaHostGetDevicePointer(&dm, hm, 0));
        I.hMirror = hm;
        V.hostMirror = dm;
        if (const char *g = getenv("CITYFLOW_B200_NO_MIRROR")) if (g[0] == '1') V.hostMirror = nullptr;
        I.lastForm[3] = V.hostMirror != nullptr;
    }
    V.kin = I.kin.p; V.nkin = I.nkin.p; V.gap = I.gap.p; V.leader = I.leader.p; V.ids = I.ids.p; V.nav = I.nav.p;
    V.nbuf = I.nbuf.p; V.count = I.count.p; V.entCnt = I.entCnt.p; V.ent = I.ent.p;
    V.waitHead = I.waitHead.p; V.waitTail = I.waitTail.p; V.inserted = I.inserted.p; V.notify = I.notify.p;
    V.curPhase = I.curPhase.p; V.remain = I.remain.p; V.rlAvail = I.rlAvail.p;
    V.mkin = I.mkin.p; V.mids = I.mids.p; V.mnav = I.mnav.p; V.finSlots = I.finSlots.p; V.ctrl = I.ctrl.p;
    ensureSlotCapacity(opt.slotCapacity);
    for (int r = 0; r < Impl::RING; ++r) CFB_CUDA(cudaEventCreateWithFlags(&I.spawnDone[r], cudaEventDisableTiming));
    for (auto &ev : I.ev) CFB_CUDA(cudaEventCreate(&ev));
    reset();
}

DeviceSim::~DeviceSim() {
    if (!impl_) return;
    Impl &I = *impl_;
    cudaStreamSynchronize(I.stream);
    for (int r = 0; r < Impl::RING; ++r) {
        if (I.hSpawn[r]) cudaFreeHost(I.hSpawn[r]);
        if (I.spawnDone[r]) cudaEventDestroy(I.spawnDone[r]);
        if (I.hPhaseRing[r]) cudaFreeHost(I.hPhaseRing[r]);
        if (I.hPhaseFlush[r]) cudaFreeHost(I.hPhaseFlush[r]);
        if (I.phaseFlushDone[r]) cudaEventDestroy(I.phaseFlushDone[r]);
    }
    for (auto &ev : I.ev) if (ev) cudaEventDestroy(ev);
    for (auto &ev : I.stepEv) cudaEventDestroy(ev);
    I.graphs.release(I.stream);
    I.shardGraphs.release(I.stream);
    if (I.hCtrl) cudaFreeHost(I.hCtrl);
    if (I.hMirror) cudaFreeHost((void *) I.hMirror);
    if (I.hInts) cudaFreeHost(I.hInts);
    if (I.stream) cudaStreamDestroy(I.stream);
    // A peer process may still have the arena mapped (cudaIpcOpenMemHandle): freeing exported memory before every
    // importer has closed it is undefined, and a barrier in a destructor can hang on a rank that died -- the arena of a
    // multi-process run is left to process exit.
    if (I.arena.p && I.p2p && I.shardWorld > 1 && I.arenaShared) { I.arena.p = nullptr; I.arena.n = 0; }
    delete impl_;
}

void DeviceSim::uploadTemplates(const std::vector<VehicleTemplate> &templates) {
    Impl &I = *impl_;
    std::vector<DTmpl> t;
    for (const auto &x : templates) t.push_back(toDevice(x, I.opt.interval));
    if (t.empty()) t.push_back(DTmpl{});
    CFB_CUDA(cudaStreamSynchronize(I.stream));
    I.tmpl.upload(t);
    I.V.tmpl = I.tmpl.p;
    I.invalidateGraphs();
    legacySync();
}

void DeviceSim::uploadPlans(const Routing &routing) {
    Impl &I = *impl_;
    const PlanTables T = planTables(routing);
    CFB_CUDA(cudaStreamSynchronize(I.stream));
    I.planBeg.upload(T.planBeg);
    I.planData.upload(T.planData);
    I.V.planBeg = I.planBeg.p;
    I.V.planData = I.planData.p;
    I.invalidateGraphs();
    legacySync();
}

void DeviceSim::ensureSlotCapacity(int slots) {
    Impl &I = *impl_;
    if (slots <= I.slotCap) return;
    if (I.arena.p) throw std::runtime_error("cityflow_b200: slot capacity of a sharded run exceeded (4 M vehicles alive or waiting)");
    int cap = std::max(I.slotCap, 1024);
    while (cap < slots) cap *= 2;
    CFB_CUDA(cudaStreamSynchronize(I.stream));
    DevBuf<int> npos, nnext;
    DevBuf<int4> ninfo;
    DevBuf<double> ncust;
    DevBuf<int> nblk, ndel;
    npos.alloc(cap); nnext.alloc(cap); ninfo.alloc(cap); ncust.alloc(cap);
    npos.fill(0xff); nnext.fill(0xff); ninfo.fill(0); ncust.fill(0xff);
    nblk.alloc(cap); ndel.alloc(cap); nblk.fill(0xff); ndel.fill(0x80);
    legacySync();   // fills before the copies (same stream, but keep the order explicit)
    if (I.slotCap) {
        CFB_CUDA(cudaMemcpy(npos.p, I.pos.p, I.slotCap * sizeof(int), cudaMemcpyDeviceToDevice));
        CFB_CUDA(cudaMemcpy(nnext.p, I.waitNext.p, I.slotCap * sizeof(int), cudaMemcpyDeviceToDevice));
        CFB_CUDA(cudaMemcpy(ninfo.p, I.slotInfo.p, I.slotCap * sizeof(int4), cudaMemcpyDeviceToDevice));
        CFB_CUDA(cudaMemcpy(ncust.p, I.slotCust.p, I.slotCap * sizeof(double), cudaMemcpyDeviceToDevice));
        CFB_CUDA(cudaMemcpy(nblk.p, I.blk.p, I.slotCap * sizeof(int), cudaMemcpyDeviceToDevice));
        CFB_CUDA(cudaMemcpy(ndel.p, I.delStep.p, I.slotCap * sizeof(int), cudaMemcpyDeviceToDevice));
    }
    std::swap(I.pos.p, npos.p); std::swap(I.pos.n, npos.n);
    std::swap(I.waitNext.p, nnext.p); std::swap(I.waitNext.n, nnext.n);
    std::swap(I.slotInfo.p, ninfo.p); std::swap(I.slotInfo.n, ninfo.n);
    std::swap(I.slotCust.p, ncust.p); std::swap(I.slotCust.n, ncust.n);
    std::swap(I.blk.p, nblk.p); std::swap(I.blk.n, nblk.n);
    std::swap(I.delStep.p, ndel.p); std::swap(I.delStep.n, ndel.n);
    if (I.V.lcOn) {
        DevBuf<LcSlot> nlc;
        nlc.alloc(cap);
        nlc.fill(0);
        if (I.slotCap) CFB_CUDA(cudaMemcpy(nlc.p, I.lcSlot.p, I.slotCap * sizeof(LcSlot), cudaMemcpyDeviceToDevice));
        std::swap(I.lcSlot.p, nlc.p); std::swap(I.lcSlot.n, nlc.n);
        I.V.lc.slot = I.lcSlot.p;
    }
    legacySync();   // ... and the copies before the old buffers are freed / the new ones are used
    I.slotCap = cap;
    I.V.pos = I.pos.p; I.V.waitNext = I.waitNext.p; I.V.slotInfo = I.slotInfo.p; I.V.slotCust = I.slotCust.p; I.V.blk = I.blk.p; I.V.delStep = I.delStep.p;
    I.invalidateGraphs();
}

void DeviceSim::reset() {
    Impl &I = *impl_;
    CFB_CUDA(cudaStreamSynchronize(I.stream));
    applyFills(resetFills(I.V, (size_t) I.P, (size_t) I.slotCap));
    CFB_CUDA(cudaMemcpy(I.remain.p, I.L.remain0.data(), I.L.remain0.size() * sizeof(double), cudaMemcpyHostToDevice));
    I.hPhase.assign(I.V.nInter, 0);
    I.phaseDirty = false;
    I.hPhaseStale = false;
    if (I.hMirror) { I.hMirror[1] = 0; I.hMirror[2] = 0; I.hMirror[3] = 0; }   // (the stream is idle: nothing else writes it now)
    I.mirrorStale = false;
    // leader = -1 everywhere is not required (only occupied positions are read)
    steps_ = 0;
    legacySync();
}

int DeviceSim::numPositions() const { return impl_->P; }
int DeviceSim::numDrivables() const { return impl_->V.nDrv; }
int DeviceSim::device() const { return impl_->opt.device; }

void DeviceSim::stageStep(const SpawnRec *recs, int n) {
    Impl &I = *impl_;
    View &V = I.V;
    cudaStream_t s = I.stream;
    // ---- stage this step's spawn records: one H2D copy of [header | records] from a pinned ring ----
    if (n + 1 > I.spawnCap) {
        CFB_CUDA(cudaStreamSynchronize(s));
        I.spawnCap = std::max(1024, (n + 1) * 2);
        I.spawn.alloc(I.spawnCap);
        I.invalidateGraphs();
    }
    V.spawn = I.spawn.p + 1;
    const int r = I.ringIdx;
    I.ringIdx = (I.ringIdx + 1) % Impl::RING;
    CFB_CUDA(cudaEventSynchronize(I.spawnDone[r]));  // ring slot r free again (RING steps in flight at most)
    if (n + 1 > I.hSpawnCap[r]) {
        if (I.hSpawn[r]) cudaFreeHost(I.hSpawn[r]);
        I.hSpawnCap[r] = std::max(1024, (n + 1) * 2);
        CFB_CUDA(cudaMallocHost(&I.hSpawn[r], I.hSpawnCap[r] * sizeof(SpawnRec)));
    }
    if (I.phaseDirty) {  // batched set_tl_phase: one H2D copy of all phases before the step
        if (!I.hPhaseRing[r]) CFB_CUDA(cudaMallocHost(&I.hPhaseRing[r], std::max(V.nInter, 1) * sizeof(int)));
        memcpy(I.hPhaseRing[r], I.hPhase.data(), V.nInter * sizeof(int));
        CFB_CUDA(cudaMemcpyAsync(V.curPhase, I.hPhaseRing[r], V.nInter * sizeof(int), cudaMemcpyHostToDevice, s));
        I.phaseDirty = false;
    }
    I.hSpawn[r][0].slot = n;
    if (n > 0) memcpy(I.hSpawn[r] + 1, recs, n * sizeof(SpawnRec));
    CFB_CUDA(cudaMemcpyAsync(I.spawn.p, I.hSpawn[r], (size_t) (n + 1) * sizeof(SpawnRec), cudaMemcpyHostToDevice, s));
    CFB_CUDA(cudaEventRecord(I.spawnDone[r], s));
    V.par = (int) (steps_ & 1);
}

void DeviceSim::step(const SpawnRec *recs, int n) {
    stageStep(recs, n);
    Impl &I = *impl_;
    View &V = I.V;
    cudaStream_t s = I.stream;
    I.ensureGrids();
    const bool tm = I.timing;
    auto launchAll = [&]() {   // with kernel timing: an event before and after each kernel
        for (int k = 0; k < 5; ++k) {
            if (tm) cudaEventRecord(I.ev[k], s);
            I.launchStep((Impl::StepKernel) k, I.pdl());
        }
        if (tm) cudaEventRecord(I.ev[5], s);
    };
    if (!tm && I.useCoop) {
        if (!I.gridStep) {
            int b = 0;
            CFB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&b, k_step, 256, 0));
            I.gridStep = std::max(b, 1) * I.numSMs;
        }
        void *args[] = {(void *) &V};
        CFB_CUDA(cudaLaunchCooperativeKernel((void *) k_step, dim3(I.gridStep), dim3(256), args, 0, s));
    } else if (tm || !I.useGraph) {
        launchAll();
    } else {
        // The five kernels of one step are replayed as one CUDA graph per list parity: one launch
        // call per step instead of five, and no host-paced gaps between the kernels.
        GraphRing &G = I.graphs;
        const int r = GraphRing::slot(steps_);
        cudaGraphExec_t &ge = G.exec[V.par][r];
        cudaGraph_t &g = G.tmpl[V.par];
        for (int attempt = 0; attempt < 2 && !ge; ++attempt) {
            if (!g) {
                CFB_CUDA(cudaStreamBeginCapture(s, cudaStreamCaptureModeThreadLocal));
                launchAll();
                if (cudaStreamEndCapture(s, &g) != cudaSuccess) g = nullptr;
            }
            if (!g || !G.instantiate(V.par, r)) {
                // a driver that cannot put programmatic dependencies into a graph: plain edges instead
                cudaGetLastError();
                if (g) { cudaGraphDestroy(g); g = nullptr; }
                ge = nullptr;
                if (!I.usePdl) throw std::runtime_error("cityflow_b200: cannot capture the step into a CUDA graph");
                I.usePdl = false;
            }
        }
        // when even the ring is exhausted: the five plain launches, which only enqueue
        if (G.busy(V.par, r)) launchAll();
        else G.launch(V.par, r, s);
    }
    CFB_CUDA(cudaGetLastError());
    {   // (a graph step that found its ring instance busy and launched plainly still counts as the graph form)
        const bool coop = !tm && I.useCoop;
        I.lastForm[0] = !tm && !coop && I.useGraph;
        I.lastForm[1] = !tm && !coop && I.usePdl;
        I.lastForm[2] = coop;
        I.lastForm[3] = V.hostMirror != nullptr;
    }
    launches_ += (!tm && I.useCoop) ? 1 : 5;
    steps_ += 1;
    I.epochHost += 1;
    I.mirrorStale = false;
    if (tm) {
        CFB_CUDA(cudaEventSynchronize(I.ev[5]));
        float ms[5];
        for (int k = 0; k < 5; ++k) cudaEventElapsedTime(&ms[k], I.ev[k], I.ev[k + 1]);
        I.times.ingest += ms[0]; I.times.notify += ms[1]; I.times.control += ms[2]; I.times.move += ms[3];
        I.times.leader += ms[4];
        I.times.launches += 1;
    }
}

static void readCtrlImpl(cudaStream_t s, Ctrl *dst, const Ctrl *src);
void DeviceSim::synchronize() { CFB_CUDA(cudaStreamSynchronize(impl_->stream)); }

// ------------------------------------------------------------------------------------------
// Sharded mode (partition.h / shard.h): the step with the seam exchanges in between (Impl::shardKernels).
void DeviceSim::configureShard(int rank, int world, const std::vector<unsigned char> &owned,
                               const std::vector<std::vector<int>> &feedPerPeer,
                               const std::vector<std::vector<int>> &ownPerPeer,
                               const std::vector<std::vector<int>> &boundarySize,
                               const std::vector<unsigned char> &ownedRoadLinks) {
    Impl &I = *impl_;
    View &V = I.V;
    CFB_CUDA(cudaStreamSynchronize(I.stream));
    I.shardRank = rank;
    I.shardWorld = world;
    I.bsize = boundarySize;
    const ShardLists SL = shardLists(V.nLanes, V.nLinks, owned, feedPerPeer, ownPerPeer, ownedRoadLinks);
    I.owned.upload(SL.owned);
    I.ownedHost = owned;
    V.owned = I.owned.p;
    I.ingBuf.upload(SL.ing);
    I.boundOut.upload(SL.boundOut);
    I.boundIn.upload(SL.boundIn);
    SL.point(V, I.ingBuf.p, I.boundOut.p, I.boundIn.p);
    I.outBeg = SL.outBeg;
    I.inBeg = SL.inBeg;
    I.tailSend.alloc(std::max(V.nBoundIn, 1));
    I.tailRecv.alloc(std::max(V.nBoundOut, 1));
    I.moverSend.alloc(std::max(V.nBoundOut, 1));
    I.moverRecv.alloc(std::max(V.nBoundIn, 1));
    I.tailSend.fill(0); I.tailRecv.fill(0); I.moverSend.fill(0); I.moverRecv.fill(0);
    V.blkUpdCap = 1 << 14;
    I.blkUpd.alloc(1 + V.blkUpdCap);
    I.blkAll.alloc((size_t) world * (1 + V.blkUpdCap));
    I.blkUpd.fill(0); I.blkAll.fill(0);
    V.blkUpd = I.blkUpd.p;
    I.useGraph = false;  // phases are launched one by one (or replayed as one sharded-step graph)
    I.useCoop = false;
    if (const char *g = getenv("CITYFLOW_B200_SHARD_GRAPH")) I.shardGraphOk = (g[0] != '0');
    legacySync();
}

ShardBuffers DeviceSim::shardBuffers() {
    Impl &I = *impl_;
    ShardBuffers b;
    b.stream = (void *) I.stream;
    b.tailSend = I.tailSend.p; b.tailRecv = I.tailRecv.p; b.moverSend = I.moverSend.p; b.moverRecv = I.moverRecv.p;
    b.tailBytes = sizeof(TailMsg); b.moverBytes = sizeof(MoverMsg);
    b.outBeg = I.outBeg; b.inBeg = I.inBeg;
    b.blkSend = I.blkUpd.p; b.blkAll = I.blkAll.p;
    b.blkBytesPerRank = (size_t) (1 + I.V.blkUpdCap) * sizeof(int2);
    return b;
}

// One step of one rank of a multi-process run (see Impl::shardKernels for the kernel sequence).
void DeviceSim::shardStep(const SpawnRec *recs, int n, ShardTransport *t) {
    Impl &I = *impl_;
    stageStep(recs, n);
    for (int attempt = 0; attempt < 2; ++attempt) {
        const int st = I.shardGraphBegin(steps_);
        if (st != 1) try {
            I.shardKernels(t, launches_);
        } catch (const std::exception &) {
            if (st != 2 || I.p2p) throw;
            // a staged exchange refused to be captured: abandon the graph, run this step plainly
        }
        if (I.shardGraphEnd(st, steps_)) break;
    }
    CFB_CUDA(cudaGetLastError());
    steps_ += 1;
    I.epochHost += 1;
}

void DeviceSim::shardSegment(int k) {
    Impl &I = *impl_;
    I.shardSegment(k, false, launches_);
    if (k == 2) {
        CFB_CUDA(cudaGetLastError());
        steps_ += 1;
        I.epochHost += 1;
    }
}

// ---- peer-memory transport (device_shard.cuh) ----
// The arena other ranks write into.  From here on the slot-indexed arrays have their final size (delStep lives in
// the arena and is mapped by the peers).
DeviceSim::ShardArena DeviceSim::shardArena() {
    Impl &I = *impl_;
    if (!I.arena.p) {
        ensureSlotCapacity(Impl::SHARD_SLOT_CAP);
        CFB_CUDA(cudaStreamSynchronize(I.stream));
        const Impl::ArenaLayout L = Impl::arenaLayout(I.shardWorld, I.V.nBoundIn, I.V.nBoundOut);
        I.arena.alloc(L.total);
        I.arena.fill(0);
        legacySync();
        CFB_CUDA(cudaMemcpy(I.arena.p + L.delStep, I.V.delStep, (size_t) Impl::SHARD_SLOT_CAP * sizeof(int), cudaMemcpyDeviceToDevice));
        legacySync();
        I.delStep.release();
        I.V.delStep = (int *) (I.arena.p + L.delStep);
        I.invalidateGraphs();
    }
    return ShardArena{I.arena.p, I.arena.n};
}

// `peerBase[q]` = rank q's arena as mapped into this process (ignored for q == me).
void DeviceSim::shardMarkArenaExported() { impl_->arenaShared = true; }
void DeviceSim::shardConnect(const std::vector<void *> &peerBase) {
    Impl &I = *impl_;
    View &V = I.V;
    const int W = I.shardWorld, me = I.shardRank;
    if (!I.arena.p || (int) peerBase.size() != W) throw std::runtime_error("shardConnect: arena missing / wrong world size");
    CFB_CUDA(cudaStreamSynchronize(I.stream));
    std::vector<ShardPeer> peers(W);
    for (int q = 0; q < W; ++q) {
        unsigned char *base = q == me ? I.arena.p : (unsigned char *) peerBase[q];
        const Impl::ArenaLayout L = Impl::arenaLayout(W, I.nInOf(q), I.nOutOf(q));
        ShardPeer &P = peers[q];
        P.flags = (int *) (base + L.flags);
        P.delStep = (int *) (base + L.delStep);
        P.blkIn = (int2 *) (base + L.blkIn) + (size_t) me * (1 + BLK_IN_CAP);
        P.moverIn = (MoverMsg *) (base + L.moverIn);
        P.tailIn = (TailMsg *) (base + L.tailIn);
        P.nIn = std::max(I.nInOf(q), 1);
        P.nOut = std::max(I.nOutOf(q), 1);
    }
    I.peers.upload(peers);
    // index tables: where my messages land in the receivers' mailboxes (partition.h)
    const SeamTables T = seamTables(I.bsize, me);
    if ((int) T.outPeer.size() != V.nBoundOut || (int) T.inPeer.size() != V.nBoundIn) throw std::runtime_error("shardConnect: boundary tables disagree");
    if ((int) T.nbr.size() > 120) throw std::runtime_error("shardConnect: too many neighbour ranks");
    const SeamIndex X = seamIndex(T);
    I.p2pInts.upload(X.ints);
    const Impl::ArenaLayout L = Impl::arenaLayout(W, V.nBoundIn, V.nBoundOut);
    ShardP2P &S = I.S;
    S.peers = I.peers.p; S.me = me; S.world = W;
    X.point(S, I.p2pInts.p);
    S.flags = (int *) (I.arena.p + L.flags);
    S.blkIn = (int2 *) (I.arena.p + L.blkIn);
    S.moverIn = (MoverMsg *) (I.arena.p + L.moverIn);
    S.tailIn = (TailMsg *) (I.arena.p + L.tailIn);
    if (V.blkUpdCap > BLK_IN_CAP) V.blkUpdCap = BLK_IN_CAP;
    if (const char *g = getenv("CITYFLOW_B200_SHARD_SPLIT")) I.shardSplit = g[0] == '1';
    I.p2p = true;
    I.invalidateGraphs();
    legacySync();
}

// Network-wide vehicle count over the peer-memory arena (k_sum_active); false: not available, use shardCounts().
bool DeviceSim::shardVehicleCount(int *activeOut) {
    Impl &I = *impl_;
    if (!I.p2p || !I.V.hostMirror) return false;
    k_sum_active<<<1, 32, 0, I.stream>>>(I.V, I.S);
    launches_ += 1;
    const auto t0 = std::chrono::steady_clock::now();
    for (long spin = 0; I.hMirror[5] < (int) I.epochHost; ++spin) {
        if ((spin & 1023) == 1023 && std::chrono::steady_clock::now() - t0 > std::chrono::seconds(5)) {
            CFB_CUDA(cudaStreamSynchronize(I.stream));
            if (I.hMirror[5] < (int) I.epochHost) return false;
        }
        __builtin_ia32_pause();
    }
    *activeOut = I.hMirror[4];
    return true;
}

void DeviceSim::shardCounts(ShardTransport *t, int32_t *laneOut, int *activeOut) {
    Impl &I = *impl_;
    const int n = laneOut ? 1 + I.V.nLanes : 1;   // the vehicle count alone is a 4-byte all-reduce
    if (I.shardScratch.n < (size_t) (1 + I.V.nLanes)) I.shardScratch.alloc(1 + I.V.nLanes);
    k_mask_counts<<<(n + 255) / 256, 256, 0, I.stream>>>(I.V, I.shardScratch.p);
    t->allReduceSumInt((void *) I.stream, I.shardScratch.p, n);
    std::vector<int> h(n);
    CFB_CUDA(cudaMemcpyAsync(h.data(), I.shardScratch.p, n * sizeof(int), cudaMemcpyDeviceToHost, I.stream));
    CFB_CUDA(cudaStreamSynchronize(I.stream));
    if (activeOut) *activeOut = h[0];
    if (laneOut) memcpy(laneOut, h.data() + 1, I.V.nLanes * sizeof(int));
}

void DeviceSim::shardWaitingCounts(ShardTransport *t, int32_t *laneOut) {
    Impl &I = *impl_;
    const int nL = I.V.nLanes;
    if (I.scratchI.n < (size_t) nL) I.scratchI.alloc(nL);
    if (I.shardScratch.n < (size_t) nL + 1) I.shardScratch.alloc(nL + 1);
    k_lane_waiting<<<(nL * 32 + 255) / 256, 256, 0, I.stream>>>(I.V, I.scratchI.p);
    k_mask_waiting<<<(nL + 255) / 256, 256, 0, I.stream>>>(I.V, I.scratchI.p, I.shardScratch.p);
    t->allReduceSumInt((void *) I.stream, I.shardScratch.p, nL);
    CFB_CUDA(cudaMemcpyAsync(laneOut, I.shardScratch.p, nL * sizeof(int), cudaMemcpyDeviceToHost, I.stream));
    CFB_CUDA(cudaStreamSynchronize(I.stream));
}

// Finished vehicles of ALL ranks since the last drain (every rank must call this at the same step).
void DeviceSim::shardGatherFinished(ShardTransport *t, std::vector<FinRec> &inout) {
    Impl &I = *impl_;
    const int cap = 1 << 16, W = t->world();
    const size_t per = (size_t) (1 + cap) * sizeof(FinRec);
    if (I.finGather.n < per * (W + 1)) I.finGather.alloc(per * (W + 1));
    if ((int) inout.size() > cap) throw std::runtime_error("cityflow_b200: too many finished vehicles between two drains (sharded capacity)");
    std::vector<FinRec> send(1 + inout.size());
    send[0].slot = (int) inout.size();
    send[0].step = 0;
    std::copy(inout.begin(), inout.end(), send.begin() + 1);
    unsigned char *mine = I.finGather.p, *all = I.finGather.p + per;
    CFB_CUDA(cudaMemcpyAsync(mine, send.data(), send.size() * sizeof(FinRec), cudaMemcpyHostToDevice, I.stream));
    t->allGather((void *) I.stream, mine, all, per);
    std::vector<FinRec> recv((size_t) W * (1 + cap));
    CFB_CUDA(cudaMemcpyAsync(recv.data(), all, per * W, cudaMemcpyDeviceToHost, I.stream));
    CFB_CUDA(cudaStreamSynchronize(I.stream));
    inout.clear();
    for (int r = 0; r < W; ++r) {
        const FinRec *p = recv.data() + (size_t) r * (1 + cap);
        for (int k = 0; k < p[0].slot; ++k) inout.push_back(p[1 + k]);
    }
}

// ---- measurement support: CUDA-event brackets on the engine's own stream ----
void DeviceSim::flushL2() {
    Impl &I = *impl_;
    const size_t bytes = (size_t) 256 << 20;  // several times the 50 MB L2 of an H100
    if (I.flushBuf.n < bytes) I.flushBuf.alloc(bytes);
    CFB_CUDA(cudaMemsetAsync(I.flushBuf.p, (int) (steps_ & 0xff), bytes, I.stream));
}
void DeviceSim::markTimed() {
    Impl &I = *impl_;
    if (I.stepEvUsed == I.stepEv.size()) {
        cudaEvent_t e;
        CFB_CUDA(cudaEventCreate(&e));
        I.stepEv.push_back(e);
    }
    CFB_CUDA(cudaEventRecord(I.stepEv[I.stepEvUsed++], I.stream));
}
double DeviceSim::collectTimedMs() {
    Impl &I = *impl_;
    CFB_CUDA(cudaStreamSynchronize(I.stream));
    double total = 0;
    for (size_t k = 0; k + 1 < I.stepEvUsed; k += 2) {
        float ms = 0;
        CFB_CUDA(cudaEventElapsedTime(&ms, I.stepEv[k], I.stepEv[k + 1]));
        total += ms;
    }
    I.stepEvUsed = 0;
    return total;
}
int DeviceSim::debugArrays(unsigned *cyc, unsigned *path) {
    Impl &I = *impl_;
    CFB_CUDA(cudaStreamSynchronize(I.stream));
    if (!I.dbgCyc.p) {  // not a CFB_DEBUG_COUNTERS build
        memset(cyc, 0, (size_t) I.P * 4);
        memset(path, 0, (size_t) I.P * 4);
        return I.P;
    }
    CFB_CUDA(cudaMemcpy(cyc, I.dbgCyc.p, (size_t) I.P * 4, cudaMemcpyDeviceToHost));
    CFB_CUDA(cudaMemcpy(path, I.dbgPath.p, (size_t) I.P * 4, cudaMemcpyDeviceToHost));
    I.dbgCyc.fill(0); I.dbgPath.fill(0);
    return I.P;
}
void DeviceSim::debugCounters(unsigned long long out[8], bool clear) {
    readCtrlImpl(impl_->stream, impl_->hCtrl, impl_->V.ctrl);
    for (int k = 0; k < 8; ++k) out[k] = impl_->hCtrl->dbg[k];
    if (clear) CFB_CUDA(cudaMemsetAsync(impl_->V.ctrl->dbg, 0, sizeof(unsigned long long) * 8, impl_->stream));
}
unsigned long long DeviceSim::vehicleSteps() {
    readCtrlImpl(impl_->stream, impl_->hCtrl, impl_->V.ctrl);
    return impl_->hCtrl->vehicleSteps;
}

void DeviceSim::launchForm(int out[4]) const {
    for (int k = 0; k < 4; ++k) out[k] = impl_->lastForm[k];
}

void DeviceSim::stepGrids(int out[5]) const {
    const Impl &I = *impl_;
    out[0] = I.gridNotify; out[1] = I.gridControl; out[2] = I.gridMove; out[3] = I.gridLeader; out[4] = I.gridStep;
}

void DeviceSim::enableKernelTiming(bool on) {
    impl_->timing = on;
    impl_->times = KernelTimes();
    for (double &x : impl_->shardMs) x = 0;
    impl_->shardTimedSteps = 0;
}
void DeviceSim::shardStepTimes(double ms[SHARD_PHASES], long long *steps) {
    for (int k = 0; k < SHARD_PHASES; ++k) ms[k] = impl_->shardMs[k];
    if (steps) *steps = impl_->shardTimedSteps;
}
DeviceSim::KernelTimes DeviceSim::kernelTimes() { return impl_->times; }

static void readCtrlImpl(cudaStream_t s, Ctrl *dst, const Ctrl *src);
static void readCtrlImpl(cudaStream_t s, Ctrl *dst, const Ctrl *src) {
    CFB_CUDA(cudaMemcpyAsync(dst, src, sizeof(Ctrl), cudaMemcpyDeviceToHost, s));
    CFB_CUDA(cudaStreamSynchronize(s));
}

// The last enqueued step's {active, error, ties} as k_leader stored them in host memory: wait for the epoch stamp instead
// of enqueuing a copy behind the step and synchronising the stream (saves a D2H round trip per get_vehicle_count()).
static bool mirrorCurrent(DeviceSim::Impl &I) {
    if (!I.V.hostMirror || I.mirrorStale) return false;
    const auto t0 = std::chrono::steady_clock::now();
    for (long spin = 0; I.hMirror[0] < (int) I.epochHost; ++spin) {
        if ((spin & 1023) == 1023) {
            if (std::chrono::steady_clock::now() - t0 > std::chrono::milliseconds(200)) return false;   // let the caller synchronise
        }
        __builtin_ia32_pause();
    }
    return true;
}

int DeviceSim::vehicleCount() {
    if (mirrorCurrent(*impl_)) return impl_->hMirror[1];
    readCtrlImpl(impl_->stream, impl_->hCtrl, impl_->V.ctrl);
    return impl_->hCtrl->active;
}

int DeviceSim::tieCount() {
    readCtrlImpl(impl_->stream, impl_->hCtrl, impl_->V.ctrl);
    return impl_->hCtrl->ties;
}

double DeviceSim::bucketSpacing() const { return impl_->L.spacing; }

int DeviceSim::errorFlags() {
    if (mirrorCurrent(*impl_)) return impl_->hMirror[2];
    readCtrlImpl(impl_->stream, impl_->hCtrl, impl_->V.ctrl);
    return impl_->hCtrl->error;
}

void DeviceSim::laneVehicleCount(int32_t *out) {
    Impl &I = *impl_;
    I.ensureHostInts(I.V.nLanes);
    CFB_CUDA(cudaMemcpyAsync(I.hInts, I.V.count, I.V.nLanes * sizeof(int), cudaMemcpyDeviceToHost, I.stream));
    CFB_CUDA(cudaStreamSynchronize(I.stream));
    memcpy(out, I.hInts, I.V.nLanes * sizeof(int));
}

void DeviceSim::laneWaitingVehicleCount(int32_t *out) {
    Impl &I = *impl_;
    if (I.scratchI.n < (size_t) I.V.nLanes) I.scratchI.alloc(I.V.nLanes);
    I.ensureHostInts(I.V.nLanes);
    const int TPB = 256;
    k_lane_waiting<<<(I.V.nLanes * 32 + TPB - 1) / TPB, TPB, 0, I.stream>>>(I.V, I.scratchI.p);
    CFB_CUDA(cudaMemcpyAsync(I.hInts, I.scratchI.p, I.V.nLanes * sizeof(int), cudaMemcpyDeviceToHost, I.stream));
    CFB_CUDA(cudaStreamSynchronize(I.stream));
    memcpy(out, I.hInts, I.V.nLanes * sizeof(int));
    launches_ += 1;
}

void DeviceSim::setPhasesFromDevice(const int32_t *phases, void *producerStream) {
    Impl &I = *impl_;
    if (I.V.owned) throw std::runtime_error("setPhasesFromDevice: not available on one rank of a sharded run");
    if (!I.actReady) {
        CFB_CUDA(cudaEventCreateWithFlags(&I.actReady, cudaEventDisableTiming));
        CFB_CUDA(cudaEventCreateWithFlags(&I.actTaken, cudaEventDisableTiming));
    }
    cudaStream_t ps = (cudaStream_t) producerStream;
    CFB_CUDA(cudaEventRecord(I.actReady, ps));
    CFB_CUDA(cudaStreamWaitEvent(I.stream, I.actReady, 0));
    if (I.V.nInter > 0) k_set_phases<<<(I.V.nInter + 127) / 128, 128, 0, I.stream>>>(I.V, phases);
    CFB_CUDA(cudaGetLastError());
    CFB_CUDA(cudaEventRecord(I.actTaken, I.stream));      // the producer may reuse its buffer after this
    CFB_CUDA(cudaStreamWaitEvent(ps, I.actTaken, 0));
    I.phaseDirty = false;    // every light was just overwritten: pending host-side changes are superseded
    I.hPhaseStale = true;
    I.mirrorStale = true;    // k_set_phases may raise ERR_PHASE_RANGE outside a step
    launches_ += 1;
}

DeviceObs DeviceSim::observeOnDevice(void *consumerStream) {
    Impl &I = *impl_;
    if (I.V.owned) throw std::runtime_error("observeOnDevice: not available on one rank of a sharded run");
    const int nL = I.V.nLanes;
    if (I.obsI.n < (size_t) 2 * nL) {
        I.obsI.alloc((size_t) 2 * std::max(nL, 1));
        I.obsD.alloc((size_t) std::max(nL, 1));
        CFB_CUDA(cudaEventCreateWithFlags(&I.obsReady, cudaEventDisableTiming));
        CFB_CUDA(cudaEventCreateWithFlags(&I.obsConsumed, cudaEventDisableTiming));
    }
    cudaStream_t cs = (cudaStream_t) consumerStream;
    // the consumer's earlier reads of the buffers finish before this refresh overwrites them ...
    CFB_CUDA(cudaEventRecord(I.obsConsumed, cs));
    CFB_CUDA(cudaStreamWaitEvent(I.stream, I.obsConsumed, 0));
    const int TPB = 256;
    if (nL > 0) k_lane_obs<<<(int) (((size_t) nL * 32 + TPB - 1) / TPB), TPB, 0, I.stream>>>(I.V, I.obsI.p, I.obsI.p + nL, I.obsD.p);
    CFB_CUDA(cudaGetLastError());
    // ... and its later reads see this refresh, without the host waiting for either stream
    CFB_CUDA(cudaEventRecord(I.obsReady, I.stream));
    CFB_CUDA(cudaStreamWaitEvent(cs, I.obsReady, 0));
    launches_ += 1;
    DeviceObs o;
    o.laneCount = I.obsI.p;
    o.laneWaiting = I.obsI.p + nL;
    o.laneSpeedSum = I.obsD.p;
    o.nLanes = nL;
    o.device = I.opt.device;
    return o;
}

// setPhase calls made since the last step act at once (trafficlight.cpp:39-41): a refresh that reads the phases sends
// them up first, on the engine's stream, through a ring of pinned buffers each guarded by the event of its last copy.
static void sendPendingPhases(DeviceSim::Impl &I) {
    View &V = I.V;
    if (!I.phaseDirty || !V.nInter) return;
    const int r = I.phaseFlushIdx;
    I.phaseFlushIdx = (r + 1) % DeviceSim::Impl::RING;
    if (!I.hPhaseFlush[r]) {
        CFB_CUDA(cudaMallocHost(&I.hPhaseFlush[r], V.nInter * sizeof(int)));
        CFB_CUDA(cudaEventCreateWithFlags(&I.phaseFlushDone[r], cudaEventDisableTiming));
    }
    CFB_CUDA(cudaEventSynchronize(I.phaseFlushDone[r]));   // its copy of RING refreshes ago has run (never waits in practice)
    memcpy(I.hPhaseFlush[r], I.hPhase.data(), V.nInter * sizeof(int));
    CFB_CUDA(cudaMemcpyAsync(V.curPhase, I.hPhaseFlush[r], V.nInter * sizeof(int), cudaMemcpyHostToDevice, I.stream));
    CFB_CUDA(cudaEventRecord(I.phaseFlushDone[r], I.stream));
    I.phaseDirty = false;
}

// The per-vehicle table's buffers, made on the first refresh (the row capacity is the position capacity, fixed when the
// engine is made), and the pointers a refresh hands out.
static void vobsMake(DeviceSim::Impl &I) {
    const size_t cap = (size_t) std::max(I.P, 1), nD = (size_t) I.V.nDrv;
    const int tiles = (int) std::max<size_t>(1, (nD + VOBS_TILE - 1) / VOBS_TILE);
    const size_t nI = 3 * cap + (nD + 1) + 2 + (size_t) tiles;
    if (I.vobsI.n < nI) {
        I.vobsI.alloc(nI);
        I.vobsD.alloc(2 * cap);
        I.vobsShadow.alloc(cap);
        CFB_CUDA(cudaMemsetAsync(I.vobsI.p, 0xff, cap * sizeof(int), I.stream));                       // slot: all padding
        CFB_CUDA(cudaMemsetAsync(I.vobsI.p + cap, 0, (nI - cap) * sizeof(int), I.stream));             // count 0
        CFB_CUDA(cudaMemsetAsync(I.vobsD.p, 0, 2 * cap * sizeof(double), I.stream));
        CFB_CUDA(cudaMemsetAsync(I.vobsShadow.p, 0, cap, I.stream));
        VehObsTable &T = I.vobs;
        T.slot = I.vobsI.p; T.priority = T.slot + cap; T.drivable = T.priority + cap;
        T.drvBegin = T.drivable + cap; T.count = T.drvBegin + nD + 1; T.prevCount = T.count + 1; T.tileSum = T.prevCount + 1;
        T.distance = I.vobsD.p; T.speed = I.vobsD.p + cap; T.shadow = I.vobsShadow.p;
        I.vobsTiles = tiles;
        if (!I.vobsReady) {
            CFB_CUDA(cudaEventCreateWithFlags(&I.vobsReady, cudaEventDisableTiming));
            CFB_CUDA(cudaEventCreateWithFlags(&I.vobsConsumed, cudaEventDisableTiming));
        }
    }
}
static DeviceVehObs vobsOut(const DeviceSim::Impl &I) {
    const VehObsTable &T = I.vobs;
    DeviceVehObs o;
    o.slot = T.slot; o.priority = T.priority; o.drivable = T.drivable;
    o.distance = T.distance; o.speed = T.speed; o.shadow = T.shadow;
    o.drivableBegin = T.drvBegin; o.count = T.count;
    o.capacity = (long long) std::max(I.P, 1);
    o.nDrv = I.V.nDrv;
    o.device = I.opt.device;
    return o;
}

DeviceVehObs DeviceSim::observeVehicles(void *consumerStream) {
    Impl &I = *impl_;
    if (I.V.owned) throw std::runtime_error("observeVehicles: not available on one rank of a sharded run");
    vobsMake(I);
    cudaStream_t cs = (cudaStream_t) consumerStream;
    CFB_CUDA(cudaEventRecord(I.vobsConsumed, cs));         // the consumer's earlier reads finish before the refresh ...
    CFB_CUDA(cudaStreamWaitEvent(I.stream, I.vobsConsumed, 0));
    k_vobs_sums<<<I.vobsTiles, VOBS_TILE, 0, I.stream>>>(I.V, I.vobs);
    k_vobs_fill<<<I.vobsTiles, VOBS_TILE, 0, I.stream>>>(I.V, I.vobs);
    CFB_CUDA(cudaGetLastError());
    CFB_CUDA(cudaEventRecord(I.vobsReady, I.stream));      // ... and its later reads see it, the host waiting for neither
    CFB_CUDA(cudaStreamWaitEvent(cs, I.vobsReady, 0));
    launches_ += 2;
    return vobsOut(I);
}

DeviceVehCtx DeviceSim::observeVehicleContext(void *consumerStream) {
    Impl &I = *impl_;
    View &V = I.V;
    if (V.owned) throw std::runtime_error("observeVehicleContext: not available on one rank of a sharded run");
    vobsMake(I);
    const size_t cap = (size_t) std::max(I.P, 1);
    if (!I.vctxI.p) {   // first call: every row counts as filled, so the first refresh writes the padding of all of them
        std::vector<int> ints(2 * cap + 2, -1);
        ints[2 * cap] = ints[2 * cap + 1] = (int) cap;
        I.vctxI.upload(ints);
        I.vctxGap.alloc(cap);
        I.vctxSignal.alloc(cap);
        legacySync();
        VehCtxTable &C = I.vctx;
        C.leader = I.vctxI.p; C.nextDrivable = C.leader + cap; C.mark = C.nextDrivable + cap; C.par = 0;
        C.gap = I.vctxGap.p; C.signal = I.vctxSignal.p;
    }
    cudaStream_t cs = (cudaStream_t) consumerStream;
    CFB_CUDA(cudaEventRecord(I.vobsConsumed, cs));         // the consumer's earlier reads finish before the refresh ...
    CFB_CUDA(cudaStreamWaitEvent(I.stream, I.vobsConsumed, 0));
    sendPendingPhases(I);
    k_vobs_sums<<<I.vobsTiles, VOBS_TILE, 0, I.stream>>>(V, I.vobs);
    k_vobs_fill<<<I.vobsTiles, VOBS_TILE, 0, I.stream>>>(V, I.vobs);
    const int grid = (int) std::min<size_t>((cap + 255) / 256, (size_t) I.numSMs * 8);
    k_vctx<<<grid, 256, 0, I.stream>>>(V, I.vobs, I.vctx);
    CFB_CUDA(cudaGetLastError());
    I.vctx.par ^= 1;
    CFB_CUDA(cudaEventRecord(I.vobsReady, I.stream));      // ... and its later reads see it, the host waiting for neither
    CFB_CUDA(cudaStreamWaitEvent(cs, I.vobsReady, 0));
    launches_ += 3;
    DeviceVehCtx o;
    o.table = vobsOut(I);
    const VehCtxTable &C = I.vctx;
    o.leader = C.leader; o.gap = C.gap; o.nextDrivable = C.nextDrivable; o.signal = C.signal;
    o.drivableLength = V.drvLength; o.drivableMaxSpeed = V.drvMaxSpeed; o.linkRoadLink = V.llRoadLink;
    o.nLanes = V.nLanes; o.nLinks = V.nLinks;
    return o;
}

void DeviceSim::setCustomSpeedsFromDevice(const int32_t *slot, const int32_t *priority, const double *speed, long long n,
                                          void *producerStream) {
    Impl &I = *impl_;
    if (I.V.owned) throw std::runtime_error("setCustomSpeedsFromDevice: not available on one rank of a sharded run");
    if (n < 0 || n > INT_MAX) throw std::runtime_error("setCustomSpeedsFromDevice: entry count out of range");
    if (!I.speedReady) {
        CFB_CUDA(cudaEventCreateWithFlags(&I.speedReady, cudaEventDisableTiming));
        CFB_CUDA(cudaEventCreateWithFlags(&I.speedTaken, cudaEventDisableTiming));
    }
    if (I.speedStamp.n < (size_t) I.slotCap) {   // first call, or the slot table grew (ensureSlotCapacity synchronised)
        I.speedStamp.alloc((size_t) I.slotCap);
        CFB_CUDA(cudaMemsetAsync(I.speedStamp.p, 0, (size_t) I.slotCap * sizeof(int), I.stream));
        I.speedCall = 0;
    }
    if (++I.speedCall == INT_MAX) {              // stamps of earlier calls must not match a later call's number
        CFB_CUDA(cudaMemsetAsync(I.speedStamp.p, 0, (size_t) I.slotCap * sizeof(int), I.stream));
        I.speedCall = 1;
    }
    cudaStream_t ps = (cudaStream_t) producerStream;
    CFB_CUDA(cudaEventRecord(I.speedReady, ps));
    CFB_CUDA(cudaStreamWaitEvent(I.stream, I.speedReady, 0));
    if (n > 0) {
        const int grid = (int) std::min<long long>((n + 255) / 256, (long long) I.numSMs * 8);
        k_vspeed<<<grid, 256, 0, I.stream>>>(I.V, slot, priority, speed, (int) n, I.speedStamp.p, I.slotCap, I.speedCall);
        CFB_CUDA(cudaGetLastError());
        launches_ += 1;
    }
    CFB_CUDA(cudaEventRecord(I.speedTaken, I.stream));     // the producer may reuse its buffers after this
    CFB_CUDA(cudaStreamWaitEvent(ps, I.speedTaken, 0));
    I.mirrorStale = true;    // k_vspeed may raise ERR_VEHICLE_* outside a step
}

DeviceIntersectionObs DeviceSim::observeIntersections(void *consumerStream) {
    Impl &I = *impl_;
    View &V = I.V;
    if (V.owned) throw std::runtime_error("observeIntersections: not available on one rank of a sharded run");
    if (!I.tobsI.p) {   // first call: the static tables and the columns as they stand before a refresh
        const IntObsLayout X = intObsLayout(I.L, V);
        I.tobsStatic.upload(X.ints.empty() ? std::vector<int>(1, 0) : X.ints);
        I.tobsI.upload(X.initialInts(V));
        I.tobsD.upload(std::vector<double>(std::max(V.nInter, 1), 0.0));
        I.tobsMv.upload(X.phaseMovements);
        legacySync();
        X.point(I.tobs, I.tobsStatic.p);
        X.pointOut(I.tobs, I.tobsOut, V, I.tobsI.p, I.tobsD.p, I.tobsMv.p);
        I.tobsOut.device = I.opt.device;
        CFB_CUDA(cudaEventCreateWithFlags(&I.tobsReady, cudaEventDisableTiming));
        CFB_CUDA(cudaEventCreateWithFlags(&I.tobsConsumed, cudaEventDisableTiming));
    }
    cudaStream_t cs = (cudaStream_t) consumerStream;
    CFB_CUDA(cudaEventRecord(I.tobsConsumed, cs));         // the consumer's earlier reads finish before the refresh ...
    CFB_CUDA(cudaStreamWaitEvent(I.stream, I.tobsConsumed, 0));
    sendPendingPhases(I);
    if (I.tobs.nTl > 0) {
        const int grid = (I.tobs.nTl + TOBS_WARPS - 1) / TOBS_WARPS;
        k_tobs<<<grid, TOBS_WARPS * 32, 0, I.stream>>>(V, I.tobs);
        CFB_CUDA(cudaGetLastError());
        launches_ += 1;
    }
    CFB_CUDA(cudaEventRecord(I.tobsReady, I.stream));      // ... and its later reads see it, the host waiting for neither
    CFB_CUDA(cudaStreamWaitEvent(cs, I.tobsReady, 0));
    return I.tobsOut;
}

DeviceIntersectionObs observeIntersectionsOf(DeviceSim &dev, void *consumerStream) { return dev.observeIntersections(consumerStream); }
DeviceVehObs observeVehiclesOf(DeviceSim &dev, void *consumerStream) { return dev.observeVehicles(consumerStream); }
DeviceVehCtx observeVehicleContextOf(DeviceSim &dev, void *consumerStream) { return dev.observeVehicleContext(consumerStream); }
void setCustomSpeedsOf(DeviceSim &dev, const int32_t *slot, const int32_t *priority, const double *speed, long long n,
                       void *producerStream) {
    dev.setCustomSpeedsFromDevice(slot, priority, speed, n, producerStream);
}

int DeviceSim::runningVehicles(std::vector<SpeedRec> &out) {
    Impl &I = *impl_;
    readCtrlImpl(I.stream, I.hCtrl, I.V.ctrl);
    const int n = I.hCtrl->active;
    out.resize(n);
    if (n == 0) return 0;
    if (I.speedOut.n < (size_t) n) I.speedOut.alloc((size_t) n * 2);
    if (I.scratchI.n < 1) I.scratchI.alloc(std::max(I.V.nLanes, 1));
    CFB_CUDA(cudaMemsetAsync(I.scratchI.p, 0, sizeof(int), I.stream));
    const int TPB = 256;
    k_gather_running<<<(int) (((size_t) I.V.nDrv * 32 + TPB - 1) / TPB), TPB, 0, I.stream>>>(I.V, I.speedOut.p, I.scratchI.p, n);
    CFB_CUDA(cudaMemcpyAsync(out.data(), I.speedOut.p, (size_t) n * sizeof(SpeedRec), cudaMemcpyDeviceToHost, I.stream));
    CFB_CUDA(cudaStreamSynchronize(I.stream));
    launches_ += 1;
    return n;
}

int DeviceSim::drainFinished(std::vector<FinRec> &slots) {
    Impl &I = *impl_;
    readCtrlImpl(I.stream, I.hCtrl, I.V.ctrl);
    const int n = std::min(I.hCtrl->finCount, I.V.finCap);
    slots.resize(n);
    if (n > 0) {
        CFB_CUDA(cudaMemcpyAsync(slots.data(), I.finSlots.p, n * sizeof(int2), cudaMemcpyDeviceToHost, I.stream));
        CFB_CUDA(cudaMemsetAsync(&I.V.ctrl->finCount, 0, sizeof(int), I.stream));
        CFB_CUDA(cudaStreamSynchronize(I.stream));
    }
    return n;
}

void DeviceSim::phases(int32_t *out) {
    Impl &I = *impl_;
    if (I.V.rl && !I.hPhaseStale) { memcpy(out, I.hPhase.data(), I.V.nInter * sizeof(int)); return; }
    CFB_CUDA(cudaMemcpyAsync(out, I.V.curPhase, I.V.nInter * sizeof(int), cudaMemcpyDeviceToHost, I.stream));
    CFB_CUDA(cudaStreamSynchronize(I.stream));
    if (I.V.rl) {
        I.hPhase.assign(out, out + I.V.nInter);
        I.hPhaseStale = false;
    }
}

int DeviceSim::leaderSlotOf(int slot) {
    Impl &I = *impl_;
    if (slot < 0 || slot >= I.slotCap) return -2;
    int p = -1;
    CFB_CUDA(cudaMemcpyAsync(&p, I.V.pos + slot, sizeof(int), cudaMemcpyDeviceToHost, I.stream));
    CFB_CUDA(cudaStreamSynchronize(I.stream));
    if (p < 0) return -2;
    int lp = -1;
    CFB_CUDA(cudaMemcpy(&lp, I.V.leader + p, sizeof(int), cudaMemcpyDeviceToHost));
    if (lp < 0) return -1;
    int4 idv;
    CFB_CUDA(cudaMemcpy(&idv, I.V.ids + lp, sizeof(int4), cudaMemcpyDeviceToHost));
    return idv.x;
}

void DeviceSim::laneVehicleSlots(std::vector<int32_t> &slots, std::vector<int32_t> &laneBeg) {
    Impl &I = *impl_;
    const int nL = I.V.nLanes;
    std::vector<int32_t> cnt(nL);
    laneVehicleCount(cnt.data());
    laneBeg.assign(nL + 1, 0);
    for (int l = 0; l < nL; ++l) laneBeg[l + 1] = laneBeg[l] + cnt[l];
    slots.resize(laneBeg[nL]);
    if (slots.empty()) return;
    DevBuf<int> dBeg, dOut;
    dBeg.upload(std::vector<int>(laneBeg.begin(), laneBeg.end()));
    dOut.alloc(slots.size());
    const int TPB = 256;
    k_lane_slots<<<(nL * 32 + TPB - 1) / TPB, TPB, 0, I.stream>>>(I.V, dOut.p, dBeg.p);
    CFB_CUDA(cudaMemcpyAsync(slots.data(), dOut.p, slots.size() * sizeof(int), cudaMemcpyDeviceToHost, I.stream));
    CFB_CUDA(cudaStreamSynchronize(I.stream));
    launches_ += 1;
}

// The arrays the debug records are assembled from (device_layout.cuh), copied to the host.
struct HostDump {
    std::vector<int> count, leader, del;
    std::vector<double2> kin;
    std::vector<double> gap;
    std::vector<int4> ids, nav;
    std::vector<LcSlot> lc;
    View V{};
};
template <class T> static void copyDown(std::vector<T> &dst, const T *src, size_t n) {
    dst.resize(n);
    if (n) CFB_CUDA(cudaMemcpy(dst.data(), src, n * sizeof(T), cudaMemcpyDeviceToHost));
}
static void dumpToHost(DeviceSim::Impl &I, HostDump &h, bool withLc) {
    CFB_CUDA(cudaStreamSynchronize(I.stream));
    const size_t P = (size_t) I.P;
    copyDown(h.del, I.V.delStep, (size_t) I.slotCap);
    readCtrlImpl(I.stream, I.hCtrl, I.V.ctrl);
    copyDown(h.count, I.V.count, (size_t) I.V.nDrv);
    copyDown(h.leader, I.V.leader, P);
    copyDown(h.kin, I.V.kin, P);
    copyDown(h.ids, I.V.ids, P);
    copyDown(h.nav, I.V.nav, P);
    if (withLc) copyDown(h.lc, I.lcSlot.p, (size_t) I.slotCap);
    else copyDown(h.gap, I.V.gap, P);
    View &V = h.V;
    V.nDrv = I.V.nDrv;
    V.off = I.L.off.data(); V.count = h.count.data(); V.leader = h.leader.data(); V.kin = h.kin.data(); V.gap = h.gap.data();
    V.ids = h.ids.data(); V.nav = h.nav.data(); V.delStep = h.del.data(); V.ctrl = I.hCtrl; V.lc.slot = h.lc.data();
}

void DeviceSim::debugDump(std::vector<DebugRec> &out) {
    HostDump h;
    dumpToHost(*impl_, h, false);
    debugRecords(h.V, impl_->ownedHost.empty() ? nullptr : impl_->ownedHost.data(), out);
}

// ---- snapshot / restore of the whole dynamic state (Archive, archive.cpp:9-151) ----
// The image stays in device memory (a D2D copy at HBM speed); toHost()/fromHost() serialise it.
struct DeviceSim::Snapshot {
    ImageHeader h;
    DevBuf<unsigned char> blob;
};

static std::vector<std::pair<void *, size_t>> snapshotRegions(DeviceSim::Impl &I) {   // device_image.cuh
    return snapshotRegions(I.V, (size_t) I.P, (size_t) I.slotCap);
}

DeviceSim::Snapshot *DeviceSim::snapshot() {
    Impl &I = *impl_;
    CFB_CUDA(cudaStreamSynchronize(I.stream));
    if (I.phaseDirty && I.V.nInter) {   // set_tl_phase calls not sent up yet are part of the state (trafficlight.cpp:39-41 acts at once)
        CFB_CUDA(cudaMemcpyAsync(I.V.curPhase, I.hPhase.data(), I.V.nInter * sizeof(int), cudaMemcpyHostToDevice, I.stream));
        CFB_CUDA(cudaStreamSynchronize(I.stream));
        I.phaseDirty = false;
    }
    auto regs = snapshotRegions(I);
    Snapshot *s = new Snapshot();
    s->h = imageHeader(steps_, I.slotCap, regs);
    s->blob.alloc(s->h.payload());
    size_t off = 0;
    for (auto &r : regs) {
        if (r.second) CFB_CUDA(cudaMemcpyAsync(s->blob.p + off, r.first, r.second, cudaMemcpyDeviceToDevice, I.stream));
        off += imagePad(r.second);
    }
    CFB_CUDA(cudaStreamSynchronize(I.stream));
    return s;
}

void DeviceSim::restore(const Snapshot *s) {
    Impl &I = *impl_;
    ensureSlotCapacity(s->h.slotCap);
    CFB_CUDA(cudaStreamSynchronize(I.stream));
    auto regs = snapshotRegions(I);
    checkImageFits(s->h, regs, I.V);
    applyFills(slotFills(I.V, (size_t) I.slotCap));   // slots beyond the archive's capacity: unused
    legacySync();   // the fills land before the image is copied over them on the engine's stream
    size_t off = 0;
    for (size_t k = 0; k < regs.size(); ++k) {
        const size_t bytes = s->h.regions[k];
        if (bytes) CFB_CUDA(cudaMemcpyAsync(regs[k].first, s->blob.p + off, bytes, cudaMemcpyDeviceToDevice, I.stream));
        off += imagePad(bytes);
    }
    I.hPhase.resize(I.V.nInter);
    if (I.V.nInter) {  // on the engine's stream: it is non-blocking, a plain cudaMemcpy would not wait for the copies above
        CFB_CUDA(cudaMemcpyAsync(I.hPhase.data(), I.V.curPhase, I.V.nInter * sizeof(int), cudaMemcpyDeviceToHost, I.stream));
        CFB_CUDA(cudaStreamSynchronize(I.stream));
    }
    I.phaseDirty = false;
    I.hPhaseStale = false;
    {   // the restored control block decides what the host mirror shows until the next step
        readCtrlImpl(I.stream, I.hCtrl, I.V.ctrl);
        I.epochHost = I.hCtrl->epoch;
        if (I.hMirror) { I.hMirror[1] = I.hCtrl->active; I.hMirror[2] = I.hCtrl->error; I.hMirror[3] = I.hCtrl->ties; I.hMirror[0] = I.hCtrl->epoch; }
        I.mirrorStale = false;
    }
    applyFills(scratchFills(I.V));
    CFB_CUDA(cudaStreamSynchronize(I.stream));
    legacySync();
    steps_ = s->h.steps;
}

void DeviceSim::freeSnapshot(Snapshot *s) { delete s; }

// The image in decoded form (device_image.cuh): the reference-schema JSON archive of host_engine.cpp goes through these.
static ImageGeometry imageGeometry(DeviceSim::Impl &I) {
    return ImageGeometry{I.L.off.data(), I.V.nDrv, I.V.nLanes, I.V.nInter, (size_t) I.P};
}
void DeviceSim::decodeSnapshot(const Snapshot *s, StateImage &out) {
    std::vector<unsigned char> blob;
    snapshotToHost(s, blob);
    decodeImage(blob, imageGeometry(*impl_), out);
}
DeviceSim::Snapshot *DeviceSim::encodeSnapshot(const StateImage &in) {
    std::vector<unsigned char> blob;
    encodeImage(in, imageGeometry(*impl_), blob);
    return snapshotFromHost(blob.data(), blob.size());
}

void DeviceSim::snapshotToHost(const Snapshot *s, std::vector<unsigned char> &out) {
    out.resize(s->h.bytes() + s->h.payload());
    writeImageHeader(s->h, out.data());
    if (s->h.payload()) CFB_CUDA(cudaMemcpy(out.data() + s->h.bytes(), s->blob.p, s->h.payload(), cudaMemcpyDeviceToHost));
}

DeviceSim::Snapshot *DeviceSim::snapshotFromHost(const unsigned char *data, size_t n) {
    Snapshot *s = new Snapshot();
    s->h = readImageHeader(data, n);
    s->blob.alloc(s->h.payload());
    if (s->h.payload()) CFB_CUDA(cudaMemcpy(s->blob.p, data + s->h.bytes(), s->h.payload(), cudaMemcpyHostToDevice));
    legacySync();
    return s;
}

int DeviceSim::slotDelStep(int slot) {
    Impl &I = *impl_;
    if (slot < 0 || slot >= I.slotCap) return INT_MIN;
    int d = INT_MIN;
    if (I.p2p) {   // every rank's finished-vehicle marks through the last completed step (they arrive as peer stores)
        k_wait_fin<<<1, 32, 0, I.stream>>>(I.V, I.S);
        CFB_CUDA(cudaStreamSynchronize(I.stream));
    }
    CFB_CUDA(cudaMemcpy(&d, I.V.delStep + slot, sizeof(int), cudaMemcpyDeviceToHost));
    return d;
}

bool DeviceSim::vehicleState(int slot, VehState &out) {
    Impl &I = *impl_;
    if (slot < 0 || slot >= I.slotCap) return false;
    CFB_CUDA(cudaStreamSynchronize(I.stream));
    int p = -1;
    CFB_CUDA(cudaMemcpy(&p, I.V.pos + slot, sizeof(int), cudaMemcpyDeviceToHost));
    if (p < 0) return false;
    double2 k;
    int4 idv, nv;
    CFB_CUDA(cudaMemcpy(&k, I.V.kin + p, sizeof(k), cudaMemcpyDeviceToHost));
    CFB_CUDA(cudaMemcpy(&idv, I.V.ids + p, sizeof(idv), cudaMemcpyDeviceToHost));
    CFB_CUDA(cudaMemcpy(&nv, I.V.nav + p, sizeof(nv), cudaMemcpyDeviceToHost));
    if (idv.x != slot) return false;
    out.pos = p;
    out.drivable = I.L.posDrv[p];
    out.planIdx = nv.x;
    out.nextDrv = idv.w;
    out.dis = k.x;
    out.speed = k.y;
    return true;
}

void DeviceSim::setCustomSpeed(int slot, double speed) {
    Impl &I = *impl_;
    CFB_CUDA(cudaStreamSynchronize(I.stream));
    int p = -1;
    CFB_CUDA(cudaMemcpy(&p, I.V.pos + slot, sizeof(int), cudaMemcpyDeviceToHost));
    double *dst = p >= 0 ? I.V.cust + p : I.V.slotCust + slot;
    double old = 0;
    CFB_CUDA(cudaMemcpy(&old, dst, sizeof(double), cudaMemcpyDeviceToHost));
    CFB_CUDA(cudaMemcpy(dst, &speed, sizeof(double), cudaMemcpyHostToDevice));
    if (old != old) {  // was unset: one more outstanding request
        readCtrlImpl(I.stream, I.hCtrl, I.V.ctrl);
        int n = I.hCtrl->nCustom + 1;
        CFB_CUDA(cudaMemcpy(&I.V.ctrl->nCustom, &n, sizeof(int), cudaMemcpyHostToDevice));
    }
    legacySync();
}

void DeviceSim::setVehiclePlan(int slot, int planId, int planIdx, int nextDrv) {
    Impl &I = *impl_;
    CFB_CUDA(cudaStreamSynchronize(I.stream));
    int p = -1;
    CFB_CUDA(cudaMemcpy(&p, I.V.pos + slot, sizeof(int), cudaMemcpyDeviceToHost));
    if (p >= 0) {
        CFB_CUDA(cudaMemcpy(&I.V.nav[p].x, &planIdx, sizeof(int), cudaMemcpyHostToDevice));
        CFB_CUDA(cudaMemcpy(&I.V.ids[p].w, &nextDrv, sizeof(int), cudaMemcpyHostToDevice));
    } else {
        CFB_CUDA(cudaMemcpy(&I.V.slotInfo[slot].z, &planId, sizeof(int), cudaMemcpyHostToDevice));
    }
    legacySync();
}

void DeviceSim::setPhase(int intersection, int phase) {
    Impl &I = *impl_;
    // TrafficLight::setPhase only changes curPhaseIndex (trafficlight.cpp:39-41).  Only reachable in
    // rlTrafficLight mode, where the device never advances phases itself, so the host copy is
    // authoritative; all changes made between two steps go up in one copy (see step()).
    if (I.hPhaseStale) {  // phases were last set on the device: start from what is there
        CFB_CUDA(cudaMemcpyAsync(I.hPhase.data(), I.V.curPhase, I.V.nInter * sizeof(int), cudaMemcpyDeviceToHost, I.stream));
        CFB_CUDA(cudaStreamSynchronize(I.stream));
        I.hPhaseStale = false;
    }
    I.hPhase[intersection] = phase;
    I.phaseDirty = true;
}

// ------------------------------------------------------------------------------------------
// Lane change (device_lc.cuh).
void DeviceSim::uploadLanePlans(const Routing &routing) {
    Impl &I = *impl_;
    CFB_CUDA(cudaStreamSynchronize(I.stream));
    const LanePlanTables T = lanePlanTables(routing);
    I.lcPlanRoute.upload(T.planRoute); I.lcPlanRoadPos.upload(T.planRoadPos); I.lcLanePlanRoad.upload(T.lanePlanRoad);
    I.lcLanePlanBeg.upload(T.lanePlanBeg); I.lcLanePlanId.upload(T.lanePlanId); I.lcRouteLastRoad.upload(T.routeLastRoad);
    LcView &C = I.V.lc;
    C.planRoute = I.lcPlanRoute.p; C.planRoadPos = I.lcPlanRoadPos.p;
    C.lanePlanRoad = I.lcLanePlanRoad.p; C.lanePlanBeg = I.lcLanePlanBeg.p; C.lanePlanId = I.lcLanePlanId.p;
    C.routeLastRoad = I.lcRouteLastRoad.p;
    legacySync();
}

void DeviceSim::enableLaneChange(const RoadNet &, const Routing &routing) {
    Impl &I = *impl_;
    View &V = I.V;
    CFB_CUDA(cudaStreamSynchronize(I.stream));
    const DeviceLayout &L = I.L;
    I.lcSegBeg.upload(L.segBeg); I.lcSegStart.upload(L.segStart); I.lcLaneIdx.upload(L.laneIdx); I.lcLaneRoadN.upload(L.laneRoadN);
    I.lcLaneWidth.upload(L.laneWidth); I.lcPosDrv.upload(L.posDrv); I.lcLaneRoad.upload(L.laneRoad);
    V.lc.laneRoad = I.lcLaneRoad.p;
    I.lcSegIdx.alloc(I.P); I.lcSegIdx.fill(0);
    I.lcCand.alloc(LC_MAX_CAND); I.lcInvolved.alloc(LC_MAX_CAND); I.lcShadowLog.alloc(LC_MAX_CAND); I.lcPrio.alloc(LC_MAX_CAND);
    I.lcCtrl.alloc(1); I.lcCtrl.fill(0);
    I.lcScratch.alloc((size_t) 4 * LC_MAX_CAND); I.lcScratch.fill(0);
    if (const char *g = getenv("CITYFLOW_B200_LC_SERIAL")) I.lcSerial = g[0] == '1';
    I.lcSlot.alloc(std::max(I.slotCap, 1)); I.lcSlot.fill(0);
    CFB_CUDA(cudaMallocHost(&I.hLcCtrl, sizeof(LcCtrl)));
    LcView &C = V.lc;
    C.slot = I.lcSlot.p; C.segIdx = I.lcSegIdx.p; C.posDrv = I.lcPosDrv.p; C.segBeg = I.lcSegBeg.p; C.segStart = I.lcSegStart.p;
    C.laneIdx = I.lcLaneIdx.p; C.laneRoadN = I.lcLaneRoadN.p; C.laneWidth = I.lcLaneWidth.p;
    C.cand = I.lcCand.p; C.involved = I.lcInvolved.p; C.shadowLog = I.lcShadowLog.p; C.ctrl = I.lcCtrl.p;
    C.scratchA = I.lcScratch.p; C.scratchB = I.lcScratch.p + LC_MAX_CAND; C.scratchC = I.lcScratch.p + 2 * LC_MAX_CAND;
    C.scratchD = I.lcScratch.p + 3 * LC_MAX_CAND;
    C.spare = nullptr; C.nSpare = 0;
    V.lcOn = 1;
    I.useGraph = false;   // the step has a host round trip in the middle (shadow priorities come from the engine RNG)
    I.useCoop = false;
    legacySync();
    uploadLanePlans(routing);
}

void DeviceSim::stepLcBegin(const SpawnRec *recs, int n, const int32_t *spare, int nSpare, std::vector<LcShadow> &created) {
    stageStep(recs, n);
    Impl &I = *impl_;
    View &V = I.V;
    cudaStream_t s = I.stream;
    const int TPB = 256;
    I.ensureGrids();
    if (nSpare > I.lcSpareCap) {
        CFB_CUDA(cudaStreamSynchronize(s));
        I.lcSpareCap = std::max(1024, nSpare * 2);
        I.lcSpare.alloc(I.lcSpareCap);
    }
    if (nSpare > 0) CFB_CUDA(cudaMemcpyAsync(I.lcSpare.p, spare, nSpare * sizeof(int), cudaMemcpyHostToDevice, s));
    V.lc.spare = I.lcSpare.p;
    V.lc.nSpare = nSpare;
    k_lc_begin<<<1, 1, 0, s>>>(V.lc);
    I.launchStep(Impl::INGEST, false);
    k_lc_admitted<<<I.gridNotify, TPB, 0, s>>>(V, V.lc);
    k_lc_segments<<<I.gridNotify, TPB, 0, s>>>(V, V.lc);
    k_lc_signal<<<I.gridControl, TPB, 0, s>>>(V, V.lc);
    if (I.lcSerial) {
        k_lc_schedule<<<1, 32, 0, s>>>(V, V.lc);
    } else {
        k_lc_order<<<1, 256, 0, s>>>(V, V.lc);
        k_lc_schedule_roads<<<LC_MAX_CAND / 128, 128, 0, s>>>(V, V.lc);
        k_lc_log<<<1, 32, 0, s>>>(V, V.lc);
    }
    CFB_CUDA(cudaMemcpyAsync(I.hLcCtrl, I.lcCtrl.p, sizeof(LcCtrl), cudaMemcpyDeviceToHost, s));
    CFB_CUDA(cudaStreamSynchronize(s));
    CFB_CUDA(cudaGetLastError());
    lcCheckCapacity(I.hLcCtrl->error);
    const int ns = I.hLcCtrl->nShadows;
    created.resize(ns);
    if (ns > 0) {
        static_assert(sizeof(LcShadow) == sizeof(int2), "LcShadow layout");
        CFB_CUDA(cudaMemcpyAsync(created.data(), I.lcShadowLog.p, ns * sizeof(int2), cudaMemcpyDeviceToHost, s));
        CFB_CUDA(cudaStreamSynchronize(s));
    }
    launches_ += 6;
}

void DeviceSim::stepLcEnd(const int32_t *priorities, int n) {
    Impl &I = *impl_;
    View &V = I.V;
    cudaStream_t s = I.stream;
    const int TPB = 256;
    if (n > 0) {
        CFB_CUDA(cudaMemcpyAsync(I.lcPrio.p, priorities, n * sizeof(int), cudaMemcpyHostToDevice, s));
        k_lc_priorities<<<(n + 127) / 128, 128, 0, s>>>(V, V.lc, I.lcPrio.p, n);
    }
    k_lc_leader<<<I.gridNotify, TPB, 0, s>>>(V, V.lc);
    I.launchStep(Impl::NOTIFY, false);
    I.launchStep(Impl::CONTROL, false);
    if (I.lcSerial) {
        k_lc_control_tail<<<1, 32, 0, s>>>(V, V.lc);
    } else {
        k_lc_tail_order<<<1, 256, 0, s>>>(V, V.lc);
        k_lc_tail_roads<<<LC_MAX_CAND / 128, 128, 0, s>>>(V, V.lc);
        k_lc_tail_clear<<<1, 32, 0, s>>>(V, V.lc);
    }
    I.launchStep(Impl::MOVE, false);
    I.launchStep(Impl::LEADER, false);
    CFB_CUDA(cudaGetLastError());
    launches_ += 6 + (n > 0);
    steps_ += 1;
    I.epochHost += 1;
}

void DeviceSim::debugDumpLc(std::vector<LcDebugRec> &out) {
    HostDump h;
    dumpToHost(*impl_, h, true);
    lcDebugRecords(h.V, out);
}

}  // namespace cfb
