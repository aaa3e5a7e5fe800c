// Device-resident simulation state + the per-step kernel sequence (implemented in
// device_sim.cu).  This is the internal C++ seam between the host engine (flows, RNG, ids; see
// host_engine.cpp) and the CUDA path; the public boundary is the C-ABI in
// include/cityflow_b200.h.  No CUDA types appear here so host-only translation units can
// include it.
#pragma once
#include <cstdint>
#include <stdexcept>
#include <string>
#include <vector>

#include "flows.h"
#include "roadnet.h"

namespace cfb {

// One vehicle handed to the device this step: it is appended to `lane`'s waiting queue
// (Lane::pushWaitingVehicle, roadnet.h:365).  Records of one step must be sorted by lane,
// stable in spawn order.
struct SpawnRec {
    int32_t slot;      // host-allocated stable vehicle handle
    int32_t lane;      // first drivable
    int32_t tmpl;      // index into the template table
    int32_t priority;  // Vehicle::priority (vehicle.cpp:45)
    int32_t plan;      // index into the plan table (route x start lane)
    int32_t pad[3];
};

struct FinRec {        // a vehicle that ran off its last road during step `step` (0-based)
    int32_t slot;
    int32_t step;
};

struct SpeedRec {      // one running vehicle for get_vehicle_speed / get_vehicle_distance
    int32_t slot;
    int32_t drivable;
    double speed;
    double dis;
};

struct DebugRec {      // full per-vehicle state for parity tests (cfb_debug_vehicles)
    int32_t slot, drivable, leaderSlot, blockerSlot, priority, enterLaneLinkTime, listIndex, pad;
    double dis, speed, gap;
};

// The dynamic state at a step boundary in decoded form: what Archive::dump writes per vehicle, drivable and
// traffic light (archive.cpp:179-343).  Vehicles are named by slot; DeviceSim::decodeSnapshot / encodeSnapshot
// translate between this and the device image (device_image.cuh).
struct StateImage {
    struct Running {
        int32_t slot, tmpl, priority;
        int32_t planIdx;            // absolute index into the plan table of the vehicle's current drivable
        int32_t nextDrivable;       // plan[planIdx + 1] (PLAN_END / PLAN_DEAD past the last road)
        int32_t prevDrivable;       // -1 none
        int32_t blockerSlot;        // -1 none
        int32_t leaderSlot;         // -1 none
        int32_t enterLaneLinkTime;
        double dis, speed, gap;     // gap: meaningful with a leader
        double len;                 // of the vehicle's template (encode only: the drivable's tail record)
    };
    struct Waiting { int32_t slot, tmpl, priority, plan; };
    std::vector<std::vector<Running>> drivables;   // per drivable, list order (front first)
    std::vector<std::vector<Waiting>> waiting;     // per lane, queue order
    std::vector<int32_t> curPhase;                 // per intersection
    std::vector<double> remain;
    long long step = 0;
    int active = 0;
    int slotCount = 0;             // slots in use: 0 .. slotCount-1
};

enum DeviceError : int {
    ERR_BUCKET_OVERFLOW = 1,    // more vehicles on a drivable than its bucket holds
    ERR_ENTRANT_OVERFLOW = 2,   // more vehicles entering one drivable in one step than staged
    ERR_MOVER_OVERFLOW = 4,
    ERR_ROUTE_DEAD_END = 8,     // lane cannot reach the next road of the route (reference asserts)
    ERR_FINISHED_OVERFLOW = 16,
    ERR_PHASE_RANGE = 32,       // a phase index handed over on the device is outside the intersection's phase list
    ERR_SHARD_TIMEOUT = 64,     // sharded run: a peer's seam message did not arrive (peer crashed or stopped stepping)
    ERR_VEHICLE_STALE = 128,    // a custom speed handed over on the device names a vehicle that is no longer running
    ERR_VEHICLE_DUPLICATE = 256,   // ... or names one vehicle twice in one call
};

struct DeviceSimOptions {
    int device = 0;
    double interval = 1.0;
    bool rlTrafficLight = false;
    int slotCapacity = 1 << 18;
    int replicas = 1;           // bench only: K independent copies of the scenario in one engine
};

// The staged exchange's device buffers (all on `stream`), for a caller of shardSegment that moves them itself.  Per peer
// q the tail / mover messages of the lanes shared with q are contiguous: entries [beg[q], beg[q+1]).
class ShardTransport;

struct ShardBuffers {
    void *stream = nullptr;
    void *tailSend = nullptr, *tailRecv = nullptr, *moverSend = nullptr, *moverRecv = nullptr;
    size_t tailBytes = 0, moverBytes = 0;       // bytes per boundary lane
    std::vector<int> outBeg, inBeg;             // lanes this rank feeds / owns, per peer (prefix sums)
    void *blkSend = nullptr, *blkAll = nullptr; // blocker changes: own list, all ranks' lists
    size_t blkBytesPerRank = 0;
};

struct DeviceObs {
    const int32_t *laneCount = nullptr;     // nLanes ints, roadnet lane order
    const int32_t *laneWaiting = nullptr;   // nLanes ints, speed < 0.1
    const double *laneSpeedSum = nullptr;   // nLanes doubles
    int nLanes = 0;
    int device = 0;
};

// The per-vehicle observation table (device_vehobs.cuh): every running vehicle, drivable-major, list order.  Rows at and
// beyond *count are padding (slot -1).
struct DeviceVehObs {
    const int32_t *slot = nullptr, *priority = nullptr, *drivable = nullptr;
    const double *distance = nullptr, *speed = nullptr;
    const uint8_t *shadow = nullptr;
    const int32_t *drivableBegin = nullptr;   // nDrv + 1 entries
    const int32_t *count = nullptr;           // device scalar
    long long capacity = 0;                   // rows
    int nDrv = 0;
    int device = 0;
};

// What lies ahead of every row of the per-vehicle table (device_vehobs.cuh, VehCtxTable), refreshed together with the
// table; capacity rows each, aligned with its rows.  The static arrays alias the engine's own tables.
struct DeviceVehCtx {
    DeviceVehObs table;
    const int32_t *leader = nullptr;          // row of the leader, -1 none
    const double *gap = nullptr;              // ControllerInfo::gap to it, +inf without a leader
    const int32_t *nextDrivable = nullptr;    // Router::getNextDrivable; PLAN_END / PLAN_DEAD where there is none
    const int8_t *signal = nullptr;           // a lane row heading for a laneLink: its roadLink available now (1) or not (0); else -1
    const double *drivableLength = nullptr, *drivableMaxSpeed = nullptr;   // static: nDrv each
    const int32_t *linkRoadLink = nullptr;    // static: nLinks
    int nLanes = 0, nLinks = 0;
};

// The per-intersection and per-movement observations (device_tlobs.cuh).  A movement is a roadLink, in RoadNet's global
// roadLink order.  The dynamic columns are refreshed by observeIntersections; the static ones are written once.
struct DeviceIntersectionObs {
    const int32_t *phase = nullptr;                // nInter: current phase index, -1 for a virtual intersection
    const double *phaseRemaining = nullptr;        // nInter: View::remain (0 for a virtual intersection)
    const int32_t *pressure = nullptr, *queue = nullptr;   // nInter
    const int32_t *movementIn = nullptr, *movementInWaiting = nullptr, *movementOut = nullptr, *movementInside = nullptr,
                  *movementPressure = nullptr;     // nRL each
    const int32_t *phasePressure = nullptr;        // nInter x maxPhases, INT32_MIN past the intersection's phase count
    const int32_t *movementBegin = nullptr;        // static: nInter + 1
    const int32_t *movementIntersection = nullptr; // static: nRL
    const int32_t *phaseCount = nullptr;           // static: nInter
    const uint8_t *phaseMovements = nullptr;       // static: nInter x maxPhases x maxMovements
    int nInter = 0, nRL = 0, maxPhases = 0, maxMovements = 0;
    int device = 0;
};

class DeviceSim {
public:
    // Throws std::runtime_error when no CUDA device / extension is usable (no CPU fallback).
    DeviceSim(const RoadNet &net, const std::vector<VehicleTemplate> &templates, const Routing &routing,
              const DeviceSimOptions &opt);
    ~DeviceSim();
    DeviceSim(const DeviceSim &) = delete;
    DeviceSim &operator=(const DeviceSim &) = delete;

    // Re-upload the (grown) template / plan tables.  A template whose length + minGap is below bucketSpacing() would
    // not fit the lane buckets: the host engine refuses it before it gets here.
    void uploadTemplates(const std::vector<VehicleTemplate> &templates);
    // The vehicle spacing (length + minGap) the lane buckets were sized for when the engine was made (device_layout.cuh)
    double bucketSpacing() const;
    void uploadPlans(const Routing &routing);
    void ensureSlotCapacity(int slots);

    // ---- sharded mode (see shard.h for the protocol) ----
    void configureShard(int rank, int world, const std::vector<unsigned char> &owned,
                        const std::vector<std::vector<int>> &feedPerPeer, const std::vector<std::vector<int>> &ownPerPeer,
                        const std::vector<std::vector<int>> &boundarySize, const std::vector<unsigned char> &ownedRoadLinks);
    // peer-memory transport (device_shard.cuh): the arena peers write into; connect once every rank's arena is mapped
    struct ShardArena { void *base; size_t bytes; };
    ShardArena shardArena();
    void shardConnect(const std::vector<void *> &peerBase);
    void shardMarkArenaExported();   // other processes map the arena: it must outlive them (never freed)
    // One step of one rank of a multi-process run (asynchronous): the whole kernel sequence with both seam exchanges,
    // over peer memory once connected, else staged through `t`; replayed as a CUDA graph from the ninth step on.
    void shardStep(const SpawnRec *recs, int n, ShardTransport *t);
    // The same step for a caller that moves the seam records itself (the loop-back group): stageStep, then segment k =
    //   0  ingest, notify, control, send (peer memory) or pack the movers
    //   1  receive or unpack the movers, move, send or pack the tails and seal the blocker list
    //   2  receive or unpack the tails, apply the blocker lists, leader; counts the step
    // with the movers' exchange between 0 and 1, and the tails' and blocker lists' between 1 and 2.
    void stageStep(const SpawnRec *recs, int n);
    void shardSegment(int k);
    ShardBuffers shardBuffers();     // what the staged exchanges move
    void shardCounts(ShardTransport *t, int32_t *laneOut, int *activeOut);   // global sums (collective)
    bool shardVehicleCount(int *activeOut);        // the same count over the peer-memory arena (no all-reduce); false = unavailable
    void shardWaitingCounts(ShardTransport *t, int32_t *laneOut);
    void shardGatherFinished(ShardTransport *t, std::vector<FinRec> &inout);

    // Enqueue one simulation step (asynchronous). `recs` must stay valid until the call returns.
    void step(const SpawnRec *recs, int n);
    void synchronize();

    // Observations left on the device for a consumer on the same GPU: refreshed on the engine's
    // stream, ordered against `consumerStream` (a cudaStream_t; null = legacy default stream) with
    // events in both directions, no host synchronisation.  Valid until the next call.
    DeviceObs observeOnDevice(void *consumerStream);
    // rlTrafficLight actions handed over on the device: `phases` = one int per intersection
    // (roadnet order, entries of virtual intersections ignored) in device memory, produced on
    // `producerStream`.  Same effect as setPhase() on every signalised intersection
    // (trafficlight.cpp:39-41); an out-of-range index leaves that light unchanged and raises
    // ERR_PHASE_RANGE.  No host synchronisation.
    void setPhasesFromDevice(const int32_t *phases, void *producerStream);
    // The table of every running vehicle, refreshed on the engine's stream with the same handshake as observeOnDevice.
    // The buffers are made once (their capacity is numPositions() rows); valid until the next call.
    DeviceVehObs observeVehicles(void *consumerStream);
    // setCustomSpeed for n vehicles at once, handed over on the device (produced on `producerStream`) as the handles of
    // observation rows: entries with slot < 0 are skipped, a handle that no longer names the running vehicle raises
    // ERR_VEHICLE_STALE, a slot named twice ERR_VEHICLE_DUPLICATE.  No host synchronisation.
    void setCustomSpeedsFromDevice(const int32_t *slot, const int32_t *priority, const double *speed, long long n,
                                   void *producerStream);
    // Every light's phase and every movement's queue and pressure, refreshed on the engine's stream with the same
    // handshake as observeOnDevice, after the setPhase calls not yet sent to the device.  The buffers are made on the
    // first call and keep their addresses for the engine's lifetime; their content is valid until the next call.
    DeviceIntersectionObs observeIntersections(void *consumerStream);
    // The per-vehicle table (as observeVehicles) and, for every row, its leader, the gap to it, its next drivable and the
    // light at its stop line, in one refresh with the same handshake, after the setPhase calls not yet sent to the
    // device.  The buffers are made on the first call and keep their addresses; their content is valid until the next call.
    DeviceVehCtx observeVehicleContext(void *consumerStream);
    // Observations (synchronise the stream).
    int vehicleCount();
    int errorFlags();
    int tieCount();                               // see cfb_tie_count
    long long stepsDone() const { return steps_; }
    void laneVehicleCount(int32_t *out);          // nLanes * replicas
    void laneWaitingVehicleCount(int32_t *out);   // speed < 0.1
    int runningVehicles(std::vector<SpeedRec> &out);
    int drainFinished(std::vector<FinRec> &out);     // vehicles that left the network since the last drain
    void phases(int32_t *out);
    int leaderSlotOf(int slot);                   // -1 none, -2 unknown/not running
    void laneVehicleSlots(std::vector<int32_t> &slots, std::vector<int32_t> &laneBeg);
    void debugDump(std::vector<DebugRec> &out);   // every running vehicle, drivable-major, list order

    struct VehState { int pos, drivable, planIdx, nextDrv; double dis, speed; };
    bool vehicleState(int slot, VehState &out);          // false: not running
    int slotDelStep(int slot);                           // step at which the slot's vehicle left (very negative: never)
    void setCustomSpeed(int slot, double speed);         // Vehicle::setCustomSpeed (running or queued vehicle)
    void setVehiclePlan(int slot, int planId, int planIdx, int nextDrv);

    // Control.
    void setPhase(int intersection, int phase);
    void reset();
    // Whole dynamic state image (device resident); see Archive in host_engine.cpp.
    struct Snapshot;
    Snapshot *snapshot();
    void restore(const Snapshot *s);
    static void freeSnapshot(Snapshot *s);
    static void snapshotToHost(const Snapshot *s, std::vector<unsigned char> &out);
    static Snapshot *snapshotFromHost(const unsigned char *data, size_t n);
    // the image in decoded form (the reference's JSON archive, host_engine.cpp); not with lane change
    void decodeSnapshot(const Snapshot *s, StateImage &out);
    Snapshot *encodeSnapshot(const StateImage &in);

    // Measurement support for bench.py / profiles (CUDA-event timing of one kernel across launches).
    struct KernelTimes { double ingest = 0, notify = 0, control = 0, move = 0, leader = 0; long long launches = 0; };
    void enableKernelTiming(bool on);
    // sharded step, phase by phase: ingest | notify+control | send movers | recv movers | move | send tails | recv tails | leader
    static constexpr int SHARD_PHASES = 8;
    void shardStepTimes(double ms[SHARD_PHASES], long long *steps);
    void flushL2();                 // 256 MiB memset on the engine stream
    void markTimed();               // record an event; brackets are (even, odd) pairs
    double collectTimedMs();        // sync; sum of bracket durations; clears the brackets
    unsigned long long vehicleSteps();
    void debugCounters(unsigned long long out[8], bool clear);
    int debugArrays(unsigned *cyc, unsigned *path);   // numPositions() entries each  // CFB_DEBUG_COUNTERS builds only  // device-side sum of the vehicle count after every step
    KernelTimes kernelTimes();
    long long launchesDone() const { return launches_; }
    // launch form of the last single-GPU step (see cfb_debug_launch_form): {graph, pdl, coop, mirror}
    void launchForm(int out[4]) const;
    // blocks of the list-driven step kernels: k_notify, k_control, k_move, k_leader, k_step (0 = not sized yet)
    void stepGrids(int out[5]) const;
    int numPositions() const;
    int numDrivables() const;
    int device() const;   // CUDA device ordinal the engine lives on

    // ---- lane change (device_lc.cuh) ----
    struct LcShadow { int32_t parentSlot, shadowSlot; };
    struct LcDebugRec {   // every running vehicle incl. shadows; mirrors oracle/harness.py LC_DTYPE with slots for identities
        int32_t slot, priority, partnerType, partnerSlot, drivable, leaderSlot, blockerSlot, flags, lastDir, pad;
        double dis, speed, gap, offset, waiting, lastChange;
    };
    // allocate the lane-change state and upload its static tables (segments, lane geometry, lane plans)
    void enableLaneChange(const RoadNet &net, const Routing &routing);
    void uploadLanePlans(const Routing &routing);
    // Candidates a step can schedule (LC_MAX_CAND, device_lc_types.cuh).  Each creates at most one shadow, so this
    // many spare slots always suffice.
    static constexpr int LC_MAX_CANDIDATES = 4096;
    // Throws for the bits the lane-change kernels set in LcCtrl::error (device_lc.cuh, device_control.cuh).
    static void lcCheckCapacity(int error) {
        if (error & 1)
            throw std::runtime_error("cityflow_b200: more than " + std::to_string(LC_MAX_CANDIDATES) +
                                     " lane-change candidates or involved vehicles in one step");
        if (error & 2) throw std::runtime_error("cityflow_b200: lane change ran out of spare slots for shadows");
    }
    // First half of a step: ingest, segment index, signals, scheduling.  `spare` = free slots lent for this
    // step's shadows; the device takes them from the front.  Synchronises and returns the shadows created, in
    // schedule order (= the order their priorities are drawn from the engine RNG, vehicle.cpp:33).  Throws when
    // the step found more than LC_MAX_CANDIDATES candidates or used up the spares.
    void stepLcBegin(const SpawnRec *recs, int n, const int32_t *spare, int nSpare, std::vector<LcShadow> &created);
    // Second half: the drawn priorities, then leader pass, notify, control (+ sequential tail), move, leader.
    void stepLcEnd(const int32_t *priorities, int n);
    void debugDumpLc(std::vector<LcDebugRec> &out);

    struct Impl;

private:
    Impl *impl_;
    long long steps_ = 0;
    long long launches_ = 0;
};

// DeviceSim::observeVehicles / setCustomSpeedsFromDevice as free functions, for the C-ABI (host_engine.cpp).  Weak: the
// host engine is also linked against a DeviceSim without the per-vehicle device path (the emulated device of the CPU
// suite), where they stay null and the C-ABI reports the entry points as unavailable.
__attribute__((weak)) DeviceVehObs observeVehiclesOf(DeviceSim &dev, void *consumerStream);
__attribute__((weak)) void setCustomSpeedsOf(DeviceSim &dev, const int32_t *slot, const int32_t *priority, const double *speed,
                                             long long n, void *producerStream);
// DeviceSim::observeIntersections, weak for the same reason.
__attribute__((weak)) DeviceIntersectionObs observeIntersectionsOf(DeviceSim &dev, void *consumerStream);
// DeviceSim::observeVehicleContext, weak for the same reason.
__attribute__((weak)) DeviceVehCtx observeVehicleContextOf(DeviceSim &dev, void *consumerStream);

}  // namespace cfb
