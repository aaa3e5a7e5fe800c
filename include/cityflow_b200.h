/* cityflow_b200 -- C ABI of the H100-native CityFlow step engine.
 *
 * The reference has no C interface: its boundary is the C++ class CityFlow::Engine
 * (src/engine/engine.h:114-183) exposed to Python by pybind11 (src/cityflow.cpp:10-48).  This
 * header is the C-ABI a binding for that class would call: one function per public Engine
 * method on the hot path, plain pointers and sizes, caller-allocated output buffers, no C++ or
 * torch types.  Every entry cites the reference method it replaces.  The pybind11 module shipped
 * in cityflow_b200/ (class `Engine`, same signatures as src/cityflow.cpp) is a thin wrapper over
 * exactly these functions; INTEGRATION.md shows the equivalent binding a reference maintainer
 * would add.
 *
 * Conventions: functions returning int return 0 on success and a negative code on failure, the
 * message is available from cfb_last_error().  An engine is not thread-safe; distinct engines
 * may be driven from distinct threads.  All simulation state lives in GPU memory; there is no
 * CPU fallback: cfb_engine_create fails when no CUDA device is usable.
 */
#ifndef CITYFLOW_B200_H
#define CITYFLOW_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct cfb_engine cfb_engine;

/* A vehicle as the reference names it: "flow_<flow>_<index>" (flow.cpp:11) or, for vehicles
 * added with push_vehicle, "manually_pushed_<index>" (engine.cpp:714; flow == -2). */
typedef struct cfb_vehicle_ref {
    int32_t flow;
    int32_t index;
} cfb_vehicle_ref;

enum {
    CFB_OK = 0,
    CFB_ERR_LOAD = -1,        /* config / roadnet / flow could not be loaded (engine.cpp:21-24) */
    CFB_ERR_DEVICE = -2,      /* CUDA error or no device */
    CFB_ERR_ARGUMENT = -3,    /* unknown id, buffer too small, ... */
    CFB_ERR_CAPACITY = -4,    /* a device-side bucket / ring overflowed */
    CFB_ERR_UNSUPPORTED = -5  /* feature of the reference not built here (laneChange, archive) */
};

/* Engine::Engine(configFile, threadNum)  engine.cpp:13-34.  thread_num is accepted for signature
 * compatibility and ignored (the kernel sequence is the thread pool).  `device` < 0 selects the
 * current CUDA device (LOCAL_RANK-aware callers pass their rank).  Returns NULL on failure; the
 * reason is then available from cfb_last_error(NULL). */
cfb_engine *cfb_engine_create(const char *config_file, int thread_num, int device);
/* Engine::~Engine  engine.cpp:762-771 */
void cfb_engine_destroy(cfb_engine *e);
/* message of the last failure on `e` (or of the last failed create when e == NULL) */
const char *cfb_last_error(const cfb_engine *e);

/* Engine::nextStep  engine.cpp:566-594.  Enqueues the kernel sequence for one step and returns
 * without waiting for the GPU; observations synchronise. */
int cfb_next_step(cfb_engine *e);
/* n consecutive steps (no reference counterpart; saves n-1 host round trips) */
int cfb_next_steps(cfb_engine *e, int n);
/* Engine::getVehicleCount  engine.cpp:615 */
int64_t cfb_get_vehicle_count(cfb_engine *e);
/* Engine::getCurrentTime  engine.cpp:678 */
double cfb_get_current_time(const cfb_engine *e);
/* Engine::getAverageTravelTime  engine.cpp:682-691 */
double cfb_get_average_travel_time(cfb_engine *e);

/* Static id tables.  Lanes are indexed in roadnet order (RoadNet::getLanes, roadnet.cpp:314-318);
 * lane ids are "<roadId>_<laneIndex>" (roadnet.h:323-325). */
int cfb_num_lanes(const cfb_engine *e);
const char *cfb_lane_id(const cfb_engine *e, int lane);
int cfb_num_intersections(const cfb_engine *e);
const char *cfb_intersection_id(const cfb_engine *e, int intersection);

/* Engine::getLaneVehicleCount  engine.cpp:628-634: out[lane] for all cfb_num_lanes() lanes */
int cfb_get_lane_vehicle_count(cfb_engine *e, int32_t *out, int n);
/* Engine::getLaneWaitingVehicleCount  engine.cpp:636-648 (speed < 0.1) */
int cfb_get_lane_waiting_vehicle_count(cfb_engine *e, int32_t *out, int n);
/* The same per-lane observations left ON THE DEVICE for a consumer on the same GPU (the policy
 * network of an RL loop): no device->host copy, no host synchronisation.  The three arrays
 * (cfb_num_lanes() entries each, roadnet lane order) are refreshed on the engine's stream and
 * ordered against `consumer_stream` (a cudaStream_t; NULL = the legacy default stream) in both
 * directions, so kernels enqueued on that stream after this call read this step's values and the
 * next refresh waits for the reads enqueued before it.  The pointers stay valid for the engine's
 * lifetime; their content is valid until the next cfb_observe_device call.
 * lane_speed_sum / lane_vehicle_count = the mean speed the reference's users derive from
 * getVehicleSpeed + getLaneVehicles (engine.cpp:650-668).  Single-GPU engines only. */
typedef struct {
    const int32_t *lane_vehicle_count;   /* engine.cpp:628-634 */
    const int32_t *lane_waiting_count;   /* engine.cpp:636-648 (speed < 0.1) */
    const double *lane_speed_sum;
    int32_t n_lanes;
    int32_t device;                      /* CUDA device ordinal the pointers live on */
} cfb_device_obs;
int cfb_observe_device(cfb_engine *e, void *consumer_stream, cfb_device_obs *out);
/* Engine::getVehicleSpeed  engine.cpp:662-668 / getVehicleDistance :670-676: running vehicles in
 * vehiclePool (priority) order.  Returns the number of running vehicles (may exceed cap; only
 * cap entries are written); any of the three output pointers may be NULL. */
int64_t cfb_get_vehicle_speed(cfb_engine *e, cfb_vehicle_ref *ids, double *speed, double *distance, int64_t cap);
/* Engine::getVehicles(includeWaiting)  engine.cpp:619-626 */
int64_t cfb_get_vehicles(cfb_engine *e, int include_waiting, cfb_vehicle_ref *ids, int64_t cap);
/* Engine::getLaneVehicles  engine.cpp:650-660: CSR over lanes, lane_begin has n_lanes+1 entries */
int64_t cfb_get_lane_vehicles(cfb_engine *e, int64_t *lane_begin, int n_lanes_plus1, cfb_vehicle_ref *ids, int64_t cap);
/* Engine::getLeader  engine.cpp:836-850: found=0 -> no leader.  Unknown vehicle -> CFB_ERR_ARGUMENT */
int cfb_get_leader(cfb_engine *e, cfb_vehicle_ref vehicle, cfb_vehicle_ref *leader, int *found);

/* Engine::setTrafficLightPhase  engine.cpp:719-725 (no-op with a message unless rlTrafficLight) */
int cfb_set_tl_phase(cfb_engine *e, const char *intersection_id, int phase);
int cfb_set_tl_phase_index(cfb_engine *e, int intersection, int phase);
/* The same for every traffic light at once, with the actions already ON THE DEVICE (the output of
 * a policy network on this GPU): `phases` = cfb_num_intersections() int32 in device memory,
 * intersection order of cfb_intersection_id(); entries of virtual intersections are ignored.
 * Consumed on the engine's stream after the work enqueued on `producer_stream` (a cudaStream_t,
 * NULL = legacy default stream) so far; that stream may reuse the buffer afterwards.  No host
 * synchronisation.  An out-of-range index leaves that light unchanged and is reported as a
 * device error by the next synchronising call.  Single-GPU engines only. */
int cfb_set_tl_phases_device(cfb_engine *e, const int32_t *phases, void *producer_stream);
/* Replay log ("saveReplay": true in the config; roadnetLogFile / replayLogFile relative to "dir").
 * Engine::setReplayLogFile engine.cpp:727-734, Engine::setSaveReplay :736-742; both only print the
 * reference's message when saveReplay is not set in the config.  File content: see the
 * cfb_replay_* functions below. */
int cfb_set_replay_file(cfb_engine *e, const char *log_file);
int cfb_set_save_replay(cfb_engine *e, int open);
/* Engine::setRandomSeed  engine.h:170 */
int cfb_set_random_seed(cfb_engine *e, int seed);
/* Engine::reset(resetRnd)  engine.cpp:744-760 */
int cfb_reset(cfb_engine *e, int reset_rnd);
/* Engine::pushVehicle(info, roads)  engine.cpp:693-717.  `values` hold, in this order: speed,
 * length, width, maxPosAcc, maxNegAcc, usualPosAcc, usualNegAcc, minGap, maxSpeed, headwayTime;
 * NaN = "not given" (struct default, vehicle.h:31-45). */
int cfb_push_vehicle(cfb_engine *e, const double values[10], const char *const *roads, int n_roads);

/* Engine::setVehicleSpeed  engine.cpp:827-834 (custom speed for the coming step) */
int cfb_set_vehicle_speed(cfb_engine *e, cfb_vehicle_ref vehicle, double speed);
/* Engine::setRoute  engine.cpp:852-866: *ok = 1 if the vehicle now follows cur_road + roads */
int cfb_set_vehicle_route(cfb_engine *e, cfb_vehicle_ref vehicle, const char *const *roads, int n_roads, int *ok);
/* Engine::getVehicleInfo  engine.cpp:868-876: "key\0value\0..." pairs; returns the bytes needed */
int64_t cfb_get_vehicle_info(cfb_engine *e, cfb_vehicle_ref vehicle, char *out, int64_t cap);

/* Archive.  Engine::snapshot() / Engine::load(archive) engine.h:176-177, Archive::dump
 * archive.cpp:153-177, Engine::loadFromFile engine.cpp:822-825.  A snapshot is a device-resident
 * image of the whole dynamic state plus the host bookkeeping (RNG, flows, id tables); it can be
 * restored into the engine that made it or into another engine built from the same config.
 * cfb_archive_dump writes one of two forms, chosen by the file name: a path ending in ".json" (what the
 * reference's users pass, tests/python/test_archive.py:99) gets the reference's JSON schema
 * (archive.cpp:153-343) -- same members, vehicle / drivable / flow / intersection names, numbers in
 * rapidjson's own spelling -- which the reference's loadFromFile reads; any other name gets this
 * engine's binary image (exact; its size follows the engine's capacity, not the vehicle count).  cfb_load_from_file accepts both and
 * tells them apart by the first bytes, so a JSON archive written by the reference loads here
 * (archive.cpp:345-550).  JSON form: not with laneChange; the engine the snapshot was taken from must
 * still exist when it is dumped (its road network names the drivables), CFB_ERR_UNSUPPORTED otherwise.
 * Note that the JSON round trip is lossy IN THE REFERENCE (its parser returns some 17-digit numbers
 * one ulp off): an engine that loads a JSON file follows the trajectory of the reference loading that
 * file, not the uninterrupted one -- tests/archive_checks.py. */
typedef struct cfb_archive cfb_archive;
cfb_archive *cfb_snapshot(cfb_engine *e);
void cfb_archive_destroy(cfb_archive *a);
int cfb_load(cfb_engine *e, const cfb_archive *a);
int cfb_archive_dump(const cfb_archive *a, const char *path);
int cfb_load_from_file(cfb_engine *e, const char *path);

/* Multi-GPU (SURVEY.md §8e; no reference counterpart -- the reference's threads share memory).
 * One process per GPU: the road graph is cut into column strips by intersection, every rank runs
 * cfb_next_step in lock step, seam records travel over NCCL on the engine's stream (shard.h).
 * `nccl_id`: the 128 bytes produced by cfb_nccl_unique_id on one rank and broadcast by the caller.
 * The two cfb_shard_* observations are collective; other getters of a sharded engine see only the
 * calling rank's part. */
int cfb_nccl_unique_id(unsigned char out[128]);
cfb_engine *cfb_engine_create_sharded(const char *config_file, int thread_num, int device, int rank, int world,
                                      const unsigned char nccl_id[128]);
int64_t cfb_shard_vehicle_count(cfb_engine *e);
int cfb_shard_lane_vehicle_count(cfb_engine *e, int32_t *out, int n, int waiting);
/* In-process loop-back group: `world` ranks on ONE GPU exchanging by device copies.  Exists so the
 * seam protocol can be checked against the unsharded engine without several GPUs. */
typedef struct cfb_shard_group cfb_shard_group;
cfb_shard_group *cfb_shard_group_create(const char *config_file, int world, int device);
void cfb_shard_group_destroy(cfb_shard_group *g);
int cfb_shard_group_step(cfb_shard_group *g, int n);
const char *cfb_shard_group_last_error(const cfb_shard_group *g);
int64_t cfb_shard_group_vehicle_count(cfb_shard_group *g);
int cfb_shard_group_lane_counts(cfb_shard_group *g, int32_t *out, int n, int waiting);
int64_t cfb_shard_group_debug_vehicles(cfb_shard_group *g, void *out, int64_t cap);
/* sums over the group's ranks: out = {cfb_vehicle_steps, cfb_tie_count} */
int cfb_shard_group_counters(cfb_shard_group *g, int64_t out[2]);
/* Test support: a loop-back group cut by `inter_owner` (the rank of every intersection, virtual ones
 * included, in roadnet order) instead of column strips.  A lane belongs to the rank of its END
 * intersection.  Returns null, with the reason in cfb_last_error, if the cut is refused. */
cfb_shard_group *cfb_debug_shard_group_create_cut(const char *config_file, int world, int device, const int32_t *inter_owner);

/* Test support: full dynamic state of every running vehicle, drivable-major in list order.
 * Record = 8 x int32 {flow, index, priority, drivable, leader flow, leader index, blocker flow,
 * blocker index}, 3 x double {distance, speed, gap}, 1 x int64 {enterLaneLinkTime}; 64 bytes. */
int64_t cfb_debug_vehicles(cfb_engine *e, void *out, int64_t cap);
/* Test support, laneChange=true runs: every running vehicle INCLUDING shadows (Vehicle::isReal() == false,
 * lanechange.cpp:71-102) in vehiclePool (priority) order; partner / leader / blocker are given as priorities (-1 none).
 * Same layout as oracle/harness.py LC_DTYPE (refdump runlc). */
typedef struct {
    int32_t flow, cnt, priority, partner_type, partner, drivable, leader, blocker, flags, last_dir;
    double dis, speed, gap, offset, waiting_time, last_change_time;
} cfb_lc_vehicle;
int64_t cfb_debug_lc_vehicles(cfb_engine *e, cfb_lc_vehicle *out, int64_t cap);
/* Test support: the launch form of the last single-GPU step, out = {graph, pdl, coop, mirror}, each 0 or 1.  graph: the
 * five step kernels were replayed as one CUDA graph; pdl: they were chained by programmatic dependent launch; coop: the
 * step ran as the one cooperative kernel k_step; mirror: the vehicle count is read from mapped host memory.  Kernel timing
 * runs plain launches without PDL.  A default engine on an H100 reports {1, 1, 0, 1}; the CITYFLOW_B200_NO_GRAPH,
 * _NO_PDL, _COOP and _NO_MIRROR variables (INTEGRATION.md) change it, and so does a driver that cannot capture
 * programmatic edges (pdl 0).  All zero but mirror before the first step, and for lane-change and sharded steps. */
int cfb_debug_launch_form(const cfb_engine *e, int32_t out[4]);
/* Test support: blocks (256 threads each) of the list-driven step kernels, out = {k_notify, k_control, k_move, k_leader,
 * k_step}: one resident wave each (occupancy x #SM), sized at the first step that launches them, 0 before. */
int cfb_debug_step_grids(const cfb_engine *e, int32_t out[5]);

/* Measurement support (bench.py): number of our kernels launched so far, per-kernel CUDA-event
 * time accumulators (ms) when enabled, and device-side size figures. */
int64_t cfb_gpu_launches(const cfb_engine *e);
/* Engine::finishedVehicleCnt (engine.h:58; the denominator part of get_average_travel_time): vehicles that completed their route */
int64_t cfb_finished_vehicle_count(cfb_engine *e);
/* Same-step entrants of one drivable with EQUAL new distance seen so far (summed over the rank's drivables).  The
 * reference orders such a pair by a non-stable std::sort over a buffer its worker threads fill in arrival order
 * (engine.cpp:247-249, :480), i.e. its result is not defined there -- two runs of the reference with different
 * thread_num differ from the first tie on.  This engine orders them by priority.  0 = the run is comparable bit for bit. */
int64_t cfb_tie_count(cfb_engine *e);
/* n steps, each bracketed by CUDA events on the engine's stream (optionally with a 256 MiB L2
 * flush before each bracket); *ms = summed device time, *vehicle_steps = sum of vehicle counts */
int cfb_timed_steps(cfb_engine *e, int n, int flush_l2, double *ms, int64_t *vehicle_steps);
/* device-side running sum of get_vehicle_count() after every step since creation.  cfb_reset sets it back to 0.  It
 * is part of the device state image, so cfb_load / cfb_load_from_file restore the value it had when the snapshot was
 * taken (the steps run after the snapshot no longer count). */
int64_t cfb_vehicle_steps(cfb_engine *e);
/* bytes copied host->device (spawn records) and device->host (control block reads) so far */
int cfb_transfer_bytes(const cfb_engine *e, int64_t *h2d, int64_t *d2h);
/* cumulative host time (ms) spent generating spawn records / enqueuing GPU work in cfb_next_step */
int cfb_host_times(const cfb_engine *e, double *gen_ms, double *enqueue_ms);
/* in-kernel debug maxima (all zero unless the library was built with -DCFB_DEBUG_COUNTERS) */
int cfb_debug_counters(cfb_engine *e, uint64_t out[8], int clear);
/* per-position cycle / path-bit samples of the control kernel (debug builds); returns #positions */
int64_t cfb_debug_arrays(cfb_engine *e, uint32_t *cyc, uint32_t *path, int64_t cap);
int cfb_enable_kernel_timing(cfb_engine *e, int on);
int cfb_kernel_times(cfb_engine *e, double ms_out[5], int64_t *steps_timed);
/* sharded run with cfb_enable_kernel_timing: accumulated device time (ms) of the eight phases of a step -- ingest, notify +
 * control, send movers, receive movers (includes waiting for the feeders), move, send tails, receive tails (includes
 * waiting for the owners), leader */
int cfb_shard_phase_times(cfb_engine *e, double ms_out[8], int64_t *steps_timed);
int cfb_synchronize(cfb_engine *e);
int64_t cfb_num_drivables(const cfb_engine *e);
/* CUDA device ordinal the engine was created on */
int cfb_device(const cfb_engine *e);

/* The replay formatter on its own (no engine, no GPU): what the engine writes with saveReplay, for
 * callers that hold vehicle states themselves.  RoadNet::convertToJson roadnet.cpp:327-394 and
 * Engine::updateLog engine.cpp:518-554.  Doubles are printed in shortest round-trip form, so every
 * token parses to the double the reference computed (the reference's own printer, dtoa_milo, does
 * not define the last digit: byte-identical files are not definable).  "Count then fill": both
 * return the bytes needed including the terminating NUL. */
typedef struct cfb_replay cfb_replay;
typedef struct {
    int32_t drivable;          /* lane index, or cfb_num_lanes() + laneLink index */
    double distance;           /* along the drivable */
    int32_t flow, index;       /* cfb_vehicle_ref */
    double length, width;      /* VehicleInfo len / width */
} cfb_replay_vehicle;
cfb_replay *cfb_replay_create(const char *roadnet_file);
void cfb_replay_destroy(cfb_replay *r);
int64_t cfb_replay_roadnet_json(cfb_replay *r, char *out, int64_t cap);
/* vehicles: running vehicles in vehiclePool (ascending priority) order; phase: current phase index
 * per intersection (cfb_num_intersections() entries) */
int64_t cfb_replay_format_step(cfb_replay *r, const cfb_replay_vehicle *vehicles, int64_t n, const int32_t *phase,
                               char *out, int64_t cap);

#ifdef __cplusplus
}
#endif
#endif /* CITYFLOW_B200_H */
