// Host side of the engine + the C-ABI of include/cityflow_b200.h.
//
// What stays on the host (and why): config / roadnet / flow loading; Flow::nextStep spawning
// and the first-lane draw, because they consume one serial std::mt19937 in a fixed order
// (flow.cpp:6-22, vehicle.cpp:45, engine.cpp:606, router.cpp:99 via engine.cpp:453-457) that the
// results depend on; vehicle id <-> slot tables; travel-time statistics.  Everything per
// vehicle / lane / intersection per step runs in device_sim.cu.  There is no CPU path for the
// simulation: without a CUDA device cfb_engine_create fails.
#include <cuda_runtime.h>

#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstring>
#include <iostream>
#include <atomic>
#include <condition_variable>
#include <map>
#include <memory>
#include <mutex>
#include <thread>
#include <random>
#include <set>
#include <sstream>
#include <fstream>
#include <functional>
#include <stdexcept>
#include <string>
#include <unordered_map>
#include <vector>

#include "../../include/cityflow_b200.h"
#include "device_sim.h"
#include "priority_map.h"
#include "replay.h"
#include "partition.h"
#include "shard.h"
#include "flows.h"
#include "json_min.h"
#include "roadnet.h"

namespace cfb {

struct FlowHot {            // the per-step fields of a Flow (flow.h:21-30), packed for the spawn loop
    double nowTime, currentTime, interval;
    int startTime, endTime;
    int cnt;
    int valid;
};

struct FlowRun {            // Flow, flow.h:17-53
    FlowDef def;
    double nowTime = 0, currentTime = 0;
    int cnt = 0;
    bool valid = true;
    int routeId = -1;
    int tmplId = -1;
};

struct SlotInfo {
    int32_t flow = -1, index = -1;   // id: flow_<flow>_<index> / manually_pushed_<index> (flow == -2)
    int32_t priority = 0;
    double enterTime = 0;
    int32_t spawnStep = 0;           // Engine::step when the vehicle was created
    int32_t routeId = -1;            // resolved route (Routing::route), for get_vehicle_info / set_vehicle_route
    int32_t firstLane = -1;          // lane whose waiting queue the vehicle was put in
    int32_t tmplId = -1;             // vehicle template (length / width for the replay log)
    bool shadow = false;             // lane change: a shadow vehicle (Vehicle::isReal() == false)
    bool live = false;
};

struct FlowStatic {         // what a spawn needs from its Flow, 12 bytes instead of a walk through FlowRun/FlowDef
    int routeId, tmplId, firstRoad;
};

struct RouteHot {           // Route's candidate first lanes (<= 4 in practice) in one cache line
    int valid, n;
    int lane[4], plan[4];
};

struct Pending {            // a vehicle created this step, waiting for planRoute (engine.cpp:450-470)
    int slot, road, routeId, tmplId, flow;
};

class HostEngine {
public:
    std::string error;
    RoadNet net;
    std::vector<FlowRun> flows;
    std::vector<FlowStatic> flowStatic;
    std::vector<RouteHot> routeHot;                          // filled on demand from routing (n = -1: not cached / too many lanes)
    std::vector<int> due;                                    // flows spawning this step, one entry per vehicle
    std::vector<FlowHot> hot;                                // hot[i] mirrors flows[i]'s runtime state (authoritative)
    std::vector<uint64_t> sortKeys;
    std::vector<int> predicted;                              // this step's priority draws, predicted on a copy of the RNG (prefetch keys)
    std::vector<Pending> pendingSorted;
    std::vector<SpawnRec> batchTmp;
    std::unique_ptr<Routing> routing;
    std::vector<VehicleTemplate> templates;
    std::map<VehicleTemplate, int> templateIndex;
    std::unique_ptr<DeviceSim> dev;
    double interval = 1.0;
    int seed = 0;
    bool rlTrafficLight = false, laneChange = false, saveReplay = false;
    bool saveReplayInConfig = false;                         // engine.h:48
    std::string dir, roadnetLogFile, replayLogFile;       // "dir" of the config: prefix of every file name
    std::unique_ptr<ReplayWriter> replay;
    std::ofstream logOut;                                    // Engine::logOut engine.h:40
    std::vector<SpeedRec> replayRecs;
    std::vector<ReplayVehicle> replayVeh;
    std::vector<int32_t> replayPhase;
    std::string replayLine;
    std::mt19937 rnd;
    size_t step = 0;
    int manuallyPushCnt = 0;
    int finishedCnt = 0;
    double cumulativeTravelTime = 0;
    std::vector<SlotInfo, HugePageAllocator<SlotInfo>> slots;
    std::vector<int> freeSlots;
    PriorityMap4 pool;                                       // priority -> slot (vehiclePool, engine.h:25)
    std::unordered_map<uint64_t, int> idToSlot;              // built lazily (get_leader)
    bool idMapValid = false;
    long long hostGenNs = 0, hostEnqueueNs = 0;
    long long genFlowsNs = 0, genCreateNs = 0, genPlanNs = 0;   // breakdown of hostGenNs: flow clocks | vehicle creation | planRoute + records
    // sharded mode
    ShardTransport *transport = nullptr;                      // not owned
    std::function<void(std::vector<FinRec> &)> finishedHook;   // local list -> list of all ranks              // host time spent generating spawns / enqueuing
    std::vector<Pending> pending;
    std::vector<SpawnRec> batch;
    std::vector<std::string> laneIds;
    size_t uploadedPlans = 0, uploadedTemplates = 0;
    bool finishedDirty = false;                              // steps enqueued since the last drain
    // ---- the spawner runs ONE STEP AHEAD of the device ----
    // Flow::nextStep / planRoute of step t+1 (prepareStep) depend on nothing step t computes -- except whether the holder of
    // a colliding priority has left, which createVehicle asks the device about -- so next_step() enqueues step t and then
    // prepares step t+1 while the GPU is busy: the host work disappears from a loop that waits for the device every step
    // (next_step(); get_vehicle_count()).  Every API call that could observe or change what the preparation touched
    // (push_vehicle, set_random_seed, reset, archives, id-based getters / setters, get_vehicles(include_waiting),
    // get_average_travel_time) first takes it back (cancelAhead), so results are those of the reference's order of events.
    std::vector<unsigned char> laneLocal;                     // sharded: lanes this rank owns or feeds
    bool ahead = false;
    bool aheadEnabled = true;
    bool undoLog = false;
    struct Undo {
        std::mt19937 rnd;
        std::vector<FlowHot> hot;
        std::vector<int> freeSlots, allocated, inserted;
        std::vector<std::pair<int, int>> erased;
        std::vector<Pending> pending;
        size_t slotsSize = 0;
        int manuallyPushCnt = 0;
    } undo;
    long long h2dBytes = 0, d2hBytes = 0;                    // host<->device traffic of the public calls (bench e2e)

    static uint64_t key(int flow, int index) { return ((uint64_t) (uint32_t) flow << 32) | (uint32_t) index; }

    // The lane buckets are sized once, from the vehicles known when the engine is made (bucketSpacing,
    // device_layout.cuh).  A vehicle that packs tighter than that could overflow a bucket: refused, not run.
    void checkFitsLayout(const VehicleTemplate &t) const {
        if (!dev || t.len + t.minGap >= dev->bucketSpacing()) return;
        std::ostringstream m;
        m << "vehicle of length " << t.len << " m with minGap " << t.minGap << " m packs tighter than the lane buckets allow: "
          << "they were sized for vehicles at least " << dev->bucketSpacing() << " m apart (length + minGap), from the "
          << "vehicles of the flow file; give the flow file a vehicle this small to run it";
        throw std::runtime_error(m.str());
    }

    int internTemplate(const VehicleTemplate &t) {
        auto it = templateIndex.find(t);
        if (it != templateIndex.end()) return it->second;
        int id = (int) templates.size();
        templates.push_back(t);
        templateIndex[t] = id;
        return id;
    }

    // Engine::loadConfig engine.cpp:37-84
    bool load(const std::string &configFile, int device) {
        bool opened = false;
        Json doc = Json::parseFile(configFile, &opened);
        if (!opened) { error = "cannot open config file!"; return false; }
        if (!doc.isObject()) { error = "wrong format of config file"; return false; }
        auto need = [&](const char *k) -> const Json & {
            const Json *v = doc.find(k);
            if (!v) throw JsonError(std::string(k) + " is required but missing in json file");
            return *v;
        };
        std::string roadnetFile, flowFile;
        try {
            const Json &iv = need("interval");
            if (!iv.isNumber()) throw JsonError("interval: expected type d");
            interval = iv.asDouble();
            const Json &rl = need("rlTrafficLight");
            if (!rl.isBool()) throw JsonError("rlTrafficLight: expected type b");
            rlTrafficLight = rl.asBool();
            const Json *lc = doc.find("laneChange");
            laneChange = lc && lc->isBool() ? lc->asBool() : false;
            const Json &sd = need("seed");
            if (!sd.isInt()) throw JsonError("seed: expected type i");
            seed = sd.asInt();
            rnd.seed(seed);
            auto str = [&](const char *k) -> std::string {
                const Json &v = need(k);
                if (!v.isString()) throw JsonError(std::string(k) + ": expected type PKc");
                return v.s;
            };
            dir = str("dir");
            roadnetFile = str("roadnetFile");
            flowFile = str("flowFile");
            const Json &sr = need("saveReplay");
            if (!sr.isBool()) throw JsonError("saveReplay: expected type b");
            saveReplayInConfig = saveReplay = sr.asBool();
            if (saveReplay) {  // engine.cpp:73-77
                roadnetLogFile = str("roadnetLogFile");
                replayLogFile = str("replayLogFile");
            }
        } catch (const JsonError &e) {
            error = e.what();
            return false;
        }
        if (!net.load(dir + roadnetFile)) { error = "loading roadnet file error!"; return false; }
        std::vector<FlowDef> defs;
        if (!loadFlows(dir + flowFile, net, defs)) { error = "loading flow file error!"; return false; }
        routing.reset(new Routing(net));
        if (laneChange) routing->enableLanePlans();   // a shadow continues the route from the lane it was inserted into
        for (auto &d : defs) {
            FlowRun f;
            f.def = d;
            f.nowTime = d.interval;  // flow.h:35
            f.routeId = routing->intern(d.anchors);
            f.tmplId = internTemplate(d.tmpl);
            hot.push_back(FlowHot{d.interval, 0.0, d.interval, d.startTime, d.endTime, 0, 1});  // nowTime = interval (flow.h:35)
            flowStatic.push_back(FlowStatic{f.routeId, f.tmplId, d.anchors[0]});
            flows.push_back(std::move(f));
        }
        if (saveReplay) {  // Engine::setLogFile engine.cpp:773-778
            replay.reset(new ReplayWriter(net));
            std::ofstream js(dir + roadnetLogFile);
            if (js) js << replay->roadnetJson();
            if (!js) std::cerr << "write roadnet log file error" << std::endl;
            logOut.open(dir + replayLogFile);
        }
        laneIds.resize(net.nLanes());
        for (int l = 0; l < net.nLanes(); ++l) laneIds[l] = net.laneName(l);
        DeviceSimOptions opt;
        opt.device = device;
        opt.interval = interval;
        opt.rlTrafficLight = rlTrafficLight;
        dev.reset(new DeviceSim(net, templates, *routing, opt));
        if (laneChange) dev->enableLaneChange(net, *routing);   // device_lc.cuh
        uploadedPlans = routing->numPlans();
        uploadedTemplates = templates.size();
        if (const char *na = getenv("CITYFLOW_B200_NO_AHEAD")) aheadEnabled = !(na[0] == '1');
        if (const char *ps = getenv("CITYFLOW_B200_PARALLEL_SPAWN_MIN")) parallelSpawnMin = atoi(ps);
        if (std::thread::hardware_concurrency() < 4) parallelSpawnMin = 0;
        return true;
    }

    double currentTime() const { return step * interval; }  // engine.cpp:678

    void checkDevice() {
        int err = dev->errorFlags();
        if (err) {
            std::string m = "device capacity/route error:";
            if (err & ERR_BUCKET_OVERFLOW) m += " lane bucket overflow;";
            if (err & ERR_ENTRANT_OVERFLOW) m += " too many vehicles entering one drivable in one step;";
            if (err & ERR_MOVER_OVERFLOW) m += " mover staging overflow;";
            if (err & ERR_ROUTE_DEAD_END) m += " a vehicle reached a lane that cannot continue its route (the reference asserts here, vehicle.cpp:60);";
            if (err & ERR_FINISHED_OVERFLOW) m += " finished ring overflow;";
            if (err & ERR_SHARD_TIMEOUT) m += " a peer rank's seam message did not arrive within 4 s (every rank of a sharded run must step in lock step);";
            if (err & ERR_PHASE_RANGE) m += " a phase index set from the device is out of range (the reference throws from phases.at(), trafficlight.cpp:17);";
            throw std::runtime_error(m);
        }
    }

    // Bring host bookkeeping up to date with the device (vehicles that left the network):
    // the tail of Engine::threadUpdateLocation (engine.cpp:296-310).
    void drain() {
        if (!finishedDirty) return;
        std::vector<FinRec> fin;
        dev->drainFinished(fin);
        if (transport) dev->shardGatherFinished(transport, fin);
        else if (finishedHook) finishedHook(fin);
        // deterministic accumulation order for the travel-time sum (ring order is atomics order)
        // a vehicle replaced by its shadow is tagged by the device (engine.cpp:297-301): it is not a
        // finished vehicle, its shadow (same name) carries on as the real one
        std::vector<char> replaced(fin.size(), 0);
        for (size_t k = 0; k < fin.size(); ++k)
            if (fin[k].slot & 0x40000000) { fin[k].slot &= ~0x40000000; replaced[k] = 1; }
        for (size_t k = 0; k < fin.size(); ++k)
            if (replaced[k]) {
                SlotInfo &s = slots[fin[k].slot];
                if (!s.live) continue;
                for (SlotInfo &o : slots)   // its shadow: same name, live, flagged (rare event: a linear search)
                    if (o.live && o.shadow && o.flow == s.flow && o.index == s.index) { o.shadow = false; break; }
                if (pool.get(s.priority) == fin[k].slot) pool.erase(s.priority);
                s.live = false;
                freeSlots.push_back(fin[k].slot);
                idMapValid = false;
            }
        std::sort(fin.begin(), fin.end(), [this](const FinRec &a, const FinRec &b) {
            return a.step != b.step ? a.step < b.step : slots[a.slot].priority < slots[b.slot].priority;
        });
        for (const FinRec &f : fin) {
            SlotInfo &s = slots[f.slot];
            if (!s.live) continue;
            finishedCnt += 1;
            cumulativeTravelTime += f.step * interval - s.enterTime;
            if (pool.get(s.priority) == f.slot) pool.erase(s.priority);   // (the priority may already be re-issued)
            s.live = false;
            freeSlots.push_back(f.slot);
        }
        if (!fin.empty()) idMapValid = false;
        finishedDirty = false;
        checkDevice();
    }

    // ---- parallel vehicle creation (large steps only: a sharded run replicates the whole network's spawns on every rank) ----
    // What a creation costs is two random cache lines (priority table cell, slot record).  The draws are known in advance
    // (RNG run ahead on a copy) as long as no draw hits a priority in use, so four threads -- each owning the quarter of the
    // priority table its keys fall into -- look up, insert and fill the slot records side by side; the first hit (a priority
    // in use, or drawn twice in this step) hands the rest of the step back to the sequential code, which asks the device and
    // redraws exactly like Vehicle::Vehicle (vehicle.cpp:45).  Same state as the sequential loop, entry by entry.
    struct Workers {
        static constexpr int T = 4;
        std::vector<std::thread> th;
        std::mutex mu;
        std::condition_variable cvGo;
        const std::function<void(int)> *job = nullptr;
        std::atomic<long long> gen{0};
        std::atomic<int> pending{0}, sleepers{0};
        std::atomic<bool> stop{false};
        // A worker spins for the next job for a while (steps follow each other every ~100 us while the engine is being
        // stepped: a condition-variable wake-up would cost more than the job), then goes to sleep.
        void start() {
            for (int w = 1; w < T; ++w)
                th.emplace_back([this, w]() {
                    long long seen = 0;
                    for (;;) {
                        long spins = 0;
                        while (gen.load(std::memory_order_acquire) == seen && !stop.load(std::memory_order_relaxed)) {
                            if (++spins < 200000) { __builtin_ia32_pause(); continue; }   // ~ a few ms
                            std::unique_lock<std::mutex> lk(mu);
                            sleepers.fetch_add(1);
                            cvGo.wait(lk, [&] { return stop.load() || gen.load() != seen; });
                            sleepers.fetch_sub(1);
                        }
                        if (stop.load()) return;
                        seen = gen.load(std::memory_order_acquire);
                        (*job)(w);
                        pending.fetch_sub(1, std::memory_order_release);
                    }
                });
        }
        void run(const std::function<void(int)> &f) {
            job = &f;
            pending.store(T - 1, std::memory_order_relaxed);
            gen.fetch_add(1);   // (sequentially consistent, like the sleepers counter: the two form a Dekker pair with the worker's wait)
            if (sleepers.load() > 0) { std::lock_guard<std::mutex> lk(mu); cvGo.notify_all(); }
            f(0);
            while (pending.load(std::memory_order_acquire) != 0) __builtin_ia32_pause();
        }
        ~Workers() {
            stop.store(true);
            { std::lock_guard<std::mutex> lk(mu); cvGo.notify_all(); }
            for (auto &t : th) t.join();
        }
    };
    std::unique_ptr<Workers> workers;
    // Used for steps that spawn at least this many vehicles (CITYFLOW_B200_PARALLEL_SPAWN_MIN; 0 = never).  The bench flows
    // spawn in bursts (every flow every 10 s), so this is every tenth step of any bench run: 1 800 creations on one GPU,
    // 14 400 on every rank of the 8-GPU run (a sharded run replicates the whole network's spawns).  The threads split the
    // creation work only (thread-local vectors, one buffer of draws: DESIGN.md section 8).  The RNG, the slot
    // hand-out and the flow clocks stay sequential.
    int parallelSpawnMin = 512;
    std::vector<int> parSlot, parIndex;

    std::vector<uint32_t> parMine[Workers::T];
    std::vector<uint32_t> parInserted[Workers::T];
    // The creation phase's share of the RNG stream, taken from the engine RNG itself before the vehicles are made (every
    // value is consumed below, in order, so the RNG ends where the sequential loop would leave it): vehicle k's priority
    // is rawDraws[2 k + drawShift], the value after it its thread index (engine.cpp:601-606); drawShift counts the
    // redraws of vehicles that hit a priority in use (each moves everybody behind it one value on).
    std::vector<uint32_t> rawDraws;
    size_t drawShift = 0, drawPos = 0;
    bool drawFromBuffer = false;
    uint32_t nextDraw() {
        if (!drawFromBuffer) return (uint32_t) rnd();
        if (drawPos == rawDraws.size()) rawDraws.push_back((uint32_t) rnd());
        return rawDraws[drawPos++];
    }
    int plannedKey(size_t k) const { return (int) rawDraws[2 * k + drawShift]; }
    // Creates the vehicles due[from .. n), whose slots / indices are in parSlot / parIndex and whose draws are plannedKey(k);
    // returns the index of the first hit (n: none).  Vehicles before the hit are complete.
    size_t createParallel(size_t from, size_t n) {
        std::atomic<size_t> firstHit{n};
        const double enter = currentTime();
        const int32_t spawnStep = (int32_t) step;
        workers->run([&](int w) {
            PriorityMap &M = pool.sub(w);
            // (the vectors' control blocks sit side by side in the member arrays: a thread works on locals and hands them back
            // at the end, or every push_back takes the cache line away from the other three -- measured 3x on the job)
            std::vector<uint32_t> mine, ins;
            mine.swap(parMine[w]);
            ins.swap(parInserted[w]);
            mine.clear(); ins.clear();
            for (size_t k = from; k < n; ++k) if (PriorityMap4::part(plannedKey(k)) == w) mine.push_back((uint32_t) k);
            constexpr size_t PF = 12;
            auto pf = [&](size_t j) { M.prefetch(plannedKey(mine[j])); __builtin_prefetch(&slots[parSlot[mine[j]]], 1); };
            for (size_t j = 0; j < std::min(PF, mine.size()); ++j) pf(j);
            for (size_t j = 0; j < mine.size(); ++j) {
                if (j + PF < mine.size()) pf(j + PF);
                const size_t k = mine[j];
                if (k >= firstHit.load(std::memory_order_relaxed)) break;
                const int key = plannedKey(k);
                if (M.get(key) >= 0) {   // in use (or drawn twice this step): from here on the sequential code decides
                    size_t cur = firstHit.load();
                    while (k < cur && !firstHit.compare_exchange_weak(cur, k)) {}
                    break;
                }
                M.insert(key, parSlot[k]);
                ins.push_back((uint32_t) k);
                const FlowStatic &fs = flowStatic[due[k]];
                SlotInfo &s = slots[parSlot[k]];
                s.flow = due[k]; s.index = parIndex[k]; s.priority = key; s.enterTime = enter; s.spawnStep = spawnStep;
                s.routeId = fs.routeId; s.firstLane = -1; s.tmplId = fs.tmplId; s.shadow = false; s.live = true;
            }
            mine.swap(parMine[w]);
            ins.swap(parInserted[w]);
        });
        const size_t c = firstHit.load();
        for (int w = 0; w < Workers::T; ++w)     // what the other threads created beyond the hit is taken back
            for (size_t j = parInserted[w].size(); j-- > 0 && parInserted[w][j] > c;) {
                const size_t k = parInserted[w][j];
                pool.erase(plannedKey(k));
                slots[parSlot[k]].live = false;
            }
        for (size_t k = from; k < c; ++k) {
            const FlowStatic &fs = flowStatic[due[k]];
            if (undoLog) { undo.inserted.push_back(plannedKey(k)); undo.allocated.push_back(parSlot[k]); }
            pending.push_back({parSlot[k], fs.firstRoad, fs.routeId, fs.tmplId, due[k]});
        }
        idMapValid = false;
        return c;
    }

    int allocSlot() {
        if (!freeSlots.empty()) {
            int s = freeSlots.back();
            freeSlots.pop_back();
            return s;
        }
        slots.emplace_back();
        return (int) slots.size() - 1;
    }

    // Vehicle ctor (vehicle.cpp:38-47) + Engine::pushVehicle (engine.cpp:605-613)
    int createVehicle(int flow, int index, int routeId, int tmplId, int firstRoad, int slotGiven = -1) {
        int priority;
        for (;;) {
            priority = (int) nextDraw();
            const int other = pool.get(priority);
            if (other < 0) break;
            // The holder of this priority may have left the network on the device already (the host
            // learns about finishes lazily).  Ask the device about that one slot -- its delStep array
            // is complete on every rank of a sharded run, so no collective drain is needed -- and let
            // the regular drain do the bookkeeping later.
            dev->synchronize();
            if (dev->slotDelStep(other) >= slots[other].spawnStep) {
                pool.erase(priority);
                if (undoLog) undo.erased.emplace_back(priority, other);
                break;
            }
        }
        (void) nextDraw();  // threadIndex = rnd() % threadNum (engine.cpp:606): drawn, not needed here
        const int slot = slotGiven >= 0 ? slotGiven : allocSlot();
        SlotInfo &s = slots[slot];
        s.flow = flow;
        s.index = index;
        s.priority = priority;
        s.enterTime = currentTime();
        s.spawnStep = (int32_t) step;
        s.routeId = routeId;
        s.firstLane = -1;
        s.tmplId = tmplId;
        s.live = true;
        pool.insert(priority, slot);
        if (undoLog) { undo.inserted.push_back(priority); undo.allocated.push_back(slot); }
        idMapValid = false;
        pending.push_back({slot, firstRoad, routeId, tmplId, flow});
        return slot;
    }

    const RouteHot &hotRoute(int id) {
        if ((size_t) id >= routeHot.size()) {
            const size_t from = routeHot.size();
            routeHot.resize(routing->numRoutes());
            for (size_t r = from; r < routeHot.size(); ++r) {
                const Route &rt = routing->route((int) r);
                RouteHot &hr = routeHot[r];
                hr.valid = rt.valid;
                hr.n = rt.valid && rt.startLanes.size() <= 4 ? (int) rt.startLanes.size() : -1;
                for (int k = 0; k < hr.n; ++k) { hr.lane[k] = rt.startLanes[k]; hr.plan[k] = rt.planOfStartLane[k]; }
            }
        }
        return routeHot[id];
    }

    // Engine::nextStep engine.cpp:566-594 (host part: P0 spawn, P1 planRoute; the rest is device work)
    // P0/P1 on the host: flows, vehicle creation, first-lane draw -> `batch` (lane-sorted spawn records)
    void prepareStep() {
        const auto t0 = std::chrono::steady_clock::now();
        const size_t nFlows = hot.size();
        FlowHot *H = hot.data();
        for (size_t i = 0; i < nFlows; ++i) {  // Flow::nextStep flow.cpp:6-22
            FlowHot &f = H[i];
            if (!f.valid) continue;
            if (f.endTime != -1 && f.currentTime > f.endTime) continue;
            if (f.currentTime >= f.startTime) {
                while (f.nowTime >= f.interval) {
                    due.push_back((int) i);   // created below, in this order (nothing a Vehicle ctor does feeds back into a Flow)
                    f.nowTime -= f.interval;
                }
                f.nowTime += interval;
            }
            f.currentTime += interval;
        }
        const auto tFlows = std::chrono::steady_clock::now();
        genFlowsNs += std::chrono::duration_cast<std::chrono::nanoseconds>(tFlows - t0).count();
        // Each creation costs a few cache misses (priority table, slot record) and nothing else; the keys are known in
        // advance because the RNG can be run ahead on a copy: priority, thread index, priority, ... (engine.cpp:601-606).
        // A priority collision makes the real sequence leave the predicted one -- then the remaining prefetches are merely
        // useless.  The prefetches run a fixed distance ahead of the creations: a core tracks only a dozen or so outstanding
        // line fills, so issuing all of a step's prefetches up front drops most of them.
        const size_t nDue = due.size();
        constexpr size_t PF = 12;
        const bool parallel = parallelSpawnMin > 0 && nDue >= (size_t) parallelSpawnMin;
        if (nDue >= 8 && !parallel) {
            std::mt19937 ahead = rnd;
            predicted.resize(nDue);
            for (size_t k = 0; k < nDue; ++k) { predicted[k] = (int) ahead(); (void) ahead(); }
        }
        const size_t nFree = freeSlots.size();
        auto prefetchFor = [&](size_t k) {
            pool.prefetch(predicted[k]);
            if (k < nFree) __builtin_prefetch(&slots[freeSlots[nFree - 1 - k]], 1);
        };
        size_t done = 0;
        if (parallel) {
            if (!workers) { workers.reset(new Workers()); workers->start(); }
            parSlot.resize(nDue); parIndex.resize(nDue);
            for (size_t k = 0; k < nDue; ++k) parIndex[k] = H[due[k]].cnt++;
            {   // allocSlot() nDue times, in the sequential loop's order: the free list from its end, then new slots
                const size_t reuse = std::min(nDue, freeSlots.size()), nF = freeSlots.size();
                for (size_t k = 0; k < reuse; ++k) parSlot[k] = freeSlots[nF - 1 - k];
                freeSlots.resize(nF - reuse);
                for (size_t k = reuse; k < nDue; ++k) { slots.emplace_back(); parSlot[k] = (int) slots.size() - 1; }
            }
            rawDraws.resize(2 * nDue);
            for (size_t i = 0; i < 2 * nDue; ++i) rawDraws[i] = (uint32_t) rnd();
            drawShift = 0;
            while (done < nDue) {
                done = createParallel(done, nDue);
                if (done == nDue) break;
                // a hit: this one vehicle goes through the sequential code (device query, redraws) reading the same stream; each
                // redraw moves the draws of everybody behind it one value on
                const FlowStatic &fs = flowStatic[due[done]];
                drawPos = 2 * done + drawShift;
                {
                    struct FromBuffer { bool &f; explicit FromBuffer(bool &b) : f(b) { f = true; } ~FromBuffer() { f = false; } } guard(drawFromBuffer);
                    createVehicle(due[done], parIndex[done], fs.routeId, fs.tmplId, fs.firstRoad, parSlot[done]);
                }
                drawShift = drawPos - 2 * (done + 1);
                ++done;
                while (rawDraws.size() < 2 * nDue + drawShift) rawDraws.push_back((uint32_t) rnd());
            }
        }
        if (done < nDue && nDue >= 8) for (size_t k = 0; k < std::min(PF, nDue); ++k) prefetchFor(k);
        for (size_t k = done; k < nDue; ++k) {
            if (nDue >= 8 && k + PF < nDue) prefetchFor(k + PF);
            const int i = due[k];
            const FlowStatic &fs = flowStatic[i];
            createVehicle(i, H[i].cnt++, fs.routeId, fs.tmplId, fs.firstRoad);
        }
        due.clear();
        batch.clear();
        const auto tCreate = std::chrono::steady_clock::now();
        genCreateNs += std::chrono::duration_cast<std::chrono::nanoseconds>(tCreate - tFlows).count();
        if (!pending.empty()) {
            // Engine::planRoute walks roads in file order, each road's buffer in spawn order
            // (road, arrival index) keys: same order as a stable sort by road, cheaper than moving structs
            bool inRoadOrder = true;   // (flows written road by road -- every generated scenario -- arrive in that order already)
            for (size_t k = 1; k < pending.size() && inRoadOrder; ++k) inRoadOrder = pending[k - 1].road <= pending[k].road;
            if (!inRoadOrder) {
                sortKeys.resize(pending.size());
                for (size_t k = 0; k < pending.size(); ++k) sortKeys[k] = ((uint64_t) (uint32_t) pending[k].road << 32) | (uint32_t) k;
                std::sort(sortKeys.begin(), sortKeys.end());
                pendingSorted.resize(pending.size());
                for (size_t k = 0; k < pending.size(); ++k) pendingSorted[k] = pending[(uint32_t) sortKeys[k]];
            }
            for (const Pending &p : inRoadOrder ? pending : pendingSorted) {
                const RouteHot &rt = hotRoute(p.routeId);
                if (rt.valid) {
                    SpawnRec r{};
                    r.slot = p.slot;
                    if (rt.n > 0) {
                        const size_t pick = rnd() % (size_t) rt.n;  // Router::selectLaneIndex router.cpp:99
                        r.lane = rt.lane[pick];
                        r.plan = rt.plan[pick];
                    } else {
                        const Route &full = routing->route(p.routeId);
                        const size_t pick = rnd() % full.startLanes.size();
                        r.lane = full.startLanes[pick];
                        r.plan = full.planOfStartLane[pick];
                    }
                    r.tmpl = p.tmplId;
                    r.priority = slots[p.slot].priority;
                    slots[p.slot].firstLane = r.lane;
                    // one rank of a sharded run ingests only the lanes it owns or feeds (k_ingest skips the others anyway)
                    if (laneLocal.empty() || laneLocal[r.lane]) batch.push_back(r);
                } else {
                    if (p.flow >= 0) {
                        if (hot[p.flow].valid)
                            std::cerr << "[warning] Invalid route '" << flows[p.flow].def.id << "'. Omitted by default." << std::endl;
                        hot[p.flow].valid = 0;
                    }
                    SlotInfo &s = slots[p.slot];
                    pool.erase(s.priority);
                    idMapValid = false;
                    s.live = false;
                    freeSlots.push_back(p.slot);
                }
            }
            pending.clear();
            bool inLaneOrder = true;
            for (size_t k = 1; k < batch.size() && inLaneOrder; ++k) inLaneOrder = batch[k - 1].lane <= batch[k].lane;
            if (!inLaneOrder) {
                sortKeys.resize(batch.size());
                for (size_t k = 0; k < batch.size(); ++k) sortKeys[k] = ((uint64_t) (uint32_t) batch[k].lane << 32) | (uint32_t) k;
                std::sort(sortKeys.begin(), sortKeys.end());
                batchTmp.resize(batch.size());
                for (size_t k = 0; k < batch.size(); ++k) batchTmp[k] = batch[(uint32_t) sortKeys[k]];
                batch.swap(batchTmp);
            }
        }
        if (templates.size() != uploadedTemplates) { dev->uploadTemplates(templates); uploadedTemplates = templates.size(); }
        if ((size_t) routing->numPlans() != uploadedPlans) { dev->uploadPlans(*routing); uploadedPlans = routing->numPlans(); }
        dev->ensureSlotCapacity((int) slots.size());
        const auto tEnd = std::chrono::steady_clock::now();
        genPlanNs += std::chrono::duration_cast<std::chrono::nanoseconds>(tEnd - tCreate).count();
        hostGenNs += std::chrono::duration_cast<std::chrono::nanoseconds>(tEnd - t0).count();
    }
    // Engine::updateLog engine.cpp:518-554: positions of the running vehicles and the light states
    // after this step, one line.  Gathers from the device (synchronises), so stepping with
    // saveReplay on is as slow as it is in the reference.
    void writeReplayLine() {
        const int n = dev->runningVehicles(replayRecs);
        std::sort(replayRecs.begin(), replayRecs.end(), [this](const SpeedRec &a, const SpeedRec &b) {
            return slots[a.slot].priority < slots[b.slot].priority;   // vehiclePool order (engine.cpp:780-790)
        });
        replayVeh.resize(n);
        for (int k = 0; k < n; ++k) {
            const SlotInfo &s = slots[replayRecs[k].slot];
            const VehicleTemplate &t = templates[s.tmplId];
            replayVeh[k] = ReplayVehicle{replayRecs[k].drivable, replayRecs[k].dis, s.flow, s.index, t.len, t.width};
        }
        replayPhase.resize(net.nInter());
        dev->phases(replayPhase.data());
        replay->formatStep(replayVeh.data(), (size_t) n, replayPhase.data(), replayLine);
        logOut << replayLine << std::endl;
    }
    void finishStep() {
        h2dBytes += (long long) batch.size() * sizeof(SpawnRec) + sizeof(int);
        finishedDirty = true;
        if (saveReplay && replay && !transport) writeReplayLine();   // before step += 1, like engine.cpp:589-593
        step += 1;
        if ((step & 255) == 0) drain();  // bound the finished ring / free slots in long unobserved runs
    }
    // One step with lane change: the shadows' priorities come from the engine RNG right after
    // this step's spawn draws (vehicle.cpp:33), so the step has a host round trip in the middle.
    void nextStepLaneChange() {
        std::vector<int32_t> spare(256);
        for (auto &x : spare) { x = allocSlot(); slots[x].live = false; }
        prepareStep();                                   // (ensures device capacity for every slot handed out so far)
        std::vector<DeviceSim::LcShadow> created;
        dev->stepLcBegin(batch.data(), (int) batch.size(), spare.data(), (int) spare.size(), created);
        std::vector<int32_t> prio(created.size());
        for (size_t k = 0; k < created.size(); ++k) {    // Vehicle copy constructor vehicle.cpp:27-36
            const SlotInfo parent = slots[created[k].parentSlot];
            int priority;
            for (;;) {
                priority = (int) rnd();
                const int other = pool.get(priority);
                if (other < 0) break;
                if (dev->slotDelStep(other) >= slots[other].spawnStep) { pool.erase(priority); break; }
            }
            SlotInfo &s = slots[created[k].shadowSlot];
            s = parent;
            s.priority = priority;
            s.spawnStep = (int32_t) step;
            s.shadow = true;
            s.live = true;
            pool.insert(priority, created[k].shadowSlot);
            prio[k] = priority;
        }
        for (size_t k = created.size(); k < spare.size(); ++k) freeSlots.push_back(spare[k]);   // the device takes spares in order
        idMapValid = false;
        dev->stepLcEnd(prio.data(), (int) prio.size());
        finishStep();
    }
    void nextStep() {
        if (laneChange) { nextStepLaneChange(); return; }
        if (!ahead) prepareStep();
        ahead = false;
        const auto t1 = std::chrono::steady_clock::now();
        if (!transport) dev->step(batch.data(), (int) batch.size());
        else dev->shardStep(batch.data(), (int) batch.size(), transport);   // one rank of a sharded run
        hostEnqueueNs += std::chrono::duration_cast<std::chrono::nanoseconds>(std::chrono::steady_clock::now() - t1).count();
        finishStep();
        prepareAhead();
    }
    void prepareAhead() {
        if (!aheadEnabled || ahead || laneChange) return;
        undo.rnd = rnd;
        undo.hot = hot;
        undo.freeSlots = freeSlots;
        undo.pending = pending;
        undo.slotsSize = slots.size();
        undo.allocated.clear(); undo.inserted.clear(); undo.erased.clear();
        undoLog = true;
        prepareStep();
        undoLog = false;
        ahead = true;
    }
    // Take the preparation of the coming step back: afterwards the host state is what it was right after the last step.
    void cancelAhead() {
        if (!ahead) return;
        ahead = false;
        rnd = undo.rnd;
        hot.swap(undo.hot);
        for (int p : undo.inserted) pool.erase(p);
        for (auto &pr : undo.erased) pool.insert(pr.first, pr.second);
        for (int s : undo.allocated) if ((size_t) s < undo.slotsSize) slots[s].live = false;
        slots.resize(undo.slotsSize);
        freeSlots = undo.freeSlots;
        pending = undo.pending;
        batch.clear();
        idMapValid = false;
    }
    // Tell the device which part of the cut `part` is ours (before the first step).
    std::string configureShard(int rank, const Partition &part) {
        if (saveReplay) {
            std::cerr << "[cityflow_b200] saveReplay is not available on one rank of a sharded run; no replay is written" << std::endl;
            saveReplay = false;
        }
        const int world = part.world;
        double look = 0;
        for (const auto &t : templates) look = std::max(look, t.maxSpeed * t.maxSpeed / t.usualNegAcc / 2 + t.maxSpeed * interval * 2);
        std::string bad = part.validate(net, look);
        if (!bad.empty()) return bad;
        std::vector<unsigned char> owned(part.drvOwner.size());
        for (size_t d = 0; d < owned.size(); ++d) owned[d] = part.drvOwner[d] == rank;
        std::vector<std::vector<int>> feed(world), own(world), bsize(world, std::vector<int>(world, 0));
        for (int q = 0; q < world; ++q) {
            feed[q] = part.boundary[rank][q];   // lanes I feed, q owns
            own[q] = part.boundary[q][rank];    // lanes q feeds, I own
            for (int p2 = 0; p2 < world; ++p2) bsize[q][p2] = (int) part.boundary[q][p2].size();
        }
        laneLocal.assign(net.nLanes(), 0);
        for (int l = 0; l < net.nLanes(); ++l) laneLocal[l] = owned[l];
        for (int q = 0; q < world; ++q) for (int l : feed[q]) laneLocal[l] = 1;
        std::vector<unsigned char> ownedRL(net.nRoadLinks(), 0);
        for (int k = 0; k < net.nLinks(); ++k)
            if (part.drvOwner[net.nLanes() + k] == rank) ownedRL[net.llRoadLink[k]] = 1;
        dev->configureShard(rank, world, owned, feed, own, bsize, ownedRL);
        return "";
    }

    // Engine::reset engine.cpp:744-760
    void reset(bool resetRnd) {
        cancelAhead();
        dev->synchronize();
        dev->reset();
        slots.clear();
        freeSlots.clear();
        pool.clear();
        idToSlot.clear();
        idMapValid = false;
        pending.clear();
        finishedCnt = 0;
        cumulativeTravelTime = 0;
        for (auto &f : hot) {  // Flow::reset flow.cpp:28-32 (valid / manuallyPushCnt are not reset)
            f.nowTime = f.interval;
            f.currentTime = 0;
            f.cnt = 0;
        }
        step = 0;
        finishedDirty = false;
        if (resetRnd) rnd.seed(seed);
    }

    int slotOfId(int flow, int index) {
        if (!idMapValid) {
            idToSlot.clear();
            for (size_t s = 0; s < slots.size(); ++s)
                if (slots[s].live) idToSlot[key(slots[s].flow, slots[s].index)] = (int) s;
            idMapValid = true;
        }
        auto it = idToSlot.find(key(flow, index));
        return it == idToSlot.end() ? -1 : it->second;
    }

    // ---- Archive (archive.cpp:9-151): host half of a snapshot ----
    struct HostState {
        std::mt19937 rnd;
        size_t step = 0;
        int manuallyPushCnt = 0, finishedCnt = 0;
        double cumulativeTravelTime = 0;
        std::vector<double> flowNow, flowCur;
        std::vector<int> flowCnt;
        std::vector<uint8_t> flowValid;
        std::vector<SlotInfo> slots;
        std::vector<int> freeSlots;
        std::vector<Pending> pending;
        // Slot records and the device image hold INDICES into the route / plan / template tables, which grow at run
        // time (push_vehicle, set_vehicle_route): the archive carries what was interned, in order, and load() re-interns
        // it -- an engine whose tables are not a prefix-compatible continuation refuses the archive.
        std::vector<std::vector<int>> routeAnchors;
        std::vector<VehicleTemplate> templates;
    };
    void saveHost(HostState &s) {
        cancelAhead();
        drain();
        s.rnd = rnd; s.step = step; s.manuallyPushCnt = manuallyPushCnt; s.finishedCnt = finishedCnt;
        s.cumulativeTravelTime = cumulativeTravelTime;
        s.flowNow.clear(); s.flowCur.clear(); s.flowCnt.clear(); s.flowValid.clear();
        for (auto &f : hot) { s.flowNow.push_back(f.nowTime); s.flowCur.push_back(f.currentTime); s.flowCnt.push_back(f.cnt); s.flowValid.push_back((uint8_t) f.valid); }
        s.slots.assign(slots.begin(), slots.end()); s.freeSlots = freeSlots; s.pending = pending;
        s.routeAnchors.clear();
        for (int r = 0; r < routing->numRoutes(); ++r) s.routeAnchors.push_back(routing->anchorsOf(r));
        s.templates = templates;
    }
    void loadHost(const HostState &s) {
        cancelAhead();
        if (s.flowNow.size() != flows.size()) throw std::runtime_error("archive does not match this engine (flows)");
        for (size_t r = 0; r < s.routeAnchors.size(); ++r) {
            if (r < (size_t) routing->numRoutes() ? routing->anchorsOf((int) r) != s.routeAnchors[r] : routing->intern(s.routeAnchors[r]) != (int) r)
                throw std::runtime_error("archive does not match this engine (route table)");
        }
        for (size_t t = templates.size(); t < s.templates.size(); ++t) checkFitsLayout(s.templates[t]);
        for (size_t t = 0; t < s.templates.size(); ++t) {
            const bool same = t < templates.size() ? (!(templates[t] < s.templates[t]) && !(s.templates[t] < templates[t])) : internTemplate(s.templates[t]) == (int) t;
            if (!same) throw std::runtime_error("archive does not match this engine (vehicle template table)");
        }
        if (templates.size() != uploadedTemplates) { dev->uploadTemplates(templates); uploadedTemplates = templates.size(); }
        if ((size_t) routing->numPlans() != uploadedPlans) { dev->uploadPlans(*routing); uploadedPlans = routing->numPlans(); }
        rnd = s.rnd; step = s.step; manuallyPushCnt = s.manuallyPushCnt; finishedCnt = s.finishedCnt;
        cumulativeTravelTime = s.cumulativeTravelTime;
        for (size_t i = 0; i < hot.size(); ++i) { hot[i].nowTime = s.flowNow[i]; hot[i].currentTime = s.flowCur[i]; hot[i].cnt = s.flowCnt[i]; hot[i].valid = s.flowValid[i]; }
        slots.assign(s.slots.begin(), s.slots.end()); freeSlots = s.freeSlots; pending = s.pending;
        pool.clear();
        for (size_t k = 0; k < slots.size(); ++k) if (slots[k].live) pool.insert(slots[k].priority, (int) k);
        idMapValid = false;
        finishedDirty = false;
    }

    // ---- Archive in the reference's JSON schema: Archive::dump (archive.cpp:153-343) and the file loader
    // Archive::Archive(Engine &, filename) (archive.cpp:345-550).  The device half goes through the decoded image
    // (StateImage, device_image.cuh); vehicles are named as the reference names them, so a file written here loads
    // in the reference and the other way round.  Not with laneChange (shadow vehicles, signals); the lanes'
    // speed history (Lane::history, read only by RouterType::DURATION routing) is written empty and ignored. ----
    std::string vehicleName(const SlotInfo &s) const {
        return s.flow == -2 ? "manually_pushed_" + std::to_string(s.index) : "flow_" + std::to_string(s.flow) + "_" + std::to_string(s.index);
    }
    std::string drivableName(int d) const {   // Lane::getId roadnet.h:323, LaneLink::getId roadnet.h:478
        if (d < net.nLanes()) return net.laneName(d);
        const int k = d - net.nLanes();
        return net.laneName(net.llStartLane[k]) + "_TO_" + net.laneName(net.llEndLane[k]);
    }

    void writeReferenceArchive(const HostState &hs, const StateImage &img, std::string &o) const {
        if (laneChange) throw std::runtime_error("an archive in the reference's JSON schema is not written with laneChange on (any other file name gets the binary form)");
        if (!laneLocal.empty()) throw std::runtime_error("an archive in the reference's JSON schema is not written by one rank of a sharded engine");
        if (!hs.pending.empty()) throw std::runtime_error("archive taken in the middle of a step");
        const int nL = net.nLanes();
        struct Ref { int priority, slot, drivable; const StateImage::Running *run; };
        std::vector<Ref> refs;
        for (int d = 0; d < (int) img.drivables.size(); ++d)
            for (const auto &r : img.drivables[d]) refs.push_back(Ref{r.priority, r.slot, d, &r});
        for (int l = 0; l < (int) img.waiting.size(); ++l)
            for (const auto &w : img.waiting[l]) refs.push_back(Ref{w.priority, w.slot, l, nullptr});
        std::sort(refs.begin(), refs.end(), [](const Ref &a, const Ref &b) { return a.priority < b.priority; });   // vehiclePool is a std::map
        auto nameOf = [&](int slot) {
            if (slot < 0 || (size_t) slot >= hs.slots.size() || !hs.slots[slot].live) throw std::runtime_error("corrupt archive (unknown vehicle)");
            return vehicleName(hs.slots[slot]);
        };
        auto key = [&o](const char *k) { o.push_back('"'); o += k; o += "\":"; };
        auto num = [&](const char *k, double v) { key(k); putJsonNumberLikeRapidjson(o, v); o.push_back(','); };
        o.clear();
        o.reserve(refs.size() * 1100 + 4096);
        o += "{\"step\":" + std::to_string(hs.step) + ",\"activeVehicleCount\":" + std::to_string(img.active) + ",\"rnd\":";
        { std::ostringstream r; r << hs.rnd; putJsonString(o, r.str()); }
        o += ",\"vehicles\":[";
        bool first = true;
        for (const Ref &v : refs) {
            const SlotInfo &si = hs.slots.at(v.slot);
            if (si.shadow) throw std::runtime_error("archive holds lane-change state");
            const VehicleTemplate &t = hs.templates.at(si.tmplId);
            if (!first) o.push_back(',');
            first = false;
            o += "{\"priority\":" + std::to_string(v.priority) + ",\"id\":";
            putJsonString(o, vehicleName(si));
            o.push_back(',');
            num("enterTime", si.enterTime);
            num("speed", v.run ? v.run->speed : t.speed);   // VehicleInfo::speed is the live speed (vehicle.cpp:119)
            num("len", t.len); num("width", t.width); num("maxPosAcc", t.maxPosAcc); num("maxNegAcc", t.maxNegAcc);
            num("usualPosAcc", t.usualPosAcc); num("usualNegAcc", t.usualNegAcc); num("minGap", t.minGap); num("maxSpeed", t.maxSpeed);
            num("headwayTime", t.headwayTime); num("yieldDistance", t.yieldDistance); num("turnSpeed", t.turnSpeed);
            key("route");
            o.push_back('[');
            const Route &rt = routing->route(si.routeId);
            for (size_t k = 0; k < rt.roads.size(); ++k) { if (k) o.push_back(','); putJsonString(o, net.roadId[rt.roads[k]]); }
            o += "],";
            num("dis", v.run ? v.run->dis : 0.0);
            key("drivable"); putJsonString(o, drivableName(v.drivable)); o.push_back(',');
            if (v.run && v.run->prevDrivable >= 0) { key("prevDrivable"); putJsonString(o, drivableName(v.run->prevDrivable)); o.push_back(','); }
            num("approachingIntersectionDistance", t.maxSpeed * t.maxSpeed / t.usualNegAcc / 2 + t.maxSpeed * interval * 2);   // vehicle.cpp:27-28
            num("gap", v.run ? v.run->gap : 0.0);
            key("enterLaneLinkTime"); o += std::to_string((unsigned) (v.run ? v.run->enterLaneLinkTime : INT_MAX)); o.push_back(',');
            if (v.run && v.run->leaderSlot >= 0) { key("leader"); putJsonString(o, nameOf(v.run->leaderSlot)); o.push_back(','); }
            if (v.run && v.run->blockerSlot >= 0) { key("blocker"); putJsonString(o, nameOf(v.run->blockerSlot)); o.push_back(','); }
            o += "\"end\":false,\"running\":";
            o += v.run ? "true" : "false";
            o += ",\"partnerType\":0,\"offset\":0.0,\"laneChangeWaitingTime\":0.0,\"laneChanging\":false,\"laneChangeLastTime\":0.0}";
        }
        o += "],\"drivables\":{";
        for (int d = 0; d < (int) img.drivables.size(); ++d) {
            if (d) o.push_back(',');
            putJsonString(o, drivableName(d));
            o += ":{\"vehicles\":[";
            for (size_t k = 0; k < img.drivables[d].size(); ++k) { if (k) o.push_back(','); putJsonString(o, nameOf(img.drivables[d][k].slot)); }
            o.push_back(']');
            if (d < nL) {
                o += ",\"waitingBuffer\":[";
                for (size_t k = 0; k < img.waiting[d].size(); ++k) { if (k) o.push_back(','); putJsonString(o, nameOf(img.waiting[d][k].slot)); }
                o += "],\"history\":[],\"historyVehicleNum\":0,\"historyAverageSpeed\":0.0";
            }
            o.push_back('}');
        }
        o += "},\"flows\":{";
        for (size_t i = 0; i < flows.size(); ++i) {
            if (i) o.push_back(',');
            putJsonString(o, flows[i].def.id);
            o += ":{";
            num("nowTime", hs.flowNow.at(i)); num("currentTime", hs.flowCur.at(i));
            o += "\"cnt\":" + std::to_string((unsigned) hs.flowCnt.at(i)) + "}";
        }
        o += "},\"trafficLights\":{";
        for (int i = 0; i < net.nInter(); ++i) {
            if (i) o.push_back(',');
            putJsonString(o, net.interId[i]);
            o += ":{";
            num("remainDuration", net.interVirtual[i] ? 0.0 : img.remain.at(i));
            o += "\"curPhaseIndex\":" + std::to_string((unsigned) (net.interVirtual[i] ? 0 : img.curPhase.at(i))) + "}";
        }
        o += "},\"finishedVehicleCnt\":" + std::to_string(hs.finishedCnt) + ",";
        key("cumulativeTravelTime");
        putJsonNumberLikeRapidjson(o, hs.cumulativeTravelTime);
        o += "}";
    }

    void readReferenceArchive(const Json &root, HostState &hs, StateImage &img) {
        if (laneChange) throw std::runtime_error("an archive in the reference's JSON schema is not read with laneChange on");
        if (!laneLocal.empty()) throw std::runtime_error("an archive in the reference's JSON schema is not read by one rank of a sharded engine");
        if (!root.isObject()) throw std::runtime_error("archive file: expected a JSON object");
        auto member = [](const Json &o, const char *name) -> const Json & {
            const Json *v = o.find(name);
            if (!v) throw std::runtime_error(std::string(name) + " is required but missing in json file");   // utility.h:113-127
            return *v;
        };
        auto dbl = [&](const Json &o, const char *name) {
            const Json &v = member(o, name);
            if (!v.isNumber()) throw std::runtime_error(std::string(name) + ": expected a number");
            return v.asDouble();
        };
        auto integer = [&](const Json &o, const char *name) -> long long {
            const Json &v = member(o, name);
            if (!v.isNumber() || v.kind == Json::Double) throw std::runtime_error(std::string(name) + ": expected an integer");
            return (v.kind == Json::Int || v.kind == Json::Int64) ? (long long) v.i : (long long) v.u;
        };
        auto str = [&](const Json &o, const char *name) -> const std::string & {
            const Json &v = member(o, name);
            if (!v.isString()) throw std::runtime_error(std::string(name) + ": expected a string");
            return v.s;
        };
        auto optStr = [](const Json &o, const char *name) -> const std::string * {
            const Json *v = o.find(name);
            return v && v->isString() ? &v->s : nullptr;
        };
        hs = HostState();
        img = StateImage();
        { std::istringstream r(str(root, "rnd")); r >> hs.rnd; if (!r) throw std::runtime_error("rnd: not a std::mt19937 state"); }
        hs.step = (size_t) integer(root, "step");
        img.step = (long long) hs.step;
        img.active = (int) integer(root, "activeVehicleCount");
        const Json &vehicles = member(root, "vehicles");
        if (!vehicles.isArray()) throw std::runtime_error("vehicles: expected an array");
        const int nL = net.nLanes(), nD = net.nDrivables(), n = (int) vehicles.arr.size();
        std::unordered_map<std::string, int> drvIndex, slotOfName;
        for (int d = 0; d < nD; ++d) drvIndex.emplace(drivableName(d), d);
        auto drivableOf = [&](const std::string &id) {
            auto it = drvIndex.find(id);
            if (it == drvIndex.end()) throw std::runtime_error("No such drivable: " + id);
            return it->second;
        };
        hs.slots.assign(n, SlotInfo());
        std::vector<double> speed(n);
        std::vector<char> running(n);
        for (int k = 0; k < n; ++k) {
            const Json &v = vehicles.arr[k];
            if (!v.isObject()) throw std::runtime_error("vehicles: expected objects");
            SlotInfo &si = hs.slots[k];
            const std::string &id = str(v, "id");
            {   // flow_<flow>_<index> (flow.cpp:14) / manually_pushed_<index> (engine.cpp:700)
                char *end = nullptr;
                if (id.compare(0, 16, "manually_pushed_") == 0) {
                    si.flow = -2;
                    si.index = (int) strtol(id.c_str() + 16, &end, 10);
                } else if (id.compare(0, 5, "flow_") == 0) {
                    si.flow = (int) strtol(id.c_str() + 5, &end, 10);
                    if (*end != '_' || si.flow < 0 || si.flow >= (int) flows.size()) throw std::runtime_error("vehicle id not understood: " + id);
                    si.index = (int) strtol(end + 1, &end, 10);
                }
                if (!end || *end != 0) throw std::runtime_error("vehicle id not understood: " + id + (id.find("shadow") != std::string::npos ? " (lane-change state is not read)" : ""));
            }
            if (!slotOfName.emplace(id, k).second) throw std::runtime_error("vehicle listed twice: " + id);
            if (integer(v, "partnerType") != 0) throw std::runtime_error("archive holds lane-change state (partner vehicles): not read");
            si.priority = (int) integer(v, "priority");
            si.enterTime = dbl(v, "enterTime");
            si.spawnStep = (int32_t) std::llround(si.enterTime / interval);
            const Json &rn = member(v, "running");
            if (!rn.isBool()) throw std::runtime_error("running: expected a bool");
            running[k] = rn.asBool();
            speed[k] = dbl(v, "speed");
            VehicleTemplate t;
            t.speed = running[k] ? 0.0 : speed[k];   // a running vehicle's initial speed is never read again
            t.len = dbl(v, "len"); t.width = dbl(v, "width"); t.maxPosAcc = dbl(v, "maxPosAcc"); t.maxNegAcc = dbl(v, "maxNegAcc");
            t.usualPosAcc = dbl(v, "usualPosAcc"); t.usualNegAcc = dbl(v, "usualNegAcc"); t.minGap = dbl(v, "minGap");
            t.maxSpeed = dbl(v, "maxSpeed"); t.headwayTime = dbl(v, "headwayTime"); t.yieldDistance = dbl(v, "yieldDistance");
            t.turnSpeed = dbl(v, "turnSpeed");
            checkFitsLayout(t);
            si.tmplId = internTemplate(t);
            const Json &rj = member(v, "route");
            if (!rj.isArray()) throw std::runtime_error("route: expected an array");
            std::vector<int> roads;
            for (const Json &r : rj.arr) {
                if (!r.isString()) throw std::runtime_error("route: expected strings");
                auto it = net.roadIndex.find(r.s);
                if (it == net.roadIndex.end()) throw std::runtime_error("No such road: " + r.s);
                roads.push_back(it->second);
            }
            si.routeId = routing->intern(roads);
            if (!routing->route(si.routeId).valid || routing->route(si.routeId).roads != roads)
                throw std::runtime_error("route of vehicle " + id + " is not a path of this road network");
            si.live = true;
        }
        auto slotOf = [&](const std::string *id) {
            if (!id) return -1;
            auto it = slotOfName.find(*id);
            if (it == slotOfName.end()) throw std::runtime_error("No such vehicle: " + *id);
            return it->second;
        };
        const Json &drivables = member(root, "drivables");
        if (!drivables.isObject()) throw std::runtime_error("drivables: expected an object");
        std::unordered_map<std::string, const Json *> drvJson;
        for (const auto &kv : drivables.obj) drvJson.emplace(kv.first, &kv.second);
        img.drivables.assign(nD, {});
        img.waiting.assign(nL, {});
        std::vector<char> placed(n, 0);
        int runningCount = 0;
        for (int d = 0; d < nD; ++d) {
            auto dj = drvJson.find(drivableName(d));
            if (dj == drvJson.end()) throw std::runtime_error(drivableName(d) + " is required but missing in json file");
            const Json &list = member(*dj->second, "vehicles");
            if (!list.isArray()) throw std::runtime_error("vehicles: expected an array");
            for (const Json &e : list.arr) {
                if (!e.isString()) throw std::runtime_error("vehicles: expected strings");
                const int k = slotOf(&e.s);
                const Json &v = vehicles.arr[k];
                if (placed[k]++ || !running[k] || drivableOf(str(v, "drivable")) != d) throw std::runtime_error("vehicle " + e.s + " is listed on a drivable it is not on");
                const SlotInfo &si = hs.slots[k];
                StateImage::Running r{};
                r.slot = k; r.tmpl = si.tmplId; r.priority = si.priority;
                const int plan = routing->planFrom(si.routeId, d);
                if (plan < 0) throw std::runtime_error("vehicle " + e.s + " is on a road that is not on its route");
                r.planIdx = routing->planBeg()[plan];
                r.nextDrivable = routing->planData()[r.planIdx + 1];
                const std::string *prev = optStr(v, "prevDrivable");
                r.prevDrivable = prev ? drivableOf(*prev) : -1;
                r.blockerSlot = slotOf(optStr(v, "blocker"));
                r.leaderSlot = slotOf(optStr(v, "leader"));
                const long long ell = integer(v, "enterLaneLinkTime");   // written as unsigned (archive.cpp:219-220); INT_MAX on a lane (engine.cpp:489)
                r.enterLaneLinkTime = ell < 0 || ell > INT_MAX ? INT_MAX : (int) ell;
                r.dis = dbl(v, "dis"); r.speed = speed[k]; r.gap = dbl(v, "gap");
                r.len = templates[si.tmplId].len;
                img.drivables[d].push_back(r);
                ++runningCount;
            }
            if (d < nL) {
                const Json &wb = member(*dj->second, "waitingBuffer");
                if (!wb.isArray()) throw std::runtime_error("waitingBuffer: expected an array");
                for (const Json &e : wb.arr) {
                    if (!e.isString()) throw std::runtime_error("waitingBuffer: expected strings");
                    const int k = slotOf(&e.s);
                    if (placed[k]++ || running[k]) throw std::runtime_error("vehicle " + e.s + " is listed twice");
                    SlotInfo &si = hs.slots[k];
                    const int plan = routing->planFrom(si.routeId, d);
                    if (plan < 0) throw std::runtime_error("vehicle " + e.s + " waits on a road that is not on its route");
                    si.firstLane = d;
                    img.waiting[d].push_back(StateImage::Waiting{k, si.tmplId, si.priority, plan});
                }
            }
        }
        for (int k = 0; k < n; ++k) if (!placed[k]) throw std::runtime_error("vehicle " + vehicleName(hs.slots[k]) + " is on no drivable");
        if (runningCount != img.active) throw std::runtime_error("activeVehicleCount does not match the drivables' lists");
        img.slotCount = n;
        const Json &fl = member(root, "flows");
        for (size_t i = 0; i < flows.size(); ++i) {
            const Json &f = member(fl, flows[i].def.id.c_str());
            hs.flowNow.push_back(dbl(f, "nowTime")); hs.flowCur.push_back(dbl(f, "currentTime")); hs.flowCnt.push_back((int) integer(f, "cnt"));
            hs.flowValid.push_back((uint8_t) hot[i].valid);     // not archived by the reference: the engine's stays
        }
        const Json &tl = member(root, "trafficLights");
        img.curPhase.assign(net.nInter(), 0);
        img.remain.assign(net.nInter(), 0.0);
        for (int i = 0; i < net.nInter(); ++i) {
            const Json &t = member(tl, net.interId[i].c_str());
            if (net.interVirtual[i]) continue;                  // TrafficLight::init leaves a virtual intersection's light alone (trafficlight.cpp:11)
            img.remain[i] = dbl(t, "remainDuration");
            const long long ph = integer(t, "curPhaseIndex");
            if (ph < 0 || ph >= net.interPhaseBeg[i + 1] - net.interPhaseBeg[i]) throw std::runtime_error("curPhaseIndex out of range");
            img.curPhase[i] = (int) ph;
        }
        hs.finishedCnt = (int) integer(root, "finishedVehicleCnt");
        hs.cumulativeTravelTime = dbl(root, "cumulativeTravelTime");
        hs.manuallyPushCnt = manuallyPushCnt;                   // not archived by the reference either
        for (int r = 0; r < routing->numRoutes(); ++r) hs.routeAnchors.push_back(routing->anchorsOf(r));
        hs.templates = templates;
    }

    cfb_vehicle_ref refOf(int slot) const { return cfb_vehicle_ref{slots[slot].flow, slots[slot].index}; }
};

}  // namespace cfb

// ------------------------------------------------------------------------------------------
// C ABI
namespace {
// Engines alive in this process.  A snapshot remembers the engine it was taken from (a JSON dump needs its road network
// for names); dumping after that engine was destroyed must fail cleanly, not touch freed memory.
std::mutex g_liveMutex;
std::map<const cfb_engine *, uint64_t> g_live;
uint64_t g_nextSerial = 1;
}  // namespace

struct cfb_engine {
    cfb_engine() {
        std::lock_guard<std::mutex> lock(g_liveMutex);
        serial = g_nextSerial++;
        g_live[this] = serial;
    }
    ~cfb_engine() {
        std::lock_guard<std::mutex> lock(g_liveMutex);
        g_live.erase(this);
    }
    cfb_engine(const cfb_engine &) = delete;
    cfb_engine &operator=(const cfb_engine &) = delete;
    uint64_t serial = 0;
    cfb::HostEngine h;
    std::string lastError;
    std::vector<cfb::SpeedRec> recs;
    std::unique_ptr<cfb::ShardTransport> transport;   // sharded run: destroyed before the device (see cfb_engine_destroy)
};

namespace {
// Every entry point runs with the engine's GPU current and leaves the caller's device as it found it: the engine may sit
// on another GPU than torch's current one, a second engine may sit on a third, and a fresh host thread starts on device 0.
struct DeviceGuard {
    int prev = -1;
    explicit DeviceGuard(const cfb_engine *e) {
        if (!e || !e->h.dev) return;
        const int want = e->h.dev->device();
        if (cudaGetDevice(&prev) != cudaSuccess) { prev = -1; cudaGetLastError(); }
        if (prev != want) cudaSetDevice(want); else prev = -1;
    }
    ~DeviceGuard() { if (prev >= 0) cudaSetDevice(prev); }
};
}  // namespace

static thread_local std::string g_createError;

#define CFB_TRY(e, ...)                                    \
    try {                                                  \
        DeviceGuard guard_(e);                             \
        __VA_ARGS__                                        \
    } catch (const std::exception &ex) {                   \
        (e)->lastError = ex.what();                        \
        const char *w = ex.what();                         \
        if (strstr(w, "CUDA")) return CFB_ERR_DEVICE;      \
        if (strstr(w, "capacity")) return CFB_ERR_CAPACITY;\
        return CFB_ERR_ARGUMENT;                           \
    }

extern "C" {

cfb_engine *cfb_engine_create(const char *config_file, int thread_num, int device) {
    (void) thread_num;
    cfb_engine *e = nullptr;
    int prevDevice = -1;   // the DeviceSim constructor selects the engine's GPU: the caller's current device is put back
    if (cudaGetDevice(&prevDevice) != cudaSuccess) { prevDevice = -1; cudaGetLastError(); }
    struct Restore { int d; ~Restore() { if (d >= 0) cudaSetDevice(d); } } restore{prevDevice};
    try {
        e = new cfb_engine();
        int dev = device;
        if (dev < 0) dev = 0;
        if (!e->h.load(config_file ? config_file : "", dev)) {
            g_createError = e->h.error.empty() ? "load config failed!" : e->h.error;
            std::cerr << g_createError << std::endl << "load config failed!" << std::endl;
            delete e;
            return nullptr;
        }
        return e;
    } catch (const std::exception &ex) {
        g_createError = ex.what();
        delete e;
        return nullptr;
    }
}

void cfb_engine_destroy(cfb_engine *e) {
    if (!e) return;
    DeviceGuard guard(e);
    e->h.transport = nullptr;
    e->transport.reset();   // NCCL communicator + peer mappings go before the device state
    delete e;
}

const char *cfb_last_error(const cfb_engine *e) { return e ? e->lastError.c_str() : g_createError.c_str(); }

int cfb_next_step(cfb_engine *e) {
    CFB_TRY(e, e->h.nextStep();)
    return CFB_OK;
}

int cfb_next_steps(cfb_engine *e, int n) {
    CFB_TRY(e, for (int i = 0; i < n; ++i) e->h.nextStep();)
    return CFB_OK;
}

int64_t cfb_get_vehicle_count(cfb_engine *e) {
    CFB_TRY(e, int c = e->h.dev->vehicleCount(); e->h.checkDevice(); e->h.d2hBytes += 16; return c;)   // {epoch, active, error, ties}: stored by k_leader into mapped host memory
}

double cfb_get_current_time(const cfb_engine *e) { return e->h.currentTime(); }

double cfb_get_average_travel_time(cfb_engine *e) {
    try {
        DeviceGuard guard(e);
        cfb::HostEngine &h = e->h;
        h.cancelAhead();
        h.drain();
        double tt = h.cumulativeTravelTime;
        int n = h.finishedCnt;
        for (auto &kv : h.pool.sorted()) {  // priority order, like vehiclePool (engine.cpp:685-689)
            tt += h.currentTime() - h.slots[kv.second].enterTime;
            n++;
        }
        return n == 0 ? 0 : tt / n;
    } catch (const std::exception &ex) {
        e->lastError = ex.what();
        return std::nan("");
    }
}

int cfb_num_lanes(const cfb_engine *e) { return e->h.net.nLanes(); }
const char *cfb_lane_id(const cfb_engine *e, int lane) {
    return lane >= 0 && lane < e->h.net.nLanes() ? e->h.laneIds[lane].c_str() : nullptr;
}
int cfb_num_intersections(const cfb_engine *e) { return e->h.net.nInter(); }
const char *cfb_intersection_id(const cfb_engine *e, int i) {
    return i >= 0 && i < e->h.net.nInter() ? e->h.net.interId[i].c_str() : nullptr;
}

int cfb_get_lane_vehicle_count(cfb_engine *e, int32_t *out, int n) {
    if (n < e->h.net.nLanes()) { e->lastError = "output buffer too small"; return CFB_ERR_ARGUMENT; }
    CFB_TRY(e, e->h.dev->laneVehicleCount(out);)
    return CFB_OK;
}

int cfb_get_lane_waiting_vehicle_count(cfb_engine *e, int32_t *out, int n) {
    if (n < e->h.net.nLanes()) { e->lastError = "output buffer too small"; return CFB_ERR_ARGUMENT; }
    CFB_TRY(e, e->h.dev->laneWaitingVehicleCount(out);)
    return CFB_OK;
}

int cfb_observe_device(cfb_engine *e, void *consumer_stream, cfb_device_obs *out) {
    if (!out) { e->lastError = "null output"; return CFB_ERR_ARGUMENT; }
    CFB_TRY(e,
        const cfb::DeviceObs o = e->h.dev->observeOnDevice(consumer_stream);
        out->lane_vehicle_count = o.laneCount;
        out->lane_waiting_count = o.laneWaiting;
        out->lane_speed_sum = o.laneSpeedSum;
        out->n_lanes = o.nLanes;
        out->device = o.device;
    )
    return CFB_OK;
}

int64_t cfb_get_vehicle_speed(cfb_engine *e, cfb_vehicle_ref *ids, double *speed, double *distance, int64_t cap) {
    CFB_TRY(e,
        cfb::HostEngine &h = e->h;
        int n = h.dev->runningVehicles(e->recs);
        // vehiclePool order = ascending priority (engine.cpp:780-790)
        std::sort(e->recs.begin(), e->recs.end(), [&h](const cfb::SpeedRec &a, const cfb::SpeedRec &b) {
            return h.slots[a.slot].priority < h.slots[b.slot].priority;
        });
        for (int64_t i = 0; i < n && i < cap; ++i) {
            if (ids) ids[i] = h.refOf(e->recs[i].slot);
            if (speed) speed[i] = e->recs[i].speed;
            if (distance) distance[i] = e->recs[i].dis;
        }
        return n;
    )
}

int64_t cfb_get_vehicles(cfb_engine *e, int include_waiting, cfb_vehicle_ref *ids, int64_t cap) {
    CFB_TRY(e,
        cfb::HostEngine &h = e->h;
        if (!include_waiting) return cfb_get_vehicle_speed(e, ids, nullptr, nullptr, cap);
        h.cancelAhead();
        h.drain();
        int64_t n = 0;
        for (auto &kv : h.pool.sorted()) {
            if (n < cap && ids) ids[n] = h.refOf(kv.second);
            ++n;
        }
        return n;
    )
}

int64_t cfb_get_lane_vehicles(cfb_engine *e, int64_t *lane_begin, int n_lanes_plus1, cfb_vehicle_ref *ids, int64_t cap) {
    if (n_lanes_plus1 < e->h.net.nLanes() + 1) { e->lastError = "output buffer too small"; return CFB_ERR_ARGUMENT; }
    CFB_TRY(e,
        std::vector<int32_t> slots; std::vector<int32_t> beg;
        e->h.dev->laneVehicleSlots(slots, beg);
        for (size_t l = 0; l < beg.size(); ++l) lane_begin[l] = beg[l];
        for (size_t i = 0; i < slots.size() && (int64_t) i < cap; ++i) ids[i] = e->h.refOf(slots[i]);
        return (int64_t) slots.size();
    )
}

int cfb_get_leader(cfb_engine *e, cfb_vehicle_ref v, cfb_vehicle_ref *leader, int *found) {
    CFB_TRY(e,
        cfb::HostEngine &h = e->h;
        h.cancelAhead();
        h.drain();
        const int vs = h.slotOfId(v.flow, v.index);
        if (vs < 0) throw std::runtime_error("Vehicle not found");
        int ls = h.dev->leaderSlotOf(vs);
        *found = ls >= 0;
        if (ls >= 0) *leader = h.refOf(ls);
    )
    return CFB_OK;
}

int cfb_set_tl_phase_index(cfb_engine *e, int intersection, int phase) {
    cfb::HostEngine &h = e->h;
    if (!h.rlTrafficLight) {  // engine.cpp:720-723
        std::cerr << "please set rlTrafficLight to true to enable traffic light control" << std::endl;
        return CFB_OK;
    }
    if (intersection < 0 || intersection >= h.net.nInter()) { e->lastError = "no such intersection"; return CFB_ERR_ARGUMENT; }
    const int nph = h.net.interPhaseBeg[intersection + 1] - h.net.interPhaseBeg[intersection];
    if (phase < 0 || phase >= nph) {
        // the reference stores the index unchecked and throws later from phases.at() inside a worker
        e->lastError = "phase index out of range";
        return CFB_ERR_ARGUMENT;
    }
    CFB_TRY(e, h.dev->setPhase(intersection, phase);)
    return CFB_OK;
}

int cfb_set_tl_phases_device(cfb_engine *e, const int32_t *phases, void *producer_stream) {
    if (!e->h.rlTrafficLight) {  // engine.cpp:720-723
        std::cerr << "please set rlTrafficLight to true to enable traffic light control" << std::endl;
        return CFB_OK;
    }
    if (!phases) { e->lastError = "null phase array"; return CFB_ERR_ARGUMENT; }
    CFB_TRY(e, e->h.dev->setPhasesFromDevice(phases, producer_stream);)
    return CFB_OK;
}

int cfb_set_tl_phase(cfb_engine *e, const char *id, int phase) {
    auto it = e->h.net.interIndex.find(id ? id : "");
    if (it == e->h.net.interIndex.end()) {
        if (!e->h.rlTrafficLight) return cfb_set_tl_phase_index(e, -1, phase);
        e->lastError = std::string("no such intersection: ") + (id ? id : "");
        return CFB_ERR_ARGUMENT;
    }
    return cfb_set_tl_phase_index(e, it->second, phase);
}

int cfb_set_replay_file(cfb_engine *e, const char *log_file) {  // Engine::setReplayLogFile engine.cpp:727-734
    cfb::HostEngine &h = e->h;
    if (!h.saveReplayInConfig) {
        std::cerr << "saveReplay is not set to true in config file!" << std::endl;
        return CFB_OK;
    }
    if (h.logOut.is_open()) h.logOut.close();
    h.logOut.clear();
    h.logOut.open(h.dir + (log_file ? log_file : ""));
    return CFB_OK;
}

int cfb_set_save_replay(cfb_engine *e, int open) {  // Engine::setSaveReplay engine.cpp:736-742
    cfb::HostEngine &h = e->h;
    if (!h.saveReplayInConfig) {
        std::cerr << "saveReplay is not set to true in config file!" << std::endl;
        return CFB_OK;
    }
    h.saveReplay = open != 0 && !h.transport && h.replay;
    return CFB_OK;
}

struct cfb_replay {
    cfb::RoadNet net;
    std::unique_ptr<cfb::ReplayWriter> w;
    std::string buf;
};

cfb_replay *cfb_replay_create(const char *roadnet_file) {
    std::unique_ptr<cfb_replay> r(new cfb_replay());
    if (!roadnet_file || !r->net.load(roadnet_file)) { g_createError = "loading roadnet file error!"; return nullptr; }
    r->w.reset(new cfb::ReplayWriter(r->net));
    return r.release();
}
void cfb_replay_destroy(cfb_replay *r) { delete r; }
static int64_t copyOut(const std::string &s, char *out, int64_t cap) {
    if (out && cap > 0) {
        const size_t n = std::min<size_t>(s.size(), (size_t) cap - 1);
        memcpy(out, s.data(), n);
        out[n] = 0;
    }
    return (int64_t) s.size() + 1;
}
int64_t cfb_replay_roadnet_json(cfb_replay *r, char *out, int64_t cap) { return copyOut(r->w->roadnetJson(), out, cap); }
int64_t cfb_replay_format_step(cfb_replay *r, const cfb_replay_vehicle *v, int64_t n, const int32_t *phase, char *out, int64_t cap) {
    static_assert(sizeof(cfb_replay_vehicle) == sizeof(cfb::ReplayVehicle), "cfb_replay_vehicle layout");
    r->w->formatStep(reinterpret_cast<const cfb::ReplayVehicle *>(v), (size_t) n, phase, r->buf);
    return copyOut(r->buf, out, cap);
}

// Test support (include/cityflow_b200.h): every running vehicle including shadows, LC_DTYPE layout.
int64_t cfb_debug_lc_vehicles(cfb_engine *e, cfb_lc_vehicle *out, int64_t cap) {
    CFB_TRY(e,
        cfb::HostEngine &h = e->h;
        std::vector<cfb::DeviceSim::LcDebugRec> recs;
        h.dev->debugDumpLc(recs);
        std::sort(recs.begin(), recs.end(), [](const cfb::DeviceSim::LcDebugRec &a, const cfb::DeviceSim::LcDebugRec &b) { return a.priority < b.priority; });
        auto prio = [&h](int slot) { return slot >= 0 ? h.slots[slot].priority : -1; };
        for (int64_t i = 0; i < (int64_t) recs.size() && i < cap; ++i) {
            const auto &r = recs[i];
            cfb_lc_vehicle &o = out[i];
            o.flow = h.slots[r.slot].flow; o.cnt = h.slots[r.slot].index; o.priority = r.priority;
            o.partner_type = r.partnerType; o.partner = prio(r.partnerSlot); o.drivable = r.drivable;
            o.leader = prio(r.leaderSlot); o.blocker = prio(r.blockerSlot); o.flags = r.flags; o.last_dir = r.lastDir;
            o.dis = r.dis; o.speed = r.speed; o.gap = r.gap; o.offset = r.offset; o.waiting_time = r.waiting;
            o.last_change_time = r.lastChange;
        }
        return (int64_t) recs.size();
    )
}

int cfb_set_random_seed(cfb_engine *e, int seed) {
    e->h.cancelAhead();
    e->h.rnd.seed(seed);
    return CFB_OK;
}

int cfb_reset(cfb_engine *e, int reset_rnd) {
    CFB_TRY(e, e->h.reset(reset_rnd != 0);)
    return CFB_OK;
}

int cfb_push_vehicle(cfb_engine *e, const double v[10], const char *const *roads, int n_roads) {
    CFB_TRY(e,
        cfb::HostEngine &h = e->h;
        h.cancelAhead();
        cfb::VehicleTemplate t;
        double *f[10] = {&t.speed, &t.len, &t.width, &t.maxPosAcc, &t.maxNegAcc, &t.usualPosAcc, &t.usualNegAcc,
                         &t.minGap, &t.maxSpeed, &t.headwayTime};
        for (int k = 0; k < 10; ++k) if (!std::isnan(v[k])) *f[k] = v[k];
        h.checkFitsLayout(t);
        std::vector<int> anchors;
        for (int k = 0; k < n_roads; ++k) {
            auto it = h.net.roadIndex.find(roads[k]);
            if (it == h.net.roadIndex.end()) throw std::runtime_error(std::string("No such road: ") + roads[k]);
            anchors.push_back(it->second);
        }
        if (anchors.empty()) throw std::runtime_error("push_vehicle needs at least one road");
        int routeId = h.routing->intern(anchors);
        int tmplId = h.internTemplate(t);
        h.createVehicle(-2, h.manuallyPushCnt++, routeId, tmplId, anchors[0]);
    )
    return CFB_OK;
}

// Full dynamic state of every running vehicle (tests only), same record layout as
// oracle/refdump's per-vehicle dump: 8 x int32, 3 x double, 1 x int64.
int64_t cfb_debug_vehicles(cfb_engine *e, void *out, int64_t cap) {
    struct Rec { int32_t flow, cnt, priority, drivable, lf, lc, bf, bc; double dis, speed, gap; int64_t enter; };
    CFB_TRY(e,
        cfb::HostEngine &h = e->h;
        std::vector<cfb::DebugRec> recs;
        h.dev->debugDump(recs);
        Rec *o = (Rec *) out;
        for (size_t i = 0; i < recs.size() && (int64_t) i < cap; ++i) {
            const cfb::DebugRec &r = recs[i];
            Rec x;
            x.flow = h.slots[r.slot].flow; x.cnt = h.slots[r.slot].index; x.priority = r.priority; x.drivable = r.drivable;
            x.lf = r.leaderSlot >= 0 ? h.slots[r.leaderSlot].flow : -1;
            x.lc = r.leaderSlot >= 0 ? h.slots[r.leaderSlot].index : -1;
            x.bf = r.blockerSlot >= 0 ? h.slots[r.blockerSlot].flow : -1;
            x.bc = r.blockerSlot >= 0 ? h.slots[r.blockerSlot].index : -1;
            x.dis = r.dis; x.speed = r.speed; x.gap = r.gap; x.enter = r.enterLaneLinkTime;
            o[i] = x;
        }
        return (int64_t) recs.size();
    )
}

// n steps, each bracketed by CUDA events on the engine stream; optional L2 flush between steps
// (outside the brackets).  Returns the summed device time in ms and the vehicle-steps done.
int cfb_timed_steps(cfb_engine *e, int n, int flush_l2, double *ms, int64_t *vehicle_steps) {
    CFB_TRY(e,
        cfb::HostEngine &h = e->h;
        h.dev->synchronize();
        const unsigned long long v0 = h.dev->vehicleSteps();
        if (flush_l2) {
            for (int i = 0; i < n; ++i) {  // one bracket per step, the flush sits between brackets
                h.dev->flushL2();
                h.dev->markTimed();
                h.nextStep();
                h.dev->markTimed();
            }
        } else {  // back to back: one bracket around all n steps (includes any host-paced gaps)
            h.dev->markTimed();
            for (int i = 0; i < n; ++i) h.nextStep();
            h.dev->markTimed();
        }
        *ms = h.dev->collectTimedMs();
        *vehicle_steps = (int64_t) (h.dev->vehicleSteps() - v0);
        h.checkDevice();
    )
    return CFB_OK;
}
int64_t cfb_vehicle_steps(cfb_engine *e) {
    CFB_TRY(e, return (int64_t) e->h.dev->vehicleSteps();)
}

int64_t cfb_finished_vehicle_count(cfb_engine *e) {
    CFB_TRY(e, e->h.cancelAhead(); e->h.drain(); return (int64_t) e->h.finishedCnt;)
}
int64_t cfb_gpu_launches(const cfb_engine *e) { return e->h.dev->launchesDone(); }
int cfb_debug_launch_form(const cfb_engine *e, int32_t out[4]) {
    int f[4];
    e->h.dev->launchForm(f);
    for (int k = 0; k < 4; ++k) out[k] = f[k];
    return CFB_OK;
}
int cfb_debug_step_grids(const cfb_engine *e, int32_t out[5]) {
    int g[5];
    e->h.dev->stepGrids(g);
    for (int k = 0; k < 5; ++k) out[k] = g[k];
    return CFB_OK;
}
int64_t cfb_tie_count(cfb_engine *e) {
    CFB_TRY(e, return (int64_t) e->h.dev->tieCount();)
}
int cfb_enable_kernel_timing(cfb_engine *e, int on) { e->h.dev->enableKernelTiming(on != 0); return CFB_OK; }
int cfb_kernel_times(cfb_engine *e, double ms[5], int64_t *steps) {
    auto t = e->h.dev->kernelTimes();
    ms[0] = t.ingest; ms[1] = t.notify; ms[2] = t.control; ms[3] = t.move; ms[4] = t.leader;
    if (steps) *steps = t.launches;
    return CFB_OK;
}
int cfb_shard_phase_times(cfb_engine *e, double ms[8], int64_t *steps) {
    long long n = 0;
    e->h.dev->shardStepTimes(ms, &n);
    if (steps) *steps = n;
    return CFB_OK;
}
int cfb_synchronize(cfb_engine *e) {
    CFB_TRY(e, e->h.dev->synchronize();)
    return CFB_OK;
}
int64_t cfb_num_drivables(const cfb_engine *e) { return e->h.dev->numDrivables(); }
int cfb_device(const cfb_engine *e) { return e->h.dev->device(); }

}  // extern "C"

// Engine::setVehicleSpeed engine.cpp:827-834
extern "C" int cfb_set_vehicle_speed(cfb_engine *e, cfb_vehicle_ref v, double speed) {
    CFB_TRY(e,
        cfb::HostEngine &h = e->h;
        h.cancelAhead();
        h.drain();
        const int s = h.slotOfId(v.flow, v.index);
        if (s < 0) throw std::runtime_error("Vehicle not found");
        h.dev->setCustomSpeed(s, speed);
    )
    return CFB_OK;
}

// Engine::setRoute engine.cpp:852-866 / Router::setRoute router.cpp:245-264.  *ok = 1 when the new
// route was accepted.
extern "C" int cfb_set_vehicle_route(cfb_engine *e, cfb_vehicle_ref v, const char *const *roads, int n_roads, int *ok) {
    *ok = 0;
    CFB_TRY(e,
        cfb::HostEngine &h = e->h;
        h.cancelAhead();
        h.drain();
        const int s = h.slotOfId(v.flow, v.index);
        if (s < 0) return CFB_OK;                       // unknown vehicle: false
        std::vector<int> anchors;
        for (int k = 0; k < n_roads; ++k) {
            auto it = h.net.roadIndex.find(roads[k]);
            if (it == h.net.roadIndex.end()) return CFB_OK;  // unknown road: false
            anchors.push_back(it->second);
        }
        cfb::DeviceSim::VehState st;
        int curLane;
        if (h.dev->vehicleState(s, st)) {
            if (st.drivable >= h.net.nLanes()) return CFB_OK;  // on a laneLink: false (router.cpp:246)
            curLane = st.drivable;
        } else {
            curLane = h.slots[s].firstLane;
            if (curLane < 0) return CFB_OK;                    // still waiting for planRoute
        }
        std::vector<int> full;
        full.push_back(h.net.laneRoad[curLane]);
        full.insert(full.end(), anchors.begin(), anchors.end());
        const int rid = h.routing->intern(full);
        const cfb::Route &rt = h.routing->route(rid);
        if (!rt.valid) return CFB_OK;
        int plan = -1;
        for (size_t k = 0; k < rt.startLanes.size(); ++k)
            if (rt.startLanes[k] == curLane) plan = rt.planOfStartLane[k];
        if (plan < 0) return CFB_OK;                           // !onValidLane(): restore the old route
        if ((size_t) h.routing->numPlans() != h.uploadedPlans) { h.dev->uploadPlans(*h.routing); h.uploadedPlans = h.routing->numPlans(); }
        const int planIdx = h.routing->planBeg()[plan];
        // onValidLane() (router.h:66-68) also fails when the lane links to the next road but none of
        // those links ends in a lane that can continue to the road after it (router.cpp:65-73)
        if (h.routing->planData()[planIdx + 1] == cfb::PLAN_DEAD) return CFB_OK;
        h.dev->setVehiclePlan(s, plan, planIdx, h.routing->planData()[planIdx + 1]);
        h.slots[s].routeId = rid;
        *ok = 1;
    )
    return CFB_OK;
}

// Engine::getVehicleInfo engine.cpp:868-876 / Vehicle::getInfo vehicle.cpp:435-457.  Fills `out`
// with "key\0value\0key\0value\0...\0"; returns the number of bytes needed.
extern "C" int64_t cfb_get_vehicle_info(cfb_engine *e, cfb_vehicle_ref v, char *out, int64_t cap) {
    CFB_TRY(e,
        cfb::HostEngine &h = e->h;
        h.cancelAhead();
        h.drain();
        const int s = h.slotOfId(v.flow, v.index);
        if (s < 0) throw std::runtime_error("Vehicle not found");
        std::string buf;
        auto put = [&buf](const std::string &k, const std::string &val) { buf += k; buf.push_back('\0'); buf += val; buf.push_back('\0'); };
        cfb::DeviceSim::VehState st;
        const bool running = h.dev->vehicleState(s, st);
        put("running", std::to_string(running));
        if (running) {
            const cfb::RoadNet &n = h.net;
            put("distance", std::to_string(st.dis));
            put("speed", std::to_string(st.speed));
            const bool onLane = st.drivable < n.nLanes();
            if (onLane) {
                put("drivable", n.laneName(st.drivable));
                const int road = n.laneRoad[st.drivable];
                put("road", n.roadId[road]);
                put("intersection", n.interId[n.roadEndInter[road]]);
            } else {
                const int ll = st.drivable - n.nLanes();
                put("drivable", n.laneName(n.llStartLane[ll]) + "_TO_" + n.laneName(n.llEndLane[ll]));
            }
            // Router::getFollowingRoads: from the current road of the route to its end
            std::string route;
            const int rid = h.slots[s].routeId;
            if (rid >= 0) {
                const auto &pb = h.routing->planBeg();
                int plan = (int) (std::upper_bound(pb.begin(), pb.end(), st.planIdx) - pb.begin()) - 1;
                const int rpos = (st.planIdx - pb[plan]) / 2;
                const auto &roads = h.routing->route(rid).roads;
                for (size_t k = rpos; k < roads.size(); ++k) route += n.roadId[roads[k]] + " ";
            }
            put("route", route);
        }
        if (out && (int64_t) buf.size() <= cap) memcpy(out, buf.data(), buf.size());
        return (int64_t) buf.size();
    )
}

extern "C" int cfb_transfer_bytes(const cfb_engine *e, int64_t *h2d, int64_t *d2h) {
    if (h2d) *h2d = e->h.h2dBytes;
    if (d2h) *d2h = e->h.d2hBytes;
    return CFB_OK;
}

extern "C" int cfb_host_times(const cfb_engine *e, double *gen_ms, double *enqueue_ms) {
    if (gen_ms) *gen_ms = e->h.hostGenNs * 1e-6;
    if (enqueue_ms) *enqueue_ms = e->h.hostEnqueueNs * 1e-6;
    if (getenv("CITYFLOW_B200_HOST_PROFILE"))
        fprintf(stderr, "[cityflow_b200] spawner: flow clocks %.3f ms, vehicle creation %.3f ms, planRoute + records %.3f ms (totals)\n",
                e->h.genFlowsNs * 1e-6, e->h.genCreateNs * 1e-6, e->h.genPlanNs * 1e-6);
    return CFB_OK;
}

extern "C" int cfb_debug_counters(cfb_engine *e, uint64_t out[8], int clear) {
    unsigned long long t[8];
    e->h.dev->debugCounters(t, clear != 0);
    for (int k = 0; k < 8; ++k) out[k] = t[k];
    return CFB_OK;
}

extern "C" int64_t cfb_debug_arrays(cfb_engine *e, uint32_t *cyc, uint32_t *path, int64_t cap) {
    if (cap < e->h.dev->numPositions()) return e->h.dev->numPositions();
    return e->h.dev->debugArrays(cyc, path);
}

// ------------------------------------------------------------------------------------------
// Archive: Engine::snapshot / load / loadFromFile, Archive::dump (engine.h:176-178, archive.cpp)
struct cfb_archive {
    cfb::HostEngine::HostState host;
    cfb::DeviceSim::Snapshot *dev = nullptr;
    cfb_engine *owner = nullptr;     // the engine the snapshot was taken from: its road network names what a JSON dump lists
    uint64_t ownerSerial = 0;
    bool ownerAlive() const {
        std::lock_guard<std::mutex> lock(g_liveMutex);
        auto it = g_live.find(owner);
        return it != g_live.end() && it->second == ownerSerial;
    }
    ~cfb_archive() { if (dev) cfb::DeviceSim::freeSnapshot(dev); }
};

namespace {
template <class T> void putVec(std::ostream &o, const std::vector<T> &v) {
    uint64_t n = v.size();
    o.write((const char *) &n, 8);
    if (n) o.write((const char *) v.data(), n * sizeof(T));
}
template <class T> void getVec(std::istream &i, std::vector<T> &v) {
    uint64_t n = 0;
    i.read((char *) &n, 8);
    v.resize(n);
    if (n) i.read((char *) v.data(), n * sizeof(T));
}
}  // namespace

extern "C" {

cfb_archive *cfb_snapshot(cfb_engine *e) {
    try {
        DeviceGuard guard(e);
        cfb_archive *a = new cfb_archive();
        e->h.saveHost(a->host);
        a->dev = e->h.dev->snapshot();
        a->owner = e;
        a->ownerSerial = e->serial;
        return a;
    } catch (const std::exception &ex) {
        e->lastError = ex.what();
        return nullptr;
    }
}

void cfb_archive_destroy(cfb_archive *a) { delete a; }

// (Not on one rank of a sharded engine: the seam mailboxes and their flags are stamped with the engine's own count of
// completed steps, which an image taken at another time would rewind.)
static void refuseShardedLoad(const cfb_engine *e) {
    if (!e->h.laneLocal.empty()) throw std::runtime_error("load / load_from_file: not supported on one rank of a sharded engine");
}

int cfb_load(cfb_engine *e, const cfb_archive *a) {
    CFB_TRY(e,
        refuseShardedLoad(e);
        e->h.dev->synchronize();
        e->h.loadHost(a->host);          // (re-interns routes / templates first: may re-upload tables)
        e->h.dev->restore(a->dev);
    )
    return CFB_OK;
}

static bool endsWithJson(const char *path) {
    const size_t n = strlen(path);
    return n >= 5 && strcmp(path + n - 5, ".json") == 0;
}

int cfb_archive_dump(const cfb_archive *a, const char *path) {
    try {
        if (endsWithJson(path)) {   // the reference's schema (Archive::dump archive.cpp:153-177): interchangeable with it
            if (!a->owner || !a->ownerAlive()) return CFB_ERR_UNSUPPORTED;
            DeviceGuard guard(a->owner);
            if (a->owner->h.laneChange) {
                a->owner->lastError = "an archive in the reference's JSON schema is not written with laneChange on (any other file name gets the binary form)";
                return CFB_ERR_UNSUPPORTED;
            }
            cfb::StateImage img;
            a->owner->h.dev->decodeSnapshot(a->dev, img);
            std::string text;
            try {
                a->owner->h.writeReferenceArchive(a->host, img, text);
            } catch (const std::exception &ex) {
                a->owner->lastError = ex.what();
                return CFB_ERR_UNSUPPORTED;
            }
            std::ofstream o(path, std::ios::binary);   // writeJsonToFile utility.cpp:103-112
            if (!o) return CFB_ERR_ARGUMENT;
            o.write(text.data(), (std::streamsize) text.size());
            return o ? CFB_OK : CFB_ERR_ARGUMENT;
        }
        std::ofstream o(path, std::ios::binary);
        if (!o) return CFB_ERR_ARGUMENT;
        const auto &s = a->host;
        const uint64_t magic = 0x3242464341ULL;  // "ACFB2"
        o.write((const char *) &magic, 8);
        std::ostringstream r;
        r << s.rnd;
        const std::string rs = r.str();
        std::vector<char> rv(rs.begin(), rs.end());
        putVec(o, rv);
        uint64_t step = s.step;
        o.write((const char *) &step, 8);
        o.write((const char *) &s.manuallyPushCnt, 4);
        o.write((const char *) &s.finishedCnt, 4);
        o.write((const char *) &s.cumulativeTravelTime, 8);
        putVec(o, s.flowNow); putVec(o, s.flowCur); putVec(o, s.flowCnt); putVec(o, s.flowValid);
        putVec(o, s.slots); putVec(o, s.freeSlots); putVec(o, s.pending);
        {
            std::vector<int> flat;   // routes: count, then (length, anchors...) each
            flat.push_back((int) s.routeAnchors.size());
            for (const auto &a : s.routeAnchors) { flat.push_back((int) a.size()); flat.insert(flat.end(), a.begin(), a.end()); }
            putVec(o, flat);
            putVec(o, s.templates);
        }
        std::vector<unsigned char> blob;
        cfb::DeviceSim::snapshotToHost(a->dev, blob);
        putVec(o, blob);
        return o ? CFB_OK : CFB_ERR_ARGUMENT;
    } catch (const std::exception &) {
        return CFB_ERR_DEVICE;
    }
}

// Engine::loadFromFile engine.cpp:822-825.  The file is either this engine's binary image or the reference's JSON
// (Archive(Engine &, file) archive.cpp:345-550), told apart by the first bytes; reading the JSON interns the routes and
// vehicle templates it lists (loadHost uploads the grown tables) and rebuilds the device image from the decoded state.
int cfb_load_from_file(cfb_engine *e, const char *path) {
    CFB_TRY(e,
        refuseShardedLoad(e);
        std::ifstream i(path, std::ios::binary);
        if (!i) throw std::runtime_error(std::string("cannot open archive file ") + path);
        uint64_t magic = 0;
        i.read((char *) &magic, 8);
        if (magic != 0x3242464341ULL) {
            i.clear();
            i.seekg(0);
            int c = i.get();
            while (c == ' ' || c == '\n' || c == '\r' || c == '\t') c = i.get();
            if (c != '{') throw std::runtime_error("not an archive: neither this engine's binary image nor the reference's JSON");
            i.close();
            const cfb::Json root = cfb::Json::parseFile(path);
            cfb_archive a;
            cfb::StateImage img;
            e->h.dev->synchronize();
            e->h.cancelAhead();
            e->h.drain();
            e->h.readReferenceArchive(root, a.host, img);
            e->h.loadHost(a.host);
            a.dev = e->h.dev->encodeSnapshot(img);
            e->h.dev->restore(a.dev);
            return CFB_OK;
        }
        cfb_archive a;
        auto &s = a.host;
        std::vector<char> rv;
        getVec(i, rv);
        std::istringstream r(std::string(rv.begin(), rv.end()));
        r >> s.rnd;
        uint64_t step = 0;
        i.read((char *) &step, 8);
        s.step = step;
        i.read((char *) &s.manuallyPushCnt, 4);
        i.read((char *) &s.finishedCnt, 4);
        i.read((char *) &s.cumulativeTravelTime, 8);
        getVec(i, s.flowNow); getVec(i, s.flowCur); getVec(i, s.flowCnt); getVec(i, s.flowValid);
        getVec(i, s.slots); getVec(i, s.freeSlots); getVec(i, s.pending);
        {
            std::vector<int> flat;
            getVec(i, flat);
            size_t k = 0;
            const int nr = flat.empty() ? 0 : flat[k++];
            for (int r = 0; r < nr && k < flat.size(); ++r) {
                const int n = flat[k++];
                if (k + n > flat.size()) throw std::runtime_error("truncated archive file");
                s.routeAnchors.emplace_back(flat.begin() + k, flat.begin() + k + n);
                k += n;
            }
            getVec(i, s.templates);
        }
        std::vector<unsigned char> blob;
        getVec(i, blob);
        if (!i) throw std::runtime_error("truncated archive file");
        a.dev = cfb::DeviceSim::snapshotFromHost(blob.data(), blob.size());
        e->h.dev->synchronize();
        e->h.loadHost(a.host);
        e->h.dev->restore(a.dev);
    )
    return CFB_OK;
}

}  // extern "C"

// ------------------------------------------------------------------------------------------
// Sharded execution (SURVEY.md §8e): one rank of a multi-GPU run over NCCL, and an in-process
// loop-back group (several ranks on one GPU, exchanges by device copies) that the parity tests use
// to check the seam protocol against the unsharded engine.

extern "C" {

int cfb_nccl_unique_id(unsigned char out[128]) {
    std::string err;
    if (!cfb::ncclUniqueIdBytes(out, err)) { g_createError = err; return CFB_ERR_DEVICE; }
    return CFB_OK;
}

cfb_engine *cfb_engine_create_sharded(const char *config_file, int thread_num, int device, int rank, int world,
                                      const unsigned char nccl_id[128]) {
    cfb_engine *e = cfb_engine_create(config_file, thread_num, device);
    if (!e || world <= 1) return e;
    DeviceGuard guard(e);
    std::string err = e->h.configureShard(rank, cfb::Partition::columnStrips(e->h.net, world));
    if (err.empty()) e->transport.reset(cfb::createNcclTransport(rank, world, nccl_id, device < 0 ? 0 : device, err));
    if (!err.empty() || !e->transport) {
        g_createError = "sharded engine: " + err;
        cfb_engine_destroy(e);
        return nullptr;
    }
    e->h.transport = e->transport.get();
    // data plane: peer memory over NVLink unless it is unavailable or CITYFLOW_B200_SHARD_TRANSPORT=nccl asks for
    // the staged NCCL send/recv form (kept for comparison)
    const char *tr = getenv("CITYFLOW_B200_SHARD_TRANSPORT");
    if (!(tr && !strcmp(tr, "nccl"))) {
        try {
            cfb::DeviceSim::ShardArena a = e->h.dev->shardArena();
            std::vector<void *> peers;
            std::string why;
            e->h.dev->shardMarkArenaExported();
            if (e->transport->shareArena(a.base, a.bytes, peers, why)) e->h.dev->shardConnect(peers);
            else std::cerr << "[cityflow_b200] sharded run falls back to NCCL send/recv: " << why << std::endl;
        } catch (const std::exception &ex) {
            g_createError = std::string("sharded engine: ") + ex.what();
            e->h.transport = nullptr;
            cfb_engine_destroy(e);
            return nullptr;
        }
    }
    return e;
}

// global observations in sharded mode (collective: every rank must call them at the same step)
int64_t cfb_shard_vehicle_count(cfb_engine *e) {
    CFB_TRY(e,
        if (!e->h.transport) return (int64_t) e->h.dev->vehicleCount();
        int a = 0;
        if (!e->h.dev->shardVehicleCount(&a)) e->h.dev->shardCounts(e->h.transport, nullptr, &a);
        e->h.d2hBytes += 8;
        e->h.checkDevice();
        return (int64_t) a;
    )
}
int cfb_shard_lane_vehicle_count(cfb_engine *e, int32_t *out, int n, int waiting) {
    if (n < e->h.net.nLanes()) { e->lastError = "output buffer too small"; return CFB_ERR_ARGUMENT; }
    CFB_TRY(e,
        if (!e->h.transport) { if (waiting) e->h.dev->laneWaitingVehicleCount(out); else e->h.dev->laneVehicleCount(out); }
        else if (waiting) e->h.dev->shardWaitingCounts(e->h.transport, out);
        else e->h.dev->shardCounts(e->h.transport, out, nullptr);
    )
    return CFB_OK;
}

}  // extern "C"

// ---- loop-back group ----
struct cfb_shard_group {
    std::vector<cfb_engine *> ranks;
    cfb::Partition part;   // the cut every rank was configured with; the getters take lane owners from it
    std::string lastError;
    bool p2p = false;
};

namespace {
// A failed copy would leave last step's records in a mailbox and the step would carry on with them: every call is checked,
// and cfb_shard_group_step reports the failure.
void loopCheck(cudaError_t err, const char *what) {
    if (err != cudaSuccess)
        throw std::runtime_error(std::string("cityflow_b200 CUDA error in the loop-back exchange (") + what + "): " + cudaGetErrorString(err));
}
// copies between the ranks' exchange buffers (same device): a[send range for b] -> b[recv range for a]
void loopExchange(std::vector<cfb::ShardBuffers> &B, bool tails) {
    const int W = (int) B.size();
    for (int a = 0; a < W; ++a) loopCheck(cudaStreamSynchronize((cudaStream_t) B[a].stream), "stream synchronize");
    for (int a = 0; a < W; ++a)
        for (int b = 0; b < W; ++b) {
            if (a == b) continue;
            if (tails) {  // owner a -> feeder b: a.tailSend over a's "own" list for peer b; b.tailRecv over b's "feed" list for peer a
                const size_t n = (size_t) (B[a].inBeg[b + 1] - B[a].inBeg[b]) * B[a].tailBytes;
                if (n) loopCheck(cudaMemcpy((char *) B[b].tailRecv + (size_t) B[b].outBeg[a] * B[b].tailBytes,
                                            (char *) B[a].tailSend + (size_t) B[a].inBeg[b] * B[a].tailBytes, n, cudaMemcpyDeviceToDevice),
                                 "tail records");
            } else {      // feeder a -> owner b
                const size_t n = (size_t) (B[a].outBeg[b + 1] - B[a].outBeg[b]) * B[a].moverBytes;
                if (n) loopCheck(cudaMemcpy((char *) B[b].moverRecv + (size_t) B[b].inBeg[a] * B[b].moverBytes,
                                            (char *) B[a].moverSend + (size_t) B[a].outBeg[b] * B[a].moverBytes, n, cudaMemcpyDeviceToDevice),
                                 "mover records");
            }
        }
    loopCheck(cudaDeviceSynchronize(), "device synchronize");   // D2D cudaMemcpy may return early; the ranks' streams are non-blocking
}
void loopAllGatherBlk(std::vector<cfb::ShardBuffers> &B) {
    const int W = (int) B.size();
    for (int a = 0; a < W; ++a) loopCheck(cudaStreamSynchronize((cudaStream_t) B[a].stream), "stream synchronize");
    for (int a = 0; a < W; ++a)
        for (int b = 0; b < W; ++b)
            loopCheck(cudaMemcpy((char *) B[b].blkAll + (size_t) a * B[a].blkBytesPerRank, B[a].blkSend, B[a].blkBytesPerRank,
                                 cudaMemcpyDeviceToDevice), "blocker records");
    loopCheck(cudaDeviceSynchronize(), "device synchronize");
}
}  // namespace

extern "C" {

// inter_owner: rank of every intersection (virtual ones included), or null for column strips
static cfb_shard_group *shardGroupCreate(const char *config_file, int world, int device, const int32_t *inter_owner) {
    std::unique_ptr<cfb_shard_group> g(new cfb_shard_group());
    auto fail = [&](const std::string &err) {
        if (!err.empty()) g_createError = "sharded engine: " + err;
        for (auto *x : g->ranks) cfb_engine_destroy(x);
        return (cfb_shard_group *) nullptr;
    };
    for (int r = 0; r < world; ++r) {
        cfb_engine *e = cfb_engine_create(config_file, 1, device);
        if (!e) return fail("");
        g->ranks.push_back(e);
        if (r == 0) {
            const cfb::RoadNet &net = e->h.net;
            if (inter_owner) {
                std::vector<int> owner(inter_owner, inter_owner + net.nInter());
                for (int i = 0; i < net.nInter(); ++i)
                    if (owner[i] < 0 || owner[i] >= world)
                        return fail("intersection " + std::to_string(i) + " is given rank " + std::to_string(owner[i]) +
                                    ", outside [0, " + std::to_string(world) + ")");
                g->part = cfb::Partition::fromOwners(net, owner, world);
            } else {
                g->part = cfb::Partition::columnStrips(net, world);
            }
        }
        std::string err = e->h.configureShard(r, g->part);
        if (!err.empty()) return fail(err);
    }
    {   // same process: the "peer mappings" are the arenas themselves
        const char *tr = getenv("CITYFLOW_B200_SHARD_TRANSPORT");
        g->p2p = !(tr && !strcmp(tr, "nccl"));
        if (g->p2p) {
            std::vector<void *> bases;
            for (auto *e : g->ranks) bases.push_back(e->h.dev->shardArena().base);
            for (auto *e : g->ranks) e->h.dev->shardConnect(bases);
        }
    }
    // finished vehicles: union over the ranks (the hook sees each rank's local list in turn)
    cfb_shard_group *gp = g.get();
    for (int r = 0; r < world; ++r) {
        gp->ranks[r]->h.finishedHook = [gp, r](std::vector<cfb::FinRec> &fin) {
            // every rank drains at the same step; collect all local lists once, hand the union to each
            static thread_local std::vector<cfb::FinRec> all;
            if (r == 0) {
                all = fin;
                for (size_t q = 1; q < gp->ranks.size(); ++q) {
                    std::vector<cfb::FinRec> f;
                    gp->ranks[q]->h.dev->drainFinished(f);
                    all.insert(all.end(), f.begin(), f.end());
                }
            }
            fin = all;
        };
    }
    return g.release();
}

cfb_shard_group *cfb_shard_group_create(const char *config_file, int world, int device) {
    return shardGroupCreate(config_file, world, device, nullptr);
}

cfb_shard_group *cfb_debug_shard_group_create_cut(const char *config_file, int world, int device, const int32_t *inter_owner) {
    if (!inter_owner) { g_createError = "sharded engine: no intersection owners given"; return nullptr; }
    return shardGroupCreate(config_file, world, device, inter_owner);
}

void cfb_shard_group_destroy(cfb_shard_group *g) {
    if (!g) return;
    for (auto *e : g->ranks) cfb_engine_destroy(e);
    delete g;
}

int cfb_shard_group_step(cfb_shard_group *g, int n) {
    try {
        const int W = (int) g->ranks.size();
        for (int it = 0; it < n; ++it) {
            std::vector<cfb::ShardBuffers> B;
            for (auto *e : g->ranks) {
                e->h.prepareStep();
                e->h.dev->stageStep(e->h.batch.data(), (int) e->h.batch.size());
                B.push_back(e->h.dev->shardBuffers());
            }
            // Between the segments the ranks' streams are drained.  Over peer memory a receive kernel then never has to
            // spin: what this checks is the protocol (indices, parities, epochs), not the waiting.
            for (int k = 0; k < 3; ++k) {
                if (k > 0) {
                    if (g->p2p) {
                        for (auto *e : g->ranks) e->h.dev->synchronize();
                    } else {
                        loopExchange(B, k == 2);
                        if (k == 2) loopAllGatherBlk(B);
                    }
                }
                for (auto *e : g->ranks) e->h.dev->shardSegment(k);
            }
            for (int r = 0; r < W; ++r) g->ranks[r]->h.finishStep();   // rank 0 first: its drain collects all lists
        }
        for (auto *e : g->ranks) e->h.checkDevice();
        return CFB_OK;
    } catch (const std::exception &ex) {
        g->lastError = ex.what();
        return CFB_ERR_DEVICE;
    }
}

const char *cfb_shard_group_last_error(const cfb_shard_group *g) { return g ? g->lastError.c_str() : g_createError.c_str(); }

int64_t cfb_shard_group_vehicle_count(cfb_shard_group *g) {
    int64_t s = 0;
    for (auto *e : g->ranks) s += e->h.dev->vehicleCount();
    return s;
}

// sums over the ranks: out = {vehicle steps (cfb_vehicle_steps), same-step entrant ties (cfb_tie_count)}
int cfb_shard_group_counters(cfb_shard_group *g, int64_t out[2]) {
    try {
        out[0] = out[1] = 0;
        for (auto *e : g->ranks) { out[0] += (int64_t) e->h.dev->vehicleSteps(); out[1] += e->h.dev->tieCount(); }
        return CFB_OK;
    } catch (const std::exception &ex) {
        g->lastError = ex.what();
        return CFB_ERR_DEVICE;
    }
}

// lane counts assembled from the owning ranks; `waiting` selects speed < 0.1 counts
int cfb_shard_group_lane_counts(cfb_shard_group *g, int32_t *out, int n, int waiting) {
    const int nL = g->ranks[0]->h.net.nLanes();
    if (n < nL) return CFB_ERR_ARGUMENT;
    const cfb::Partition &part = g->part;
    std::vector<int32_t> tmp(nL);
    for (size_t r = 0; r < g->ranks.size(); ++r) {
        if (waiting) g->ranks[r]->h.dev->laneWaitingVehicleCount(tmp.data()); else g->ranks[r]->h.dev->laneVehicleCount(tmp.data());
        for (int l = 0; l < nL; ++l) if (part.drvOwner[l] == (int) r) out[l] = tmp[l];
    }
    return CFB_OK;
}

// every running vehicle of the owning ranks (same record as cfb_debug_vehicles)
int64_t cfb_shard_group_debug_vehicles(cfb_shard_group *g, void *out, int64_t cap) {
    const cfb::Partition &part = g->part;
    struct Rec { int32_t w[8]; double d[3]; int64_t e; };
    int64_t total = 0;
    std::vector<Rec> tmp;
    for (size_t r = 0; r < g->ranks.size(); ++r) {
        int64_t n = cfb_debug_vehicles(g->ranks[r], nullptr, 0);
        tmp.resize(n);
        cfb_debug_vehicles(g->ranks[r], tmp.data(), n);
        for (auto &x : tmp) {
            if (part.drvOwner[x.w[3]] != (int) r) continue;  // ghost copies
            if (total < cap && out) ((Rec *) out)[total] = x;
            ++total;
        }
    }
    return total;
}

}  // extern "C"
