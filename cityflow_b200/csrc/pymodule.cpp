// pybind11 module: the `cityflow.Engine` Python surface of the reference (src/cityflow.cpp:10-48),
// same method names, keyword names and defaults, implemented as a thin wrapper over the C-ABI in
// include/cityflow_b200.h.  Dict results are built in std::map key order (sorted by id), as
// pybind11's stl caster does for the reference's std::map return values.
#include <pybind11/pybind11.h>
#include <pybind11/stl.h>

#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <limits>
#include <map>
#include <memory>
#include <numeric>
#include <string>
#include <vector>

#include "../../include/cityflow_b200.h"

namespace py = pybind11;
using namespace py::literals;

namespace {

std::string vehicleName(const cfb_vehicle_ref &r) {
    if (r.flow == -2) return "manually_pushed_" + std::to_string(r.index);
    return "flow_" + std::to_string(r.flow) + "_" + std::to_string(r.index);
}

bool parseVehicleName(const std::string &id, cfb_vehicle_ref &out) {
    try {
        if (id.compare(0, 16, "manually_pushed_") == 0) {
            out.flow = -2;
            out.index = std::stoi(id.substr(16));
            return true;
        }
        if (id.compare(0, 5, "flow_") == 0) {
            size_t us = id.find('_', 5);
            if (us == std::string::npos) return false;
            out.flow = std::stoi(id.substr(5, us - 5));
            out.index = std::stoi(id.substr(us + 1));
            return vehicleName(out) == id;
        }
    } catch (...) {
    }
    return false;
}

class Engine;

class Archive {
public:
    explicit Archive(Engine &e);
    explicit Archive(cfb_archive *a) : a_(a) {}
    ~Archive() { if (a_) cfb_archive_destroy(a_); }
    Archive(const Archive &) = delete;
    void dump(const std::string &path) {
        if (cfb_archive_dump(a_, path.c_str()) < 0) throw std::runtime_error("cannot write archive to " + path);
    }
    cfb_archive *a_ = nullptr;
};

class Engine {
public:
    Engine(const std::string &configFile, int threadNum, int device, int shardRank, int shardWorld, const py::bytes &ncclId) {
        if (device < 0) {
            const char *env = std::getenv("CITYFLOW_B200_DEVICE");
            device = env ? std::atoi(env) : 0;
        }
        const std::string id = ncclId;
        sharded_ = shardWorld > 1;
        if (sharded_ && id.size() != 128) throw std::runtime_error("nccl_id must be the 128 bytes of cityflow_b200.nccl_unique_id()");
        {
            py::gil_scoped_release rel;
            e_ = sharded_ ? cfb_engine_create_sharded(configFile.c_str(), threadNum, device, shardRank, shardWorld,
                                                      (const unsigned char *) id.data())
                          : cfb_engine_create(configFile.c_str(), threadNum, device);
        }
        if (!e_) throw std::runtime_error(std::string("load config failed! ") + cfb_last_error(nullptr));
        const int n = cfb_num_lanes(e_);
        std::vector<std::string> ids(n);
        for (int i = 0; i < n; ++i) ids[i] = cfb_lane_id(e_, i);
        laneOrder_.resize(n);
        std::iota(laneOrder_.begin(), laneOrder_.end(), 0);
        std::sort(laneOrder_.begin(), laneOrder_.end(), [&](int a, int b) { return ids[a] < ids[b]; });
        laneKeys_.reserve(n);
        for (int i = 0; i < n; ++i) laneKeys_.push_back(py::str(ids[laneOrder_[i]]));
        laneBuf_.resize(n);
    }
    ~Engine() {
        if (e_) cfb_engine_destroy(e_);
    }
    Engine(const Engine &) = delete;

    void check(int rc) const {
        if (rc < 0) throw std::runtime_error(cfb_last_error(e_));
    }
    void nextStep() {
        py::gil_scoped_release rel;
        int rc = cfb_next_step(e_);
        if (rc < 0) {
            py::gil_scoped_acquire acq;
            check(rc);
        }
    }
    void nextSteps(int n) {
        int rc;
        {
            py::gil_scoped_release rel;
            rc = cfb_next_steps(e_, n);
        }
        check(rc);
    }
    size_t getVehicleCount() {
        int64_t c = sharded_ ? cfb_shard_vehicle_count(e_) : cfb_get_vehicle_count(e_);
        if (c < 0) check((int) c);
        return (size_t) c;
    }
    py::dict laneDict(bool waiting) {
        int rc = sharded_ ? cfb_shard_lane_vehicle_count(e_, laneBuf_.data(), (int) laneBuf_.size(), waiting)
                 : waiting ? cfb_get_lane_waiting_vehicle_count(e_, laneBuf_.data(), (int) laneBuf_.size())
                           : cfb_get_lane_vehicle_count(e_, laneBuf_.data(), (int) laneBuf_.size());
        check(rc);
        py::dict d;
        for (size_t i = 0; i < laneOrder_.size(); ++i) d[laneKeys_[i]] = py::int_(laneBuf_[laneOrder_[i]]);
        return d;
    }
    std::vector<std::string> laneIds() {
        std::vector<std::string> ids(cfb_num_lanes(e_));
        for (size_t i = 0; i < ids.size(); ++i) ids[i] = cfb_lane_id(e_, (int) i);
        return ids;
    }
    // device pointers of the per-lane observation arrays, ordered against CUDA stream `stream`
    py::dict observeDevice(uintptr_t stream) {
        cfb_device_obs o{};
        check(cfb_observe_device(e_, (void *) stream, &o));
        py::dict d;
        d["lane_vehicle_count"] = py::int_((uintptr_t) o.lane_vehicle_count);
        d["lane_waiting_count"] = py::int_((uintptr_t) o.lane_waiting_count);
        d["lane_speed_sum"] = py::int_((uintptr_t) o.lane_speed_sum);
        d["n_lanes"] = py::int_(o.n_lanes);
        d["device"] = py::int_(o.device);
        return d;
    }
    py::dict getLaneVehicleCount() { return laneDict(false); }
    py::dict getLaneWaitingVehicleCount() { return laneDict(true); }

    py::dict vehicleDict(bool distance) {
        int64_t n = cfb_get_vehicle_speed(e_, nullptr, nullptr, nullptr, 0);
        if (n < 0) check((int) n);
        std::vector<cfb_vehicle_ref> ids(n);
        std::vector<double> val(n);
        n = cfb_get_vehicle_speed(e_, ids.data(), distance ? nullptr : val.data(), distance ? val.data() : nullptr, n);
        if (n < 0) check((int) n);
        std::vector<std::pair<std::string, double>> items(n);
        for (int64_t i = 0; i < n; ++i) items[i] = {vehicleName(ids[i]), val[i]};
        std::sort(items.begin(), items.end(), [](const auto &a, const auto &b) { return a.first < b.first; });
        py::dict d;
        for (auto &kv : items) d[py::str(kv.first)] = py::float_(kv.second);
        return d;
    }
    py::dict getVehicleSpeed() { return vehicleDict(false); }
    py::dict getVehicleDistance() { return vehicleDict(true); }

    std::vector<std::string> getVehicles(bool includeWaiting) {
        int64_t n = cfb_get_vehicles(e_, includeWaiting, nullptr, 0);
        if (n < 0) check((int) n);
        std::vector<cfb_vehicle_ref> ids(n);
        n = cfb_get_vehicles(e_, includeWaiting, ids.data(), n);
        if (n < 0) check((int) n);
        std::vector<std::string> out(n);
        for (int64_t i = 0; i < n; ++i) out[i] = vehicleName(ids[i]);
        return out;
    }
    py::dict getLaneVehicles() {
        const int nl = (int) laneOrder_.size();
        std::vector<int64_t> beg(nl + 1);
        int64_t n = cfb_get_lane_vehicles(e_, beg.data(), nl + 1, nullptr, 0);
        if (n < 0) check((int) n);
        std::vector<cfb_vehicle_ref> ids(n);
        n = cfb_get_lane_vehicles(e_, beg.data(), nl + 1, ids.data(), n);
        if (n < 0) check((int) n);
        py::dict d;
        for (int i = 0; i < nl; ++i) {
            const int l = laneOrder_[i];
            py::list lst;
            for (int64_t k = beg[l]; k < beg[l + 1] && k < n; ++k) lst.append(py::str(vehicleName(ids[k])));
            d[laneKeys_[i]] = lst;
        }
        return d;
    }
    std::string getLeader(const std::string &id) {
        cfb_vehicle_ref v, l{};
        int found = 0;
        if (!parseVehicleName(id, v) || cfb_get_leader(e_, v, &l, &found) < 0)
            throw std::runtime_error("Vehicle '" + id + "' not found");  // engine.cpp:839
        return found ? vehicleName(l) : "";
    }
    double getCurrentTime() const { return cfb_get_current_time(e_); }
    double getAverageTravelTime() { return cfb_get_average_travel_time(e_); }
    void setTrafficLightPhase(const std::string &id, int phase) { check(cfb_set_tl_phase(e_, id.c_str(), phase)); }
    void setRandomSeed(int seed) { check(cfb_set_random_seed(e_, seed)); }
    void reset(bool seed) { check(cfb_reset(e_, seed)); }
    void pushVehicle(const std::map<std::string, double> &info, const std::vector<std::string> &roads) {
        static const char *names[10] = {"speed", "length", "width", "maxPosAcc", "maxNegAcc", "usualPosAcc",
                                        "usualNegAcc", "minGap", "maxSpeed", "headwayTime"};
        double v[10];
        for (int k = 0; k < 10; ++k) {
            auto it = info.find(names[k]);
            v[k] = it == info.end() ? std::numeric_limits<double>::quiet_NaN() : it->second;
        }
        std::vector<const char *> r;
        for (auto &s : roads) r.push_back(s.c_str());
        check(cfb_push_vehicle(e_, v, r.data(), (int) r.size()));
    }
    void setReplayLogFile(const std::string &f) { check(cfb_set_replay_file(e_, f.c_str())); }  // engine.cpp:727-734
    void setSaveReplay(bool open) { check(cfb_set_save_replay(e_, open)); }                    // engine.cpp:736-742
    void setVehicleSpeed(const std::string &id, double speed) {
        cfb_vehicle_ref v;
        if (!parseVehicleName(id, v) || cfb_set_vehicle_speed(e_, v, speed) < 0)
            throw std::runtime_error("Vehicle '" + id + "' not found");  // engine.cpp:830
    }
    bool setVehicleRoute(const std::string &id, const std::vector<std::string> &route) {
        cfb_vehicle_ref v;
        if (!parseVehicleName(id, v)) return false;
        std::vector<const char *> r;
        for (auto &s : route) r.push_back(s.c_str());
        int ok = 0;
        check(cfb_set_vehicle_route(e_, v, r.data(), (int) r.size(), &ok));
        return ok != 0;
    }
    std::map<std::string, std::string> getVehicleInfo(const std::string &id) {
        cfb_vehicle_ref v;
        int64_t n = -1;
        if (parseVehicleName(id, v)) n = cfb_get_vehicle_info(e_, v, nullptr, 0);
        if (n < 0) throw std::runtime_error("Vehicle '" + id + "' not found");  // engine.cpp:871
        std::string buf((size_t) n, '\0');
        cfb_get_vehicle_info(e_, v, &buf[0], n);
        std::map<std::string, std::string> out;
        size_t i = 0;
        while (i < buf.size()) {
            std::string k(buf.c_str() + i);
            i += k.size() + 1;
            std::string val(buf.c_str() + i);
            i += val.size() + 1;
            out[k] = val;
        }
        return out;
    }
    std::unique_ptr<Archive> snapshot() {
        cfb_archive *a = cfb_snapshot(e_);
        if (!a) throw std::runtime_error(cfb_last_error(e_));
        return std::unique_ptr<Archive>(new Archive(a));
    }
    void load(const Archive &a) { check(cfb_load(e_, a.a_)); }
    void loadFromFile(const std::string &path) { check(cfb_load_from_file(e_, path.c_str())); }
    cfb_engine *raw() { return e_; }
    [[noreturn]] void unsupported(const char *what) const {
        throw std::runtime_error(std::string(what) + " is not implemented by the GPU engine yet");
    }
    // measurement helpers (not part of the reference surface)
    int64_t gpuLaunches() const { return cfb_gpu_launches(e_); }
    int64_t tieCount() { return cfb_tie_count(e_); }
    void enableKernelTiming(bool on) { cfb_enable_kernel_timing(e_, on); }
    py::tuple kernelTimes() {
        double ms[5];
        int64_t n = 0;
        cfb_kernel_times(e_, ms, &n);
        return py::make_tuple(py::make_tuple(ms[0], ms[1], ms[2], ms[3], ms[4]), n);
    }
    py::tuple timedSteps(int n, bool flushL2) {
        double ms = 0;
        int64_t vs = 0;
        int rc;
        {
            py::gil_scoped_release rel;
            rc = cfb_timed_steps(e_, n, flushL2, &ms, &vs);
        }
        check(rc);
        return py::make_tuple(ms, vs);
    }
    int64_t vehicleSteps() { return cfb_vehicle_steps(e_); }
    int64_t numDrivables() const { return cfb_num_drivables(e_); }
    py::tuple hostTimes() { double a = 0, b = 0; cfb_host_times(e_, &a, &b); return py::make_tuple(a, b); }
    py::tuple transferBytes() { int64_t a = 0, b = 0; cfb_transfer_bytes(e_, &a, &b); return py::make_tuple(a, b); }
    void synchronize() {
        py::gil_scoped_release rel;
        cfb_synchronize(e_);
    }

private:
    cfb_engine *e_ = nullptr;
    bool sharded_ = false;
    std::vector<int> laneOrder_;
    std::vector<py::str> laneKeys_;
    std::vector<int32_t> laneBuf_;
};

Archive::Archive(Engine &e) : a_(cfb_snapshot(e.raw())) {
    if (!a_) throw std::runtime_error(cfb_last_error(e.raw()));
}

}  // namespace

PYBIND11_MODULE(_cityflow_b200, m) {
    m.doc() = "H100-native CityFlow step engine (drop-in for cityflow.Engine)";
    py::class_<Engine>(m, "Engine")
        .def(py::init<const std::string &, int, int, int, int, const py::bytes &>(), "config_file"_a, "thread_num"_a = 1,
             "device"_a = -1, "shard_rank"_a = 0, "shard_world"_a = 1, "nccl_id"_a = py::bytes())
        .def("next_step", &Engine::nextStep)
        .def("get_vehicle_count", &Engine::getVehicleCount)
        .def("get_vehicles", &Engine::getVehicles, "include_waiting"_a = false)
        .def("get_lane_vehicle_count", &Engine::getLaneVehicleCount)
        .def("get_lane_waiting_vehicle_count", &Engine::getLaneWaitingVehicleCount)
        .def("get_lane_vehicles", &Engine::getLaneVehicles)
        .def("get_vehicle_speed", &Engine::getVehicleSpeed)
        .def("get_vehicle_info", &Engine::getVehicleInfo, "vehicle_id"_a)
        .def("get_vehicle_distance", &Engine::getVehicleDistance)
        .def("get_leader", &Engine::getLeader, "vehicle_id"_a)
        .def("get_current_time", &Engine::getCurrentTime)
        .def("get_average_travel_time", &Engine::getAverageTravelTime)
        .def("set_tl_phase", &Engine::setTrafficLightPhase, "intersection_id"_a, "phase_id"_a)
        .def("set_vehicle_speed", &Engine::setVehicleSpeed, "vehicle_id"_a, "speed"_a)
        .def("set_replay_file", &Engine::setReplayLogFile, "replay_file"_a)
        .def("set_random_seed", &Engine::setRandomSeed, "seed"_a)
        .def("set_save_replay", &Engine::setSaveReplay, "open"_a)
        .def("push_vehicle", &Engine::pushVehicle)
        .def("reset", &Engine::reset, "seed"_a = false)
        .def("load", &Engine::load, "archive"_a)
        .def("snapshot", &Engine::snapshot)
        .def("load_from_file", &Engine::loadFromFile, "path"_a)
        .def("set_vehicle_route", &Engine::setVehicleRoute, "vehicle_id"_a, "route"_a)
        // extras
        .def("next_steps", &Engine::nextSteps, "n"_a)
        .def("gpu_launches", &Engine::gpuLaunches)
        .def("tie_count", &Engine::tieCount)
        .def("shard_phase_times", [](Engine &e) {
            double ms[8] = {0}; int64_t n = 0;
            cfb_shard_phase_times(e.raw(), ms, &n);
            return py::make_tuple(std::vector<double>(ms, ms + 8), n);
        })
        .def("enable_kernel_timing", &Engine::enableKernelTiming, "on"_a = true)
        .def("kernel_times", &Engine::kernelTimes)
        .def("timed_steps", &Engine::timedSteps, "n"_a, "flush_l2"_a = false)
        .def("vehicle_steps", &Engine::vehicleSteps)
        .def("transfer_bytes", &Engine::transferBytes)
        .def("num_drivables", [](Engine &e) { return e.numDrivables(); })
        .def("host_times", &Engine::hostTimes)
        .def("lane_ids", &Engine::laneIds)
        .def("intersection_ids", [](Engine &e) {
            std::vector<std::string> ids(cfb_num_intersections(e.raw()));
            for (size_t i = 0; i < ids.size(); ++i) ids[i] = cfb_intersection_id(e.raw(), (int) i);
            return ids;
        })
        .def("num_intersections", [](Engine &e) { return cfb_num_intersections(e.raw()); })
        .def("set_tl_phases_device", [](Engine &e, uintptr_t phases, uintptr_t stream) {
            if (cfb_set_tl_phases_device(e.raw(), (const int32_t *) phases, (void *) stream) < 0)
                throw std::runtime_error(cfb_last_error(e.raw()));
        }, "phases_ptr"_a, "stream"_a = 0)
        .def("device", [](Engine &e) { return cfb_device(e.raw()); })
        .def("observe_device", &Engine::observeDevice, "stream"_a = 0)
        .def("synchronize", &Engine::synchronize);
    py::class_<Archive>(m, "Archive")
        .def(py::init<Engine &>())
        .def("dump", &Archive::dump, "path"_a);
    m.def("nccl_unique_id", []() {
        unsigned char id[128];
        if (cfb_nccl_unique_id(id) < 0) throw std::runtime_error(cfb_last_error(nullptr));
        return py::bytes((const char *) id, 128);
    }, "128-byte id for Engine(..., shard_world=N, nccl_id=...): create on one rank, broadcast to all");
    m.attr("__version__") = "b200-dev";
}
