"""The intersection observations (cfb_observe_intersections_device, cfb_road_link_info) through the C-ABI over the
emulated device: the kernel body of csrc/device_tlobs.cuh on the emulated warp (tests/device_sim_emu_intobs.cpp), under
the real host engine.  Every column is compared with a restatement of its definition built from the roadnet JSON itself
and the engine's dict getters; the emulated device's "device memory" is host memory, so the pointers are read with numpy."""
import ctypes
import json
import os
import subprocess

import numpy as np
import pytest

from test_cpu import _HAVE_CUDA_SDK

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INT32_MIN = -2 ** 31
TYPES = {"turn_right": 1, "turn_left": 2, "go_straight": 3}

pytestmark = pytest.mark.skipif(not _HAVE_CUDA_SDK, reason="needs the CUDA headers and libcudart to build the host-check library")


@pytest.fixture(autouse=True)
def _emulated(monkeypatch):
    monkeypatch.setenv("CFB_EMULATED_DEVICE_FOR_TESTS", "1")


def _intobs_lib():
    """oracle/_build/libcfb_hostcheck_intobs.so: the host engine and C-ABI (csrc/host_engine.cpp) over the emulated
    device with the intersection observations (tests/device_sim_emu_intobs.cpp).  Test infrastructure, built like
    test_cpu.py's host-check library."""
    os.makedirs(os.path.join(ROOT, "oracle", "_build"), exist_ok=True)
    lib = os.path.join(ROOT, "oracle", "_build", "libcfb_hostcheck_intobs.so")
    csrc = os.path.join(ROOT, "cityflow_b200", "csrc")
    tests = os.path.join(ROOT, "tests")
    srcs = [os.path.join(tests, "device_sim_emu_intobs.cpp")] + [os.path.join(csrc, f) for f in
            ("host_engine.cpp", "roadnet.cpp", "flows.cpp", "partition.cpp", "shard.cpp", "replay.cpp", "json_write.cpp")]
    deps = srcs + [os.path.join(csrc, f) for f in os.listdir(csrc) if f.endswith((".cuh", ".h"))] + \
        [os.path.join(tests, f) for f in ("device_emu.h", "device_hostsim.h", "device_sim_emu.cpp")] + \
        [os.path.join(ROOT, "include", "cityflow_b200.h")]
    if not os.path.exists(lib) or os.path.getmtime(lib) < max(os.path.getmtime(f) for f in deps):
        tmp = lib + ".%d.tmp" % os.getpid()
        subprocess.check_call(["g++", "-std=c++17", "-O1", "-fPIC", "-shared", "-ffp-contract=off", "-I/usr/local/cuda/include",
                               "-I" + csrc, "-I" + tests, "-I" + os.path.join(ROOT, "include")] + srcs +
                              ["-L/usr/local/cuda/lib64", "-lcudart", "-ldl", "-o", tmp])
        os.replace(tmp, lib)
    return lib


def _emulated_engine(cfg):
    from cityflow_b200 import capi
    path = _intobs_lib()

    class EmulatedEngine(capi.CEngine):
        def _library(self):
            return capi.bind(ctypes.CDLL(path))

    return EmulatedEngine(cfg, 0)


def _host(ptr, n, ctype):
    return np.ctypeslib.as_array((ctype * max(n, 1)).from_address(ptr))[:n].copy()


def table(eng):
    """The refreshed observations as numpy arrays."""
    o = eng.observe_intersections_device()
    nI, nR, mP, mM = o.n_intersections, o.n_road_links, o.max_phases, o.max_movements
    i32, f64 = ctypes.c_int32, ctypes.c_double
    t = {k: _host(getattr(o, k), nI, i32) for k in ("phase", "pressure", "queue", "phase_count")}
    t["phase_remaining"] = _host(o.phase_remaining, nI, f64)
    for k in ("movement_in", "movement_in_waiting", "movement_out", "movement_inside", "movement_pressure",
              "movement_intersection"):
        t[k] = _host(getattr(o, k), nR, i32)
    t["movement_begin"] = _host(o.movement_begin, nI + 1, i32)
    t["phase_pressure"] = _host(o.phase_pressure, nI * mP, i32).reshape(nI, mP)
    t["phase_movements"] = _host(o.phase_movements, nI * mP * mM, ctypes.c_uint8).reshape(nI, mP, mM)
    t["ptrs"] = tuple(getattr(o, k) for k, _ in o._fields_ if k not in ("device",))
    return t


class Restatement:
    """The definitions, from the roadnet JSON alone: movements, their distinct in / out lanes, laneLinks and phases."""

    def __init__(self, cfg):
        c = json.load(open(cfg))
        net = json.load(open(c["dir"] + c["roadnetFile"]))
        self.interval = c["interval"]
        self.rl = c.get("rlTrafficLight", False)
        lane0, n = {}, 0
        for r in net["roads"]:
            lane0[r["id"]] = n
            n += len(r["lanes"])
        self.n_lanes = n
        self.inters = net["intersections"]
        self.ids = [i["id"] for i in self.inters]
        self.virtual = [bool(i["virtual"]) for i in self.inters]
        self.mv = []            # per movement: (intersection, index, type, start road, end road, in, out, laneLinks)
        self.begin = [0]
        self.phases = []        # per intersection: [(time, set of local movement indices)]
        ll = 0
        for k, inter in enumerate(self.inters):
            if not inter["virtual"]:
                for j, rl in enumerate(inter["roadLinks"]):
                    ins, outs, links = [], [], []
                    for x in rl["laneLinks"]:
                        a = lane0[rl["startRoad"]] + x["startLaneIndex"]
                        b = lane0[rl["endRoad"]] + x["endLaneIndex"]
                        ins += [a] if a not in ins else []
                        outs += [b] if b not in outs else []
                        links.append(ll)
                        ll += 1
                    self.mv.append((k, j, TYPES[rl["type"]], rl["startRoad"], rl["endRoad"], ins, outs, links))
                self.phases.append([(ph["time"], set(ph["availableRoadLinks"])) for ph in inter["trafficLight"]["lightphases"]])
            else:
                self.phases.append([])
            self.begin.append(len(self.mv))
        self.n_links = ll
        self.max_phases = max([1] + [len(p) for p in self.phases])
        self.max_movements = max([1] + [self.begin[k + 1] - self.begin[k] for k in range(len(self.inters))])
        # fixed-time plan (TrafficLight::init / passTime): phase 0 with its full time, then remain -= dt
        self.cur = [0] * len(self.inters)
        self.remain = [0.0 if v else p[0][0] for v, p in zip(self.virtual, self.phases)]

    def pass_time(self):
        if self.rl:
            return
        for k, ph in enumerate(self.phases):
            if self.virtual[k]:
                continue
            rem, cur = self.remain[k] - self.interval, self.cur[k]
            while rem <= 0.0:
                cur = (cur + 1) % len(ph)
                rem += ph[cur][0]
            self.remain[k], self.cur[k] = rem, cur

    def movement_columns(self, count, waiting, drv_count):
        cols = {k: [] for k in ("movement_in", "movement_in_waiting", "movement_out", "movement_inside")}
        for (_, _, _, _, _, ins, outs, links) in self.mv:
            cols["movement_in"].append(sum(count[l] for l in ins))
            cols["movement_in_waiting"].append(sum(waiting[l] for l in ins))
            cols["movement_out"].append(sum(count[l] for l in outs))
            cols["movement_inside"].append(sum(drv_count[self.n_lanes + x] for x in links))
        cols = {k: np.array(v, np.int32) for k, v in cols.items()}
        cols["movement_pressure"] = cols["movement_in"] - cols["movement_out"]
        return cols

    def phase_pressure(self, count):
        mp = [sum(count[l] for l in ins) - sum(count[l] for l in outs) for (_, _, _, _, _, ins, outs, _) in self.mv]
        out = np.full((len(self.inters), self.max_phases), INT32_MIN, np.int64)
        for k, ph in enumerate(self.phases):
            for p, (_, avail) in enumerate(ph):
                out[k, p] = sum(mp[self.begin[k] + m] for m in avail)
        return out

    def intersection_columns(self, count, waiting):
        pressure, queue = [], []
        for k in range(len(self.inters)):
            ins, outs = [], []
            for (_, _, _, _, _, a, b, _) in self.mv[self.begin[k]:self.begin[k + 1]]:
                ins += [l for l in a if l not in ins]
                outs += [l for l in b if l not in outs]
            pressure.append(sum(count[l] for l in ins) - sum(count[l] for l in outs))
            queue.append(sum(waiting[l] for l in ins))
        return np.array(pressure, np.int32), np.array(queue, np.int32)

    def max_pressure(self, count):
        """The MaxPressure action of every light: the first phase of largest pressure (virtual: -1)."""
        pp = self.phase_pressure(count)
        return [-1 if v else int(np.argmax(pp[k])) for k, v in enumerate(self.virtual)]


def drivable_counts(eng, lane_change):
    """Vehicles per drivable (lanes, then laneLinks) from the full per-vehicle records, shadows included."""
    if lane_change:
        from oracle.harness import LC_DTYPE
        n = eng._check(eng.lib.cfb_debug_lc_vehicles(eng.h, None, 0))
        recs = np.zeros(n, LC_DTYPE)
        if n:
            eng._check(eng.lib.cfb_debug_lc_vehicles(eng.h, recs.ctypes.data, n))
    else:
        recs = eng.debug_vehicles()
    return np.bincount(recs["drivable"], minlength=eng.n_drivables)


def check_static(eng, R, t):
    assert len(t["phase"]) == len(R.inters) and len(t["movement_in"]) == len(R.mv)
    assert (t["movement_begin"] == R.begin).all()
    assert (t["movement_intersection"] == [m[0] for m in R.mv]).all()
    assert (t["phase_count"] == [len(p) for p in R.phases]).all()
    assert t["phase_pressure"].shape[1] == R.max_phases and t["phase_movements"].shape[2] == R.max_movements
    want = np.zeros((len(R.inters), R.max_phases, R.max_movements), np.uint8)
    for k, ph in enumerate(R.phases):
        for p, (_, avail) in enumerate(ph):
            want[k, p, list(avail)] = 1
    assert (t["phase_movements"] == want).all()
    assert eng.road_links() == [(m[0], m[1], m[2], m[3], m[4]) for m in R.mv]
    assert eng.lib.cfb_num_road_links(eng.h) == len(R.mv)
    assert eng.lib.cfb_road_link_info(eng.h, len(R.mv), None) < 0


def check_table(eng, R, t, lane_change, phases=True):
    """Every dynamic column against the restatement, from the dict getters of the same engine."""
    count, waiting = eng.lane_vehicle_count(), eng.lane_waiting_count()
    drv = drivable_counts(eng, lane_change)
    assert (drv[:eng.n_lanes] == count).all()
    for k, v in R.movement_columns(count, waiting, drv).items():
        assert (t[k] == v).all(), k
    pressure, queue = R.intersection_columns(count, waiting)
    assert (t["pressure"] == pressure).all() and (t["queue"] == queue).all()
    assert (t["phase_pressure"] == R.phase_pressure(count)).all()
    if phases:
        assert (t["phase"] == [-1 if v else c for v, c in zip(R.virtual, R.cur)]).all()
        assert (t["phase_remaining"].view(np.int64) == np.array(R.remain, np.float64).view(np.int64)).all()


def check_dump(eng, R, t, path):
    """phase / phase_remaining against the trafficLights of the engine's own JSON archive, bit for bit."""
    eng.dump(path)
    tl = json.load(open(path))["trafficLights"]
    for k, i in enumerate(R.ids):
        if R.virtual[k]:
            assert t["phase"][k] == -1 and t["phase_remaining"][k] == 0.0
        else:
            assert t["phase"][k] == tl[i]["curPhaseIndex"]
            assert t["phase_remaining"][k].tobytes() == np.float64(tl[i]["remainDuration"]).tobytes()


def _dense_3x3(directory, lane_change=False, rl=False):
    from cityflow_b200 import scenario
    return scenario.make_grid_scenario(directory, 3, 3, dense=dict(frac=1.0, interval=3.0, seed=3), name="io33%d%d" % (lane_change, rl),
                                       lane_change=lane_change, rl_traffic_light=rl)


def _irregular(directory):
    import conftest
    from cityflow_b200 import scenario
    net = conftest._irregular_net()
    flows = scenario.random_walk_flows(net, frac=1.0, interval=4.0, seed=9)
    return scenario.write_scenario(directory, net, flows, seed=7, name="ioirr")


def _fuzzed(directory, seed=7):
    import randnet
    from cityflow_b200 import scenario
    net = randnet.random_roadnet(seed, rows=2 + seed % 3, cols=3 + seed % 2)
    flows = randnet.random_flows(net, seed + 100, n_flows=40 + seed % 50)
    return scenario.write_scenario(directory, net, flows, seed=seed, interval=1.0, name="iof%d" % seed)


def _star(directory):
    import edgenet
    return edgenet.write("star", directory)


NETS = {"dense_3x3": _dense_3x3, "irregular": _irregular, "fuzzed": _fuzzed, "star": _star,
        "dense_3x3_lane_change": lambda d: _dense_3x3(d, lane_change=True)}


@pytest.mark.parametrize("net", sorted(NETS))
def test_table_every_step(net, tmp_path):
    """Every column, every step, equals the restatement from the roadnet JSON and the dict getters; phase and
    phase_remaining follow the fixed-time plan bit for bit and (without lane change) equal the JSON archive's."""
    cfg = NETS[net](str(tmp_path))
    lane_change = net.endswith("lane_change")
    eng = _emulated_engine(cfg)
    R = Restatement(cfg)
    t = table(eng)
    check_static(eng, R, t)
    check_table(eng, R, t, lane_change)
    steps = 150 if net == "star" else 250
    seen = dict(inside=0, waiting=0, pressure=set(), advanced=0)
    for s in range(steps):
        eng.next_step()
        R.pass_time()
        t2 = table(eng)
        assert t2["ptrs"] == t["ptrs"]
        t = t2
        check_table(eng, R, t, lane_change)
        if not lane_change and s % 50 == 49:
            check_dump(eng, R, t, str(tmp_path / "x.json"))
        seen["inside"] += int(t["movement_inside"].sum())
        seen["waiting"] += int(t["queue"].sum())
        seen["pressure"].update(t["pressure"].tolist())
        seen["advanced"] += int((t["phase"] > 0).sum())
    assert seen["inside"] > 100 and seen["waiting"] > 100 and seen["advanced"] > 10, seen
    assert max(seen["pressure"]) > 0 and (net == "star" or min(seen["pressure"]) < 0), seen["pressure"]
    if net == "star":   # more movements at one light than a warp has lanes: the kernel's movement loop goes round
        assert R.max_movements > 32, R.max_movements
    if net == "irregular":
        assert any(r != int(r) for r in R.remain), R.remain


def test_no_flows_gives_zeros(tmp_path):
    from cityflow_b200 import scenario
    cfg = scenario.write_scenario(str(tmp_path), scenario.grid_roadnet(2, 3), [], name="ioempty")
    eng = _emulated_engine(cfg)
    R = Restatement(cfg)
    for _ in range(3):
        eng.next_step()
        R.pass_time()
        t = table(eng)
        for k in ("pressure", "queue", "movement_in", "movement_in_waiting", "movement_out", "movement_inside",
                  "movement_pressure"):
            assert not t[k].any(), k
        real = ~np.array(R.virtual)
        pc = t["phase_count"]
        for k in np.nonzero(real)[0]:
            assert (t["phase_pressure"][k, :pc[k]] == 0).all() and (t["phase_pressure"][k, pc[k]:] == INT32_MIN).all()
        assert (t["phase_pressure"][~real] == INT32_MIN).all()
        check_table(eng, R, t, False)


def test_rl_phases_show_at_once_and_after_reset_and_load(tmp_path):
    """rlTrafficLight: a set_tl_phase made before a refresh shows in it, before any step; after reset() every light is
    back at phase 0, after load(snapshot) at the snapshot's phases."""
    cfg = _dense_3x3(str(tmp_path), rl=True)
    eng = _emulated_engine(cfg)
    R = Restatement(cfg)
    real = [k for k, v in enumerate(R.virtual) if not v]
    eng.next_step(20)
    table(eng)
    want = {k: (3 * n + 1) % len(R.phases[k]) for n, k in enumerate(real)}
    for k, ph in want.items():
        eng.set_tl_phase(k, ph)
    t = table(eng)
    assert [int(t["phase"][k]) for k in real] == [want[k] for k in real]
    remain0 = [R.phases[k][0][0] for k in real]
    assert [float(t["phase_remaining"][k]) for k in real] == remain0   # (the device never advances a light in this mode)
    snap = eng.snapshot()
    eng.next_step(5)
    eng.set_tl_phase(real[0], (want[real[0]] + 1) % len(R.phases[real[0]]))
    eng.next_step(5)
    eng.set_tl_phase(real[1], (want[real[1]] + 1) % len(R.phases[real[1]]))   # pending when the snapshot is loaded
    eng.load(snap)
    t = table(eng)
    assert [int(t["phase"][k]) for k in real] == [want[k] for k in real]
    check_table(eng, R, t, False, phases=False)
    eng.set_tl_phase(real[2], 0)
    eng.reset()
    t = table(eng)
    assert [int(t["phase"][k]) for k in real] == [0] * len(real)
    assert not t["movement_in"].any()


def test_max_pressure_lock_step(tmp_path):
    """Engine A is driven by the dict getters, MaxPressure restated from the roadnet JSON and set_tl_phase per light;
    engine B by the phase_pressure column (first maximum, as numpy's argmax).  Same phases and bit-equal full state
    every step."""
    cfg = _dense_3x3(str(tmp_path), rl=True)
    a, b = _emulated_engine(cfg), _emulated_engine(cfg)
    R = Restatement(cfg)
    switches = 0
    prev = None
    for s in range(250):
        act_a = R.max_pressure(a.lane_vehicle_count())
        t = table(b)
        act_b = [-1 if v else int(np.argmax(t["phase_pressure"][k])) for k, v in enumerate(R.virtual)]
        assert act_a == act_b, "step %d" % s
        for k, p in enumerate(act_a):
            if p >= 0:
                a.set_tl_phase(k, p)
                b.set_tl_phase(k, p)
        assert (table(b)["phase"] == act_b).all()
        switches += prev is not None and act_a != prev
        prev = act_a
        a.next_step()
        b.next_step()
        assert a.debug_vehicles().tobytes() == b.debug_vehicles().tobytes(), "step %d" % s
    assert switches > 20, switches
    assert a.vehicle_count() > 50
