"""TEST INFRASTRUCTURE ONLY: Python access to the two checkers.

* ``RefDump``    -- runs ``oracle/_ref/refdump`` (the compiled, UNMODIFIED reference with a
                    white-box state dumper, built by ``oracle/Makefile``) and parses its output.
* ``PortOracle`` -- ctypes wrapper around ``oracle/_build/libcityflow_oracle.so``, the CPU
                    restatement in ``oracle/cityflow_oracle.cpp``.

Only tests/, ``__graft_entry__.smoke()`` and ``bench.py``'s cpu_baseline / ``--impl reference`` leg
may import this module.  The product package never does.
"""
from __future__ import annotations

import ctypes
import json
import os
import subprocess
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REF_DIR = os.path.join(HERE, "_ref")
REFDUMP = os.path.join(REF_DIR, "refdump")
PORT_LIB = os.path.join(HERE, "_build", "libcityflow_oracle.so")

VEH_DTYPE = np.dtype([
    ("flow", "<i4"), ("cnt", "<i4"), ("priority", "<i4"), ("drivable", "<i4"),
    ("leader_flow", "<i4"), ("leader_cnt", "<i4"), ("blocker_flow", "<i4"), ("blocker_cnt", "<i4"),
    ("dis", "<f8"), ("speed", "<f8"), ("gap", "<f8"), ("enter_ll_time", "<i8"),
])


LC_DTYPE = np.dtype([   # `refdump runlc` / cfo_lc_vehicles: every running vehicle incl. shadows, keyed by priority
    ("flow", "<i4"), ("cnt", "<i4"), ("priority", "<i4"), ("partner_type", "<i4"), ("partner", "<i4"),
    ("drivable", "<i4"), ("leader", "<i4"), ("blocker", "<i4"), ("flags", "<i4"), ("last_dir", "<i4"),
    ("dis", "<f8"), ("speed", "<f8"), ("gap", "<f8"), ("offset", "<f8"), ("waiting_time", "<f8"),
    ("last_change_time", "<f8"),
])
REFDUMP_LC = os.path.join(os.path.dirname(REFDUMP), "refdump_lcorder")


REF_TIMEOUT = 900   # seconds: a reference run that does not come back fails the test instead of blocking the suite


def have_lc_ref() -> bool:
    return os.path.exists(REFDUMP_LC)


def load_reference_module():
    """The reference's own pybind11 module (oracle/_ref/cityflow*.so), loaded without touching
    sys.modules['cityflow'] (that name is this repository's drop-in package)."""
    import glob
    import importlib.machinery
    import importlib.util
    so = glob.glob(os.path.join(os.path.dirname(REFDUMP), "cityflow*.so"))
    if not so:
        return None
    loader = importlib.machinery.ExtensionFileLoader("cityflow", so[0])
    spec = importlib.util.spec_from_loader("cityflow", loader)
    mod = importlib.util.module_from_spec(spec)
    loader.exec_module(mod)
    return mod


def have_ref() -> bool:
    return os.path.exists(REFDUMP)


def have_port() -> bool:
    return os.path.exists(PORT_LIB)


def build(ref: bool = True) -> None:
    """Compile the checkers (building the checker is not using it)."""
    targets = ["port"]
    if ref and os.path.isdir("/root/reference/src"):
        targets.append("ref")
    subprocess.check_call(["make", "-s", "-C", HERE] + targets)


class StepState:
    """State after one step, as dumped by refdump / produced by PortOracle.snapshot()."""
    __slots__ = ("step", "vehicle_count", "pool_size", "finished", "cum_travel_time", "lane_count",
                 "lane_waiting", "lane_queue", "phases", "vehicles", "order")

    def key_sorted(self):
        v = self.vehicles
        idx = np.lexsort((v["cnt"], v["flow"]))
        return v[idx]


def parse_static(path: str) -> dict:
    buf = open(path, "rb").read()
    off = 0

    def i32(n=1):
        nonlocal off
        a = np.frombuffer(buf, "<i4", n, off)
        off += 4 * n
        return a if n > 1 else int(a[0])

    def f64(n=1):
        nonlocal off
        a = np.frombuffer(buf, "<f8", n, off)
        off += 8 * n
        return a if n > 1 else float(a[0])

    assert i32() == 0x43465331
    n_roads, n_inter, n_lanes, n_links, n_rl, n_cross = (i32() for _ in range(6))
    lanes = []
    for _ in range(n_lanes):
        length, max_speed = f64(), f64()
        road, idx, m = i32(), i32(), i32()
        links = [i32() for _ in range(m)]
        lanes.append(dict(length=length, max_speed=max_speed, road=road, idx=idx, links=links))
    links = []
    for _ in range(n_links):
        length = f64()
        start, end, rl, typ, m = i32(), i32(), i32(), i32(), i32()
        crosses = []
        for _ in range(m):
            c, side, other = i32(), i32(), i32()
            d0, d1 = f64(), f64()
            crosses.append((c, side, other, d0, d1))
        links.append(dict(length=length, start=start, end=end, road_link=rl, type=typ, crosses=crosses))
    inters = []
    for _ in range(n_inter):
        virt, nrl, nph = i32(), i32(), i32()
        phases = []
        for _ in range(nph):
            t = f64()
            av = [i32() for _ in range(nrl)]
            phases.append((t, av))
        inters.append(dict(virtual=virt, n_road_links=nrl, phases=phases))
    assert off == len(buf)
    return dict(n_roads=n_roads, n_cross=n_cross, n_road_links=n_rl, lanes=lanes, links=links, inters=inters)


def parse_run(path: str, n_inter: int, n_drivables: int):
    buf = open(path, "rb").read()
    off = 0
    magic, n_lanes = np.frombuffer(buf, "<i4", 2, off)
    off += 8
    assert magic == 0x43464431
    out = []
    while off < len(buf):
        st = StepState()
        hdr = np.frombuffer(buf, "<i4", 5, off)
        off += 20
        st.step, st.vehicle_count, n_run, st.pool_size, st.finished = (int(x) for x in hdr)
        st.cum_travel_time = float(np.frombuffer(buf, "<f8", 1, off)[0])
        off += 8
        st.lane_count = np.frombuffer(buf, "<i4", n_lanes, off); off += 4 * n_lanes
        st.lane_waiting = np.frombuffer(buf, "<i4", n_lanes, off); off += 4 * n_lanes
        st.lane_queue = np.frombuffer(buf, "<i4", n_lanes, off); off += 4 * n_lanes
        st.phases = np.frombuffer(buf, "<i4", n_inter, off); off += 4 * n_inter
        st.vehicles = np.frombuffer(buf, VEH_DTYPE, n_run, off); off += VEH_DTYPE.itemsize * n_run
        order = []
        for _ in range(n_drivables):
            m = int(np.frombuffer(buf, "<i4", 1, off)[0]); off += 4
            order.append(np.frombuffer(buf, "<i4", 2 * m, off).reshape(m, 2)); off += 8 * m
        st.order = order
        out.append(st)
    return out


def parse_runlc(path: str, n_inter: int, n_drivables: int):
    buf = open(path, "rb").read()
    off = 0
    magic, n_lanes = np.frombuffer(buf, "<i4", 2, off)
    off += 8
    assert magic == 0x43464C31
    out = []
    while off < len(buf):
        st = StepState()
        hdr = np.frombuffer(buf, "<i4", 5, off)
        off += 20
        st.step, st.vehicle_count, n_run, st.pool_size, st.finished = (int(x) for x in hdr)
        st.cum_travel_time = float(np.frombuffer(buf, "<f8", 1, off)[0])
        off += 8
        st.lane_count = np.frombuffer(buf, "<i4", n_lanes, off); off += 4 * n_lanes
        st.lane_waiting = st.lane_queue = None
        st.phases = np.frombuffer(buf, "<i4", n_inter, off); off += 4 * n_inter
        st.vehicles = np.frombuffer(buf, LC_DTYPE, n_run, off); off += LC_DTYPE.itemsize * n_run
        order = []
        for _ in range(n_drivables):
            m = int(np.frombuffer(buf, "<i4", 1, off)[0]); off += 4
            order.append(np.frombuffer(buf, "<i4", m, off)); off += 4 * m
        st.order = order
        out.append(st)
    return out


def parse_counts(path: str) -> dict:
    """`refdump counts`: {"vehicle_count": int32[steps], "dumps": {step: (lane_count, lane_waiting, lane_speed_sum)}}"""
    buf = open(path, "rb").read()
    magic, n_lanes, steps, every = (int(x) for x in np.frombuffer(buf, "<i4", 4, 0))
    assert magic == 0x43464E31
    off = 16
    vc = np.zeros(steps, np.int64)
    dumps = {}
    for s in range(steps):
        vc[s] = int(np.frombuffer(buf, "<i4", 1, off)[0]); off += 4
        if (s + 1) % every != 0 and s + 1 != steps:
            continue
        st = int(np.frombuffer(buf, "<i4", 1, off)[0]); off += 4
        assert st == s + 1
        cnt = np.frombuffer(buf, "<i4", n_lanes, off); off += 4 * n_lanes
        wait = np.frombuffer(buf, "<i4", n_lanes, off); off += 4 * n_lanes
        ssum = np.frombuffer(buf, "<f8", n_lanes, off); off += 8 * n_lanes
        dumps[st] = (cnt, wait, ssum)
    assert off == len(buf)
    return {"vehicle_count": vc, "dumps": dumps, "n_lanes": n_lanes}


class RefDump:
    """The compiled reference (oracle/_ref/refdump)."""

    @staticmethod
    def counts(config: str, steps: int, threads: int = 1, every: int = 25, out_path: str = None) -> dict:
        """Vehicle count after every step + per-lane observables every `every` steps (cheap at 1e6 vehicles)."""
        path = out_path or tempfile.mktemp(suffix=".bin")
        try:
            subprocess.check_call([REFDUMP, "counts", config, str(steps), str(threads), path, str(every)], timeout=3600)
            return parse_counts(path)
        finally:
            if out_path is None and os.path.exists(path):
                os.unlink(path)

    @staticmethod
    def static(config: str) -> dict:
        with tempfile.NamedTemporaryFile(suffix=".bin") as f:
            subprocess.check_call([REFDUMP, "static", config, f.name], timeout=REF_TIMEOUT)
            return parse_static(f.name)

    @staticmethod
    def run(config: str, steps: int, threads: int = 1, every: int = 1, *, n_inter: int, n_drivables: int):
        with tempfile.NamedTemporaryFile(suffix=".bin") as f:
            subprocess.check_call([REFDUMP, "run", config, str(steps), str(threads), f.name, str(every)], timeout=REF_TIMEOUT)
            return parse_run(f.name, n_inter, n_drivables)

    @staticmethod
    def archive(config: str, steps: int, out_json: str, threads: int = 1) -> None:
        """The reference's own JSON archive (Archive::dump) after `steps` steps."""
        subprocess.check_call([REFDUMP, "archive", config, str(steps), str(threads), out_json], timeout=REF_TIMEOUT)

    @staticmethod
    def resume(config: str, archive_json: str, steps: int, threads: int = 1, every: int = 1, *, n_inter: int, n_drivables: int):
        """Engine::loadFromFile(archive_json) in the reference, then `steps` steps dumped like run()."""
        with tempfile.NamedTemporaryFile(suffix=".bin") as f:
            subprocess.check_call([REFDUMP, "resume", config, archive_json, str(steps), str(threads), f.name, str(every)], timeout=REF_TIMEOUT)
            return parse_run(f.name, n_inter, n_drivables)

    @staticmethod
    def runlc(config: str, steps: int, every: int = 1, *, n_inter: int, n_drivables: int, patched: bool = True, threads: int = 1):
        """laneChange=true run of the reference with the priority-ordered worker set (`patched`,
        oracle/lc_order_patch.sh) or of the unmodified build; states incl. shadows."""
        with tempfile.NamedTemporaryFile(suffix=".bin") as f:
            subprocess.check_call([REFDUMP_LC if patched else REFDUMP, "runlc", config, str(steps), str(threads), f.name, str(every)], timeout=REF_TIMEOUT)
            return parse_runlc(f.name, n_inter, n_drivables)

    @staticmethod
    def bench(config: str, steps: int, threads: int, warmup: int = 0) -> dict:
        out = subprocess.check_output([REFDUMP, "bench", config, str(steps), str(threads), str(warmup)], timeout=3600)
        return json.loads(out.decode().strip().splitlines()[-1])


class PortOracle:
    """CPU restatement (oracle/cityflow_oracle.cpp) through its plain C interface."""

    def __init__(self, config: str):
        lib = ctypes.CDLL(PORT_LIB)
        self.lib = lib
        lib.cfo_create.restype = ctypes.c_void_p
        lib.cfo_create.argtypes = [ctypes.c_char_p]
        for name in ("cfo_destroy", "cfo_next_step", "cfo_reset", "cfo_lane_vehicle_count", "cfo_lane_waiting_count",
                     "cfo_lane_queue_size", "cfo_phases", "cfo_set_tl_phase"):
            getattr(lib, name).restype = None
        lib.cfo_destroy.argtypes = [ctypes.c_void_p]
        lib.cfo_next_step.argtypes = [ctypes.c_void_p, ctypes.c_int]
        lib.cfo_reset.argtypes = [ctypes.c_void_p, ctypes.c_int]
        lib.cfo_set_tl_phase.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int]
        for name in ("cfo_lane_vehicle_count", "cfo_lane_waiting_count", "cfo_lane_queue_size", "cfo_phases"):
            getattr(lib, name).argtypes = [ctypes.c_void_p, ctypes.c_void_p]
        for name in ("cfo_num_lanes", "cfo_num_drivables", "cfo_num_intersections", "cfo_vehicle_count",
                     "cfo_pool_size", "cfo_finished_count", "cfo_tie_count"):
            getattr(lib, name).restype = ctypes.c_int
            getattr(lib, name).argtypes = [ctypes.c_void_p]
        for name in ("cfo_cumulative_travel_time", "cfo_current_time"):
            getattr(lib, name).restype = ctypes.c_double
            getattr(lib, name).argtypes = [ctypes.c_void_p]
        lib.cfo_vehicles.restype = ctypes.c_int
        lib.cfo_vehicles.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int]
        lib.cfo_drivable_vehicles.restype = ctypes.c_int
        lib.cfo_drivable_vehicles.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_int]
        self.h = lib.cfo_create(config.encode())
        if not self.h:
            raise RuntimeError("oracle: load config failed: %s" % config)
        self.n_lanes = lib.cfo_num_lanes(self.h)
        self.n_drivables = lib.cfo_num_drivables(self.h)
        self.n_inter = lib.cfo_num_intersections(self.h)
        self.steps = 0

    def __del__(self):
        if getattr(self, "h", None):
            self.lib.cfo_destroy(self.h)
            self.h = None

    def next_step(self, n: int = 1):
        self.lib.cfo_next_step(self.h, n)
        self.steps += n

    def reset(self, seed: bool = False):
        self.lib.cfo_reset(self.h, int(seed))
        self.steps = 0

    def set_tl_phase(self, inter: int, phase: int):
        self.lib.cfo_set_tl_phase(self.h, inter, phase)

    def vehicle_count(self) -> int:
        return self.lib.cfo_vehicle_count(self.h)

    def set_random_seed(self, seed: int):
        self.lib.cfo_set_random_seed.restype = None
        self.lib.cfo_set_random_seed.argtypes = [ctypes.c_void_p, ctypes.c_int]
        self.lib.cfo_set_random_seed(self.h, seed)

    def set_vehicle_speed(self, flow: int, cnt: int, speed: float) -> bool:
        self.lib.cfo_set_vehicle_speed.restype = ctypes.c_int
        self.lib.cfo_set_vehicle_speed.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_double]
        return self.lib.cfo_set_vehicle_speed(self.h, flow, cnt, speed) == 0

    def set_vehicle_route(self, flow: int, cnt: int, roads: list) -> bool:
        self.lib.cfo_road_index.restype = ctypes.c_int
        self.lib.cfo_road_index.argtypes = [ctypes.c_void_p, ctypes.c_char_p]
        r = np.array([self.lib.cfo_road_index(self.h, x.encode()) for x in roads], np.int32)
        if (r < 0).any():
            return False            # unknown road id (engine.cpp:859-861)
        self.lib.cfo_set_vehicle_route.restype = ctypes.c_int
        self.lib.cfo_set_vehicle_route.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_int]
        return self.lib.cfo_set_vehicle_route(self.h, flow, cnt, r.ctypes.data, len(r)) == 1

    def get_leader(self, flow: int, cnt: int):
        """(flow, cnt) of the leader, None if there is none; KeyError for an unknown vehicle."""
        self.lib.cfo_get_leader.restype = ctypes.c_int
        self.lib.cfo_get_leader.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p]
        a, b = ctypes.c_int32(), ctypes.c_int32()
        rc = self.lib.cfo_get_leader(self.h, flow, cnt, ctypes.byref(a), ctypes.byref(b))
        if rc < 0:
            raise KeyError((flow, cnt))
        return (a.value, b.value) if rc else None

    def average_travel_time(self) -> float:
        self.lib.cfo_average_travel_time.restype = ctypes.c_double
        self.lib.cfo_average_travel_time.argtypes = [ctypes.c_void_p]
        return float(self.lib.cfo_average_travel_time(self.h))

    def push_vehicle(self, info: dict, roads: list):
        names = ["speed", "length", "width", "maxPosAcc", "maxNegAcc", "usualPosAcc", "usualNegAcc", "minGap", "maxSpeed", "headwayTime"]
        v = np.array([info.get(k, float("nan")) for k in names], np.float64)
        self.lib.cfo_road_index.restype = ctypes.c_int
        self.lib.cfo_road_index.argtypes = [ctypes.c_void_p, ctypes.c_char_p]
        r = np.array([self.lib.cfo_road_index(self.h, x.encode()) for x in roads], np.int32)
        assert (r >= 0).all()
        self.lib.cfo_push_vehicle.restype = None
        self.lib.cfo_push_vehicle.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int]
        self.lib.cfo_push_vehicle(self.h, v.ctypes.data, r.ctypes.data, len(r))

    def tie_count(self) -> int:
        return self.lib.cfo_tie_count(self.h)

    def max_refused_cross_index(self) -> int:
        """Highest position in its laneLink's cross list at which Cross::canPass has refused a vehicle so far (-1: none)."""
        self.lib.cfo_max_refused_cross_index.restype = ctypes.c_int
        self.lib.cfo_max_refused_cross_index.argtypes = [ctypes.c_void_p]
        return self.lib.cfo_max_refused_cross_index(self.h)

    def _lane_array(self, fn, n=None):
        a = np.zeros(n or self.n_lanes, np.int32)
        getattr(self.lib, fn)(self.h, a.ctypes.data)
        return a

    def lane_vehicle_count(self):
        return self._lane_array("cfo_lane_vehicle_count")

    def lane_waiting_count(self):
        return self._lane_array("cfo_lane_waiting_count")

    def vehicles(self):
        n = self.lib.cfo_vehicles(self.h, None, 0)
        a = np.zeros(n, VEH_DTYPE)
        self.lib.cfo_vehicles(self.h, a.ctypes.data, n)
        return a

    def lc_snapshot(self) -> StepState:
        """State in the shape of parse_runlc (laneChange runs)."""
        lib = self.lib
        lib.cfo_lc_vehicles.restype = ctypes.c_int
        lib.cfo_lc_vehicles.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int]
        lib.cfo_drivable_priorities.restype = ctypes.c_int
        lib.cfo_drivable_priorities.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_int]
        st = StepState()
        st.step = self.steps
        st.vehicle_count = self.vehicle_count()
        st.pool_size = lib.cfo_pool_size(self.h)
        st.finished = lib.cfo_finished_count(self.h)
        st.cum_travel_time = lib.cfo_cumulative_travel_time(self.h)
        st.lane_count = self.lane_vehicle_count()
        st.lane_waiting = st.lane_queue = None
        st.phases = self._lane_array("cfo_phases", self.n_inter)
        n = lib.cfo_lc_vehicles(self.h, None, 0)
        a = np.zeros(n, LC_DTYPE)
        lib.cfo_lc_vehicles(self.h, a.ctypes.data, n)
        st.vehicles = a
        st.order = []
        tmp = np.zeros(4096, np.int32)
        for d in range(self.n_drivables):
            m = lib.cfo_drivable_priorities(self.h, d, tmp.ctypes.data, len(tmp))
            st.order.append(tmp[:m].copy())
        return st

    def snapshot(self, with_order: bool = False) -> StepState:
        st = StepState()
        st.step = self.steps
        st.vehicle_count = self.vehicle_count()
        st.pool_size = self.lib.cfo_pool_size(self.h)
        st.finished = self.lib.cfo_finished_count(self.h)
        st.cum_travel_time = self.lib.cfo_cumulative_travel_time(self.h)
        st.lane_count = self.lane_vehicle_count()
        st.lane_waiting = self.lane_waiting_count()
        st.lane_queue = self._lane_array("cfo_lane_queue_size")
        st.phases = self._lane_array("cfo_phases", self.n_inter)
        st.vehicles = self.vehicles()
        st.order = None
        if with_order:
            st.order = []
            tmp = np.zeros(2 * 4096, np.int32)
            for d in range(self.n_drivables):
                m = self.lib.cfo_drivable_vehicles(self.h, d, tmp.ctypes.data, 4096)
                st.order.append(tmp[:2 * m].reshape(m, 2).copy())
        return st


def compare_states(a: StepState, b: StepState, *, speed_tol: float = 0.0, check_order: bool = True) -> list:
    """Returns a list of human-readable mismatches (empty = parity)."""
    bad = []
    for name in ("vehicle_count", "pool_size", "finished"):
        if getattr(a, name) != getattr(b, name):
            bad.append("%s: %s != %s" % (name, getattr(a, name), getattr(b, name)))
    if a.cum_travel_time != b.cum_travel_time:
        bad.append("cum_travel_time: %r != %r" % (a.cum_travel_time, b.cum_travel_time))
    for name in ("lane_count", "lane_waiting", "lane_queue", "phases"):
        x, y = getattr(a, name), getattr(b, name)
        if x is None or y is None:
            continue
        if not np.array_equal(x, y):
            w = np.nonzero(x != y)[0]
            bad.append("%s differs at %d entries, first idx %d: %d != %d" % (name, len(w), w[0], x[w[0]], y[w[0]]))
    va, vb = a.key_sorted(), b.key_sorted()
    if len(va) != len(vb):
        bad.append("running vehicles: %d != %d" % (len(va), len(vb)))
        return bad
    for f in ("flow", "cnt", "priority", "drivable", "leader_flow", "leader_cnt", "blocker_flow", "blocker_cnt",
              "enter_ll_time"):
        if not np.array_equal(va[f], vb[f]):
            w = np.nonzero(va[f] != vb[f])[0]
            bad.append("veh.%s differs at %d vehicles, first (flow %d cnt %d): %d != %d" %
                       (f, len(w), va["flow"][w[0]], va["cnt"][w[0]], va[f][w[0]], vb[f][w[0]]))
    for f in ("dis", "speed", "gap"):
        x, y = va[f], vb[f]
        if speed_tol == 0.0:
            neq = x.view(np.int64) != y.view(np.int64)
            neq &= ~((x == 0) & (y == 0))  # +0 / -0
        else:
            neq = np.abs(x - y) > speed_tol
        if neq.any():
            w = np.nonzero(neq)[0]
            bad.append("veh.%s differs at %d vehicles, first (flow %d cnt %d): %r != %r" %
                       (f, len(w), va["flow"][w[0]], va["cnt"][w[0]], float(x[w[0]]), float(y[w[0]])))
    if check_order and a.order is not None and b.order is not None:
        for d, (x, y) in enumerate(zip(a.order, b.order)):
            if not np.array_equal(x, y):
                bad.append("list order differs in drivable %d" % d)
                break
    return bad


def compare_lc_states(ref: StepState, got: StepState) -> list:
    """Lane-change runs: bit-equal or a list of differences (vehicles keyed by priority)."""
    bad = []
    for f in ("step", "vehicle_count", "pool_size", "finished"):
        if getattr(ref, f) != getattr(got, f):
            bad.append("%s: ref %s got %s" % (f, getattr(ref, f), getattr(got, f)))
    if ref.cum_travel_time != got.cum_travel_time:
        bad.append("cum_travel_time: ref %r got %r" % (ref.cum_travel_time, got.cum_travel_time))
    if not np.array_equal(ref.lane_count, got.lane_count):
        bad.append("lane counts differ on %d lanes" % int((np.asarray(ref.lane_count) != np.asarray(got.lane_count)).sum()))
    if not np.array_equal(ref.phases, got.phases):
        bad.append("phases differ")
    a, b = ref.vehicles, got.vehicles
    if len(a) != len(b):
        bad.append("running vehicles: ref %d got %d" % (len(a), len(b)))
    else:
        for f in LC_DTYPE.names:
            ne = np.nonzero(a[f] != b[f])[0]
            if len(ne):
                k = ne[0]
                bad.append("%s differs for %d vehicles, first flow_%d_%d prio %d: ref %r got %r" %
                           (f, len(ne), a["flow"][k], a["cnt"][k], a["priority"][k], a[f][k], b[f][k]))
    for d, (x, y) in enumerate(zip(ref.order, got.order)):
        if not np.array_equal(x, y):
            bad.append("list order differs on drivable %d" % d)
            break
    return bad
