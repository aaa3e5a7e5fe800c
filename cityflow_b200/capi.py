"""ctypes binding of the C-ABI (include/cityflow_b200.h) -- what a foreign-language host would
bind.  Used by the parity tests so they exercise the exported symbols directly."""
from __future__ import annotations

import ctypes
import re
import os

import numpy as np

from . import LIB_PATH

HEADER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "cityflow_b200.h")

VEH_DTYPE = np.dtype([
    ("flow", "<i4"), ("cnt", "<i4"), ("priority", "<i4"), ("drivable", "<i4"),
    ("leader_flow", "<i4"), ("leader_cnt", "<i4"), ("blocker_flow", "<i4"), ("blocker_cnt", "<i4"),
    ("dis", "<f8"), ("speed", "<f8"), ("gap", "<f8"), ("enter_ll_time", "<i8"),
])
REF_DTYPE = np.dtype([("flow", "<i4"), ("index", "<i4")])
REPLAY_DTYPE = np.dtype([("drivable", "<i4"), ("distance", "<f8"), ("flow", "<i4"), ("index", "<i4"),
                         ("length", "<f8"), ("width", "<f8")], align=True)   # cfb_replay_vehicle
REPLAY_LC_DTYPE = np.dtype([("v", REPLAY_DTYPE), ("shadow_depth", "<i4"), ("lane_change_dir", "<i4"),
                            ("offset", "<f8")], align=True)                     # cfb_replay_vehicle_lc
REF_SHADOW_SHIFT = 24          # CFB_REF_SHADOW_SHIFT: bits 24-30 of cfb_vehicle_ref.index count "_shadow" suffixes
REF_INDEX_MASK = 0x00ffffff    # CFB_REF_INDEX_MASK


def vehicle_name(flow: int, index: int) -> str:
    """The reference's id of a cfb_vehicle_ref (include/cityflow_b200.h)."""
    base = "manually_pushed_%d" % (index & REF_INDEX_MASK) if flow == -2 else "flow_%d_%d" % (flow, index & REF_INDEX_MASK)
    return base + "_shadow" * (index >> REF_SHADOW_SHIFT)


def parse_vehicle_name(name: str):
    """(flow, index) of a reference id, shadow suffixes in index's bits 24-30; None if it names no vehicle."""
    depth = 0
    while name.endswith("_shadow") and depth < 127:
        name, depth = name[:-7], depth + 1
    m = re.fullmatch(r"flow_(\d+)_(\d+)|manually_pushed_(\d+)", name)
    if not m:
        return None
    flow, index = (int(m.group(1)), int(m.group(2))) if m.group(3) is None else (-2, int(m.group(3)))
    if index > REF_INDEX_MASK:
        return None
    return flow, index | (depth << REF_SHADOW_SHIFT)


def declared_symbols() -> list:
    """Every function name the header declares."""
    txt = open(HEADER).read()
    txt = re.sub(r"/\*.*?\*/", "", txt, flags=re.S)
    return sorted(set(re.findall(r"\b(cfb_[a-z0-9_]+)\s*\(", txt)))


def load_library() -> ctypes.CDLL:
    """The product library (libcityflow_b200.so next to this file); there is no other path to load from."""
    if not os.path.exists(LIB_PATH):
        raise RuntimeError("cityflow_b200: %s is missing -- build it first (__graft_entry__.build())" % LIB_PATH)
    return bind(ctypes.CDLL(LIB_PATH))


def bind(lib: ctypes.CDLL) -> ctypes.CDLL:
    """Attach the argument / result types of include/cityflow_b200.h to an opened library."""
    c = ctypes
    vp, i32, i64, dbl, cp = c.c_void_p, c.c_int, c.c_int64, c.c_double, c.c_char_p
    sig = {
        "cfb_engine_create": (vp, [cp, i32, i32]),
        "cfb_engine_destroy": (None, [vp]),
        "cfb_last_error": (cp, [vp]),
        "cfb_next_step": (i32, [vp]),
        "cfb_next_steps": (i32, [vp, i32]),
        "cfb_get_vehicle_count": (i64, [vp]),
        "cfb_get_current_time": (dbl, [vp]),
        "cfb_get_average_travel_time": (dbl, [vp]),
        "cfb_num_lanes": (i32, [vp]),
        "cfb_lane_id": (cp, [vp, i32]),
        "cfb_num_intersections": (i32, [vp]),
        "cfb_intersection_id": (cp, [vp, i32]),
        "cfb_get_lane_vehicle_count": (i32, [vp, vp, i32]),
        "cfb_get_lane_waiting_vehicle_count": (i32, [vp, vp, i32]),
        "cfb_get_vehicle_speed": (i64, [vp, vp, vp, vp, i64]),
        "cfb_get_vehicles": (i64, [vp, i32, vp, i64]),
        "cfb_get_lane_vehicles": (i64, [vp, vp, i32, vp, i64]),
        "cfb_set_tl_phase": (i32, [vp, cp, i32]),
        "cfb_set_tl_phase_index": (i32, [vp, i32, i32]),
        "cfb_set_random_seed": (i32, [vp, i32]),
        "cfb_reset": (i32, [vp, i32]),
        "cfb_debug_vehicles": (i64, [vp, vp, i64]),
        "cfb_gpu_launches": (i64, [vp]),
        "cfb_tie_count": (i64, [vp]),
        "cfb_enable_kernel_timing": (i32, [vp, i32]),
        "cfb_kernel_times": (i32, [vp, vp, vp]),
        "cfb_synchronize": (i32, [vp]),
        "cfb_num_drivables": (i64, [vp]),
        "cfb_shard_group_create": (vp, [cp, i32, i32]),
        "cfb_shard_group_destroy": (None, [vp]),
        "cfb_shard_group_step": (i32, [vp, i32]),
        "cfb_shard_group_last_error": (cp, [vp]),
        "cfb_shard_group_vehicle_count": (i64, [vp]),
        "cfb_shard_group_lane_counts": (i32, [vp, vp, i32, i32]),
        "cfb_shard_group_debug_vehicles": (i64, [vp, vp, i64]),
        "cfb_replay_create": (vp, [cp]),
        "cfb_replay_destroy": (None, [vp]),
        "cfb_replay_roadnet_json": (i64, [vp, vp, i64]),
        "cfb_replay_format_step": (i64, [vp, vp, i64, vp, vp, i64]),
        "cfb_replay_format_step_lc": (i64, [vp, vp, i64, vp, vp, i64]),
        "cfb_push_vehicle": (i32, [vp, vp, vp, i32]),
        "cfb_snapshot": (vp, [vp]),
        "cfb_archive_destroy": (None, [vp]),
        "cfb_load": (i32, [vp, vp]),
        "cfb_archive_dump": (i32, [vp, cp]),
        "cfb_load_from_file": (i32, [vp, cp]),
        "cfb_set_replay_file": (i32, [vp, cp]),
        "cfb_set_save_replay": (i32, [vp, i32]),
        "cfb_timed_steps": (i32, [vp, i32, i32, vp, vp]),
        "cfb_vehicle_steps": (i64, [vp]),
        "cfb_transfer_bytes": (i32, [vp, vp, vp]),
        "cfb_debug_launch_form": (i32, [vp, vp]),
        "cfb_debug_step_grids": (i32, [vp, vp]),
        "cfb_shard_group_counters": (i32, [vp, vp]),
        "cfb_debug_shard_group_create_cut": (vp, [cp, i32, i32, vp]),
        "cfb_observe_vehicles_device": (i32, [vp, vp, vp]),
        "cfb_set_vehicle_speeds_device": (i32, [vp, vp, vp, vp, i64, vp]),
        "cfb_vehicle_refs": (i32, [vp, vp, i64, vp]),
        "cfb_drivable_id": (cp, [vp, i64]),
        "cfb_observe_intersections_device": (i32, [vp, vp, vp]),
        "cfb_num_road_links": (i32, [vp]),
        "cfb_road_link_info": (i32, [vp, i32, vp]),
        "cfb_observe_vehicle_context_device": (i32, [vp, vp, vp]),
    }
    for name, (res, args) in sig.items():
        if not hasattr(lib, name):
            continue   # (a test build may lack optional entry points)
        fn = getattr(lib, name)
        fn.restype = res
        fn.argtypes = args
    return lib


class DeviceVehicleObs(ctypes.Structure):
    """cfb_device_vehicle_obs: device pointers of the per-vehicle observation table (include/cityflow_b200.h)."""
    _fields_ = [("slot", ctypes.c_void_p), ("priority", ctypes.c_void_p), ("drivable", ctypes.c_void_p),
                ("distance", ctypes.c_void_p), ("speed", ctypes.c_void_p), ("shadow", ctypes.c_void_p),
                ("drivable_begin", ctypes.c_void_p), ("count", ctypes.c_void_p), ("capacity", ctypes.c_int64),
                ("n_drivables", ctypes.c_int32), ("device", ctypes.c_int32)]


class DeviceVehicleContext(ctypes.Structure):
    """cfb_device_vehicle_context: the per-vehicle table and what lies ahead of each row (include/cityflow_b200.h)."""
    _fields_ = [("table", DeviceVehicleObs)] + [(k, ctypes.c_void_p) for k in (
        "leader", "gap", "next_drivable", "signal", "drivable_length", "drivable_max_speed", "link_road_link")] + \
        [("n_lanes", ctypes.c_int32), ("n_links", ctypes.c_int32)]


class DeviceIntersectionObs(ctypes.Structure):
    """cfb_device_intersection_obs: device pointers of the intersection / movement observations (include/cityflow_b200.h)."""
    _fields_ = [(k, ctypes.c_void_p) for k in (
        "phase", "phase_remaining", "pressure", "queue", "movement_in", "movement_in_waiting", "movement_out",
        "movement_inside", "movement_pressure", "phase_pressure", "movement_begin", "movement_intersection",
        "phase_count", "phase_movements")] + \
        [(k, ctypes.c_int32) for k in ("n_intersections", "n_road_links", "max_phases", "max_movements", "device")]


class RoadLink(ctypes.Structure):
    """cfb_road_link: one movement as the roadnet file lists it."""
    _fields_ = [("intersection", ctypes.c_int32), ("index", ctypes.c_int32), ("type", ctypes.c_int32),
                ("pad", ctypes.c_int32), ("start_road", ctypes.c_char_p), ("end_road", ctypes.c_char_p)]


class CEngine:
    """Minimal object wrapper over the raw C calls (numpy in / out)."""

    def _library(self) -> ctypes.CDLL:
        return load_library()

    def __init__(self, config: str, device: int = 0):
        self.lib = self._library()
        self.h = self.lib.cfb_engine_create(config.encode(), 1, device)
        if not self.h:
            raise RuntimeError("cfb_engine_create failed: %s" % self.lib.cfb_last_error(None).decode())
        self.n_lanes = self.lib.cfb_num_lanes(self.h)
        self.n_inter = self.lib.cfb_num_intersections(self.h)
        self.n_drivables = int(self.lib.cfb_num_drivables(self.h))

    def close(self):
        if getattr(self, "h", None):
            self.lib.cfb_engine_destroy(self.h)
            self.h = None

    __del__ = close

    def _check(self, rc):
        if rc < 0:
            raise RuntimeError(self.lib.cfb_last_error(self.h).decode())
        return rc

    def next_step(self, n: int = 1):
        self._check(self.lib.cfb_next_steps(self.h, n))

    def vehicle_count(self) -> int:
        return int(self._check(self.lib.cfb_get_vehicle_count(self.h)))

    def lane_ids(self):
        return [self.lib.cfb_lane_id(self.h, i).decode() for i in range(self.n_lanes)]

    def lane_vehicle_count(self):
        a = np.zeros(self.n_lanes, np.int32)
        self._check(self.lib.cfb_get_lane_vehicle_count(self.h, a.ctypes.data, self.n_lanes))
        return a

    def lane_waiting_count(self):
        a = np.zeros(self.n_lanes, np.int32)
        self._check(self.lib.cfb_get_lane_waiting_vehicle_count(self.h, a.ctypes.data, self.n_lanes))
        return a

    def vehicle_speed(self):
        n = self._check(self.lib.cfb_get_vehicle_speed(self.h, None, None, None, 0))
        ids = np.zeros(n, REF_DTYPE)
        sp = np.zeros(n)
        ds = np.zeros(n)
        self._check(self.lib.cfb_get_vehicle_speed(self.h, ids.ctypes.data, sp.ctypes.data, ds.ctypes.data, n))
        return ids, sp, ds

    def debug_vehicles(self):
        n = self._check(self.lib.cfb_debug_vehicles(self.h, None, 0))
        a = np.zeros(n, VEH_DTYPE)
        if n:
            self._check(self.lib.cfb_debug_vehicles(self.h, a.ctypes.data, n))
        return a

    def set_tl_phase(self, inter: int, phase: int):
        self._check(self.lib.cfb_set_tl_phase_index(self.h, inter, phase))

    def reset(self, seed: bool = False):
        self._check(self.lib.cfb_reset(self.h, int(seed)))

    def set_vehicle_speed(self, flow: int, index: int, speed: float) -> bool:
        """Engine::setVehicleSpeed (engine.cpp:827-834); False = no such vehicle."""
        class Ref(ctypes.Structure):
            _fields_ = [("flow", ctypes.c_int32), ("index", ctypes.c_int32)]
        self.lib.cfb_set_vehicle_speed.restype = ctypes.c_int
        self.lib.cfb_set_vehicle_speed.argtypes = [ctypes.c_void_p, Ref, ctypes.c_double]
        return self.lib.cfb_set_vehicle_speed(self.h, Ref(flow, index), speed) >= 0

    def set_vehicle_route(self, flow: int, index: int, roads: list) -> bool:
        """Engine::setRoute (engine.cpp:852-866)."""
        class Ref(ctypes.Structure):
            _fields_ = [("flow", ctypes.c_int32), ("index", ctypes.c_int32)]
        arr = (ctypes.c_char_p * len(roads))(*[r.encode() for r in roads])
        ok = ctypes.c_int(0)
        self.lib.cfb_set_vehicle_route.restype = ctypes.c_int
        self.lib.cfb_set_vehicle_route.argtypes = [ctypes.c_void_p, Ref, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p]
        self._check(self.lib.cfb_set_vehicle_route(self.h, Ref(flow, index), arr, len(roads), ctypes.byref(ok)))
        return ok.value == 1

    def set_random_seed(self, seed: int):
        self._check(self.lib.cfb_set_random_seed(self.h, seed))

    def push_vehicle(self, info: dict, roads: list):
        """Engine::pushVehicle (engine.cpp:693-717); missing keys keep the reference's defaults."""
        names = ["speed", "length", "width", "maxPosAcc", "maxNegAcc", "usualPosAcc", "usualNegAcc", "minGap", "maxSpeed", "headwayTime"]
        v = np.array([info.get(k, float("nan")) for k in names], np.float64)
        arr = (ctypes.c_char_p * len(roads))(*[r.encode() for r in roads])
        self._check(self.lib.cfb_push_vehicle(self.h, v.ctypes.data, arr, len(roads)))

    def dump(self, path: str):
        """engine.snapshot().dump(path): the reference's JSON schema when `path` ends in .json, else the binary image."""
        a = self.lib.cfb_snapshot(self.h)
        if not a:
            raise RuntimeError(self.lib.cfb_last_error(self.h).decode())
        try:
            if self.lib.cfb_archive_dump(a, path.encode()) < 0:
                raise RuntimeError("cannot write archive to %s: %s" % (path, self.lib.cfb_last_error(self.h).decode()))
        finally:
            self.lib.cfb_archive_destroy(a)

    def load_from_file(self, path: str):
        self._check(self.lib.cfb_load_from_file(self.h, path.encode()))

    def average_travel_time(self) -> float:
        return float(self.lib.cfb_get_average_travel_time(self.h))

    def gpu_launches(self) -> int:
        return int(self.lib.cfb_gpu_launches(self.h))

    def tie_count(self) -> int:
        return int(self._check(self.lib.cfb_tie_count(self.h)))

    def launch_form(self) -> tuple:
        """(graph, pdl, coop, mirror) of the last step (cfb_debug_launch_form)."""
        a = np.zeros(4, np.int32)
        self._check(self.lib.cfb_debug_launch_form(self.h, a.ctypes.data))
        return tuple(int(x) for x in a)

    def step_grids(self) -> dict:
        """Blocks of the list-driven step kernels (cfb_debug_step_grids); 0 = not launched yet."""
        a = np.zeros(5, np.int32)
        self._check(self.lib.cfb_debug_step_grids(self.h, a.ctypes.data))
        return dict(zip(("k_notify", "k_control", "k_move", "k_leader", "k_step"), (int(x) for x in a)))

    def timed_steps(self, n: int, flush_l2: bool = False):
        """(device ms, vehicle steps) of n event-bracketed steps (cfb_timed_steps)."""
        ms, vs = ctypes.c_double(0.0), ctypes.c_int64(0)
        self._check(self.lib.cfb_timed_steps(self.h, n, int(flush_l2), ctypes.byref(ms), ctypes.byref(vs)))
        return ms.value, vs.value

    def vehicle_steps(self) -> int:
        return int(self._check(self.lib.cfb_vehicle_steps(self.h)))

    def enable_kernel_timing(self, on: bool = True):
        self._check(self.lib.cfb_enable_kernel_timing(self.h, int(on)))

    def kernel_times(self):
        """(ms per kernel: ingest, notify, control, move, leader; steps timed)"""
        ms, n = np.zeros(5), ctypes.c_int64(0)
        self._check(self.lib.cfb_kernel_times(self.h, ms.ctypes.data, ctypes.byref(n)))
        return ms, n.value

    def transfer_bytes(self):
        """(host->device, device->host) bytes so far"""
        h2d, d2h = ctypes.c_int64(0), ctypes.c_int64(0)
        self._check(self.lib.cfb_transfer_bytes(self.h, ctypes.byref(h2d), ctypes.byref(d2h)))
        return h2d.value, d2h.value

    def observe_vehicles_device(self, stream: int = 0) -> DeviceVehicleObs:
        """Refresh the per-vehicle observation table (cfb_observe_vehicles_device) and return its pointers."""
        o = DeviceVehicleObs()
        self._check(self.lib.cfb_observe_vehicles_device(self.h, stream, ctypes.byref(o)))
        return o

    def set_vehicle_speeds_device(self, slot: int, priority: int, speed: int, n: int, stream: int = 0):
        """cfb_set_vehicle_speeds_device: slot / priority / speed are device addresses of n entries each."""
        self._check(self.lib.cfb_set_vehicle_speeds_device(self.h, slot, priority, speed, n, stream))

    def observe_vehicle_context_device(self, stream: int = 0) -> DeviceVehicleContext:
        """Refresh the per-vehicle table with each row's leader, gap, next drivable and light
        (cfb_observe_vehicle_context_device) and return their pointers."""
        o = DeviceVehicleContext()
        self._check(self.lib.cfb_observe_vehicle_context_device(self.h, stream, ctypes.byref(o)))
        return o

    def observe_intersections_device(self, stream: int = 0) -> DeviceIntersectionObs:
        """Refresh the intersection observations (cfb_observe_intersections_device) and return their pointers."""
        o = DeviceIntersectionObs()
        self._check(self.lib.cfb_observe_intersections_device(self.h, stream, ctypes.byref(o)))
        return o

    def road_links(self):
        """cfb_road_link_info of every movement: (intersection, index, type, start road, end road) tuples."""
        out = []
        for r in range(self.lib.cfb_num_road_links(self.h)):
            x = RoadLink()
            self._check(self.lib.cfb_road_link_info(self.h, r, ctypes.byref(x)))
            out.append((x.intersection, x.index, x.type, x.start_road.decode(), x.end_road.decode()))
        return out

    def vehicle_refs(self, slots):
        """cfb_vehicle_refs: REF_DTYPE record per slot, (-1, -1) where the slot holds no vehicle."""
        s = np.ascontiguousarray(slots, np.int32)
        out = np.zeros(len(s), REF_DTYPE)
        self._check(self.lib.cfb_vehicle_refs(self.h, s.ctypes.data, len(s), out.ctypes.data))
        return out

    def drivable_ids(self):
        return [self.lib.cfb_drivable_id(self.h, d).decode() for d in range(self.n_drivables)]

    def snapshot(self) -> "CArchive":
        a = self.lib.cfb_snapshot(self.h)
        if not a:
            raise RuntimeError(self.lib.cfb_last_error(self.h).decode())
        return CArchive(self.lib, a)

    def load(self, archive: "CArchive"):
        self._check(self.lib.cfb_load(self.h, archive.h))


class CArchive:
    """A cfb_snapshot image, freed with the object."""

    def __init__(self, lib, h):
        self.lib, self.h = lib, h

    def close(self):
        if getattr(self, "h", None):
            self.lib.cfb_archive_destroy(self.h)
            self.h = None

    __del__ = close


class CShardGroup:
    """`world` ranks of one simulation on ONE GPU (loop-back exchanges): checks the seam protocol.  `owners`: the rank of
    every intersection (virtual ones included), for a cut other than column strips."""

    def _library(self) -> ctypes.CDLL:
        return load_library()

    def __init__(self, config: str, world: int, owners=None, device: int = 0):
        self.lib = self._library()
        if owners is None:
            self.h = self.lib.cfb_shard_group_create(config.encode(), world, device)
        else:
            owners = np.ascontiguousarray(owners, np.int32)
            self.h = self.lib.cfb_debug_shard_group_create_cut(config.encode(), world, device, owners.ctypes.data)
        if not self.h:
            raise RuntimeError("cfb_shard_group_create failed: %s" % self.lib.cfb_last_error(None).decode())
        self.world = world

    def close(self):
        if getattr(self, "h", None):
            self.lib.cfb_shard_group_destroy(self.h)
            self.h = None

    __del__ = close

    def next_step(self, n: int = 1):
        if self.lib.cfb_shard_group_step(self.h, n) < 0:
            raise RuntimeError(self.lib.cfb_shard_group_last_error(self.h).decode())

    def vehicle_count(self) -> int:
        return int(self.lib.cfb_shard_group_vehicle_count(self.h))

    def lane_counts(self, n_lanes: int, waiting: bool = False):
        a = np.zeros(n_lanes, np.int32)
        rc = self.lib.cfb_shard_group_lane_counts(self.h, a.ctypes.data, n_lanes, int(waiting))
        assert rc == 0
        return a

    def counters(self):
        """(vehicle steps, ties) summed over the ranks"""
        a = np.zeros(2, np.int64)
        if self.lib.cfb_shard_group_counters(self.h, a.ctypes.data) < 0:
            raise RuntimeError(self.lib.cfb_shard_group_last_error(self.h).decode())
        return int(a[0]), int(a[1])

    def debug_vehicles(self):
        n = int(self.lib.cfb_shard_group_debug_vehicles(self.h, None, 0))
        a = np.zeros(n, VEH_DTYPE)
        if n:
            self.lib.cfb_shard_group_debug_vehicles(self.h, a.ctypes.data, n)
        return a


class CReplay:
    """The replay formatter on its own (cfb_replay_*): needs the roadnet file only, no GPU."""

    def __init__(self, roadnet_file: str):
        self.lib = load_library()
        self.h = self.lib.cfb_replay_create(roadnet_file.encode())
        if not self.h:
            raise RuntimeError("cfb_replay_create failed: %s" % self.lib.cfb_last_error(None).decode())

    def close(self):
        if getattr(self, "h", None):
            self.lib.cfb_replay_destroy(self.h)
            self.h = None

    __del__ = close

    def roadnet_json(self) -> str:
        n = int(self.lib.cfb_replay_roadnet_json(self.h, None, 0))
        buf = ctypes.create_string_buffer(n)
        self.lib.cfb_replay_roadnet_json(self.h, buf, n)
        return buf.value.decode()

    def format_step(self, vehicles: np.ndarray, phases: np.ndarray) -> str:
        v = np.ascontiguousarray(vehicles, REPLAY_DTYPE)
        ph = np.ascontiguousarray(phases, np.int32)
        n = int(self.lib.cfb_replay_format_step(self.h, v.ctypes.data, len(v), ph.ctypes.data, None, 0))
        buf = ctypes.create_string_buffer(n)
        self.lib.cfb_replay_format_step(self.h, v.ctypes.data, len(v), ph.ctypes.data, buf, n)
        return buf.value.decode()

    def format_step_lc(self, vehicles: np.ndarray, phases: np.ndarray) -> str:
        """format_step with lane change (cfb_replay_format_step_lc): REPLAY_LC_DTYPE records."""
        v = np.ascontiguousarray(vehicles, REPLAY_LC_DTYPE)
        ph = np.ascontiguousarray(phases, np.int32)
        n = int(self.lib.cfb_replay_format_step_lc(self.h, v.ctypes.data, len(v), ph.ctypes.data, None, 0))
        buf = ctypes.create_string_buffer(n)
        self.lib.cfb_replay_format_step_lc(self.h, v.ctypes.data, len(v), ph.ctypes.data, buf, n)
        return buf.value.decode()
