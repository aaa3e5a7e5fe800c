"""The per-vehicle observation table and the batched custom speed (cfb_observe_vehicles_device,
cfb_set_vehicle_speeds_device, cfb_vehicle_refs) through the C-ABI over the emulated device: the kernel bodies of
csrc/device_vehobs.cuh on the emulated warp (tests/device_sim_emu_vehobs.cpp), under the real host engine.  The emulated
device's "device memory" is host memory, so the returned pointers are read with numpy and the actions are passed as
numpy arrays."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from test_cpu import _HAVE_CUDA_SDK

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

pytestmark = pytest.mark.skipif(not _HAVE_CUDA_SDK, reason="needs the CUDA headers and libcudart to build the host-check library")

SHADOW = 1 << 24   # capi.REF_SHADOW_SHIFT


@pytest.fixture(autouse=True)
def _emulated(monkeypatch):
    monkeypatch.setenv("CFB_EMULATED_DEVICE_FOR_TESTS", "1")


def _vehobs_lib():
    """oracle/_build/libcfb_hostcheck_vehobs.so: the host engine and C-ABI (csrc/host_engine.cpp) over the emulated device with the per-vehicle entry points (tests/device_sim_emu_vehobs.cpp).  Test infrastructure,
    built like test_cpu.py's host-check library."""
    os.makedirs(os.path.join(ROOT, "oracle", "_build"), exist_ok=True)
    lib = os.path.join(ROOT, "oracle", "_build", "libcfb_hostcheck_vehobs.so")
    csrc = os.path.join(ROOT, "cityflow_b200", "csrc")
    tests = os.path.join(ROOT, "tests")
    srcs = [os.path.join(tests, "device_sim_emu_vehobs.cpp")] + [os.path.join(csrc, f) for f in
            ("host_engine.cpp", "roadnet.cpp", "flows.cpp", "partition.cpp", "shard.cpp", "replay.cpp", "json_write.cpp")]
    deps = srcs + [os.path.join(csrc, f) for f in os.listdir(csrc) if f.endswith((".cuh", ".h"))] + \
        [os.path.join(tests, f) for f in ("device_emu.h", "device_hostsim.h", "device_sim_emu.cpp")]
    if not os.path.exists(lib) or os.path.getmtime(lib) < max(os.path.getmtime(f) for f in deps):
        subprocess.check_call(["g++", "-std=c++17", "-O1", "-fPIC", "-shared", "-ffp-contract=off", "-I/usr/local/cuda/include",
                               "-I" + csrc, "-I" + tests, "-I" + os.path.join(ROOT, "include")] + srcs +
                              ["-L/usr/local/cuda/lib64", "-lcudart", "-ldl", "-o", lib])
    return lib


def _emulated_engine(cfg):
    from cityflow_b200 import capi
    path = _vehobs_lib()

    class EmulatedEngine(capi.CEngine):
        def _library(self):
            return capi.bind(ctypes.CDLL(path))

    return EmulatedEngine(cfg, 0)


def _host(ptr, n, ctype):
    return np.ctypeslib.as_array((ctype * max(n, 1)).from_address(ptr))[:n].copy()


def _table(eng):
    """The refreshed table as numpy columns (rows in use only) + the padding check."""
    o = eng.observe_vehicles_device()
    n = int(_host(o.count, 1, ctypes.c_int32)[0])
    cap = o.capacity
    slot = _host(o.slot, cap, ctypes.c_int32)
    assert 0 <= n <= cap and (slot[n:] == -1).all()
    t = dict(slot=slot[:n], priority=_host(o.priority, n, ctypes.c_int32), drivable=_host(o.drivable, n, ctypes.c_int32),
             distance=_host(o.distance, n, ctypes.c_double), speed=_host(o.speed, n, ctypes.c_double),
             shadow=_host(o.shadow, n, ctypes.c_uint8), begin=_host(o.drivable_begin, o.n_drivables + 1, ctypes.c_int32))
    assert o.n_drivables == eng.n_drivables and t["begin"][-1] == n
    return t


def _lane_vehicles(eng):
    beg = np.zeros(eng.n_lanes + 1, np.int64)
    from cityflow_b200.capi import REF_DTYPE
    n = eng._check(eng.lib.cfb_get_lane_vehicles(eng.h, beg.ctypes.data, eng.n_lanes + 1, None, 0))
    ids = np.zeros(n, REF_DTYPE)
    eng._check(eng.lib.cfb_get_lane_vehicles(eng.h, beg.ctypes.data, eng.n_lanes + 1, ids.ctypes.data, n))
    return beg, ids


def _check_table(eng, lane_change):
    """Every semantic the table promises, against the host getters of the same engine."""
    t = _table(eng)
    n = len(t["slot"])
    assert n == eng.vehicle_count()
    assert (np.diff(t["begin"]) >= 0).all()
    assert (t["drivable"] == np.repeat(np.arange(eng.n_drivables), np.diff(t["begin"]))).all()
    refs = eng.vehicle_refs(t["slot"])
    assert (refs["flow"] != -1).all()
    # lanes: exactly get_lane_vehicles, names and order, shadows included
    beg, ids = _lane_vehicles(eng)
    nl = eng.n_lanes
    assert (t["begin"][:nl + 1] == beg).all()
    assert (refs[:beg[-1]] == ids).all()
    # shadows: named "<id>_shadow" while they change lanes, never without lane change
    assert ((refs["index"] >= SHADOW) == (t["shadow"] == 1)).all()
    if not lane_change:
        assert not t["shadow"].any()
    # the real vehicles in priority order: get_vehicles / get_vehicle_speed, bit for bit
    real = t["shadow"] == 0
    order = np.argsort(t["priority"][real], kind="stable")
    vids, sp, ds = eng.vehicle_speed()
    assert (refs[real][order] == vids).all()
    assert (t["speed"][real][order].view(np.int64) == sp.view(np.int64)).all()
    assert (t["distance"][real][order].view(np.int64) == ds.view(np.int64)).all()
    # laneLinks too: every running vehicle's full record
    if lane_change:
        lc = _lc_vehicles(eng)
        o = np.argsort(t["priority"], kind="stable")
        assert (lc["priority"] == t["priority"][o]).all() and (lc["drivable"] == t["drivable"][o]).all()
        assert (lc["dis"] == t["distance"][o]).all() and (lc["speed"] == t["speed"][o]).all()
        assert ((lc["partner_type"] == 2) == (t["shadow"][o] == 1)).all()
    else:
        dbg = eng.debug_vehicles()
        assert (dbg["priority"] == t["priority"]).all() and (dbg["drivable"] == t["drivable"]).all()
        assert (dbg["dis"] == t["distance"]).all() and (dbg["speed"] == t["speed"]).all()
        assert (dbg["flow"] == refs["flow"]).all() and (dbg["cnt"] == refs["index"]).all()
    return t


def _lc_vehicles(eng):
    from oracle.harness import LC_DTYPE
    n = eng._check(eng.lib.cfb_debug_lc_vehicles(eng.h, None, 0))
    a = np.zeros(n, LC_DTYPE)
    if n:
        eng._check(eng.lib.cfb_debug_lc_vehicles(eng.h, a.ctypes.data, n))
    return a


def _dense_3x3(directory, lane_change):
    from cityflow_b200 import scenario
    return scenario.make_grid_scenario(directory, 3, 3, dense=dict(frac=1.0, interval=3.0, seed=3), name="vo33",
                                       lane_change=lane_change)


def _fuzzed(directory, lane_change, seed=7):
    import randnet
    from cityflow_b200 import scenario
    net = randnet.random_roadnet(seed, rows=2 + seed % 3, cols=3 + seed % 2)
    flows = randnet.random_flows(net, seed + 100, n_flows=40 + seed % 50)
    return scenario.write_scenario(directory, net, flows, seed=seed, interval=1.0, lane_change=lane_change, name="vof%d" % seed)


@pytest.mark.parametrize("lane_change", [False, True])
@pytest.mark.parametrize("net", ["dense_3x3", "fuzzed"])
def test_vehicle_table_every_step(net, lane_change, tmp_path):
    """The table against get_lane_vehicles, get_vehicle_speed / _distance, get_vehicles and the debug records, every
    step of 150, with and without lane change."""
    cfg = (_dense_3x3 if net == "dense_3x3" else _fuzzed)(str(tmp_path), lane_change)
    eng = _emulated_engine(cfg)
    ids = [eng.lib.cfb_drivable_id(eng.h, d).decode() for d in range(eng.n_drivables)]
    assert ids[:eng.n_lanes] == eng.lane_ids() and all("_TO_" in i for i in ids[eng.n_lanes:])
    assert eng.lib.cfb_drivable_id(eng.h, eng.n_drivables) is None
    rows = links = shadows = 0
    for _ in range(150):
        eng.next_step()
        t = _check_table(eng, lane_change)
        rows += len(t["slot"])
        links += int((t["drivable"] >= eng.n_lanes).sum())
        shadows += int(t["shadow"].sum())
    assert rows > 3000 and links > 200, (rows, links)
    assert (shadows > 20) == lane_change, shadows


def test_vehicle_table_of_an_empty_network_and_a_long_queue(tmp_path):
    """Before the first step the table is empty (count 0, all padding); on edgenet's long_queue a lane holds more than
    32 vehicles (the warp's bucket loop), and the rows the queue leaves behind go back to padding."""
    import edgenet
    eng = _emulated_engine(edgenet.write("long_queue", str(tmp_path)))
    t = _table(eng)
    assert len(t["slot"]) == 0 and (t["begin"] == 0).all()
    most = 0
    for _ in range(400):
        eng.next_step()
        t = _table(eng)
        most = max(most, int(np.diff(t["begin"]).max()))
        assert len(t["slot"]) == eng.vehicle_count()
    assert most > 32, most
    _check_table(eng, False)


def _same_state(a, b, lane_change):
    if lane_change:
        x, y = _lc_vehicles(a), _lc_vehicles(b)
    else:
        x, y = a.debug_vehicles(), b.debug_vehicles()
    assert x.tobytes() == y.tobytes()


def _act(dev, host, rng, extra_host=0):
    """One random action on both engines: `host` through cfb_set_vehicle_speed per id, `dev` through one
    cfb_set_vehicle_speeds_device call with padded columns (slot -1 entries mixed in).  `extra_host` vehicles first get
    a host-side request on both engines, which the device call then overrides for some of them."""
    t = _table(dev)
    n = len(t["slot"])
    if n == 0:
        return 0
    refs = dev.vehicle_refs(t["slot"])
    pick = rng.choice(n, size=rng.integers(1, n + 1), replace=False)
    speed = rng.uniform(0.0, 15.0, len(pick))
    for k in rng.choice(n, size=min(extra_host, n), replace=False):
        for e in (dev, host):
            assert e.set_vehicle_speed(int(refs["flow"][k]), int(refs["index"][k]), 3.5)
    for k, v in zip(pick, speed):
        assert host.set_vehicle_speed(int(refs["flow"][k]), int(refs["index"][k]), float(v))
    slot = np.concatenate([t["slot"][pick], [-1, -1]]).astype(np.int32)
    prio = np.concatenate([t["priority"][pick], [0, 7]]).astype(np.int32)
    spd = np.concatenate([speed, [1.0, 2.0]])
    perm = rng.permutation(len(slot))
    slot, prio, spd = slot[perm].copy(), prio[perm].copy(), spd[perm].copy()
    dev.set_vehicle_speeds_device(slot.ctypes.data, prio.ctypes.data, spd.ctypes.data, len(slot))
    return len(pick)


@pytest.mark.parametrize("lane_change", [False, True])
def test_batched_speed_equals_per_vehicle_calls(lane_change, tmp_path):
    """Two engines in lock step over 200 steps: one gets set_vehicle_speed per id, the other one
    set_vehicle_speeds_device call with the same vehicles and speeds every few steps, sometimes on top of host-side
    requests for the same vehicles in the same step.  Every vehicle's full state is equal after every step."""
    cfg = _dense_3x3(str(tmp_path), lane_change)
    dev, host = _emulated_engine(cfg), _emulated_engine(cfg)
    rng = np.random.default_rng(11)
    acted = 0
    for s in range(200):
        if s % 3 == 2:
            acted += _act(dev, host, rng, extra_host=3 if s % 2 else 0)
        dev.next_step()
        host.next_step()
        assert dev.vehicle_count() == host.vehicle_count()
        _same_state(dev, host, lane_change)
    assert acted > 1000, acted


def test_stale_handle_and_duplicate_slot_are_refused(tmp_path):
    """Handles of vehicles that have left, a priority that does not match the slot's vehicle, a slot outside the slot
    table and a slot named twice in one call each raise a RuntimeError at the next synchronising call; the ids of slots
    whose vehicle left are no longer that vehicle's."""
    cfg = _dense_3x3(str(tmp_path), False)
    eng = _emulated_engine(cfg)
    eng.next_step(30)
    old = _table(eng)
    old_refs = eng.vehicle_refs(old["slot"])
    eng.next_step(120)
    left = ~np.isin(old["slot"], _table(eng)["slot"])
    assert left.sum() > 5
    assert (eng.vehicle_refs(old["slot"][left]) != old_refs[left]).all()
    assert (eng.vehicle_refs([1 << 30, -5])["flow"] == -1).all()
    cases = {"left": ("Vehicle not found", lambda s, p: (old["slot"][left], old["priority"][left])),
             "priority": ("Vehicle not found", lambda s, p: ([s[0]], [p[0] + 1])),
             "outside": ("Vehicle not found", lambda s, p: ([1 << 30], [p[0]])),
             "twice": ("twice", lambda s, p: ([s[0], s[1], s[0]], [p[0], p[1], p[0]]))}
    for name, (msg, make) in cases.items():
        eng = _emulated_engine(cfg)
        eng.next_step(150)
        t = _table(eng)
        slot, prio = (np.ascontiguousarray(x, np.int32) for x in make(t["slot"], t["priority"]))
        spd = np.full(len(slot), 5.0)
        eng.set_vehicle_speeds_device(slot.ctypes.data, prio.ctypes.data, spd.ctypes.data, len(slot))
        with pytest.raises(RuntimeError, match=msg):
            eng.vehicle_count()
