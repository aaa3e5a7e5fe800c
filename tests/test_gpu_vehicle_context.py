"""What lies ahead of every vehicle on the GPU (VehicleObservations(context=True), cfb_observe_vehicle_context_device):
leader, gap, next drivable and light of every row against the compiled reference and the engine's debug records, at the
30x30 bench point against the debug records and the IntersectionObservations join, and through the public Python
surface: zero copy, side-stream ordering, the default launch form and CITYFLOW_B200_NO_GRAPH=1."""
import ctypes
import tempfile

import numpy as np
import pytest

import test_cpu_vehicle_context as C

pytestmark = pytest.mark.gpu

_TYPESTR = {ctypes.c_int32: "<i4", ctypes.c_double: "<f8", ctypes.c_int8: "|i1", ctypes.c_uint8: "|u1"}


def _engine(cfg):
    """The C-ABI engine, whose pointers are device memory: `read` copies them down after the engine's work."""
    import torch
    import cityflow_b200
    from cityflow_b200.capi import CEngine

    class DeviceEngine(CEngine):
        def read(self, ptr, n, ctype):
            if n == 0:
                return np.zeros(0, np.dtype(_TYPESTR[ctype]))
            torch.cuda.synchronize()
            return torch.as_tensor(cityflow_b200._DeviceArray(self, ptr, n, _TYPESTR[ctype]), device="cuda").cpu().numpy()

    return DeviceEngine(cfg, 0)


def _run_against_reference(cfg, steps, lane_change, tmp):
    if not C._have_ref(lane_change):
        pytest.skip("the compiled reference (oracle/_ref) is not built")
    eng = _engine(cfg)
    states, ctxs = C.reference(cfg, steps, lane_change, eng.n_inter, eng.n_drivables, tmp)
    t = C.context(eng)
    C.check_static(eng, cfg)
    seen = {}
    for s in range(1, steps + 1):
        eng.next_step()
        t2 = C.context(eng)
        assert t2["ptrs"] == t["ptrs"]
        t = t2
        for k, x in C.check_self(eng, t, lane_change).items():
            seen[k] = seen.get(k, 0) + x
        C.check_reference(t, states[s], ctxs[s], lane_change)
    return seen


def test_context_on_the_6x6_dense_grid_against_the_reference(cfg_6x6_dense, tmp_path):
    seen = _run_against_reference(cfg_6x6_dense, 300, False, str(tmp_path))
    assert seen["leaders"] > 20000 and seen["cross"] > 1000 and seen["green"] > 1000 and seen["red"] > 1000, seen


def test_context_with_lane_change_against_the_priority_ordered_reference(tmp_path):
    cfg = C._dense_3x3(str(tmp_path), lane_change=True)
    seen = _run_against_reference(cfg, 250, True, str(tmp_path))
    assert seen["leaders"] > 1000 and seen["cross"] > 100, seen


def _movement_light(eng):
    """Per movement: available in its intersection's current phase, from the IntersectionObservations columns
    (phase, movement_begin, movement_intersection, phase_movements)."""
    o = eng.observe_intersections_device()
    ni, nrl, mp, mm = o.n_intersections, o.n_road_links, o.max_phases, o.max_movements
    phase = eng.read(o.phase, ni, ctypes.c_int32)
    beg = eng.read(o.movement_begin, ni + 1, ctypes.c_int32)
    inter = eng.read(o.movement_intersection, nrl, ctypes.c_int32)
    pm = eng.read(o.phase_movements, ni * mp * mm, ctypes.c_uint8).reshape(ni, mp, mm)
    r = np.arange(nrl)
    return pm[inter, phase[inter], r - beg[inter]]


def test_context_at_the_bench_operating_point():
    """30x30 grid after bench.py's prefill (about 1.3e5 rows): leader and gap equal the debug records, and the light
    of every row equals the join of IntersectionObservations' phase and phase_movements over the row's movement."""
    from cityflow_b200 import scenario
    cfg = scenario.make_grid_scenario(tempfile.mkdtemp(), 30, 30, name="vcbench",
                                      dense=dict(frac=0.5, interval=10.0, seed=1, fleet_spread=0.02))
    eng = _engine(cfg)
    eng.next_step(1205)
    for _ in range(3):
        t = C.context(eng)
        n = t["n"]
        assert n > 100000, n
        seen = C.check_self(eng, t, False)
        assert seen["cross"] > 1000 and seen["green"] > 1000 and seen["red"] > 1000, seen
        light = _movement_light(eng)
        heads = (t["drivable"][:n] < eng.n_lanes) & (t["next"][:n] >= eng.n_lanes)
        rl = C.static(eng)["road_link"][t["next"][:n][heads] - eng.n_lanes]
        assert (t["signal"][:n][heads] == light[rl]).all()
        eng.next_step()


@pytest.mark.parametrize("form", ["default", "no_graph"])
def test_public_surface_in_lock_step(form, cfg_6x6_dense, monkeypatch):
    """VehicleObservations(context=True) of a cityflow.Engine against the C-ABI context of a second engine on the same
    scenario: equal columns every step, the tensors keep their storage, a refresh on a side stream orders a reduction
    on that stream, and a plain VehicleObservations on the same engine leaves the context's padding intact."""
    import torch
    import cityflow
    import cityflow_b200
    if form == "no_graph":
        monkeypatch.setenv("CITYFLOW_B200_NO_GRAPH", "1")
    pub = cityflow.Engine(cfg_6x6_dense, thread_num=1)
    ref = _engine(cfg_6x6_dense)
    obs = cityflow_b200.VehicleObservations(pub, context=True)
    plain = cityflow_b200.VehicleObservations(pub)
    assert not hasattr(plain, "leader") and not hasattr(plain, "drivable_length")
    cols = ("slot", "priority", "drivable", "leader", "gap", "next_drivable", "signal", "drivable_begin", "count",
            "drivable_length", "drivable_max_speed", "link_road_link")
    ptrs = [getattr(obs, k).data_ptr() for k in cols]
    assert obs.leader.dtype == torch.int32 and obs.gap.dtype == torch.float64 and obs.signal.dtype == torch.int8
    side = torch.cuda.Stream()
    C.context(ref)
    st = C.static(ref)
    assert (obs.drivable_length.cpu().numpy() == st["length"]).all()
    assert (obs.drivable_max_speed.cpu().numpy() == st["max_speed"]).all()
    assert (obs.link_road_link.cpu().numpy() == st["road_link"]).all() and obs.n_lanes == ref.n_lanes
    for s in range(150):
        pub.next_step()
        ref.next_step()
        if s % 3 == 0:
            plain.refresh()
        obs.refresh(stream=side)
        with torch.cuda.stream(side):
            led = (obs.leader >= 0).sum()
            green = (obs.signal == 1).sum()
        t = C.context(ref)
        side.synchronize()
        n = t["n"]
        assert int(led.item()) == int((t["leader"] >= 0).sum()) and int(green.item()) == int((t["signal"] == 1).sum())
        assert int(obs.count.item()) == n
        for k, ck in (("slot", "slot"), ("leader", "leader"), ("next_drivable", "next"), ("signal", "signal")):
            assert (getattr(obs, k).cpu().numpy() == t[ck]).all(), (s, k)
        assert obs.gap.cpu().numpy().tobytes() == t["gap"].tobytes()
    assert ptrs == [getattr(obs, k).data_ptr() for k in cols]
    assert int(obs.count.item()) > 500
