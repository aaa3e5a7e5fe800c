"""IntersectionObservations on the GPU, through the public Python surface: every column against the restatement of
tests/test_cpu_intersection_obs.py (the roadnet JSON plus the dict getters of the same engine), zero copy, stream
ordering, pending set_tl_phase calls, and MaxPressure run on the device in lock step with MaxPressure run from the
dicts, in the default launch form (graph + PDL) and without graphs."""
import json
import tempfile

import numpy as np
import pytest

from test_cpu_intersection_obs import INT32_MIN, Restatement

pytestmark = pytest.mark.gpu

_COLUMNS = ("phase", "phase_remaining", "pressure", "queue", "movement_in", "movement_in_waiting", "movement_out",
            "movement_inside", "movement_pressure", "phase_pressure", "movement_begin", "movement_intersection",
            "phase_count", "phase_movements")


def _engine(cfg):
    import cityflow
    return cityflow.Engine(cfg, thread_num=1)


def _grid(rows, cols, name, **kw):
    from cityflow_b200 import scenario
    return scenario.make_grid_scenario(tempfile.mkdtemp(), rows, cols, name=name, **kw)


def _lanes(eng, d):
    return np.array([d[l] for l in eng.lane_ids()], np.int64)


def _check(eng, obs, vobs, R, phases=True):
    """Refresh both tables and compare every dynamic column with the restatement."""
    obs.refresh()
    vobs.refresh()
    count, waiting = _lanes(eng, eng.get_lane_vehicle_count()), _lanes(eng, eng.get_lane_waiting_vehicle_count())
    drv = np.diff(vobs.drivable_begin.cpu().numpy())
    assert (drv[:len(count)] == count).all()
    for k, v in R.movement_columns(count, waiting, drv).items():
        assert (getattr(obs, k).cpu().numpy() == v).all(), k
    pressure, queue = R.intersection_columns(count, waiting)
    assert (obs.pressure.cpu().numpy() == pressure).all() and (obs.queue.cpu().numpy() == queue).all()
    assert (obs.phase_pressure.cpu().numpy() == R.phase_pressure(count)).all()
    if phases:
        assert (obs.phase.cpu().numpy() == [-1 if v else c for v, c in zip(R.virtual, R.cur)]).all()
        assert (obs.phase_remaining.cpu().numpy().view(np.int64) == np.array(R.remain).view(np.int64)).all()
    return int(obs.queue.sum().item())


def _check_static(eng, obs, R):
    assert (obs.movement_begin.cpu().numpy() == R.begin).all()
    assert (obs.movement_intersection.cpu().numpy() == [m[0] for m in R.mv]).all()
    assert (obs.phase_count.cpu().numpy() == [len(p) for p in R.phases]).all()
    types = {1: "turn_right", 2: "turn_left", 3: "go_straight"}
    assert obs.road_links == [dict(intersection=R.ids[m[0]], index=m[1], start_road=m[3], end_road=m[4], type=types[m[2]])
                              for m in R.mv]
    pm = obs.phase_movements.cpu().numpy()
    for k, ph in enumerate(R.phases):
        for p, (_, avail) in enumerate(ph):
            assert sorted(np.flatnonzero(pm[k, p])) == sorted(avail)


def _check_dump(eng, obs, R, path):
    import cityflow_b200
    cityflow_b200.Archive(eng).dump(path)
    tl = json.load(open(path))["trafficLights"]
    ph, rem = obs.phase.cpu().numpy(), obs.phase_remaining.cpu().numpy()
    for k, i in enumerate(R.ids):
        if not R.virtual[k]:
            assert ph[k] == tl[i]["curPhaseIndex"] and rem[k].tobytes() == np.float64(tl[i]["remainDuration"]).tobytes()


def _irregular():
    import conftest
    from cityflow_b200 import scenario
    net = conftest._irregular_net()
    return scenario.write_scenario(tempfile.mkdtemp(), net, scenario.random_walk_flows(net, frac=1.0, interval=4.0, seed=9),
                                   seed=7, name="gioirr")


@pytest.mark.parametrize("net", ["dense_6x6", "irregular", "lane_change"])
def test_table_every_step(net, cfg_6x6_dense, tmp_path):
    import cityflow_b200
    cfg = {"dense_6x6": lambda: cfg_6x6_dense, "irregular": _irregular,
           "lane_change": lambda: _grid(4, 4, "giolc", dense=dict(frac=1.0, interval=2.0, seed=7), lane_change=True)}[net]()
    eng = _engine(cfg)
    R = Restatement(cfg)
    obs, vobs = cityflow_b200.IntersectionObservations(eng), cityflow_b200.VehicleObservations(eng)
    _check_static(eng, obs, R)
    ptrs = [getattr(obs, k).data_ptr() for k in _COLUMNS]
    queued = 0
    for s in range(300):
        eng.next_step()
        R.pass_time()
        queued += _check(eng, obs, vobs, R)
        if net != "lane_change" and s % 100 == 99:
            _check_dump(eng, obs, R, str(tmp_path / "x.json"))
    assert queued > 1000, queued
    assert ptrs == [getattr(obs, k).data_ptr() for k in _COLUMNS]


def test_table_at_the_bench_operating_point():
    """30x30 grid after bench.py's prefill and warm-up, checked at a few step counts past 1200; a refresh ordered on a
    side stream feeds a reduction on that stream with no host wait in between."""
    import torch
    import cityflow_b200
    cfg = _grid(30, 30, "giobench", dense=dict(frac=0.5, interval=10.0, seed=1, fleet_spread=0.02))
    eng = _engine(cfg)
    R = Restatement(cfg)
    eng.next_steps(1200)
    for _ in range(1200):
        R.pass_time()
    obs, vobs = cityflow_b200.IntersectionObservations(eng), cityflow_b200.VehicleObservations(eng)
    _check_static(eng, obs, R)
    ptrs = [getattr(obs, k).data_ptr() for k in _COLUMNS]
    for n in (1, 4, 45):
        eng.next_steps(n)
        for _ in range(n):
            R.pass_time()
        assert _check(eng, obs, vobs, R) > 1000
    side = torch.cuda.Stream()
    for _ in range(5):
        eng.next_step()
        R.pass_time()
        obs.refresh(stream=side)
        with torch.cuda.stream(side):
            total = obs.movement_in.sum() + obs.movement_inside.sum()
            best = obs.phase_pressure.max(1).values
        side.synchronize()
        count = _lanes(eng, eng.get_lane_vehicle_count())
        want = R.movement_columns(count, count, np.diff(vobs.refresh().drivable_begin.cpu().numpy()))
        assert int(total.item()) == int(want["movement_in"].sum() + want["movement_inside"].sum())
        assert (best.cpu().numpy() == R.phase_pressure(count).max(1)).all()
    assert ptrs == [getattr(obs, k).data_ptr() for k in _COLUMNS]


def test_pending_phases_show_in_the_next_refresh(cfg_6x6_rl):
    """set_tl_phase then refresh; set_tl_phases_tensor then set_tl_phase then refresh; and many refreshes each after one
    more set_tl_phase (each flush stages its own copy): every refresh shows every call made before it."""
    import torch
    import cityflow_b200
    eng = _engine(cfg_6x6_rl)
    R = Restatement(cfg_6x6_rl)
    ids = eng.intersection_ids()
    real = [k for k, v in enumerate(R.virtual) if not v]
    eng.next_steps(30)
    obs = cityflow_b200.IntersectionObservations(eng)
    want = torch.zeros(len(ids), dtype=torch.int32)
    for k in real:
        want[k] = (k * 5 + 3) % len(R.phases[k])
        eng.set_tl_phase(ids[k], int(want[k]))
    obs.refresh()
    assert (obs.phase.cpu()[real] == want[real]).all()
    dev = ((want + 1) % 4).cuda()
    cityflow_b200.set_tl_phases_tensor(eng, dev)
    eng.set_tl_phase(ids[real[0]], 2)
    obs.refresh()
    expect = dev.cpu().clone()
    expect[real[0]] = 2
    assert (obs.phase.cpu()[real] == expect[real]).all()
    for n in range(200):   # more refreshes than the staging ring holds, without a step in between
        k = real[n % len(real)]
        expect[k] = n % len(R.phases[k])
        eng.set_tl_phase(ids[k], int(expect[k]))
        obs.refresh()
        assert int(obs.phase[k].item()) == int(expect[k])
    assert (obs.phase.cpu()[real] == expect[real]).all()
    eng.next_step()
    obs.refresh()
    assert (obs.phase.cpu()[real] == expect[real]).all()
    eng.reset()
    obs.refresh()
    assert not obs.phase.cpu()[real].any() and not obs.movement_in.any()
    assert (obs.phase.cpu()[[k for k in range(len(ids)) if R.virtual[k]]] == -1).all()


@pytest.mark.parametrize("form", ["default", "no_graph"])
def test_max_pressure_lock_step(form, cfg_6x6_rl, monkeypatch):
    """Engine A: get_lane_vehicle_count + MaxPressure in Python + set_tl_phase per light.  Engine B: refresh +
    phase_pressure.argmax (the first maximum, as the Python side takes) + set_tl_phases_tensor.  Equal phases and
    equal state every step for 400 steps; equal JSON archives every 50."""
    import torch
    import cityflow_b200
    if form == "no_graph":
        monkeypatch.setenv("CITYFLOW_B200_NO_GRAPH", "1")
    a, b = _engine(cfg_6x6_rl), _engine(cfg_6x6_rl)
    R = Restatement(cfg_6x6_rl)
    ids = a.intersection_ids()
    real = [k for k, v in enumerate(R.virtual) if not v]
    obs = cityflow_b200.IntersectionObservations(b)
    changes, prev = 0, None
    with tempfile.TemporaryDirectory() as d:
        for s in range(400):
            act_a = R.max_pressure(_lanes(a, a.get_lane_vehicle_count()))
            for k in real:
                a.set_tl_phase(ids[k], act_a[k])
            obs.refresh()
            act_b = obs.phase_pressure.argmax(1).to(torch.int32)
            cityflow_b200.set_tl_phases_tensor(b, act_b)
            got = act_b.cpu().tolist()
            assert [got[k] for k in real] == [act_a[k] for k in real], "step %d" % s
            changes += prev is not None and got != prev
            prev = got
            a.next_step()
            b.next_step()
            assert a.get_vehicle_speed() == b.get_vehicle_speed() and a.get_lane_vehicles() == b.get_lane_vehicles(), s
            assert a.get_vehicle_distance() == b.get_vehicle_distance(), "step %d" % s
            if s % 50 == 49:   # every vehicle's full state and every light, decoded (the binary image also holds the
                #                work lists in atomics order, which two equal engines need not share)
                cityflow_b200.Archive(a).dump(d + "/a.json")
                cityflow_b200.Archive(b).dump(d + "/b.json")
                assert open(d + "/a.json", "rb").read() == open(d + "/b.json", "rb").read(), "step %d" % s
    assert changes > 50, changes
    assert (obs.phase_pressure[[k for k in range(len(ids)) if R.virtual[k]]] == INT32_MIN).all()
