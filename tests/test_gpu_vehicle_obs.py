"""VehicleObservations and set_vehicle_speeds_tensor on the GPU, through the public Python surface: the table against
the dict getters of the same engine, zero copy, stream ordering, and the batched custom speed in lock step with an
engine that gets the same speeds through set_vehicle_speed, in the default launch form (graph + PDL) and without graphs."""
import math
import tempfile

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _engine(cfg):
    import cityflow
    return cityflow.Engine(cfg, thread_num=1)


def _rows(obs):
    """(n, slot, priority, drivable, distance, speed, shadow, drivable_begin) on the host, after a refresh."""
    n = int(obs.count.item())
    slot = obs.slot.cpu().numpy()
    assert (slot[n:] == -1).all()
    cols = [c.cpu().numpy()[:n] for c in (obs.priority, obs.drivable, obs.distance, obs.speed, obs.shadow)]
    return [n, slot[:n]] + cols + [obs.drivable_begin.cpu().numpy()]


def _check(eng, obs, lane_change=False):
    obs.refresh()
    n, slot, prio, drv, dist, speed, shadow, beg = _rows(obs)
    assert n == eng.get_vehicle_count() and beg[-1] == n
    assert (drv == np.repeat(np.arange(len(beg) - 1), np.diff(beg))).all()
    names = obs.vehicle_ids(slot)
    assert None not in names
    lanes = eng.get_lane_vehicles()
    for l, lid in enumerate(eng.lane_ids()):
        assert names[beg[l]:beg[l + 1]] == lanes[lid], lid
    assert [nm.endswith("_shadow") for nm in names] == [bool(s) for s in shadow]
    assert lane_change or not shadow.any()
    real = np.flatnonzero(shadow == 0)
    real = real[np.argsort(prio[real], kind="stable")]
    assert [names[i] for i in real] == eng.get_vehicles()
    sp, ds = eng.get_vehicle_speed(), eng.get_vehicle_distance()
    assert all(sp[names[i]] == speed[i] and ds[names[i]] == dist[i] for i in real)
    return n, int((drv >= len(eng.lane_ids())).sum()), int(shadow.sum())


def _grid(rows, cols, name, **kw):
    from cityflow_b200 import scenario
    d = tempfile.mkdtemp()
    return scenario.make_grid_scenario(d, rows, cols, name=name, **kw)


def test_vehicle_table_on_a_dense_grid_every_step(cfg_6x6_dense):
    import cityflow_b200
    eng = _engine(cfg_6x6_dense)
    obs = cityflow_b200.VehicleObservations(eng)
    assert obs.drivable_ids[:len(eng.lane_ids())] == eng.lane_ids()
    assert int(obs.count.item()) == 0 and (obs.slot == -1).all()
    rows = links = 0
    for _ in range(300):
        eng.next_step()
        n, k, _ = _check(eng, obs)
        rows += n
        links += k
    assert rows > 50000 and links > 1000, (rows, links)


def test_vehicle_table_with_lane_change():
    import cityflow_b200
    eng = _engine(_grid(4, 4, "vlc", dense=dict(frac=1.0, interval=2.0, seed=7), lane_change=True))
    obs = cityflow_b200.VehicleObservations(eng)
    shadows = 0
    for _ in range(300):
        eng.next_step()
        shadows += _check(eng, obs, lane_change=True)[2]
    assert shadows > 50, shadows


def test_vehicle_table_at_the_bench_operating_point():
    """30x30 grid after bench.py's prefill and warm-up (about 1.3e5 rows, ~170 tiles of the cross-block scan); the
    storage stays the same across refreshes and a refresh on a side stream orders a reduction on that stream."""
    import torch
    import cityflow_b200
    eng = _engine(_grid(30, 30, "vbench", dense=dict(frac=0.5, interval=10.0, seed=1, fleet_spread=0.02)))
    for _ in range(1205):
        eng.next_step()
    obs = cityflow_b200.VehicleObservations(eng)
    ptrs = [t.data_ptr() for t in (obs.slot, obs.priority, obs.drivable, obs.distance, obs.speed, obs.shadow,
                                   obs.drivable_begin, obs.count)]
    n = _check(eng, obs)[0]
    assert n > 100000, n
    side = torch.cuda.Stream()
    for _ in range(5):
        eng.next_step()
        obs.refresh(stream=side)
        with torch.cuda.stream(side):
            live = obs.slot >= 0
            cnt = live.sum()
            tot = torch.where(live, obs.speed, torch.zeros_like(obs.speed)).sum()
        side.synchronize()
        sp = eng.get_vehicle_speed()
        assert int(cnt.item()) == eng.get_vehicle_count()
        assert math.isclose(float(tot.item()), math.fsum(sp.values()), rel_tol=1e-9)
    assert ptrs == [t.data_ptr() for t in (obs.slot, obs.priority, obs.drivable, obs.distance, obs.speed, obs.shadow,
                                           obs.drivable_begin, obs.count)]


def _state(eng):
    return eng.get_vehicle_speed(), eng.get_vehicle_distance(), eng.get_lane_vehicles(), eng.get_vehicle_count()


@pytest.mark.parametrize("form", ["default", "no_graph"])
def test_batched_speed_in_lock_step_with_per_vehicle_calls(form, cfg_6x6_dense, monkeypatch):
    """Engine A gets set_vehicle_speed per id, engine B one set_vehicle_speeds_tensor call with the same random subset
    and speeds every third step (on top of host-side requests for some of the same vehicles); equal states every step."""
    import torch
    import cityflow_b200
    if form == "no_graph":
        monkeypatch.setenv("CITYFLOW_B200_NO_GRAPH", "1")
    a, b = _engine(cfg_6x6_dense), _engine(cfg_6x6_dense)
    obs = cityflow_b200.VehicleObservations(b)
    g = torch.Generator(device="cuda").manual_seed(3)
    acted = 0
    for s in range(200):
        if s % 3 == 2:
            obs.refresh()
            n = int(obs.count.item())
            if n:
                pick = torch.randperm(n, device="cuda", generator=g)[:max(1, n // 3)]
                speed = torch.rand(len(pick), device="cuda", dtype=torch.float64, generator=g) * 15
                slot, prio = obs.slot[pick].contiguous(), obs.priority[pick].contiguous()
                names = obs.vehicle_ids(slot)
                for nm in names[:3] if s % 2 else []:
                    a.set_vehicle_speed(nm, 2.5)
                    b.set_vehicle_speed(nm, 2.5)
                for nm, v in zip(names, speed.tolist()):
                    a.set_vehicle_speed(nm, v)
                cityflow_b200.set_vehicle_speeds_tensor(b, slot, prio, speed)
                acted += len(pick)
        a.next_step()
        b.next_step()
        assert _state(a) == _state(b), "step %d" % s
    assert acted > 2000, acted
    assert b.get_vehicle_count() > 0


def test_fixed_shape_policy_loop(cfg_6x6_dense):
    """observe -> torch policy over the padded columns -> set_vehicle_speeds_tensor -> next_step, 100 steps, with no
    host copy in the loop; kept in lock step with an engine that gets the same speeds through set_vehicle_speed."""
    import cityflow_b200
    a, b = _engine(cfg_6x6_dense), _engine(cfg_6x6_dense)
    obs = cityflow_b200.VehicleObservations(b)
    for _ in range(50):
        a.next_step()
        b.next_step()
    for s in range(100):
        obs.refresh()
        speed = (obs.speed * 0.5 + (obs.distance % 7.0)).contiguous()   # any function of the row
        cityflow_b200.set_vehicle_speeds_tensor(b, obs.slot, obs.priority, speed)
        n, slot = int(obs.count.item()), obs.slot
        for nm, v in zip(obs.vehicle_ids(slot[:n]), speed[:n].tolist()):
            a.set_vehicle_speed(nm, v)
        a.next_step()
        b.next_step()
        assert _state(a) == _state(b), "step %d" % s


def test_batched_speed_refuses_stale_and_duplicate_handles(cfg_6x6_dense):
    import torch
    import cityflow_b200
    for case in ("stale", "twice"):
        eng = _engine(cfg_6x6_dense)
        obs = cityflow_b200.VehicleObservations(eng)
        for _ in range(40):
            eng.next_step()
        obs.refresh()
        slot, prio = obs.slot[:2].clone(), obs.priority[:2].clone()
        if case == "stale":
            prio[0] += 1
        else:
            slot[1], prio[1] = slot[0], prio[0]
        cityflow_b200.set_vehicle_speeds_tensor(eng, slot, prio, torch.ones(2, dtype=torch.float64, device="cuda"))
        with pytest.raises(RuntimeError, match="Vehicle not found" if case == "stale" else "twice"):
            eng.get_vehicle_count()
    with pytest.raises(ValueError):
        cityflow_b200.set_vehicle_speeds_tensor(eng, slot.long(), prio, torch.ones(2, dtype=torch.float64, device="cuda"))
