"""A short tour of every kernel for compute-sanitizer (run on the GPU box):

    compute-sanitizer --tool memcheck  python tools/sanitize_run.py
    compute-sanitizer --tool racecheck python tools/sanitize_run.py
    compute-sanitizer --tool initcheck python tools/sanitize_run.py

Small networks so the instrumented kernels finish in seconds: single engine (step kernels, spawn
ring, observation kernels, archive, vehicle setters, the per-vehicle table with and without its context and batched custom speed), rlTrafficLight engine (host and device phase
setting, device-resident observations, the intersection observations with pending host phases), lane change (its per-road
kernels run roads concurrently: racecheck is the interesting tool there) and a 2-rank loop-back shard group
(pack/unpack/seal kernels).
Exit code 0 and the sanitizer's "ERROR SUMMARY: 0 errors" are the result."""
import os
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from cityflow_b200 import scenario  # noqa: E402


def main():
    steps = int(sys.argv[1]) if len(sys.argv) > 1 else 150
    d = tempfile.mkdtemp()
    cfg = scenario.make_grid_scenario(d, 3, 3, dense=dict(frac=1.0, interval=2.0, seed=3), name="san")
    cfg_rl = scenario.make_grid_scenario(d, 3, 3, dense=dict(frac=1.0, interval=2.0, seed=4), name="sanrl", rl_traffic_light=True)
    cfg_sh = scenario.make_grid_scenario(d, 3, 4, dense=dict(frac=1.0, interval=2.0, seed=5), name="sansh")
    import cityflow
    import cityflow_b200
    from cityflow_b200.capi import CShardGroup

    eng = cityflow.Engine(cfg, thread_num=1)
    for _ in range(steps):
        eng.next_step()
    n = eng.get_vehicle_count()
    speeds = eng.get_vehicle_speed()
    eng.get_lane_vehicle_count(); eng.get_lane_waiting_vehicle_count(); eng.get_lane_vehicles()
    eng.get_vehicle_distance(); eng.get_vehicles(include_waiting=True); eng.get_average_travel_time()
    vid = next(iter(speeds))
    eng.get_vehicle_info(vid); eng.get_leader(vid); eng.set_vehicle_speed(vid, 1.0)
    snap = eng.snapshot()
    for _ in range(20):
        eng.next_step()
    eng.load(snap)
    for _ in range(20):
        eng.next_step()
    eng.reset()
    for _ in range(30):
        eng.next_step()
    print("engine ok, vehicles", n, eng.get_vehicle_count())

    # per-vehicle table and batched custom speed (device_vehobs.cuh), padded columns passed as they are
    if os.environ.get("SAN_NO_TORCH") != "1":
        import torch
        vo = cityflow_b200.VehicleObservations(eng)
        for _ in range(20):
            vo.refresh()
            cityflow_b200.set_vehicle_speeds_tensor(eng, vo.slot, vo.priority, (vo.speed * 0.5).contiguous())
            eng.next_step()
        vc = cityflow_b200.VehicleObservations(eng, context=True)   # what lies ahead of each row (k_vctx), plain refreshes between
        for k in range(20):
            vc.refresh()
            if k % 2:
                vo.refresh()
            eng.next_step()
        torch.cuda.synchronize()
        print("vehicle table ok, rows", int(vo.count.item()), eng.get_vehicle_count())

    rl = cityflow.Engine(cfg_rl, thread_num=1)
    inters = rl.intersection_ids()
    try:
        if os.environ.get("SAN_NO_TORCH") == "1":
            raise RuntimeError("SAN_NO_TORCH=1")
        import torch
        obs = cityflow_b200.LaneObservations(rl)
        tobs = cityflow_b200.IntersectionObservations(rl)
        idx = torch.arange(rl.num_intersections(), device="cuda", dtype=torch.int32)
    except Exception as e:  # noqa: BLE001
        obs = None
        print("torch tensors unavailable:", e)
    for t in range(steps):
        if obs is not None and t % 3 == 0:
            obs.refresh()
            cityflow_b200.set_tl_phases_tensor(rl, ((idx + t // 10) % 8).to(torch.int32))
        elif t % 3 == 1:
            for i in inters[:4]:
                try:
                    rl.set_tl_phase(i, (t // 7) % 8)
                except RuntimeError:
                    pass  # virtual intersection
            if obs is not None:   # the refresh sends the pending set_tl_phase calls up first (device_tlobs.cuh)
                tobs.refresh()
                cityflow_b200.set_tl_phases_tensor(rl, tobs.phase_pressure.argmax(1).to(torch.int32))
        rl.next_step()
    print("rl ok, vehicles", rl.get_vehicle_count())

    # lane change: its per-road kernels run roads concurrently (racecheck is the interesting tool here)
    from cityflow_b200.capi import CEngine
    cfg_lc = scenario.make_grid_scenario(d, 3, 3, dense=dict(frac=1.0, interval=2.0, seed=6), name="sanlc", lane_change=True)
    lc = CEngine(cfg_lc)
    for _ in range(steps):
        lc.next_step()
    print("lane change ok, vehicles (shadows included)", lc.vehicle_count())

    grp = CShardGroup(cfg_sh, 2)
    grp.next_step(steps)
    print("shard group ok, vehicles", grp.vehicle_count())


if __name__ == "__main__":
    main()
