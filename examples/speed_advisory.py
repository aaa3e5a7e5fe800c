"""Per-vehicle observations and actions on the GPU (INTEGRATION.md section 4): every step, each lane's queue within 50 m
of its stop line is counted in torch from the vehicle table, and the vehicles approaching a queue of two or more
cars in front of a red light get an advisory speed of 5 m/s for the coming step -- one set_vehicle_speeds_tensor call,
nothing copied to the host inside the loop.  Lane lengths and each vehicle's light come from the table's context
columns (VehicleObservations(context=True))."""
import os
import sys
import tempfile
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import cityflow  # noqa: E402
import cityflow_b200  # noqa: E402
from cityflow_b200 import scenario  # noqa: E402

with tempfile.TemporaryDirectory() as d:
    cfg = scenario.make_grid_scenario(d, 10, 10, dense=dict(frac=1.0, interval=5.0, seed=1))
    eng = cityflow.Engine(cfg)
    obs = cityflow_b200.VehicleObservations(eng, context=True)    # tensors are created once
    n_lanes = obs.n_lanes
    lane_len = obs.drivable_length[:n_lanes]
    steps, advised = 500, torch.zeros((), dtype=torch.int64, device="cuda")
    t0 = time.perf_counter()
    for _ in range(steps):
        obs.refresh()                                               # the table and its context, ordered against torch's stream
        on_lane = (obs.slot >= 0) & (obs.drivable < n_lanes)        # padding rows have slot -1
        lane = obs.drivable.clamp(0, n_lanes - 1).long()
        near = on_lane & (lane_len[lane] - obs.distance < 50.0)
        queue = torch.zeros(n_lanes, dtype=torch.int64, device="cuda").index_add_(0, lane, (near & (obs.speed < 0.1)).long())
        act = near & (obs.speed >= 0.1) & (queue[lane] >= 2) & (obs.signal == 0)   # red ahead: signal 0
        slot = torch.where(act, obs.slot, torch.full_like(obs.slot, -1))   # slot -1: no action for that row
        cityflow_b200.set_vehicle_speeds_tensor(eng, slot, obs.priority, torch.full_like(obs.speed, 5.0))
        advised += act.sum()
        eng.next_step()
    torch.cuda.synchronize()
    eng.synchronize()
    dt = time.perf_counter() - t0
    print("%d steps in %.2f s (%.0f steps/s), %d vehicles, %d speed advisories, longest queue now %d" % (
        steps, dt, steps / dt, eng.get_vehicle_count(), int(advised), int(queue.max())))
