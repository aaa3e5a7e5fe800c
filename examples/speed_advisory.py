"""Per-vehicle observations and actions on the GPU (INTEGRATION.md section 4): every step, each lane's queue within 50 m
of its stop line is counted in torch from the vehicle table, and the vehicles approaching a queue of two or more
cars get an advisory speed of 5 m/s for the coming step -- one set_vehicle_speeds_tensor call, nothing copied to the
host inside the loop."""
import json
import math
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
    c = json.load(open(cfg))
    roads = {r["id"]: r for r in json.load(open(os.path.join(c["dir"], c["roadnetFile"])))["roads"]}

    def road_length(r):   # the grid's roads are straight: the lanes are as long as their road
        pts = r["points"]
        return sum(math.hypot(b["x"] - a["x"], b["y"] - a["y"]) for a, b in zip(pts, pts[1:]))
    lane_ids = eng.lane_ids()
    lane_len = torch.tensor([road_length(roads[l.rsplit("_", 1)[0]]) for l in lane_ids], dtype=torch.float64, device="cuda")
    n_lanes = len(lane_ids)

    obs = cityflow_b200.VehicleObservations(eng)                  # tensors are created once
    steps, advised = 500, torch.zeros((), dtype=torch.int64, device="cuda")
    t0 = time.perf_counter()
    for _ in range(steps):
        obs.refresh()                                               # the table, ordered against torch's stream
        on_lane = (obs.slot >= 0) & (obs.drivable < n_lanes)        # padding rows have slot -1
        lane = obs.drivable.clamp(0, n_lanes - 1).long()
        near = on_lane & (lane_len[lane] - obs.distance < 50.0)
        queue = torch.zeros(n_lanes, dtype=torch.int64, device="cuda").index_add_(0, lane, (near & (obs.speed < 0.1)).long())
        act = near & (obs.speed >= 0.1) & (queue[lane] >= 2)
        slot = torch.where(act, obs.slot, torch.full_like(obs.slot, -1))   # slot -1: no action for that row
        cityflow_b200.set_vehicle_speeds_tensor(eng, slot, obs.priority, torch.full_like(obs.speed, 5.0))
        advised += act.sum()
        eng.next_step()
    torch.cuda.synchronize()
    eng.synchronize()
    dt = time.perf_counter() - t0
    print("%d steps in %.2f s (%.0f steps/s), %d vehicles, %d speed advisories, longest queue now %d" % (
        steps, dt, steps / dt, eng.get_vehicle_count(), int(advised), int(queue.max())))
