"""Intersection observations at the bench operating point: the device time of one IntersectionObservations refresh, and
a 1000-step MaxPressure loop run on the device (refresh + argmax + set_tl_phases_tensor) against the same loop run
through the host (get_lane_vehicle_count() + pressure in Python + set_tl_phase per light).  Prints one JSON line.

    python tools/intersection_obs_timing.py [--calls 1000] [--steps 1000]

Workload: bench.py's 30x30 grid (random-walk flows frac=0.5 interval=10 s seed=1, +-2 % vehicle parameters).  The
refresh is timed on the fixed-time engine after bench.py's 1200 prefill and 5 warm-up steps.  The MaxPressure loops run
on an rlTrafficLight copy of the scenario, brought to the same step count by the device loop first; both loops choose
among the phases that serve a movement other than a right turn, the first of largest pressure.  Host-clock figures end
in a device synchronise; the refresh is timed with CUDA events.  Needs a CUDA device (there is no CPU path)."""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def host_plan(cfg):
    """What a host-side MaxPressure controller builds from the roadnet JSON: per light, per phase it may choose, the
    lane ids counted in (+1) and out (-1) of the movements the phase serves."""
    c = json.load(open(cfg))
    net = json.load(open(c["dir"] + c["roadnetFile"]))
    plan = []
    for inter in net["intersections"]:
        if inter["virtual"]:
            continue
        rls, phases = inter["roadLinks"], []
        for k, ph in enumerate(inter["trafficLight"]["lightphases"]):
            served = [rls[r] for r in sorted(set(ph["availableRoadLinks"]))]
            if all(rl["type"] == "turn_right" for rl in served):
                continue
            terms = []
            for rl in served:
                terms += [(+1, l) for l in sorted({"%s_%d" % (rl["startRoad"], x["startLaneIndex"]) for x in rl["laneLinks"]})]
                terms += [(-1, l) for l in sorted({"%s_%d" % (rl["endRoad"], x["endLaneIndex"]) for x in rl["laneLinks"]})]
            phases.append((k, terms))
        plan.append((inter["id"], phases))
    return plan


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--calls", type=int, default=1000)
    p.add_argument("--steps", type=int, default=1000)
    p.add_argument("--prefill", type=int, default=1205)
    a = p.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("intersection_obs_timing.py: no CUDA device")
    import cityflow
    import cityflow_b200
    from cityflow_b200 import scenario
    d = tempfile.mkdtemp()
    dense = dict(frac=0.5, interval=10.0, seed=1, fleet_spread=0.02)
    sync = torch.cuda.synchronize

    eng = cityflow.Engine(scenario.make_grid_scenario(d, 30, 30, name="iot", dense=dense), thread_num=1)
    eng.next_steps(a.prefill)
    r = {"gpu": card(), "vehicles": eng.get_vehicle_count(), "intersections": eng.num_intersections()}
    obs = cityflow_b200.IntersectionObservations(eng)
    r["road_links"] = len(obs.road_links)
    for _ in range(20):
        obs.refresh()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    sync()
    s.record()
    for _ in range(a.calls):
        obs.refresh()
    e.record()
    sync()
    r["refresh_device_ms"] = s.elapsed_time(e) / a.calls
    del obs, eng

    cfg = scenario.make_grid_scenario(d, 30, 30, name="iotrl", dense=dense, rl_traffic_light=True)
    eng = cityflow.Engine(cfg, thread_num=1)
    obs = cityflow_b200.IntersectionObservations(eng)
    other = torch.tensor([rl["type"] != "turn_right" for rl in obs.road_links], device=obs.phase.device)
    local = (obs.movement_begin[:-1, None] + torch.arange(obs.phase_movements.shape[2], device=other.device)).clamp(max=len(other) - 1)
    masked = ~(obs.phase_movements.bool() & other[local][:, None, :]).any(2)
    low = torch.iinfo(torch.int32).min

    def device_loop(n):
        for _ in range(n):
            obs.refresh()
            cityflow_b200.set_tl_phases_tensor(eng, obs.phase_pressure.masked_fill(masked, low).argmax(1).to(torch.int32))
            eng.next_step()

    plan = host_plan(cfg)

    def dict_loop(n):
        for _ in range(n):
            count = eng.get_lane_vehicle_count()
            for iid, phases in plan:
                best, arg = None, 0
                for k, terms in phases:
                    pr = sum(sg * count[l] for sg, l in terms)
                    if best is None or pr > best:
                        best, arg = pr, k
                eng.set_tl_phase(iid, arg)
            eng.next_step()

    device_loop(a.prefill)
    eng.get_vehicle_count()
    r["max_pressure_vehicles"] = eng.get_vehicle_count()
    loops = {"max_pressure_device_ms_per_step": [], "max_pressure_dict_ms_per_step": []}
    for _ in range(2):   # alternated: other work on the host moves both
        loops["max_pressure_device_ms_per_step"].append(host_ms(lambda: device_loop(a.steps), sync, eng) / a.steps)
        loops["max_pressure_dict_ms_per_step"].append(host_ms(lambda: dict_loop(a.steps), sync, eng) / a.steps)
    r.update(loops)
    r["max_pressure_vehicles_after"] = eng.get_vehicle_count()
    print(json.dumps(r))


def host_ms(f, sync, eng):
    sync()
    eng.synchronize()
    t0 = time.perf_counter()
    f()
    sync()
    eng.synchronize()
    return 1e3 * (time.perf_counter() - t0)


if __name__ == "__main__":
    main()
