"""Per-vehicle observations and speed actions at the bench operating point: the host dict getters against the device
table (VehicleObservations) and set_vehicle_speed against set_vehicle_speeds_tensor.  Prints one JSON line.

    python tools/vehicle_obs_timing.py [--calls 1000]

Workload: bench.py's 30x30 grid (random-walk flows frac=0.5 interval=10 s seed=1, +-2 % vehicle parameters) after its
1200 prefill and 5 warm-up steps, about 1.3e5 running vehicles.  Host-clock figures end in a device synchronise; device
figures are CUDA events on the consumer stream.  Needs a CUDA device (there is no CPU path)."""
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


def host_ms(f, sync):
    sync()
    t0 = time.perf_counter()
    f()
    sync()
    return 1e3 * (time.perf_counter() - t0)


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--calls", type=int, default=1000)
    p.add_argument("--prefill", type=int, default=1205)
    a = p.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("vehicle_obs_timing.py: no CUDA device")
    import cityflow
    import cityflow_b200
    from cityflow_b200 import scenario
    d = tempfile.mkdtemp()
    cfg = scenario.make_grid_scenario(d, 30, 30, name="vot", dense=dict(frac=0.5, interval=10.0, seed=1, fleet_spread=0.02))
    eng = cityflow.Engine(cfg, thread_num=1)
    for _ in range(a.prefill):
        eng.next_step()
    sync = torch.cuda.synchronize
    eng.get_vehicle_count()
    r = {"gpu": card(), "vehicles": eng.get_vehicle_count()}
    for name in ("get_vehicle_speed", "get_vehicle_distance", "get_lane_vehicles"):
        getattr(eng, name)()                                  # (first call: allocations)
        r[name + "_ms"] = host_ms(getattr(eng, name), sync)

    obs = cityflow_b200.VehicleObservations(eng)
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
    r["rows"] = int(obs.count.item())

    def steps(with_refresh):
        for _ in range(a.calls):
            eng.next_step()
            if with_refresh:
                obs.refresh()
    # alternate the two loops twice: other work on the host moves both
    loops = {"step_ms": [], "step_refresh_ms": []}
    for _ in range(2):
        loops["step_ms"].append(host_ms(lambda: steps(False), sync) / a.calls)
        loops["step_refresh_ms"].append(host_ms(lambda: steps(True), sync) / a.calls)
    r.update(loops)
    eng.get_vehicle_count()

    obs.refresh()
    n = int(obs.count.item())
    names = obs.vehicle_ids(obs.slot[:1000])
    r["set_vehicle_speed_x1000_ms"] = host_ms(lambda: [eng.set_vehicle_speed(nm, 5.0) for nm in names], sync)
    eng.next_step()
    for k in (1000, 100000):
        obs.refresh()
        k = min(k, int(obs.count.item()))
        slot, prio = obs.slot[:k].clone(), obs.priority[:k].clone()
        speed = torch.full((k,), 5.0, dtype=torch.float64, device="cuda")
        cityflow_b200.set_vehicle_speeds_tensor(eng, slot, prio, speed)   # warm
        sync()
        s.record()
        cityflow_b200.set_vehicle_speeds_tensor(eng, slot, prio, speed)
        e.record()
        sync()
        r["set_vehicle_speeds_tensor_%d_device_ms" % k] = s.elapsed_time(e)
        r["set_vehicle_speeds_tensor_%d_host_ms" % k] = host_ms(
            lambda: cityflow_b200.set_vehicle_speeds_tensor(eng, slot, prio, speed), sync)
        eng.get_vehicle_count()                               # (raises if a handle were refused)
        eng.next_step()
    r["rows_at_actions"] = n
    print(json.dumps(r))


if __name__ == "__main__":
    main()
