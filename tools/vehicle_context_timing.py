"""The per-vehicle context refresh (VehicleObservations(context=True)) against the plain table refresh at the bench
operating point, in device time.  Prints one JSON line.

    python tools/vehicle_context_timing.py [--calls 1000]

Workload: bench.py's 30x30 grid (random-walk flows frac=0.5 interval=10 s seed=1, +-2 % vehicle parameters) after 1205
steps, about 1.3e5 running vehicles.  Each figure is CUDA events around `--calls` back-to-back refreshes on the
consumer stream, divided by the calls; the two kinds alternate twice, since other work on the machine moves both.  The
card's name, power limit and top SM clock are read in the same run.  Needs a CUDA device (there is no CPU path)."""
import argparse
import json
import os
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from vehicle_obs_timing import card  # noqa: E402


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--calls", type=int, default=1000)
    p.add_argument("--prefill", type=int, default=1205)
    a = p.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("vehicle_context_timing.py: no CUDA device")
    import cityflow
    import cityflow_b200
    from cityflow_b200 import scenario
    cfg = scenario.make_grid_scenario(tempfile.mkdtemp(), 30, 30, name="vct",
                                      dense=dict(frac=0.5, interval=10.0, seed=1, fleet_spread=0.02))
    eng = cityflow.Engine(cfg, thread_num=1)
    for _ in range(a.prefill):
        eng.next_step()
    r = {"gpu": card(), "vehicles": eng.get_vehicle_count(), "calls": a.calls}
    plain = cityflow_b200.VehicleObservations(eng)
    ctx = cityflow_b200.VehicleObservations(eng, context=True)
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    def device_ms(obs):
        for _ in range(20):
            obs.refresh()
        torch.cuda.synchronize()
        s.record()
        for _ in range(a.calls):
            obs.refresh()
        e.record()
        torch.cuda.synchronize()
        return s.elapsed_time(e) / a.calls

    r["plain_refresh_device_ms"], r["context_refresh_device_ms"] = [], []
    for _ in range(2):
        r["plain_refresh_device_ms"].append(device_ms(plain))
        r["context_refresh_device_ms"].append(device_ms(ctx))
    r["rows"] = int(ctx.count.item())
    r["rows_with_leader"] = int((ctx.leader >= 0).sum().item())
    r["rows_at_a_light"] = int((ctx.signal >= 0).sum().item())
    print(json.dumps(r))


if __name__ == "__main__":
    main()
