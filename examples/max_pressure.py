"""MaxPressure signal control with nothing crossing to the host: IntersectionObservations gives every phase's pressure
(the incoming minus the outgoing vehicles of the movements it serves) as a torch CUDA tensor, argmax picks each light's
phase, set_tl_phases_tensor hands the choice back (INTEGRATION.md section 4).  Prints the average travel time against
the same grid under its fixed-time plan.

The grid generator's phase lists start with a phase that serves right turns only (and every other phase serves the
right turns too), so a right-turn-only phase never relieves more than the phases beside it.  The controller chooses
among the phases that serve at least one movement other than a right turn."""
import os
import sys
import tempfile
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import cityflow  # noqa: E402
import cityflow_b200  # noqa: E402
from cityflow_b200 import scenario  # noqa: E402

STEPS = 1800
DENSE = dict(frac=1.0, interval=4.0, seed=1)

with tempfile.TemporaryDirectory() as d:
    fixed = cityflow.Engine(scenario.make_grid_scenario(d, 8, 8, dense=DENSE, name="fixed"))
    fixed.next_steps(STEPS)
    eng = cityflow.Engine(scenario.make_grid_scenario(d, 8, 8, dense=DENSE, name="mp", rl_traffic_light=True))
    obs = cityflow_b200.IntersectionObservations(eng)
    # the phases to choose among: those that serve a movement other than a right turn (static, computed once)
    other = torch.tensor([rl["type"] != "turn_right" for rl in obs.road_links], device=obs.phase.device)
    local = obs.movement_begin[:-1, None] + torch.arange(obs.phase_movements.shape[2], device=other.device)
    served = obs.phase_movements.bool() & other[local.clamp(max=len(other) - 1)][:, None, :]
    allowed = served.any(2)
    t0 = time.perf_counter()
    for _ in range(STEPS):
        obs.refresh()                                               # k_tobs, ordered against torch's stream
        act = obs.phase_pressure.masked_fill(~allowed, torch.iinfo(torch.int32).min).argmax(1).to(torch.int32)
        cityflow_b200.set_tl_phases_tensor(eng, act)                # virtual intersections' entries are ignored
        eng.next_step()
    torch.cuda.synchronize()
    eng.synchronize()
    dt = time.perf_counter() - t0
    print("8x8 dense grid, %d steps: average travel time %.1f s under MaxPressure (%.0f steps/s), %.1f s under the "
          "fixed-time plan" % (STEPS, eng.get_average_travel_time(), STEPS / dt, fixed.get_average_travel_time()))
