"""Lane change on the GPU where its per-road kernels run wide, on irregular networks, and past 256 new shadows in one step,
against the restatement (oracle/cityflow_oracle.cpp in its device form) every step: every lane-change field of every
running vehicle, shadows included, vehicle and lane counts.

The small networks of the other lane-change tests stay inside one block of every lane-change kernel.  Here:
* k_lc_order / k_lc_tail_order sort a step's candidates / involved vehicles in one block of 256 threads, one entry per
  thread per pass: more than 256 of them take a second pass;
* k_lc_schedule_roads / k_lc_tail_roads run blocks of 128 threads, one per entry: past 128 entries the roads are
  served from different blocks at once, and shadows take their slots from one counter by atomicAdd across them;
* more than 256 new shadows in one step use more spare slots than a step was once lent.
K disjoint copies of one small scenario (tests/edgenet.py, replicated) reach these sizes; the restatement reports what a
run reached (edgenet.LcReach).  CITYFLOW_B200_LC_SERIAL=1 selects the one-thread scheduling and control tail; it runs in
lock step with the default form, and both must equal the restatement (records are keyed by priority: a shadow's slot
comes from atomic order in the per-road form).

Irregular networks (tests/randnet.py: 1-3 lanes per road, lanes of one road with different lengths, bent roads,
dead-end lanes) and the star / short_hops edge shapes run with lane change here for the first time on the GPU."""
import pytest

import edgenet

pytestmark = pytest.mark.gpu


def _engine(cfg, monkeypatch, serial=False):
    """A CEngine made with CITYFLOW_B200_LC_SERIAL set or not (DeviceSim reads it in enableLaneChange)."""
    from cityflow_b200.capi import CEngine
    monkeypatch.delenv("CITYFLOW_B200_LC_SERIAL", raising=False)
    if serial:
        monkeypatch.setenv("CITYFLOW_B200_LC_SERIAL", "1")
    eng = CEngine(cfg)
    monkeypatch.delenv("CITYFLOW_B200_LC_SERIAL", raising=False)
    return eng


def _engines(cfg, monkeypatch, serial):
    engines = {"default": _engine(cfg, monkeypatch)}
    if serial:
        engines["lc_serial"] = _engine(cfg, monkeypatch, serial=True)
    return engines


# ------------------------------------------------------------------------------------------
# 64 copies of the dense 2x2 grid with flow seed 8: about ten candidates, eight new shadows and twenty involved vehicles
# per copy in one step within 40 steps -- past the one-pass sort of k_lc_order / k_lc_tail_order, over several blocks of
# the per-road kernels, past 256 new shadows.
def test_replicated_grid_wide_default_and_serial(tmp_path, monkeypatch):
    cfg = edgenet.write_replicated(str(tmp_path), 64, "grid2x2", seed=8)
    reach = edgenet.lc_vs_restatement(_engines(cfg, monkeypatch, serial=True), cfg, 200)
    print("grid2x2 (flow seed 8) x 64, default and one-thread forms in lock step: %s" % reach)
    s = reach.stats()
    assert s["candidates"] > 256 and s["involved"] > 256 and reach.new_shadows > 256, str(reach)


# 96 copies with flow seed 3: three new shadows per copy in step 175, 288 in all, after the network has filled
# (60 k vehicles).
def test_replicated_grid_more_than_256_shadows_in_one_step(tmp_path, monkeypatch):
    cfg = edgenet.write_replicated(str(tmp_path), 96, "grid2x2", seed=3)
    reach = edgenet.lc_vs_restatement(_engines(cfg, monkeypatch, serial=False), cfg, 180)
    print("grid2x2 (flow seed 3) x 96: %s" % reach)
    assert reach.new_shadows > 256, str(reach)


# 4 copies of long_queue: buckets of 3+ warp chunks with 30+ candidates on one road, so one thread of k_lc_schedule_roads
# walks a long list of entries and inserts many shadows into one bucket while other roads do the same.
def test_replicated_long_queue(tmp_path, monkeypatch):
    cfg = edgenet.write_replicated(str(tmp_path), 4, "long_queue")
    reach = edgenet.lc_vs_restatement(_engines(cfg, monkeypatch, serial=False), cfg, 700)
    print("long_queue x 4: %s" % reach)
    s = reach.stats()
    assert s["candidates"] > 256 and s["involved"] > 256 and s["candidates_on_a_road"] > 32, str(reach)


# ------------------------------------------------------------------------------------------
# The networks of tests/test_gpu_parity.py::test_fuzzed_irregular_networks_vs_port, with lane change; seed 1 also in the
# one-thread form.
@pytest.mark.parametrize("seed", [1, 2, 3, 5, 8, 11])
def test_fuzzed_irregular_networks_with_lane_change(seed, tmp_path, monkeypatch):
    import randnet
    from cityflow_b200 import scenario
    net = randnet.random_roadnet(seed, rows=2 + seed % 3, cols=3 + seed % 2)
    flows = randnet.random_flows(net, seed + 100, n_flows=40 + seed % 50)
    cfg = scenario.write_scenario(str(tmp_path), net, flows, seed=seed, interval=[1.0, 0.5, 2.0, 1.0][seed % 4], lane_change=True,
                                  name="g%d_lc" % seed)
    reach = edgenet.lc_vs_restatement(_engines(cfg, monkeypatch, serial=seed == 1), cfg, 500)
    print("irregular network %d with lane change: %s" % (seed, reach))
    assert reach.shadow_states > 0, str(reach)


@pytest.mark.parametrize("shape,steps", [("star", 400), ("short_hops", 500)])
def test_edge_shapes_with_lane_change(shape, steps, tmp_path, monkeypatch):
    """star: 4-lane roads into 8- and 6-leg intersections, 60 candidates in one step.  On short_hops' 8-25 m lanes nobody
    asks to change lanes (the restatement finds no candidate in 500 steps): what runs is the lane-change step's own kernel
    sequence around vehicles crossing 3+ drivables per step."""
    cfg = edgenet.write(shape, str(tmp_path), lane_change=True)
    reach = edgenet.lc_vs_restatement(_engines(cfg, monkeypatch, serial=False), cfg, steps)
    print("%s with lane change: %s" % (shape, reach))
    if shape == "star":
        assert reach.stats()["candidates"] > 32 and reach.shadow_states > 1000, str(reach)
