"""Lane change at widths the small networks never reach, without a GPU: K disjoint copies of one small scenario in one
roadnet (tests/edgenet.py, replicated).  The copies evolve side by side, so a step's lane-change candidates, involved
vehicles and new shadows grow K-fold while the restatement stays affordable.

The replicated networks are pinned to the reference here (loader tables, and the restatement against the
priority-ordered reference with lane change), and the real host engine runs over the emulated device past 256 new
shadows in one step: the spare slots a step lends the device for its shadows come from csrc/host_engine.cpp, which the
emulated device links too.  tests/test_gpu_lane_change_wide.py runs the same networks on the GPU."""
import pytest

import edgenet
from oracle import harness as H
from test_cpu import _HAVE_CUDA_SDK, _check_loader_tables, _emulated_engine

# (unit, copies, steps) pinned to the reference; small enough for refdump to run quickly
PINNED = [("grid2x2", 4, 200), ("long_queue", 2, 400)]


@pytest.mark.skipif(not H.have_lc_ref(), reason="needs oracle/_ref/refdump_lcorder")
@pytest.mark.parametrize("unit,k,steps", PINNED, ids=["%s-x%d" % (u, k) for u, k, _ in PINNED])
def test_replicated_network_loader_and_restatement_vs_reference(unit, k, steps, tmp_path):
    """The replicated roadnet through the product's loader: static tables bit-identical to the reference's, and the copies
    disjoint (no laneLink ends in another copy).  With lane change, the restatement in its device form equal to the
    priority-ordered reference every step, shadows included."""
    cfg = edgenet.write_replicated(str(tmp_path), k, unit)
    mine = _check_loader_tables(cfg)
    per_copy = mine["n_lanes"] // k
    assert mine["n_lanes"] == per_copy * k
    owner = lambda lane: lane // per_copy     # roads (and their lanes) are listed copy by copy
    for lane, links in enumerate(mine["lane_out"]):
        assert all(owner(mine["link_end"][x]) == owner(lane) for x in links), lane
    ora = edgenet.device_form_restatement(cfg)
    run = H.RefDump.runlc(cfg, steps, 1, n_inter=ora.n_inter, n_drivables=ora.n_drivables)
    assert len(run) == steps
    reach = edgenet.LcReach(ora)
    for st in run:
        ora.next_step()
        got = ora.lc_snapshot()
        bad = H.compare_lc_states(st, got)
        assert not bad, "step %d: %s" % (st.step, "; ".join(bad[:5]))
        reach.add(got.vehicles)
    print("%s x %d with lane change, equal to the priority-ordered reference: %s" % (unit, k, reach))
    assert reach.new_shadows >= k


# With flow seed 8 the dense 2x2 grid changes lanes early: 48 copies create up to 390 shadows in one step within 40 steps,
# past the 256 spare slots a step was once lent, where the step threw instead of carrying on.
SHADOW_K, SHADOW_SEED, SHADOW_STEPS = 48, 8, 40


@pytest.mark.skipif(not _HAVE_CUDA_SDK, reason="needs the CUDA headers and libcudart to build the host-check library")
@pytest.mark.parametrize("lc_serial", [False, True], ids=["per_road", "lc_serial"])
def test_more_than_256_shadows_in_one_step_over_emulated_device(lc_serial, tmp_path, monkeypatch):
    """The real host engine (spare slots, shadow priorities, name take-over) over the emulated device on 48 copies of the
    dense 2x2 grid, equal to the restatement every step in every lane-change field, past 256 new shadows in one step; with
    the per-road scheduling kernels and with the one-thread ones (CITYFLOW_B200_LC_SERIAL=1)."""
    monkeypatch.setenv("CFB_EMULATED_DEVICE_FOR_TESTS", "1")
    if lc_serial:
        monkeypatch.setenv("CITYFLOW_B200_LC_SERIAL", "1")
    else:
        monkeypatch.delenv("CITYFLOW_B200_LC_SERIAL", raising=False)
    cfg = edgenet.write_replicated(str(tmp_path), SHADOW_K, "grid2x2", seed=SHADOW_SEED)
    reach = edgenet.lc_vs_restatement({"emulated": _emulated_engine(cfg)}, cfg, SHADOW_STEPS)
    print("grid2x2 (flow seed %d) x %d over the emulated device: %s" % (SHADOW_SEED, SHADOW_K, reach))
    assert reach.new_shadows > 256, str(reach)
