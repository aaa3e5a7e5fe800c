"""GPU test: lane change at the public surface of the `cityflow` drop-in on the device -- shadows' ids, lookups by id,
binary snapshots and the replay log (k_gather_running_lc) -- against the priority-ordered reference's own module
(oracle/_ref/lcorder/, which travels with the tree), through tests/lc_surface_main.py.  A child process: the two
reference modules define the same C++ types, so this one is not loaded next to oracle/_ref/cityflow*.so."""
import json
import os
import subprocess
import sys

import pytest

import lc_surface_main as S
from test_cpu import _golden_module, _hetero_lane_change_config

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.skipif(not S.have_lc_module(), reason="needs oracle/_ref/lcorder/cityflow*.so")
@pytest.mark.parametrize("kind", ["lc3_default", "lc4_dense", "bent_roads"])
def test_lane_change_surface_vs_reference_module(kind, tmp_path):
    d = str(tmp_path)
    cfg = S.with_replay(_hetero_lane_change_config(d) if kind == "bent_roads" else _golden_module().make_lc_config(kind, d))
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.path.join(ROOT, "tests"))
    out = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "lc_surface_main.py"), cfg, "500"],
                         env=env, capture_output=True, text=True, timeout=3000, cwd=d)
    assert out.returncode == 0 and out.stdout.startswith("OK"), out.stdout[-1500:] + out.stderr[-3000:]
    stats = json.loads(out.stdout[3:out.stdout.index(" with ")])
    assert os.path.join(ROOT, "cityflow") in out.stdout   # the product module, not a test build
    assert stats["shadow_ids"] > 0 and stats["takeovers"] > 0 and stats["stale_refused"] > 0, stats
    assert stats["shadow_lookups"] > 0 and stats["snapshot_steps"] == 10 and stats["replay_dirs"] > 0, stats
