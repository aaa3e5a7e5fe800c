"""Lane change at the public surface over the emulated device: vehicle ids of shadows, lookups by id, binary snapshots
and the replay log against the priority-ordered reference's own Python module (tests/lc_surface_main.py)."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import lc_surface_main as S
from test_cpu import _HAVE_CUDA_SDK, _golden_module, _hetero_lane_change_config, _pyemu_dir

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _scenario(kind, directory):
    if kind == "bent_roads":
        return _hetero_lane_change_config(directory)
    return _golden_module().make_lc_config(kind, directory)


@pytest.mark.skipif(not _HAVE_CUDA_SDK or not S.have_lc_module(), reason="needs the CUDA SDK and oracle/_ref/lcorder/cityflow*.so")
@pytest.mark.parametrize("kind", ["lc3_default", "lc4_dense", "bent_roads"])
def test_lane_change_surface_vs_reference_module_over_emulated_device(kind, tmp_path):
    cfg = S.with_replay(_scenario(kind, str(tmp_path)))
    env = dict(os.environ, CFB_EMULATED_DEVICE_FOR_TESTS="1", PYTHONPATH=_pyemu_dir() + os.pathsep + os.path.join(ROOT, "tests"))
    out = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "lc_surface_main.py"), cfg, "500"],
                         env=env, capture_output=True, text=True, timeout=3000, cwd=str(tmp_path))
    assert out.returncode == 0 and out.stdout.startswith("OK"), out.stdout[-1500:] + out.stderr[-3000:]
    stats = json.loads(out.stdout[3:out.stdout.index(" with ")])
    assert "pyemu" in out.stdout
    assert stats["shadow_ids"] > 0 and stats["takeovers"] > 0 and stats["stale_refused"] > 0, stats
    assert stats["shadow_lookups"] > 0 and stats["snapshot_steps"] == 10 and stats["replay_dirs"] > 0, stats


def _replay_fixture(tmp_path):
    from cityflow_b200 import scenario
    from cityflow_b200.capi import REPLAY_DTYPE, REPLAY_LC_DTYPE
    cfg = scenario.make_grid_scenario(str(tmp_path), 2, 2, name="rp")
    c = json.load(open(cfg))
    v = np.zeros(3, REPLAY_DTYPE)
    v["drivable"] = [0, 1, 2]            # lanes 0 and 1 of the first road, lane 2 (its outermost)
    v["distance"] = [10.0, 55.5, 3.25]
    v["flow"] = [0, 1, -2]
    v["index"] = [4, 7, 2]
    v["length"] = 5.0
    v["width"] = 2.0
    lc = np.zeros(3, REPLAY_LC_DTYPE)
    lc["v"] = v
    net = c["dir"] + c["roadnetFile"]
    return net, v, lc, np.zeros(len(json.load(open(net))["intersections"]), np.int32)


def test_lane_change_replay_formatter_without_lane_change_state_is_the_plain_one(tmp_path):
    """No offset, no direction, no suffix: cfb_replay_format_step_lc writes the bytes cfb_replay_format_step writes."""
    from cityflow_b200.capi import CReplay
    net, v, lc, phases = _replay_fixture(tmp_path)
    rp = CReplay(net)
    assert rp.format_step_lc(lc, phases) == rp.format_step(v, phases)


def test_lane_change_replay_formatter_draws_the_offset_direction_and_suffix(tmp_path):
    """Vehicle::getPoint (vehicle.cpp:81-105): a car half-way to the next lane is drawn half-way between the two lanes'
    points; the id gets its "_shadow" suffixes and the line its change direction."""
    from cityflow_b200.capi import CReplay
    net, v, lc, phases = _replay_fixture(tmp_path)
    rp = CReplay(net)
    centre = [t.split(" ") for t in rp.format_step(v, phases).split(";")[0].split(",")[:3]]
    w = json.load(open(net))["roads"][0]["lanes"]
    lc["offset"] = [(w[0]["width"] + w[1]["width"]) / 4, 0.0, 0.0]   # half-way from lane 0 to lane 1
    lc["lane_change_dir"] = [1, -1, 0]
    lc["shadow_depth"] = [0, 1, 0]
    toks = [t.split(" ") for t in rp.format_step_lc(lc, phases).split(";")[0].split(",")[:3]]
    v2 = v.copy()
    v2["drivable"][0] = 1
    v2["distance"][0] = v["distance"][0]
    next_lane = rp.format_step(v2, phases).split(";")[0].split(",")[0].split(" ")
    for i in (0, 1):
        assert float(toks[0][i]) == 0.5 * float(next_lane[i]) + 0.5 * float(centre[0][i])
    assert toks[0][2] == centre[0][2]                       # heading: the current lane's direction
    assert toks[0][3:5] == ["flow_0_4", "1"]
    assert toks[1][3:5] == ["flow_1_7_shadow", "-1"] and toks[1][:3] == centre[1][:3]
    assert toks[2] == centre[2]


def test_vehicle_ids_of_the_c_abi_round_trip():
    """cfb_vehicle_ref: "_shadow" suffixes in bits 24-30 of index (include/cityflow_b200.h)."""
    from cityflow_b200 import capi
    for name in ("flow_0_0", "flow_12_16777215", "manually_pushed_3", "flow_3_5_shadow", "manually_pushed_9_shadow"):
        assert capi.vehicle_name(*capi.parse_vehicle_name(name)) == name
    assert capi.parse_vehicle_name("flow_3_5_shadow") == (3, 5 | 1 << capi.REF_SHADOW_SHIFT)
    assert capi.parse_vehicle_name("flow_3_16777216_shadow") is None
    assert capi.parse_vehicle_name("flow_3_5_shadowx") is None and capi.parse_vehicle_name("_shadow") is None
