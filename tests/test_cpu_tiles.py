"""k_notify and k_move serve two drivables per warp, one per 16-lane tile: every loop around a warp primitive runs to
the larger trip count of the two tiles and predicates its work.  The whole-step tests meet unequal tiles only as the
work lists happen to fall; here tests/tile_pair_probe.cpp pairs them on purpose (heaviest drivable next to the
lightest in every warp) and requires the restatement's full state after every step."""
import os
import re
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _tile_pair_probe():
    os.makedirs(os.path.join(ROOT, "oracle", "_build"), exist_ok=True)
    probe = os.path.join(ROOT, "oracle", "_build", "tile_pair_probe")
    csrc = os.path.join(ROOT, "cityflow_b200", "csrc")
    tests = os.path.join(ROOT, "tests")
    srcs = [os.path.join(tests, "tile_pair_probe.cpp"), os.path.join(csrc, "roadnet.cpp"), os.path.join(csrc, "flows.cpp")]
    deps = srcs + [os.path.join(csrc, f) for f in os.listdir(csrc) if f.endswith((".cuh", ".h"))] + \
        [os.path.join(ROOT, "oracle", "cityflow_oracle.cpp")] + \
        [os.path.join(tests, f) for f in ("device_emu.h", "device_hostsim.h", "device_step_probe.cpp")]
    if not os.path.exists(probe) or os.path.getmtime(probe) < max(os.path.getmtime(f) for f in deps):
        subprocess.check_call(["g++", "-std=c++17", "-O1", "-ffp-contract=off", "-I/usr/local/cuda/include", "-I" + csrc, "-I" + tests]
                              + srcs + ["-o", probe])
    return probe


@pytest.mark.skipif(not os.path.exists("/usr/local/cuda/include/vector_types.h"), reason="needs the CUDA headers")
@pytest.mark.parametrize("shape", ["long_queue", "star", "merge_ties"])
def test_unequal_tiles_of_one_warp_match_the_restatement(shape, tmp_path):
    """long_queue: a lane of up to ~190 vehicles (a dozen k_move chunks) next to a drivable holding one.  star: laneLinks
    with far more than 16 crosses (several k_notify chunks) next to lanes that trigger none.  merge_ties: up to 6
    entrants, some tied at equal distance, sorted in one tile while the other tile has fewer or none."""
    import edgenet
    cfg = edgenet.write(shape, str(tmp_path))
    out = subprocess.run([_tile_pair_probe(), cfg, "400"], capture_output=True, text=True, timeout=900)
    assert out.returncode == 0 and out.stdout.startswith("OK"), out.stdout[-2000:] + out.stderr[-500:]
    states = int(out.stdout.split(" steps, ")[1].split(" vehicle states")[0])
    assert states > 20000, out.stdout
    m = re.search(r"notify (\d+), (\d+) with different cross chunks \(max (\d+) crosses\); move (\d+), (\d+) with different "
                  r"bucket chunks \(max (\d+) vehicles\), (\d+) with different entrant counts \(max (\d+) entrants\)", out.stdout)
    assert m, out.stdout
    _, notify_differ, max_crosses, _, move_differ, max_vehicles, ent_differ, max_entrants = (int(x) for x in m.groups())
    if shape == "long_queue":
        assert move_differ > 1000 and max_vehicles > 32, out.stdout
    elif shape == "star":
        assert notify_differ > 1000 and max_crosses > 32, out.stdout
    else:
        ties = int(out.stdout.split(" failures, ")[1].split(" ties")[0])
        assert ent_differ > 100 and max_entrants >= 4 and ties > 100, out.stdout
