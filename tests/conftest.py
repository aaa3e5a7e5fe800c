import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100)")


@pytest.fixture(scope="session")
def scenario_dir(tmp_path_factory):
    return str(tmp_path_factory.mktemp("scenarios"))


def _make(scenario_dir, rows, cols, name, dense=None, **cfg):
    from cityflow_b200 import scenario
    return scenario.make_grid_scenario(scenario_dir, rows, cols, dense=dense, name=name, **cfg)


@pytest.fixture(scope="session")
def cfg_1x1(scenario_dir):
    return _make(scenario_dir, 1, 1, "g1")


@pytest.fixture(scope="session")
def cfg_3x3_dense(scenario_dir):
    return _make(scenario_dir, 3, 3, "g3d", dense=dict(frac=1.0, interval=3.0, seed=3))


@pytest.fixture(scope="session")
def cfg_6x6(scenario_dir):
    return _make(scenario_dir, 6, 6, "g6")


@pytest.fixture(scope="session")
def cfg_6x6_dense(scenario_dir):
    return _make(scenario_dir, 6, 6, "g6d", dense=dict(frac=1.0, interval=4.0, seed=1))


@pytest.fixture(scope="session")
def cfg_6x6_rl(scenario_dir):
    return _make(scenario_dir, 6, 6, "g6rl", dense=dict(frac=1.0, interval=5.0, seed=2), rl_traffic_light=True)


@pytest.fixture(scope="session")
def cfg_hetero_halfstep(scenario_dir):
    """4x4 grid, interval = 0.5 s, every flow with its own (seeded) vehicle parameters: exercises the
    dt-dependent formulas (vehicle.cpp:244, :257-266, :278-281) and the per-template gathers."""
    import random
    from cityflow_b200 import scenario
    net = scenario.grid_roadnet(4, 4)
    flows = scenario.random_walk_flows(net, frac=1.0, interval=4.0, seed=7)
    rng = random.Random(11)
    for f in flows:
        f["vehicle"] = {
            "length": rng.choice([4.0, 5.0, 6.5, 12.0]), "width": 2.0,
            "maxPosAcc": rng.choice([1.5, 2.0, 3.0]), "maxNegAcc": rng.choice([3.5, 4.5, 6.0]),
            "usualPosAcc": rng.choice([1.0, 2.0, 2.5]), "usualNegAcc": rng.choice([2.5, 3.5, 4.5]),
            "minGap": rng.choice([1.5, 2.5, 3.0]), "maxSpeed": rng.choice([8.0, 11.11, 16.67, 20.0]),
            "headwayTime": rng.choice([1.0, 1.5, 2.0]),
        }
        f["interval"] = float(rng.choice([3, 4, 5, 7]))
        f["startTime"] = rng.choice([0, 0, 10, 50])
        f["endTime"] = rng.choice([-1, -1, 400])
    return scenario.write_scenario(scenario_dir, net, flows, interval=0.5, seed=3, name="hetero")


def _irregular_net(seed=5):
    """A 3x3 grid bent out of shape: road polylines with interior points, unequal lane widths and
    speed limits, laneLinks WITHOUT explicit points (the loader's default curve, roadnet.cpp:212-247),
    odd intersection widths and phase times.  Exercises the geometry code the generator's tidy
    output never reaches."""
    import random
    from cityflow_b200 import scenario
    rng = random.Random(seed)
    net = scenario.grid_roadnet(3, 3)
    for road in net["roads"]:
        a, b = road["points"]
        mx, my = (a["x"] + b["x"]) / 2, (a["y"] + b["y"]) / 2
        dx, dy = b["x"] - a["x"], b["y"] - a["y"]
        k = rng.uniform(-0.08, 0.08)
        road["points"] = [a, {"x": mx - dy * k, "y": my + dx * k}, b]          # a bend
        road["lanes"] = [{"width": rng.choice([3, 3.5, 4]), "maxSpeed": rng.choice([11.11, 13.89, 16.67])} for _ in road["lanes"]]
    for inter in net["intersections"]:
        if inter["virtual"]:
            continue
        inter["width"] = rng.choice([20, 25, 30, 12.5])
        for i, rl in enumerate(inter["roadLinks"]):
            for j, ll in enumerate(rl["laneLinks"]):
                if (i + j) % 2 == 0:
                    ll.pop("points")                                             # default curve
                elif (i + j) % 5 == 0:
                    ll["points"] = []                                            # empty list = default curve too
        for ph in inter["trafficLight"]["lightphases"]:
            ph["time"] = rng.choice([5, 17, 30, 12.5])
    return net


@pytest.fixture(scope="session")
def cfg_irregular(scenario_dir):
    from cityflow_b200 import scenario
    net = _irregular_net()
    flows = scenario.random_walk_flows(net, frac=1.0, interval=4.0, seed=9)
    return scenario.write_scenario(scenario_dir, net, flows, seed=7, name="irregular")


@pytest.fixture(scope="session")
def cfg_replay(scenario_dir):
    """saveReplay on, on the irregular network, with vehicles of assorted lengths and widths
    (the replay line carries both).  Returns the config path; the log files land next to it."""
    import random
    from cityflow_b200 import scenario
    net = _irregular_net(seed=11)
    flows = scenario.random_walk_flows(net, frac=1.0, interval=5.0, seed=3)
    rng = random.Random(2)
    for f in flows:
        f["vehicle"]["length"] = rng.choice([4.0, 5.0, 7.5, 12.25])
        f["vehicle"]["width"] = rng.choice([1.8, 2.0, 2.55])
    return scenario.write_scenario(scenario_dir, net, flows, seed=4, save_replay=True, name="replay")
