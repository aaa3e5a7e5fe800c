"""More seeds of the fuzz / API parity checks that `pytest -m gpu` runs (tests/test_gpu_parity.py: test_fuzzed_irregular_networks_vs_port,
test_fuzzed_network_vs_compiled_reference, test_vehicle_setters_step_by_step_vs_port):

    python tools/gpu_fuzz_check.py [first_seed last_seed]

1. random irregular networks (tests/randnet.py): GPU engine vs the restatement, full state every step -- including networks
   where a vehicle starts on a lane that cannot continue its route (the reference parks it at the end of the lane,
   vehicle.cpp:323-329, and so does the engine).
2. set_vehicle_speed / set_vehicle_route step by step against the restatement (pinned against the reference's Python module
   by tests/test_cpu.py::test_port_oracle_vs_reference_python_api).
"""
import os
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from cityflow_b200 import scenario  # noqa: E402
from oracle import harness as H  # noqa: E402


def gpu_state(eng, step):
    st = H.StepState()
    st.step = step
    st.vehicle_count = eng.vehicle_count()
    st.pool_size = st.finished = 0
    st.cum_travel_time = 0.0
    st.lane_count = eng.lane_vehicle_count()
    st.lane_waiting = eng.lane_waiting_count()
    st.lane_queue = st.phases = st.order = None
    st.vehicles = eng.debug_vehicles()
    return st


def relax(ref):
    ref.pool_size = ref.finished = 0
    ref.cum_travel_time = 0.0
    return ref


def fuzz(first, last, steps=500):
    import randnet
    from cityflow_b200.capi import CEngine
    d = tempfile.mkdtemp()
    summary = {"equal": 0, "dead_end_divergence": 0, "UNEXPECTED": 0}
    for seed in range(first, last):
        net = randnet.random_roadnet(seed, rows=2 + seed % 3, cols=3 + seed % 2)
        flows = randnet.random_flows(net, seed + 100, n_flows=40 + seed % 50)
        cfg = scenario.write_scenario(d, net, flows, seed=seed, interval=[1.0, 0.5, 2.0, 1.0][seed % 4], name="g%d" % seed)
        eng, ora = CEngine(cfg), H.PortOracle(cfg)
        verdict = "equal"
        for s in range(1, steps + 1):
            ora.next_step()
            try:
                eng.next_step()
                bad = H.compare_states(relax(ora.snapshot()), gpu_state(eng, s))
            except RuntimeError as e:
                verdict = "dead_end_divergence" if "cannot continue its route" in str(e) else "UNEXPECTED"
                print("seed %d step %d: engine error: %s" % (seed, s, str(e)[:120]))
                break
            if bad:
                # a vehicle braking for the end of a dead-end lane changes everything behind it: a mismatch is
                # the known divergence iff the restatement holds such a vehicle at this point
                ora.lib.cfo_invalid_lane_vehicles.restype = __import__('ctypes').c_int; ora.lib.cfo_invalid_lane_vehicles.argtypes = [__import__('ctypes').c_void_p]
                verdict = "dead_end_divergence" if ora.lib.cfo_invalid_lane_vehicles(ora.h) > 0 else "UNEXPECTED"
                print("seed %d step %d: %s" % (seed, s, "; ".join(bad[:3])))
                break
        summary[verdict] += 1
        print("seed %d: %s" % (seed, verdict))
    print("fuzz summary:", summary)
    return summary["UNEXPECTED"] == 0


def api_vs_restatement(steps=400):
    import json
    import cityflow
    d = tempfile.mkdtemp()
    cfg = scenario.make_grid_scenario(d, 4, 4, dense=dict(frac=1.0, interval=3.0, seed=2), name="api")
    flows = json.load(open(os.path.join(d, "flow_api.json")))
    eng, ora = cityflow.Engine(cfg, thread_num=1), H.PortOracle(cfg)

    def vid(f, k):
        return "manually_pushed_%d" % k if f == -2 else "flow_%d_%d" % (f, k)

    ok = True
    for s in range(1, steps + 1):
        v = ora.vehicles()
        if s % 20 == 3:
            for j in range(0, len(v), max(1, len(v) // 6)):
                f, k, sp = int(v["flow"][j]), int(v["cnt"][j]), float(v["speed"][j]) * 0.5
                eng.set_vehicle_speed(vid(f, k), sp)
                assert ora.set_vehicle_speed(f, k, sp)
        if s % 30 == 7:
            for j in range(1, len(v), max(1, len(v) // 8)):
                f, k = int(v["flow"][j]), int(v["cnt"][j])
                target = flows[(s + j) % len(flows)]["route"][-1:]
                a, b = eng.set_vehicle_route(vid(f, k), target), ora.set_vehicle_route(f, k, target)
                if a != b:
                    print("step %d %s -> %s: engine %s restatement %s" % (s, vid(f, k), target, a, b))
                    ok = False
        eng.next_step()
        ora.next_step()
        v = ora.vehicles()
        mine = eng.get_vehicle_speed()
        theirs = {vid(f, k): sp for f, k, sp in zip(v["flow"], v["cnt"], v["speed"])}
        if mine != theirs:
            diff = [k for k in theirs if mine.get(k) != theirs[k]][:3]
            print("step %d: speeds differ, e.g. %s" % (s, [(k, mine.get(k), theirs[k]) for k in diff]))
            ok = False
            break
    print("set_vehicle_speed / set_vehicle_route vs restatement:", "equal" if ok else "DIFFERENT")
    return ok


if __name__ == "__main__":
    a, b = (int(sys.argv[1]), int(sys.argv[2])) if len(sys.argv) > 2 else (1, 13)
    r1 = fuzz(a, b)
    r2 = api_vs_restatement()
    sys.exit(0 if (r1 and r2) else 1)
