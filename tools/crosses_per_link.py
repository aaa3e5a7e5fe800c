"""Crosses per laneLink of the bench roadnet (30x30 grid), from the product loader's static tables: the number of lanes
k_notify puts on one laneLink (one per cross, in chunks of its 16-lane tile).

    python tools/crosses_per_link.py
"""
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    from cityflow_b200 import scenario
    csrc = os.path.join(ROOT, "cityflow_b200", "csrc")
    with tempfile.TemporaryDirectory() as d:
        probe = os.path.join(d, "loader_probe")
        subprocess.check_call(["g++", "-std=c++17", "-O1", os.path.join(ROOT, "tests", "loader_probe.cpp"),
                               os.path.join(csrc, "roadnet.cpp"), os.path.join(csrc, "flows.cpp"), "-o", probe])
        cfg = scenario.make_grid_scenario(d, 30, 30, dense=dict(frac=0.5, interval=10.0, seed=1), name="bench")
        t = json.loads(subprocess.check_output([probe, cfg]))
    per = np.zeros(t["n_links"], np.int64)
    # an entry is [cross, side, crossing link, ...]: every cross of link l appears once on the crossing link's list
    # with l as ITS crossing link, so a link's own count is how often it is named as the crossing link
    for c in t["crosses"]:
        per[c[2] - t["n_lanes"]] += 1
    print(json.dumps({"links": int(len(per)), "crosses": int(per.sum()), "mean": float(per.mean()), "max": int(per.max()),
                      "share_le_16": float((per <= 16).mean()),
                      "hist": {int(k): int(v) for k, v in enumerate(np.bincount(per)) if v}}))


if __name__ == "__main__":
    main()
