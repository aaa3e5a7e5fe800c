"""Seeded road networks in the reference's JSON format, each built to push the step kernels past a loop bound or a
fixed capacity that the grid generator and tests/randnet.py never reach:

* ``long_queue`` -- a corridor with 600-1500 m roads, 2-4 lanes and one intersection up to 80 m wide, a fleet of
  1.5-2.0 m vehicles with a 0.5 m minGap (and a few 12 m trucks on the other direction).  Long fixed-time red phases
  fill lanes end to end and back the queue up onto the wide intersection's laneLinks: buckets with more than 96
  vehicles (3+ warp chunks, more than bumper-to-bumper 2.5 m vehicles fit) and laneLinks with more than 32.
* ``star`` -- intersections with 8 and 6 legs of 4 lanes each, most lane pairs linked, phases that let conflicting
  movements run together: laneLinks with more than 64 crosses (three 32-bit mask words) and lanes fed by 12 or
  more laneLinks.
* ``short_hops`` -- 8-25 m lanes between intersections 3-6 m wide, fast vehicles with short headways and a 2 s
  step: vehicles crossing 3 or more drivables in one step, leader searches over many drivables, and several
  entrants per lane per step.

* ``merge_ties`` -- the opposite: parallel, bit-equal approaches whose flows share one vehicle template per group and
  run in lockstep, so that 2, 3 and 4 vehicles enter one lane in the same step at the same distance, on an empty
  lane and behind survivors, and (two target lanes) vehicles on neighbouring lanes share a distance.  It exercises
  the tie rule: same-step entrants with equal distance are ordered by ascending priority.

In the first three shapes every flow has its own vehicle parameters (as scenario.random_walk_flows' fleet_spread
does), so that two entrants never tie and the unmodified reference's result is defined.  The unmodified reference
breaks ties by heap address, so merge_ties is compared with it only up to its first tie, and beyond that with the
priority-ordered build (oracle/lc_order_patch.sh), whose tie order is ascending priority while at most 16 vehicles
change drivable per step.  Flow intervals are at least 1 s (flow.h:34 asserts it).  The fixed-time plans hold the
approaches red, not rlTrafficLight: the unmodified reference is run from the JSON alone.

The ``reach`` helpers measure what a run actually reached, so that a test can assert its edge."""
import math
import random

import numpy as np


def _heading(road, at_end):
    p = road["points"]
    a, b = (p[-2], p[-1]) if at_end else (p[0], p[1])
    return math.atan2(b["y"] - a["y"], b["x"] - a["x"])


def _network(pos, virtual, widths, edges, lanes_of, speed_of, link_frac, rng):
    """Roads for every directed (s, e) in `edges` (both directions), laneLinks with the loader's default curve for a
    fraction `link_frac` of the lane pairs of every non-U-turn roadLink.  Intersections get no phases here."""
    roads, out_of, in_to = [], {}, {}
    for a, b in edges:
        for s, e in ((a, b), (b, a)):
            rid = "r_%s__%s" % (s, e)
            road = {"id": rid, "points": [{"x": pos[s][0], "y": pos[s][1]}, {"x": pos[e][0], "y": pos[e][1]}],
                    "lanes": [{"width": 3.5, "maxSpeed": speed_of(s, e)} for _ in range(lanes_of(s, e))],
                    "startIntersection": "n_%s" % s, "endIntersection": "n_%s" % e}
            roads.append(road)
            out_of.setdefault(s, []).append(road)
            in_to.setdefault(e, []).append(road)
    inters = {}
    for node in pos:
        ins, outs = in_to.get(node, []), out_of.get(node, [])
        inter = {"id": "n_%s" % node, "point": {"x": pos[node][0], "y": pos[node][1]},
                 "width": 0 if virtual[node] else widths[node], "roads": [r["id"] for r in ins + outs], "roadLinks": [],
                 "trafficLight": {"roadLinkIndices": [], "lightphases": []}, "virtual": virtual[node]}
        if not virtual[node]:
            for ra in ins:
                for rb in outs:
                    if rb["endIntersection"] == ra["startIntersection"]:
                        continue                                    # no U-turns
                    turn = (_heading(rb, False) - _heading(ra, True) + math.pi) % (2 * math.pi) - math.pi
                    kind = "go_straight" if abs(turn) < 0.6 else ("turn_left" if turn > 0 else "turn_right")
                    na, nb = len(ra["lanes"]), len(rb["lanes"])
                    pairs = [(c, d) for c in range(na) for d in range(nb) if rng.random() < link_frac]
                    if not pairs:
                        pairs = [(rng.randrange(na), rng.randrange(nb))]
                    inter["roadLinks"].append({"type": kind, "startRoad": ra["id"], "endRoad": rb["id"], "direction": 0,
                                               "laneLinks": [{"startLaneIndex": c, "endLaneIndex": d} for c, d in pairs]})
        inters[node] = inter
    return {"intersections": [inters[n] for n in sorted(pos)], "roads": roads}


def _set_phases(inter, phases):
    n = len(inter["roadLinks"])
    inter["trafficLight"] = {"roadLinkIndices": list(range(n)),
                             "lightphases": [{"time": t, "availableRoadLinks": sorted(set(a))} for t, a in phases]}


def _vehicle(rng, length, min_gap, max_speed, headway):
    """Own parameters for one flow: nothing two flows share, so entrants never tie."""
    return {"length": length, "width": 2.0,
            "maxPosAcc": rng.uniform(1.8, 3.0), "maxNegAcc": rng.uniform(4.0, 6.0),
            "usualPosAcc": rng.uniform(1.5, 2.5), "usualNegAcc": rng.uniform(2.5, 4.0),
            "minGap": min_gap, "maxSpeed": max_speed, "headwayTime": headway}


def _next_roads(net):
    nxt = {}
    for inter in net["intersections"]:
        for rl in inter["roadLinks"]:
            nxt.setdefault(rl["startRoad"], set()).add(rl["endRoad"])
    return {k: sorted(v) for k, v in nxt.items()}


def _entry_roads(net):
    """Roads that start at a virtual intersection (the network's edge), sorted."""
    virtual = {i["id"]: i["virtual"] for i in net["intersections"]}
    return sorted(r["id"] for r in net["roads"] if virtual[r["startIntersection"]])


def long_queue(seed: int):
    """(roadnet, flows): W - A - B - E corridor along x, a north and a south leg at A and at B.  A is 60-80 m wide;
    A gives the movements into the A-B road 400 s of green (and everything else 30 s); B holds that road red for
    300 s, so it fills end to end and its queue backs up onto A's laneLinks."""
    rng = random.Random(seed)
    L = lambda: rng.uniform(600, 1500)
    xa = L()
    xb = xa + rng.uniform(600, 700)            # the corridor that fills: short enough to fill within a few hundred steps
    xe = xb + L()
    pos = {"W": (0.0, 0.0), "A": (xa, 0.0), "B": (xb, 0.0), "E": (xe, 0.0),
           "AN": (xa, L()), "AS": (xa, -L()), "BN": (xb, L()), "BS": (xb, -L())}
    virtual = {k: k not in ("A", "B") for k in pos}
    widths = {"A": rng.uniform(60, 80), "B": rng.uniform(20, 30)}
    edges = [("W", "A"), ("A", "B"), ("B", "E"), ("AN", "A"), ("AS", "A"), ("BN", "B"), ("BS", "B")]
    nl = {e: rng.choice([2, 3, 4]) for e in edges}
    net = _network(pos, virtual, widths, edges, lambda s, e: nl.get((s, e), nl.get((e, s))),
                   lambda s, e: 13.89, 0.7, rng)
    for inter in net["intersections"]:
        rls = inter["roadLinks"]
        if inter["id"] == "n_A":
            east = [i for i, rl in enumerate(rls) if rl["endRoad"] == "r_A__B"]
            _set_phases(inter, [(400, east), (30, [i for i in range(len(rls)) if i not in east])])
        elif inter["id"] == "n_B":
            held = [i for i, rl in enumerate(rls) if rl["startRoad"] == "r_A__B"]
            _set_phases(inter, [(300, [i for i in range(len(rls)) if i not in held]), (60, held)])
    nxt = _next_roads(net)
    flows = []
    # eastbound through the wide intersection: small vehicles, each flow its own
    for start in ("r_W__A", "r_AN__A", "r_AS__A"):
        for k in range(10):
            end = rng.choice(["r_B__E", "r_B__BN", "r_B__BS"])
            flows.append({"vehicle": _vehicle(rng, rng.uniform(1.5, 2.0), 0.5, rng.uniform(11.0, 16.0), rng.uniform(1.0, 1.6)),
                          "route": [start, "r_A__B", end], "interval": rng.uniform(1.0, 2.0),
                          "startTime": rng.choice([0, 0, 5, 20]), "endTime": -1})
    # westbound: small vehicles with a few trucks among them, red at A for 300 s
    for k in range(12):
        truck = k % 4 == 0
        start = rng.choice(["r_E__B", "r_BN__B", "r_BS__B"])
        veh = _vehicle(rng, 12.0, 2.0, rng.uniform(9.0, 11.0), rng.uniform(1.5, 2.0)) if truck else \
            _vehicle(rng, rng.uniform(1.5, 2.0), 0.5, rng.uniform(11.0, 16.0), rng.uniform(1.0, 1.6))
        flows.append({"vehicle": veh, "route": [start, "r_B__A", rng.choice(nxt["r_B__A"])],
                      "interval": rng.uniform(5.0, 9.0) if truck else rng.uniform(1.5, 3.0), "startTime": 0, "endTime": -1})
    return net, flows


def star(seed: int):
    """(roadnet, flows): an 8-leg and a 6-leg intersection joined by one road, 4 lanes everywhere, 85 % of all lane
    pairs linked; three phases that each release a random half of the roadLinks, conflicting ones included."""
    rng = random.Random(seed)
    pos = {"C1": (0.0, 0.0), "C2": (400.0, 0.0)}
    virtual = {"C1": False, "C2": False}
    widths = {"C1": rng.uniform(30, 40), "C2": rng.uniform(25, 35)}
    edges = [("C1", "C2")]
    for c, legs, skip in (("C1", 8, 0), ("C2", 6, 3)):
        cx, cy = pos[c]
        for j in range(legs):
            if j == skip and c == "C2":
                continue                                    # the leg towards C1 is the joining road
            if j == 0 and c == "C1":
                continue
            ang = (math.pi if c == "C1" else 0.0) + 2 * math.pi * j / legs + rng.uniform(-0.1, 0.1)
            leg = "%s_%d" % (c, j)
            r = rng.uniform(200, 300)
            pos[leg] = (cx + r * math.cos(ang), cy + r * math.sin(ang))
            virtual[leg] = True
            edges.append((leg, c))
    net = _network(pos, virtual, widths, edges, lambda s, e: 4, lambda s, e: rng.choice([11.11, 13.89, 16.67]), 0.85, rng)
    for inter in net["intersections"]:
        if inter["virtual"]:
            continue
        n = len(inter["roadLinks"])
        _set_phases(inter, [(rng.choice([15, 20, 30]), [i for i in range(n) if i % 3 == k or rng.random() < 0.3]) for k in range(3)])
    nxt = _next_roads(net)
    starts = _entry_roads(net)
    flows = []
    for k in range(70):
        s = rng.choice(starts)
        route = [s, rng.choice(nxt[s])]
        while route[-1] in nxt and len(route) < 3:
            route.append(rng.choice(nxt[route[-1]]))
        flows.append({"vehicle": _vehicle(rng, rng.uniform(4.0, 5.0), rng.uniform(1.5, 2.5), rng.uniform(10.0, 16.0), rng.uniform(1.0, 1.5)),
                      "route": route, "interval": rng.uniform(1.0, 4.0), "startTime": rng.choice([0, 0, 10]), "endTime": -1})
    return net, flows


def short_hops(seed: int, rows: int = 4, cols: int = 5):
    """(roadnet, flows): a lattice of intersections 3-6 m wide whose lanes are 8-25 m long, lanes allowing 30 m/s,
    fast vehicles with 0.3-0.6 s headways; long walks through the lattice.  Meant for a 2 s step.  Every lane pair is
    linked: a vehicle this fast cannot always stop at the end of a lane that does not continue its route, and the
    reference asserts when it passes one (vehicle.cpp:60)."""
    rng = random.Random(seed)
    R, C = rows + 2, cols + 2
    widths = {(i, j): rng.uniform(3, 6) for i in range(R) for j in range(C)}
    gx = [0.0]
    for j in range(1, C):
        gx.append(gx[-1] + rng.uniform(8, 25) + widths.get((1, j - 1), 0) + widths.get((1, j), 0))
    gy = [0.0]
    for i in range(1, R):
        gy.append(gy[-1] + rng.uniform(8, 25) + widths.get((i - 1, 1), 0) + widths.get((i, 1), 0))
    interior = lambda i, j: 0 < i < R - 1 and 0 < j < C - 1
    pos, virtual = {}, {}
    for i in range(R):
        for j in range(C):
            if (i in (0, R - 1)) and (j in (0, C - 1)):
                continue
            pos["%d_%d" % (i, j)] = (gx[j], gy[i])
            virtual["%d_%d" % (i, j)] = not interior(i, j)
    w = {"%d_%d" % k: v for k, v in widths.items()}
    edges = []
    for i in range(R):
        for j in range(C):
            a = "%d_%d" % (i, j)
            for di, dj in ((0, 1), (1, 0)):
                b = "%d_%d" % (i + di, j + dj)
                if a in pos and b in pos and (not virtual[a] or not virtual[b]):
                    edges.append((a, b))
    nl = {e: rng.choice([1, 2]) for e in edges}
    net = _network(pos, virtual, w, edges, lambda s, e: nl.get((s, e), nl.get((e, s))), lambda s, e: 30.0, 1.0, rng)
    for inter in net["intersections"]:
        if inter["virtual"]:
            continue
        n = len(inter["roadLinks"])
        _set_phases(inter, [(60, list(range(n))), (rng.choice([4, 6]), [i for i in range(n) if i % 2 == 0])])
    nxt = _next_roads(net)
    starts = _entry_roads(net)
    flows = []
    for k in range(40):
        route = [rng.choice(starts)]
        while len(route) < 9:                               # no road twice: the router's quirks with revisits stay out
            options = [r for r in nxt.get(route[-1], []) if r not in route]
            if not options:
                break
            route.append(rng.choice(options))
        flows.append({"vehicle": _vehicle(rng, rng.uniform(4.0, 5.0), rng.uniform(1.0, 2.0), rng.uniform(27.0, 32.0), rng.uniform(0.3, 0.6)),
                      "route": route, "interval": rng.uniform(2.0, 5.0), "startTime": rng.choice([0, 0, 10]), "endTime": -1})
    for f in flows:
        f["vehicle"]["maxPosAcc"] = rng.uniform(5.0, 8.0)
        f["vehicle"]["usualPosAcc"] = rng.uniform(4.0, 5.0)
    return net, flows


MERGE_GROUPS = {"P": (0, 0, 1, 1), "Q": (0, 0, 0), "R": (1, 1, 1, 1)}   # target lane on I -> J of every approach road


def merge_ties(seed: int):
    """(roadnet, flows): single-lane approach roads into one merge intersection I, then a two-lane road I -> J to a
    second real intersection J and an exit road.  The approach roads are parallel translates of each other along y
    (lane lengths are then computed from x alone, so they are bit-equal), and so are their laneLinks into I -> J:
    explicit two-point horizontal polylines of equal x span, so they are parallel, have no crosses, and leave nothing
    at I that could tell two approaches apart.  One phase releases every movement at I and at J.

    Every merge group of MERGE_GROUPS has one vehicle template and one (interval, startTime) shared by its flows, one
    flow per approach road: its vehicles run in lockstep and enter their target lane in the same step at the same
    distance.  P sends a pair into each lane (equal distances on neighbouring lanes), Q three and R four vehicles into
    one lane.  Two background flows with their own parameters use approaches of their own, one per target lane, so
    that ties also land behind survivors."""
    rng = random.Random(seed)
    w_i, w_j = rng.uniform(10, 14), rng.uniform(8, 12)
    d_ij, l_app, l_exit = rng.uniform(220, 260), 300.0, 300.0
    approaches = [("%s%d" % (g, k), t) for g, lanes in sorted(MERGE_GROUPS.items()) for k, t in enumerate(lanes)]
    approaches += [("B0", 0), ("B1", 1)]
    inters = {"I": {"id": "n_I", "point": {"x": 0.0, "y": 0.0}, "width": w_i, "roads": [], "roadLinks": [], "virtual": False},
              "J": {"id": "n_J", "point": {"x": d_ij, "y": 0.0}, "width": w_j, "roads": [], "roadLinks": [], "virtual": False},
              "X": {"id": "n_X", "point": {"x": d_ij + l_exit, "y": 0.0}, "width": 0, "roads": [], "roadLinks": [], "virtual": True}}
    lane = lambda: {"width": 3.5, "maxSpeed": 13.89}

    def road(rid, a, b, pa, pb, n):
        inters[a]["roads"].append(rid)
        inters[b]["roads"].append(rid)
        return {"id": rid, "points": [{"x": pa[0], "y": pa[1]}, {"x": pb[0], "y": pb[1]}], "lanes": [lane() for _ in range(n)],
                "startIntersection": inters[a]["id"], "endIntersection": inters[b]["id"]}

    roads = []
    for k, (name, target) in enumerate(approaches):
        y = 12.0 * (k + 1)
        inters[name] = {"id": "n_%s" % name, "point": {"x": -l_app, "y": y}, "width": 0, "roads": [], "roadLinks": [], "virtual": True}
        roads.append(road("r_%s__I" % name, name, "I", (-l_app, y), (0.0, y), 1))
        inters["I"]["roadLinks"].append({"type": "go_straight", "startRoad": "r_%s__I" % name, "endRoad": "r_I__J", "direction": 0,
                                         "laneLinks": [{"startLaneIndex": 0, "endLaneIndex": target,
                                                        "points": [{"x": -w_i, "y": y}, {"x": w_i, "y": y}]}]})
    roads.append(road("r_I__J", "I", "J", (0.0, 0.0), (d_ij, 0.0), 2))
    roads.append(road("r_J__X", "J", "X", (d_ij, 0.0), (d_ij + l_exit, 0.0), 2))
    inters["J"]["roadLinks"].append({"type": "go_straight", "startRoad": "r_I__J", "endRoad": "r_J__X", "direction": 0,
                                     "laneLinks": [{"startLaneIndex": 0, "endLaneIndex": 0}, {"startLaneIndex": 1, "endLaneIndex": 1}]})
    for inter in inters.values():
        inter["trafficLight"] = {"roadLinkIndices": [], "lightphases": []}
        if not inter["virtual"]:
            _set_phases(inter, [(60, list(range(len(inter["roadLinks"]))))])
    net = {"intersections": [inters[k] for k in sorted(inters)], "roads": roads}
    flows = []
    timing = {"P": (12.0, 0), "Q": (16.0, 4), "R": (20.0, 8)}
    for g in sorted(MERGE_GROUPS):
        veh = _vehicle(rng, rng.uniform(4.0, 5.0), rng.uniform(2.0, 2.5), rng.uniform(11.0, 13.0), rng.uniform(1.0, 1.5))
        interval, start = timing[g]
        for k in range(len(MERGE_GROUPS[g])):
            flows.append({"vehicle": dict(veh), "route": ["r_%s%d__I" % (g, k), "r_I__J", "r_J__X"], "interval": interval,
                          "startTime": start, "endTime": -1})
    for name in ("B0", "B1"):
        flows.append({"vehicle": _vehicle(rng, rng.uniform(4.0, 6.0), rng.uniform(2.0, 2.5), rng.uniform(10.0, 14.0), rng.uniform(1.0, 1.5)),
                      "route": ["r_%s__I" % name, "r_I__J", "r_J__X"], "interval": rng.uniform(15.0, 25.0), "startTime": rng.choice([0, 2]),
                      "endTime": -1})
    return net, flows


def merge_approach_lanes(cfg: str) -> dict:
    """{group: lane indices of its approach roads} of a merge_ties config ("B": the background approaches)."""
    import json
    c = json.load(open(cfg))
    lane, out = 0, {}
    for r in json.load(open(c["dir"] + c["roadnetFile"]))["roads"]:
        if r["id"].endswith("__I"):
            out.setdefault(r["id"][2], []).append(lane)
        lane += len(r["lanes"])
    return out


SHAPES = {"long_queue": (long_queue, 1.0), "star": (star, 1.0), "short_hops": (short_hops, 2.0), "merge_ties": (merge_ties, 1.0)}


def write(shape: str, directory: str, seed: int = 1, lane_change: bool = False) -> str:
    """The config of `shape` (seeded) in `directory`, with the step interval the shape is built for."""
    from cityflow_b200 import scenario
    make, interval = SHAPES[shape]
    net, flows = make(seed)
    return scenario.write_scenario(directory, net, flows, interval=interval, seed=seed, lane_change=lane_change,
                                   name="%s%d%s" % (shape, seed, "_lc" if lane_change else ""))


def write_spawn_burst(directory: str, n_flows: int = 2200) -> str:
    """A 4x4 grid with `n_flows` single-vehicle flows that all start at t = 0, so that the first step hands the device more
    spawn records than k_ingest stages in shared memory (SPAWN_SMEM = 2048)."""
    from cityflow_b200 import scenario
    net = scenario.grid_roadnet(4, 4)
    base = scenario.random_walk_flows(net, frac=1.0, interval=5.0, seed=4)
    flows = []
    for k in range(n_flows):
        f = dict(base[k % len(base)])
        f["vehicle"] = dict(f["vehicle"])
        f["interval"], f["startTime"], f["endTime"] = 1.0, 0, 0
        flows.append(f)
    return scenario.write_scenario(directory, net, flows, seed=5, name="burst")


def loader_tables(cfg: str) -> dict:
    """The static tables of the product's loader (tests/loader_probe.cpp, built into oracle/_build like
    tests/test_cpu.py's _dump_static): lane_out, link_end, link_cross_count, ..."""
    import json
    import os
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    probe = os.path.join(root, "oracle", "_build", "loader_probe")
    src = os.path.join(root, "tests", "loader_probe.cpp")
    csrc = os.path.join(root, "cityflow_b200", "csrc")
    os.makedirs(os.path.dirname(probe), exist_ok=True)
    if not os.path.exists(probe) or os.path.getmtime(probe) < max(os.path.getmtime(src), os.path.getmtime(os.path.join(csrc, "roadnet.cpp"))):
        subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", src, os.path.join(csrc, "roadnet.cpp"),
                               os.path.join(csrc, "flows.cpp"), "-o", probe])
    return json.loads(subprocess.check_output([probe, cfg]))


# ---------------------------------------------------------------- what a run reached
class Reach:
    """Maxima over a run, fed one state after the other: vehicles on one drivable, entrants into one drivable in one
    step, drivables crossed by one vehicle in one step (a lower bound: the shortest path between the two drivables)."""

    def __init__(self, static):
        self.n_lanes = static["n_lanes"]
        self.lane_out = static["lane_out"]
        self.link_end = static["link_end"]
        self.lane_occ = self.link_occ = self.entrants = self.hops = 0
        self.prev = None
        self._dist = {}

    def _hops(self, a, b):
        """Drivables entered on the shortest way from drivable a to drivable b (lanes -> laneLinks -> end lanes)."""
        if (a, b) in self._dist:
            return self._dist[(a, b)]
        frontier, seen, k = [a], {a}, 0
        while frontier and b not in seen and k < 64:
            k += 1
            nxt = []
            for d in frontier:
                succ = [self.n_lanes + x for x in self.lane_out[d]] if d < self.n_lanes else [self.link_end[d - self.n_lanes]]
                for s in succ:
                    if s not in seen:
                        seen.add(s)
                        nxt.append(s)
            frontier = nxt
        self._dist[(a, b)] = k if b in seen else 0
        return self._dist[(a, b)]

    def add(self, vehicles):
        """`vehicles`: VEH_DTYPE (or LC_DTYPE) records of one step, shadows excluded."""
        drv = vehicles["drivable"]
        if len(drv):
            occ = np.bincount(drv)
            self.lane_occ = max(self.lane_occ, int(occ[:self.n_lanes].max(initial=0)))
            self.link_occ = max(self.link_occ, int(occ[self.n_lanes:].max(initial=0)))
        now = {(int(f), int(c)): int(d) for f, c, d in zip(vehicles["flow"], vehicles["cnt"], drv)}
        if self.prev is not None:
            into = {}
            for key, d in now.items():
                p = self.prev.get(key)
                if p is not None and p != d:
                    into[d] = into.get(d, 0) + 1
                    self.hops = max(self.hops, self._hops(p, d))
            self.entrants = max([self.entrants] + list(into.values()))
        self.prev = now

    def __str__(self):
        return "max vehicles on a lane %d, on a laneLink %d; max entrants into one drivable in one step %d; max drivables " \
               "crossed in one step %d" % (self.lane_occ, self.link_occ, self.entrants, self.hops)
