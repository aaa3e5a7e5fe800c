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

``replicated`` puts K disjoint copies of a small scenario (a dense 2x2 grid, or long_queue) into one roadnet, so that the
per-step counts of lane change (candidates, involved vehicles, new shadows) grow K-fold while the restatement stays
affordable.

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


def merge_ties(seed: int, groups=MERGE_GROUPS, background=True):
    """(roadnet, flows): single-lane approach roads into one merge intersection I, then a two-lane road I -> J to a
    second real intersection J and an exit road.  The approach roads are parallel translates of each other along y
    (lane lengths are then computed from x alone, so they are bit-equal), and so are their laneLinks into I -> J:
    explicit two-point horizontal polylines of equal x span, so they are parallel, have no crosses, and leave nothing
    at I that could tell two approaches apart.  One phase releases every movement at I and at J.

    Every merge group of MERGE_GROUPS has one vehicle template and one (interval, startTime) shared by its flows, one
    flow per approach road: its vehicles run in lockstep and enter their target lane in the same step at the same
    distance.  P sends a pair into each lane (equal distances on neighbouring lanes), Q three and R four vehicles into
    one lane.  Two background flows with their own parameters use approaches of their own, one per target lane, so
    that ties also land behind survivors.  `groups` / `background` replace the merge groups and drop the background
    flows (merge_16)."""
    rng = random.Random(seed)
    w_i, w_j = rng.uniform(10, 14), rng.uniform(8, 12)
    d_ij, l_app, l_exit = rng.uniform(220, 260), 300.0, 300.0
    approaches = [("%s%d" % (g, k), t) for g, lanes in sorted(groups.items()) for k, t in enumerate(lanes)]
    if background:
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
    for g in sorted(groups):
        veh = _vehicle(rng, rng.uniform(4.0, 5.0), rng.uniform(2.0, 2.5), rng.uniform(11.0, 13.0), rng.uniform(1.0, 1.5))
        interval, start = timing.get(g, (20.0, 0))
        for k in range(len(groups[g])):
            flows.append({"vehicle": dict(veh), "route": ["r_%s%d__I" % (g, k), "r_I__J", "r_J__X"], "interval": interval,
                          "startTime": start, "endTime": -1})
    for name in ("B0", "B1") if background else ():
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


# merge_16: sixteen approaches in lockstep into lane 0 of I -> J -- ENT_CAP = 16 entrants of one lane in one step, one
# full mover message when I -> J is a seam lane.  No background flows: a 17th entrant would overflow ENT_CAP.
SHAPES = {"long_queue": (long_queue, 1.0), "star": (star, 1.0), "short_hops": (short_hops, 2.0), "merge_ties": (merge_ties, 1.0),
          "merge_16": (lambda seed: merge_ties(seed, {"W": (0,) * 16}, background=False), 1.0)}


def write(shape: str, directory: str, seed: int = 1, lane_change: bool = False) -> str:
    """The config of `shape` (seeded) in `directory`, with the step interval the shape is built for."""
    from cityflow_b200 import scenario
    make, interval = SHAPES[shape]
    net, flows = make(seed)
    return scenario.write_scenario(directory, net, flows, interval=interval, seed=seed, lane_change=lane_change,
                                   name="%s%d%s" % (shape, seed, "_lc" if lane_change else ""))


def _grid2x2_unit(seed):
    """A dense 2x2 grid: every road with a successor starts a flow, one vehicle every 2 s."""
    from cityflow_b200 import scenario
    net = scenario.grid_roadnet(2, 2)
    return net, scenario.random_walk_flows(net, frac=1.0, interval=2.0, seed=seed)


# unit: (roadnet and flows of a seed, default seed, step interval)
REPLICA_UNITS = {"grid2x2": (_grid2x2_unit, 3, 1.0), "long_queue": (long_queue, 1, 1.0)}


def replicated(unit: str, k: int, seed=None, dx: float = 5000.0):
    """(roadnet, flows): `k` disjoint copies of `unit`, copy c prefixed "c<c>_" in every intersection, road and route id
    and moved by c * dx along x (every point: roads, intersections, laneLinks).  Nothing joins two copies, so a run
    carries k independent scenarios and its per-step counts (vehicles, lane-change candidates, shadows) grow k-fold."""
    import copy
    make, default_seed, _ = REPLICA_UNITS[unit]
    net, flows = make(default_seed if seed is None else seed)

    def moved(p, c):
        return {**p, "x": p["x"] + c * dx}

    out_net, out_flows = {"intersections": [], "roads": []}, []
    for c in range(k):
        pre = "c%d_" % c
        for inter in net["intersections"]:
            i = copy.deepcopy(inter)
            i["id"] = pre + i["id"]
            i["point"] = moved(i["point"], c)
            i["roads"] = [pre + r for r in i["roads"]]
            for rl in i["roadLinks"]:
                rl["startRoad"], rl["endRoad"] = pre + rl["startRoad"], pre + rl["endRoad"]
                for ll in rl["laneLinks"]:
                    if "points" in ll:
                        ll["points"] = [moved(p, c) for p in ll["points"]]
            out_net["intersections"].append(i)
        for road in net["roads"]:
            r = copy.deepcopy(road)
            r["id"] = pre + r["id"]
            r["startIntersection"], r["endIntersection"] = pre + r["startIntersection"], pre + r["endIntersection"]
            r["points"] = [moved(p, c) for p in r["points"]]
            out_net["roads"].append(r)
        for f in flows:
            g = copy.deepcopy(f)
            g["route"] = [pre + r for r in g["route"]]
            out_flows.append(g)
    return out_net, out_flows


def write_replicated(directory: str, k: int, unit: str = "grid2x2", lane_change: bool = True, seed=None, dx: float = 5000.0) -> str:
    """The config of `k` disjoint copies of `unit` (see replicated) in `directory`, at the unit's step interval."""
    from cityflow_b200 import scenario
    net, flows = replicated(unit, k, seed, dx)
    s = REPLICA_UNITS[unit][1] if seed is None else seed
    return scenario.write_scenario(directory, net, flows, interval=REPLICA_UNITS[unit][2], seed=s, lane_change=lane_change,
                                   name="%s_x%d%s" % (unit, k, "_lc" if lane_change else ""))


def device_form_restatement(cfg: str):
    """The restatement (oracle.harness.PortOracle) in the decomposition the device runs (cfo_set_device_form): bit-equal
    to the default form, and it counts the sizes of the lane-change step's sequential parts (cfo_device_form_stats)."""
    import ctypes
    from oracle import harness as H
    o = H.PortOracle(cfg)
    o.lib.cfo_set_device_form.restype = None
    o.lib.cfo_set_device_form.argtypes = [ctypes.c_void_p, ctypes.c_int]
    o.lib.cfo_set_device_form(o.h, 1)
    return o


def lc_records(eng):
    """cfb_debug_lc_vehicles of a CEngine: every running vehicle, shadows included, as oracle.harness.LC_DTYPE records in
    ascending priority.  Identities are priorities, never slots."""
    import ctypes
    from oracle import harness as H
    lib = eng.lib
    lib.cfb_debug_lc_vehicles.restype = ctypes.c_int64
    lib.cfb_debug_lc_vehicles.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int64]
    n = int(lib.cfb_debug_lc_vehicles(eng.h, None, 0))
    got = np.zeros(n, H.LC_DTYPE)
    if n:
        lib.cfb_debug_lc_vehicles(eng.h, got.ctypes.data, n)
    return got


class LcReach:
    """What a lane-change run reached, from the device-form restatement (device_form_restatement): the most candidates
    (vehicles asking to change lanes) and involved vehicles (caught up in a change) in one step, the most candidates on
    one road, and the most shadows created in one step (shadow priorities the step before did not have)."""

    def __init__(self, ora):
        import ctypes
        self.ora = ora
        ora.lib.cfo_device_form_stats.restype = None
        ora.lib.cfo_device_form_stats.argtypes = [ctypes.c_void_p, ctypes.c_void_p]
        self.new_shadows = self.shadow_states = self.steps = self.max_vehicles = 0
        self.prev = set()

    def add(self, records):
        sh = set(records["priority"][records["partner_type"] == 2].tolist())
        self.new_shadows = max(self.new_shadows, len(sh - self.prev))
        self.shadow_states += len(sh)
        self.max_vehicles = max(self.max_vehicles, len(records))
        self.prev = sh
        self.steps += 1

    def stats(self):
        import ctypes
        out = (ctypes.c_double * 6)()
        self.ora.lib.cfo_device_form_stats(self.ora.h, out)
        return dict(candidates=int(out[1]), candidates_on_a_road=int(out[2]), involved=int(out[4]))

    def __str__(self):
        s = self.stats()
        return ("%d steps, up to %d running vehicles: at most %d candidates (%d on one road), %d involved vehicles and %d new "
                "shadows in one step; %d shadow states" % (self.steps, self.max_vehicles, s["candidates"], s["candidates_on_a_road"],
                                                         s["involved"], self.new_shadows, self.shadow_states))


def lc_vs_restatement(engines: dict, cfg: str, steps: int) -> LcReach:
    """Step the lane-change engines of `engines` (name -> CEngine or its emulated-device form) and the device-form
    restatement together.  After every step, each engine's vehicle count, lane counts and records (lc_records: every
    field, shadows included, keyed by priority) must equal the restatement's.  Returns what the run reached."""
    import ctypes
    from oracle import harness as H
    ora = device_form_restatement(cfg)
    reach = LcReach(ora)
    lib = ora.lib
    lib.cfo_lc_vehicles.restype = ctypes.c_int
    lib.cfo_lc_vehicles.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int]
    for s in range(1, steps + 1):
        for eng in engines.values():
            eng.next_step()
        ora.next_step()
        want = np.zeros(lib.cfo_lc_vehicles(ora.h, None, 0), H.LC_DTYPE)   # lc_snapshot's records, without the list orders
        lib.cfo_lc_vehicles(ora.h, want.ctypes.data, len(want))
        count, lanes = ora.vehicle_count(), ora.lane_vehicle_count()
        reach.add(want)
        for name, eng in engines.items():
            got = lc_records(eng)
            assert eng.vehicle_count() == count, "%s, step %d" % (name, s)
            assert np.array_equal(eng.lane_vehicle_count(), lanes), "%s, lane counts, step %d" % (name, s)
            assert len(got) == len(want), "%s, step %d: %d records, restatement %d" % (name, s, len(got), len(want))
            for f in H.LC_DTYPE.names:
                bad = np.nonzero(got[f] != want[f])[0]
                assert not len(bad), "%s, step %d, field %s differs for %d vehicles, first priority %d: %r, restatement %r" % (
                    name, s, f, len(bad), want["priority"][bad[0]], got[f][bad[0]], want[f][bad[0]])
    return reach


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


# ---------------------------------------------------------------- cuts of a sharded run and what a run reached at them
def partition(cfg: str, world: int, owners=None) -> dict:
    """The product's partition of `cfg` (tests/partition_probe.cpp, built into oracle/_build like loader_tables): column
    strips, or Partition::fromOwners of `owners` (one rank per intersection, virtual ones included).  Keys: inter_owner,
    inter_virtual, lane_owner, lane_feeder, lane_start, lane_end, boundary[a][b] (lanes fed by a, owned by b)."""
    import json
    import os
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    probe = os.path.join(root, "oracle", "_build", "partition_probe")
    csrc = os.path.join(root, "cityflow_b200", "csrc")
    srcs = [os.path.join(root, "tests", "partition_probe.cpp"), os.path.join(csrc, "partition.cpp"), os.path.join(csrc, "roadnet.cpp")]
    os.makedirs(os.path.dirname(probe), exist_ok=True)
    deps = srcs + [os.path.join(csrc, "partition.h"), os.path.join(csrc, "roadnet.h")]
    if not os.path.exists(probe) or os.path.getmtime(probe) < max(os.path.getmtime(f) for f in deps):
        subprocess.check_call(["g++", "-std=c++17", "-O1"] + srcs + ["-o", probe])
    args = [probe, cfg, str(world)]
    if owners is not None:
        args += ["-1", ",".join(str(int(o)) for o in owners)]
    return json.loads(subprocess.check_output(args))


def look_ahead(cfg: str) -> float:
    """How far beyond its lane end a vehicle of `cfg` may look (HostEngine::configureShard's formula over the flows'
    vehicles): Partition::validate refuses a seam lane no longer than this."""
    import json
    c = json.load(open(cfg))
    look = 0.0
    for f in json.load(open(c["dir"] + c["flowFile"])):
        v = f["vehicle"]
        look = max(look, v["maxSpeed"] * v["maxSpeed"] / v["usualNegAcc"] / 2 + v["maxSpeed"] * c["interval"] * 2)
    return look


def scattered_owners(cfg: str, world: int, seed: int) -> list:
    """A seeded random rank for every intersection, with both ends of every road that has a lane no longer than the
    look-ahead put on one rank (so that Partition::validate accepts the cut), and every rank given at least one real
    intersection where the network has enough of them."""
    p, static = partition(cfg, 1), loader_tables(cfg)
    length = [float.fromhex(x) for x in static["lane_length"]]
    look = look_ahead(cfg)
    rng = random.Random(seed)
    n = len(p["inter_owner"])
    real = [i for i in range(n) if not p["inter_virtual"][i]]
    own = [rng.randrange(world) for _ in range(n)]
    for k, i in enumerate(rng.sample(real, min(world, len(real)))):
        own[i] = k
    root = list(range(n))

    def find(i):
        while root[i] != i:
            root[i] = root[root[i]]
            i = root[i]
        return i
    for l in range(p["n_lanes"]):
        if length[l] <= look:
            a, b = find(p["lane_start"][l]), find(p["lane_end"][l])
            root[max(a, b)] = min(a, b)
    return [own[find(i)] for i in range(n)]


def checkerboard_owners(cfg: str, world: int = 2) -> list:
    """Rank (column + row) % world of every intersection, columns and rows counted over the distinct x and y of the
    intersections' points: on a grid, every road is a seam road and every rank has seams in all four directions."""
    import json
    c = json.load(open(cfg))
    pts = [(i["point"]["x"], i["point"]["y"]) for i in json.load(open(c["dir"] + c["roadnetFile"]))["intersections"]]
    xs, ys = sorted({x for x, _ in pts}), sorted({y for _, y in pts})
    return [(xs.index(x) + ys.index(y)) % world for x, y in pts]


class SeamReach:
    """What a sharded run reached at its seams, fed the restatement's state (VEH_DTYPE records) after every step:

    * ``crossed``: vehicles entering a seam lane, per direction (feeder, owner) -> (total, most in one step);
    * ``max_movers``: the most vehicles entering one seam lane in one step (one mover message, ENT_CAP = 16 records);
    * ``max_queue``: the longest queue on a seam lane, as the share of the lane's length from its end back to the last
      of the halted (speed < 0.1) vehicles that follow its head without a moving one between them, and ``halted_feeding``: the most halted vehicles on laneLinks into a seam
      lane whose queue covered 90 % of it (they wait on the ghost tail);
    * ``spawns`` / ``finishes``: vehicles appearing on / leaving the network from a seam lane, ``virtual_spawns``: those
      spawns onto a seam lane fed by a virtual intersection;
    * ``max_blk_sent``: the most blocker changes one rank sends in one step (a changed blocker of a vehicle on one of
      its drivables, or one of its vehicles leaving the network), and ``foreign_blockers``: vehicle steps whose blocker
      is on a drivable of another rank (a chain that leaves the rank);
    * from the cut alone: ``neighbours`` per rank, ``virtual_fed`` seam lanes (their feeder is a virtual intersection),
      ``empty_ranks`` (ranks without a real intersection) and the seam lanes each rank feeds and owns."""

    def __init__(self, static, part):
        self.n_lanes = static["n_lanes"]
        self.length = [float.fromhex(x) for x in static["lane_length"]]
        self.link_end = static["link_end"]
        lane_owner = part["lane_owner"]
        link_owner = [0] * len(self.link_end)
        for l, links in enumerate(static["lane_out"]):
            for k in links:
                link_owner[k] = lane_owner[l]          # a laneLink sits in the intersection its start lane ends at
        self.owner = np.array(list(lane_owner) + link_owner)
        W = part["world"]
        self.world = W
        self.seam = {l: (a, b) for a in range(W) for b in range(W) for l in part["boundary"][a][b]}
        self.neighbours = [sum(1 for q in range(W) if q != r and part["boundary"][r][q] + part["boundary"][q][r]) for r in range(W)]
        self.feeds = [sum(len(part["boundary"][r][q]) for q in range(W)) for r in range(W)]
        self.owns = [sum(len(part["boundary"][q][r]) for q in range(W)) for r in range(W)]
        virt = part["inter_virtual"]
        self.virtual_lanes = {l for l in self.seam if virt[part["lane_start"][l]]}
        self.virtual_fed = len(self.virtual_lanes)
        has_real = {o for o, v in zip(part["inter_owner"], virt) if not v}
        self.empty_ranks = [r for r in range(W) if r not in has_real]
        self.crossed = {}
        self.max_movers = self.spawns = self.virtual_spawns = self.finishes = self.max_blk_sent = self.foreign_blockers = self.halted_feeding = 0
        self.max_queue = 0.0
        self.prev = {}

    def add(self, vehicles):
        nl = self.n_lanes
        now = {(int(f), int(c)): (int(d), (int(bf), int(bc))) for f, c, d, bf, bc in
               zip(vehicles["flow"], vehicles["cnt"], vehicles["drivable"], vehicles["blocker_flow"], vehicles["blocker_cnt"])}
        into, pairs, sent = {}, {}, [0] * self.world
        for key, (d, blk) in now.items():
            p = self.prev.get(key)
            if p is None:
                self.spawns += d in self.seam
                self.virtual_spawns += d in self.virtual_lanes
            elif p[0] != d and d in self.seam:
                into[d] = into.get(d, 0) + 1
                pairs[self.seam[d]] = pairs.get(self.seam[d], 0) + 1
            if p is not None and p[1] != blk:
                sent[self.owner[d]] += 1
            if blk[0] >= 0 or blk[1] >= 0:
                b = now.get(blk)
                self.foreign_blockers += b is not None and self.owner[b[0]] != self.owner[d]
        for key, (d, _) in self.prev.items():
            if key not in now:
                self.finishes += d in self.seam
                sent[self.owner[d]] += 1
        self.max_movers = max([self.max_movers] + list(into.values()))
        self.max_blk_sent = max([self.max_blk_sent] + sent)
        for pr, n in pairs.items():
            tot, most = self.crossed.get(pr, (0, 0))
            self.crossed[pr] = (tot + n, max(most, n))
        drv, dis, spd = vehicles["drivable"], vehicles["dis"], vehicles["speed"]
        halted = spd < 0.1
        full = set()
        for l in set(int(x) for x in drv[halted]) & set(self.seam):
            on = np.nonzero(drv == l)[0]
            on = on[np.argsort(-dis[on], kind="stable")]
            run = np.cumprod(halted[on])                 # the halted vehicles from the head back, up to the first moving one
            if run[0]:
                q = (self.length[l] - float(dis[on[int(run.sum()) - 1]])) / self.length[l]
                self.max_queue = max(self.max_queue, q)
                if q >= 0.9:
                    full.add(l)
        if full:
            on_links = drv[halted & (drv >= nl)]
            self.halted_feeding = max(self.halted_feeding, int(sum(self.link_end[d - nl] in full for d in on_links)))
        self.prev = now

    def __str__(self):
        crossed = ", ".join("%d->%d %d (%d in one step)" % (a, b, t, m) for (a, b), (t, m) in sorted(self.crossed.items()))
        return ("seam lanes fed / owned per rank %s / %s, neighbours per rank %s, %d seam lanes fed by a virtual intersection, "
                "ranks without a real intersection %s; crossings %s; at most %d movers into one seam lane in one step; "
                "longest halted queue on a seam lane %.3f of its length, %d halted vehicles on laneLinks into a full one; "
                "%d spawns onto seam lanes (%d onto virtual-fed ones), %d finishes on seam lanes; at most %d blocker changes sent by one rank in one step, "
                "%d vehicle steps blocked across ranks" %
                (self.feeds, self.owns, self.neighbours, self.virtual_fed, self.empty_ranks, crossed or "none", self.max_movers,
                 self.max_queue, self.halted_feeding, self.spawns, self.virtual_spawns, self.finishes, self.max_blk_sent, self.foreign_blockers))


def group_vs_restatement(grp, cfg, steps, reach=None, check=lambda s: True):
    """Step a loop-back group (cityflow_b200.capi.CShardGroup, or its emulated-device form) and the restatement together.
    At every step `check(s)` accepts: vehicle count, lane and waiting counts, the ranks' summed counters (vehicle steps,
    ties), and every running vehicle -- every field, and the order of every drivable's list (the group lists each rank's
    vehicles drivable by drivable in list order) -- must be equal.  `reach` (SeamReach) is fed every step.  Returns the
    restatement."""
    from oracle import harness as H
    ora = H.PortOracle(cfg)
    vehicle_steps = 0
    for s in range(1, steps + 1):
        grp.next_step()
        ora.next_step()
        st = ora.snapshot(with_order=check(s))
        vehicle_steps += st.vehicle_count
        if reach is not None:
            reach.add(st.vehicles)
        if not check(s):
            continue
        assert grp.vehicle_count() == st.vehicle_count, "step %d" % s
        assert grp.counters() == (vehicle_steps, ora.tie_count()), "counters, step %d" % s
        assert np.array_equal(grp.lane_counts(ora.n_lanes), st.lane_count), "lane counts, step %d" % s
        assert np.array_equal(grp.lane_counts(ora.n_lanes, True), st.lane_waiting), "waiting counts, step %d" % s
        mine = grp.debug_vehicles()
        a, b = np.sort(mine, order=["flow", "cnt"]), np.sort(st.vehicles, order=["flow", "cnt"])
        assert len(a) == len(b), "step %d" % s
        for f in ("flow", "cnt", "priority", "drivable", "dis", "speed", "leader_flow", "leader_cnt", "blocker_flow",
                  "blocker_cnt", "gap", "enter_ll_time"):
            assert np.array_equal(a[f], b[f]), "step %d field %s" % (s, f)
        listed = mine[np.argsort(mine["drivable"], kind="stable")]
        want = np.concatenate([o for o in st.order if len(o)] or [np.zeros((0, 2), np.int32)])
        assert np.array_equal(np.stack([listed["flow"], listed["cnt"]], 1), want), "list order, step %d" % s
    return ora
