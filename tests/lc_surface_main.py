"""Lane change at the Python surface, object for object: the reference's own module built from the priority-ordered
copy of the reference (oracle/lc_module.mk -> oracle/_ref/lcorder/, the same build refdump_lcorder pins the lane-change
state to) and whatever `import cityflow` resolves to get the same calls on a laneChange=true scenario and must return
EQUAL objects every step: the id lists of get_vehicles (running and all) and get_lane_vehicles (shadows "<id>_shadow"
included, lane order included), the dicts of get_vehicle_speed / get_vehicle_distance, get_leader and get_vehicle_info by
a shadow's id and by its parent's, set_vehicle_speed on both, the same refusals for the id of a shadow whose change has
completed; a binary snapshot taken while cars change lanes gives the same names when it is loaded again; and the two
replay logs agree (ids, change directions and light states exact, numbers as doubles).  TEST INFRASTRUCTURE.

Run as a script (`python tests/lc_surface_main.py <config.json> <steps>`) it prints "OK <stats>" -- the CPU suite does
that in a child process whose PYTHONPATH puts the emulated-device build of the module first; the GPU suite calls
compare_lc_surface() in-process with the real module."""
import glob
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LC_MODULE_DIR = os.path.join(ROOT, "oracle", "_ref", "lcorder")


def have_lc_module() -> bool:
    return bool(glob.glob(os.path.join(LC_MODULE_DIR, "cityflow*.so")))


def load_lc_reference_module():
    """oracle/_ref/lcorder/cityflow*.so, loaded without touching sys.modules['cityflow']."""
    import importlib.machinery
    import importlib.util
    so = glob.glob(os.path.join(LC_MODULE_DIR, "cityflow*.so"))[0]
    loader = importlib.machinery.ExtensionFileLoader("cityflow", so)
    spec = importlib.util.spec_from_file_location("cityflow", so, loader=loader)
    mod = importlib.util.module_from_spec(spec)
    loader.exec_module(mod)
    return mod


def with_replay(cfg: str) -> str:
    """A copy of the config with saveReplay on (log files next to it)."""
    c = json.load(open(cfg))
    c.update(saveReplay=True, roadnetLogFile="replay_roadnet.json", replayLogFile="replay.txt")
    out = cfg[:-5] + "_replay.json"
    json.dump(c, open(out, "w"))
    return out


def same_replay_line(ours: str, ref: str, where: str):
    """Token-wise: ids, change directions and light states identical, numbers equal as doubles (the reference's
    printer does not define the last digit, cityflow_b200/csrc/replay.h)."""
    (va, la), (vb, lb) = [x.split(";") for x in (ours, ref)]
    assert la == lb, where + ": traffic-light part differs"
    a, b = va.split(","), vb.split(",")
    assert len(a) == len(b), (where, len(a), len(b))
    for x, y in zip(a, b):
        tx, ty = x.split(" "), y.split(" ")
        assert len(tx) == len(ty), (where, x, y)
        if len(tx) < 7:
            assert tx == ty
            continue
        assert tx[3] == ty[3] and tx[4] == ty[4], (where, x, y)
        for i in (0, 1, 2, 5, 6):
            fa, fb = float(tx[i]), float(ty[i])
            assert fa == fb or abs(fa - fb) <= 1e-12 * max(1.0, abs(fb)), (where, x, y)


def _base(vid: str) -> str:
    while vid.endswith("_shadow"):
        vid = vid[:-7]
    return vid


def compare_lc_surface(ours_mod, ref_mod, cfg: str, steps: int) -> dict:
    c = json.load(open(cfg))
    ref = ref_mod.Engine(cfg, thread_num=1)
    eng = ours_mod.Engine(cfg, thread_num=1)
    replay = c.get("saveReplay", False)
    if replay:
        ref.set_replay_file("replay_ref.txt")
        eng.set_replay_file("replay_ours.txt")
    stats = dict(steps=0, shadow_ids=0, takeovers=0, stale_refused=0, shadow_lookups=0, custom=0, leaders=0,
                 snapshot_steps=0, replay_lines=0, replay_dirs=0)

    def same(name, *args, **kw):
        a, b = getattr(ref, name)(*args, **kw), getattr(eng, name)(*args, **kw)
        assert a == b, (name, args, stats["steps"], _first_difference(a, b))
        return a

    def both(name, *args, **kw):
        """a call that may raise: same return value or the same kind of exception"""
        out = []
        for e in (ref, eng):
            try:
                out.append(("ok", getattr(e, name)(*args, **kw)))
            except Exception as ex:   # noqa: BLE001
                out.append(("raised", type(ex).__name__))
        assert out[0] == out[1], (name, args, stats["steps"], out)
        return out[0]

    def observe():
        lanes = same("get_lane_vehicles")
        running = same("get_vehicles")
        every = same("get_vehicles", include_waiting=True)
        same("get_vehicle_speed")
        same("get_vehicle_distance")
        same("get_vehicle_count")
        same("get_lane_vehicle_count")
        return lanes, running, every

    snap, snap_step, recorded = None, None, []
    prev_shadows = set()
    for s in range(1, steps + 1):
        stats["steps"] = s
        if s % 20 == 5:   # custom speeds on cars changing lanes and on their shadows
            for sid in sorted(prev_shadows)[:3]:
                both("set_vehicle_speed", sid, 2.0)
                both("set_vehicle_speed", _base(sid), 3.0)
                stats["custom"] += 2
        both("next_step")
        lanes, running, every = observe()
        on_lanes = [v for lst in lanes.values() for v in lst]
        shadows = {v for v in on_lanes if v.endswith("_shadow")}
        assert not (shadows & set(every)), "a shadow still changing is not a real vehicle"
        stats["shadow_ids"] += len(shadows)
        for sid in sorted(shadows):
            for vid in (sid, _base(sid)):
                same("get_leader", vid)
                same("get_vehicle_info", vid)
                stats["shadow_lookups"] += 1
        for vid in on_lanes[::7] + running[::11]:
            same("get_leader", vid)
            stats["leaders"] += 1
        for sid in sorted(prev_shadows - shadows):   # completed (or given up): the shadow's own id is gone
            if _base(sid) in every:
                stats["takeovers"] += 1
            for name in ("get_leader", "get_vehicle_info"):
                assert both(name, sid)[0] == "raised", (name, sid, s)
            assert both("set_vehicle_speed", sid, 1.0)[0] == "raised"
            stats["stale_refused"] += 1
        prev_shadows = shadows
        # a snapshot taken while cars change lanes names them the same way when it is loaded again
        if snap is None and s >= steps // 2 and len(shadows) >= 2:
            snap, snap_step = eng.snapshot(), s
        elif snap is not None and s <= snap_step + 10:
            recorded.append((lanes, every))
            if s == snap_step + 10:
                if replay:
                    eng.set_save_replay(False)
                eng.load(snap)
                for k in range(10):
                    eng.next_step()
                    assert (eng.get_lane_vehicles(), eng.get_vehicles(include_waiting=True)) == recorded[k], k
                    stats["snapshot_steps"] += 1
                if replay:
                    eng.set_save_replay(True)
    del ref, eng
    if replay:
        ours = open(c["dir"] + "replay_ours.txt").read().split("\n")
        theirs = open(c["dir"] + "replay_ref.txt").read().split("\n")
        assert len(ours) == len(theirs) == steps + 1
        for k, (a, b) in enumerate(zip(ours[:-1], theirs[:-1])):
            same_replay_line(a, b, "replay step %d" % (k + 1))
            stats["replay_dirs"] += sum(1 for v in b.split(";")[0].split(",") if v and v.split(" ")[4] != "0")
        stats["replay_lines"] = steps
    return stats


def _first_difference(a, b):
    if isinstance(a, dict) and isinstance(b, dict):
        for k in a:
            if k not in b or a[k] != b[k]:
                return (k, a[k], b.get(k))
        return ("extra keys", sorted(set(b) - set(a))[:5])
    if isinstance(a, list) and isinstance(b, list):
        if len(a) != len(b):
            return ("lengths", len(a), len(b))
        for k, (x, y) in enumerate(zip(a, b)):
            if x != y:
                return (k, x, y)
    return (a, b)


if __name__ == "__main__":
    import cityflow
    print("OK", json.dumps(compare_lc_surface(cityflow, load_lc_reference_module(), sys.argv[1], int(sys.argv[2]))),
          "with", cityflow.__file__)
