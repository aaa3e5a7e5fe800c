"""What lies ahead of every vehicle (cfb_observe_vehicle_context_device): each row's leader, gap, next drivable and the
light at its stop line, through the C-ABI over the emulated device -- the kernel body of csrc/device_vehobs.cuh
(vctxFill) on the emulated warp (tests/device_sim_emu_vehctx.cpp), under the real host engine.  Every column is checked
every step against the compiled reference (`refdump run` / `runlc` for leader and gap, `oracle/refctx.cpp` for the
next drivable and the light) and against the engine's own debug records.  The emulated device's "device memory" is host
memory, so the returned pointers are read with numpy."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from test_cpu import _HAVE_CUDA_SDK

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

pytestmark = pytest.mark.skipif(not _HAVE_CUDA_SDK, reason="needs the CUDA headers and libcudart to build the host-check library")


@pytest.fixture(autouse=True)
def _emulated(monkeypatch):
    monkeypatch.setenv("CFB_EMULATED_DEVICE_FOR_TESTS", "1")


def _ctx_lib():
    """oracle/_build/libcfb_hostcheck_vehctx.so: the host engine and C-ABI (csrc/host_engine.cpp) over the emulated
    device with the per-vehicle entry points and the context (tests/device_sim_emu_vehctx.cpp).  Test infrastructure,
    built like test_cpu_vehicle_obs.py's library."""
    os.makedirs(os.path.join(ROOT, "oracle", "_build"), exist_ok=True)
    lib = os.path.join(ROOT, "oracle", "_build", "libcfb_hostcheck_vehctx.so")
    csrc = os.path.join(ROOT, "cityflow_b200", "csrc")
    tests = os.path.join(ROOT, "tests")
    srcs = [os.path.join(tests, "device_sim_emu_vehctx.cpp")] + [os.path.join(csrc, f) for f in
            ("host_engine.cpp", "roadnet.cpp", "flows.cpp", "partition.cpp", "shard.cpp", "replay.cpp", "json_write.cpp")]
    deps = srcs + [os.path.join(csrc, f) for f in os.listdir(csrc) if f.endswith((".cuh", ".h"))] + \
        [os.path.join(tests, f) for f in ("device_emu.h", "device_hostsim.h", "device_sim_emu.cpp", "device_sim_emu_vehobs.cpp")]
    if not os.path.exists(lib) or os.path.getmtime(lib) < max(os.path.getmtime(f) for f in deps):
        subprocess.check_call(["g++", "-std=c++17", "-O1", "-fPIC", "-shared", "-ffp-contract=off", "-I/usr/local/cuda/include",
                               "-I" + csrc, "-I" + tests, "-I" + os.path.join(ROOT, "include")] + srcs +
                              ["-L/usr/local/cuda/lib64", "-lcudart", "-ldl", "-o", lib])
    return lib


def _emulated_engine(cfg):
    from cityflow_b200 import capi
    path = _ctx_lib()

    class EmulatedEngine(capi.CEngine):
        def _library(self):
            return capi.bind(ctypes.CDLL(path))

    return EmulatedEngine(cfg, 0)


def _host(ptr, n, ctype):
    return np.ctypeslib.as_array((ctype * max(n, 1)).from_address(ptr))[:n].copy()


def _read(eng, ptr, n, ctype):
    """n elements at a pointer the engine handed out: host memory on the emulated device; an engine whose pointers are
    device memory brings its own `read` (tests/test_gpu_vehicle_context.py)."""
    return eng.read(ptr, n, ctype) if hasattr(eng, "read") else _host(ptr, n, ctype)


def context(eng, plain=False):
    """One refresh (plain=True: the table alone, cfb_observe_vehicles_device) as numpy columns of capacity length,
    after checking that every row from count on holds the padding values.  Context columns are read from the buffers
    the context refresh hands out, whichever refresh ran."""
    if plain:
        o = eng.observe_vehicles_device()
    else:
        c = eng.observe_vehicle_context_device()
        o = c.table
        eng._ctx_ptrs = c
    c = eng._ctx_ptrs
    cap = o.capacity
    n = int(_read(eng, o.count, 1, ctypes.c_int32)[0])
    t = dict(n=n, cap=cap, slot=_read(eng, o.slot, cap, ctypes.c_int32), priority=_read(eng, o.priority, cap, ctypes.c_int32),
             drivable=_read(eng, o.drivable, cap, ctypes.c_int32), begin=_read(eng, o.drivable_begin, o.n_drivables + 1, ctypes.c_int32),
             leader=_read(eng, c.leader, cap, ctypes.c_int32), gap=_read(eng, c.gap, cap, ctypes.c_double),
             next=_read(eng, c.next_drivable, cap, ctypes.c_int32), signal=_read(eng, c.signal, cap, ctypes.c_int8),
             ptrs=(c.leader, c.gap, c.next_drivable, c.signal, c.drivable_length, c.drivable_max_speed, c.link_road_link))
    assert 0 <= n <= cap and (t["slot"][n:] == -1).all() and t["begin"][-1] == n
    if not plain:
        assert (t["leader"][n:] == -1).all() and np.isposinf(t["gap"][n:]).all()
        assert (t["next"][n:] == -1).all() and (t["signal"][n:] == -1).all()
        assert c.n_lanes == eng.n_lanes and c.n_lanes + c.n_links == eng.n_drivables
    return t


def static(eng):
    c = eng._ctx_ptrs
    nd = eng.n_drivables
    return dict(length=_read(eng, c.drivable_length, nd, ctypes.c_double), max_speed=_read(eng, c.drivable_max_speed, nd, ctypes.c_double),
                road_link=_read(eng, c.link_road_link, c.n_links, ctypes.c_int32))


def _lc_vehicles(eng):
    from oracle.harness import LC_DTYPE
    n = eng._check(eng.lib.cfb_debug_lc_vehicles(eng.h, None, 0))
    a = np.zeros(n, LC_DTYPE)
    if n:
        eng._check(eng.lib.cfb_debug_lc_vehicles(eng.h, a.ctypes.data, n))
    return a


def check_self(eng, t, lane_change):
    """The columns against the engine's own debug records and tables (no reference needed)."""
    n, nl = t["n"], eng.n_lanes
    leader, gap, nxt, sig = t["leader"][:n], t["gap"][:n], t["next"][:n], t["signal"][:n]
    prio, drv = t["priority"][:n], t["drivable"][:n]
    has = leader >= 0
    assert (leader < n).all() and (leader != np.arange(n)).all()
    assert (np.isposinf(gap) == ~has).all()
    lp = np.where(has, prio[np.maximum(leader, 0)], -1)
    if lane_change:   # every running vehicle incl. shadows, by priority (leader / gap as the vehicle keeps them)
        lc = _lc_vehicles(eng)
        o = np.argsort(prio, kind="stable")
        assert (lc["priority"] == prio[o]).all()
        assert (lc["leader"] == lp[o]).all()
        assert (lc["gap"][has[o]].view(np.int64) == gap[o][has[o]].view(np.int64)).all()
    else:             # the debug records run in table order: drivable-major, list order
        dbg = eng.debug_vehicles()
        assert (dbg["priority"] == prio).all() and (dbg["drivable"] == drv).all()
        refs = eng.vehicle_refs(t["slot"][:n])
        lref = refs[np.maximum(leader, 0)]
        assert (np.where(has, lref["flow"], -1) == dbg["leader_flow"]).all()
        assert (np.where(has, lref["index"], -1) == dbg["leader_cnt"]).all()
        assert (dbg["gap"][has].view(np.int64) == gap[has].view(np.int64)).all()
    # next drivable: from a lane a laneLink (or none), from a laneLink a lane; a light only on lanes heading for a laneLink
    st = static(eng)
    on_lane = drv < nl
    assert ((nxt >= nl) | (nxt < 0))[on_lane].all() and (nxt[~on_lane] >= 0).all() and (nxt[~on_lane] < nl).all()
    assert ((nxt >= -2) & (nxt < eng.n_drivables)).all()
    heads = on_lane & (nxt >= nl)
    assert ((sig >= 0) == heads).all() and np.isin(sig, (-1, 0, 1)).all()
    assert (st["road_link"] >= 0).all()
    return dict(leaders=int(has.sum()), cross=int((has & (drv[np.maximum(leader, 0)] != drv)).sum()),
                green=int((sig == 1).sum()), red=int((sig == 0).sum()), dead=int((nxt == -2).sum()),
                end=int((on_lane & (nxt == -1)).sum()), links=int((~on_lane).sum()))


# ---------------------------------------------------------------------------------------------------------------------
# the compiled reference
REFCTX = os.path.join(ROOT, "oracle", "_ref", "refctx")   # oracle/refctx.cpp, built by oracle/refctx.mk


def _have_ref(lane_change):
    from oracle import harness as H
    if lane_change:
        return H.have_lc_ref() and os.path.exists(REFCTX + "_lcorder")
    return H.have_ref() and os.path.exists(REFCTX)


CTX_REC = np.dtype([("priority", "<i4"), ("drivable", "<i4"), ("next", "<i4"), ("signal", "<i4"),
                    ("dis", "<f8"), ("speed", "<f8")])


def parse_ctx(path):
    buf = open(path, "rb").read()
    assert np.frombuffer(buf, "<i4", 1, 0)[0] == 0x43464331
    off, out = 4, {}
    while off < len(buf):
        step, n = (int(x) for x in np.frombuffer(buf, "<i4", 2, off))
        off += 8
        out[step] = np.frombuffer(buf, CTX_REC, n, off)
        off += CTX_REC.itemsize * n
    return out


def _by_priority(a):
    return a[np.argsort(a["priority"], kind="stable")]


def reference(cfg, steps, lane_change, n_inter, n_drivables, tmp):
    """(per-step vehicle states of `refdump run` / `runlc`, per-step records of `refctx`), from the unmodified
    reference, or its priority-ordered build with lane change.  Every step, refctx's vehicles -- priority, drivable,
    distance and speed, bit for bit -- are run's: asking for the next drivable does not change the reference's course."""
    from oracle import harness as H
    out = os.path.join(tmp, "ctx.bin")
    subprocess.check_call([REFCTX + ("_lcorder" if lane_change else ""), cfg, str(steps), "1", out], timeout=H.REF_TIMEOUT)
    ctxs = parse_ctx(out)
    if lane_change:
        states = H.RefDump.runlc(cfg, steps, 1, n_inter=n_inter, n_drivables=n_drivables)
    else:
        states = H.RefDump.run(cfg, steps, 1, 1, n_inter=n_inter, n_drivables=n_drivables)
    states = {st.step: st for st in states}
    assert sorted(ctxs) == sorted(states) == list(range(1, steps + 1))
    for s, c in ctxs.items():
        v, c = _by_priority(states[s].vehicles), _by_priority(c)
        assert len(v) == len(c) and (v["priority"] == c["priority"]).all() and (v["drivable"] == c["drivable"]).all(), s
        assert v["dis"].tobytes() == c["dis"].tobytes() and v["speed"].tobytes() == c["speed"].tobytes(), s
    return states, ctxs


def check_reference(t, state, ctx, lane_change):
    """Leader, gap, next drivable and light of every vehicle, bit for bit, matched by priority."""
    n = t["n"]
    prio, leader, gap = t["priority"][:n], t["leader"][:n], t["gap"][:n]
    v = state.vehicles
    assert len(v) == n and len(ctx) == n
    o = np.argsort(prio, kind="stable")
    vo = v[np.argsort(v["priority"], kind="stable")]
    co = ctx[np.argsort(ctx["priority"], kind="stable")]
    assert (vo["priority"] == prio[o]).all() and (co["priority"] == prio[o]).all()
    has = (leader >= 0)[o]
    lp = np.where(leader >= 0, prio[np.maximum(leader, 0)], -1)[o]
    if lane_change:
        assert (vo["leader"] == lp).all()
    else:
        key = {(int(f), int(c)): int(p) for f, c, p in zip(v["flow"], v["cnt"], v["priority"])}
        want = np.array([key[(int(f), int(c))] if f != -1 or c != -1 else -1 for f, c in zip(vo["leader_flow"], vo["leader_cnt"])],
                        np.int64)
        assert (want == lp).all()
    assert (vo["gap"][has].view(np.int64) == gap[o][has].view(np.int64)).all()
    assert (co["next"] == t["next"][:n][o]).all()
    assert (co["signal"] == t["signal"][:n][o]).all()


def check_static(eng, cfg):
    from oracle import harness as H
    R = H.RefDump.static(cfg)
    st = static(eng)
    want_len = [l["length"] for l in R["lanes"]] + [l["length"] for l in R["links"]]
    want_max = [l["max_speed"] for l in R["lanes"]] + [10000.0] * len(R["links"])
    assert st["length"].tobytes() == np.array(want_len, np.float64).tobytes()
    assert st["max_speed"].tobytes() == np.array(want_max, np.float64).tobytes()
    assert (st["road_link"] == np.array([l["road_link"] for l in R["links"]], np.int32)).all()


def _dense_3x3(directory, lane_change=False, rl=False):
    from cityflow_b200 import scenario
    return scenario.make_grid_scenario(directory, 3, 3, dense=dict(frac=1.0, interval=3.0, seed=3), name="vc33%d%d" % (lane_change, rl),
                                       lane_change=lane_change, rl_traffic_light=rl)


def _irregular(directory):
    import conftest
    from cityflow_b200 import scenario
    net = conftest._irregular_net()
    flows = scenario.random_walk_flows(net, frac=1.0, interval=4.0, seed=9)
    return scenario.write_scenario(directory, net, flows, seed=7, name="vcirr")


def _fuzzed(directory, seed=7):
    import randnet
    from cityflow_b200 import scenario
    net = randnet.random_roadnet(seed, rows=2 + seed % 3, cols=3 + seed % 2)
    flows = randnet.random_flows(net, seed + 100, n_flows=40 + seed % 50)
    return scenario.write_scenario(directory, net, flows, seed=seed, interval=1.0, name="vcf%d" % seed)


NETS = {"dense_3x3": _dense_3x3, "irregular": _irregular, "fuzzed": _fuzzed,
        "dense_3x3_lane_change": lambda d: _dense_3x3(d, lane_change=True)}


@pytest.mark.parametrize("net", sorted(NETS))
def test_context_every_step_against_the_reference(net, tmp_path):
    """Every column, every step of 200, equals the compiled reference's (leader and gap from `run` / `runlc`, next
    drivable and light from `refctx`, matched by priority) and the engine's debug records; the static columns equal
    `refdump static`; the buffers keep their addresses."""
    lane_change = net.endswith("lane_change")
    if not _have_ref(lane_change):
        pytest.skip("the compiled reference (oracle/_ref) is not built here")
    cfg = NETS[net](str(tmp_path))
    eng = _emulated_engine(cfg)
    steps = 200
    states, ctxs = reference(cfg, steps, lane_change, eng.n_inter, eng.n_drivables, str(tmp_path))
    t = context(eng)
    check_static(eng, cfg)
    seen = {}
    for s in range(1, steps + 1):
        eng.next_step()
        t2 = context(eng)
        assert t2["ptrs"] == t["ptrs"]
        t = t2
        for k, x in check_self(eng, t, lane_change).items():
            seen[k] = seen.get(k, 0) + x
        check_reference(t, states[s], ctxs[s], lane_change)
    assert seen["leaders"] > 1000 and seen["cross"] > 100 and seen["green"] > 100 and seen["red"] > 100, seen
    assert seen["end"] > 10 and seen["links"] > 100, seen
    if net == "fuzzed":   # parked vehicles: lanes that cannot continue their route
        assert seen["dead"] > 0, seen


def test_set_tl_phase_shows_before_the_next_step(tmp_path):
    """rlTrafficLight: set_tl_phase between steps shows in `signal` at the next refresh, before any step: the light of
    every lane row heading for a laneLink is that roadLink's availability in the phase just set (the phase table of
    `refdump static`), which is what RoadLink::isAvailable answers in the reference between steps."""
    from oracle import harness as H
    if not H.have_ref():
        pytest.skip("the compiled reference (oracle/_ref) is not built here")
    cfg = _dense_3x3(str(tmp_path), rl=True)
    eng = _emulated_engine(cfg)
    R = H.RefDump.static(cfg)
    real = [i for i, it in enumerate(R["inters"]) if not it["virtual"]]
    owner, idx = [], []   # roadLink -> (intersection, index in it)
    for i, it in enumerate(R["inters"]):
        for k in range(it["n_road_links"]):
            owner.append(i)
            idx.append(k)
    eng.next_step(30)
    changed = 0
    for rnd in range(6):
        before = context(eng)
        phases = {i: (rnd * 3 + 1 + i) % len(R["inters"][i]["phases"]) for i in real}
        for i, ph in phases.items():
            eng.set_tl_phase(i, ph)
        t = context(eng)
        n = t["n"]
        assert (t["slot"][:n] == before["slot"][:n]).all()
        heads = (t["drivable"][:n] < eng.n_lanes) & (t["next"][:n] >= eng.n_lanes)
        rl = static(eng)["road_link"][t["next"][:n][heads] - eng.n_lanes]
        want = [R["inters"][owner[r]]["phases"][phases[owner[r]]][1][idx[r]] for r in rl]
        assert (t["signal"][:n][heads] == np.array(want, np.int8)).all()
        changed += int((t["signal"][:n] != before["signal"][:n]).sum())
        check_self(eng, t, False)
        eng.next_step(7)
    assert changed > 10, changed


def test_plain_and_context_refreshes_interleaved_while_the_fleet_drains(tmp_path):
    """A plain refresh moves the table's own padding mark too; the context refresh keeps its own, so interleaving the
    two -- as two VehicleObservations on one engine do -- leaves correct padding in every row of every column while
    the row count rises and falls (the flows stop at 100 s and the network empties)."""
    from cityflow_b200 import scenario
    net = scenario.grid_roadnet(2, 2)
    flows = scenario.random_walk_flows(net, frac=1.0, interval=5.0, seed=5)
    for f in flows:
        f["endTime"] = 100
    cfg = scenario.write_scenario(str(tmp_path), net, flows, name="vcdrain")
    eng = _emulated_engine(cfg)
    rng = np.random.default_rng(3)
    most = 0
    for s in range(700):
        eng.next_step()
        k = rng.integers(0, 3)
        if k == 0:
            context(eng, plain=True)
        elif k == 1:
            context(eng, plain=True)
            check_self(eng, context(eng), False)
        else:
            t = context(eng)
            check_self(eng, t, False)
            most = max(most, t["n"])
            if s % 2:
                context(eng, plain=True)
    t = context(eng)
    assert most > 30 and t["n"] == eng.vehicle_count() and t["n"] < most // 4, (most, t["n"])


def test_empty_network(tmp_path):
    """No flows: every row is padding, before and after steps; the static columns are there all the same."""
    from cityflow_b200 import scenario
    cfg = scenario.write_scenario(str(tmp_path), scenario.grid_roadnet(2, 3), [], name="vcempty")
    eng = _emulated_engine(cfg)
    for _ in range(3):
        t = context(eng)
        assert t["n"] == 0
        eng.next_step()
    st = static(eng)
    assert (st["length"] > 0).all() and len(st["road_link"]) == eng.n_drivables - eng.n_lanes
