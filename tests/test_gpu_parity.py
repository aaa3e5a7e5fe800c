"""GPU parity tests proper: the CUDA path, called through the C-ABI (ctypes), against the
checkers on identical seeded inputs -- the compiled unmodified reference (oracle/_ref/refdump)
when it travelled to this box, and the CPU restatement (oracle/cityflow_oracle.cpp).

Bar (BASELINE.json north_star): per-lane vehicle counts bit-exact every step, per-vehicle speeds
within 1e-6.  What is asserted here is stronger: every running vehicle's (drivable, distance,
speed, leader, gap, blocker, enterLaneLinkTime) is bit-equal every step.
"""
import numpy as np
import pytest

from oracle import harness as H

pytestmark = pytest.mark.gpu


def _gpu_state(eng, step):
    st = H.StepState()
    st.step = step
    st.vehicle_count = eng.vehicle_count()
    st.pool_size = st.finished = 0
    st.cum_travel_time = 0.0
    st.lane_count = eng.lane_vehicle_count()
    st.lane_waiting = eng.lane_waiting_count()
    st.lane_queue = None
    st.phases = None
    st.vehicles = eng.debug_vehicles()
    st.order = None
    return st


def _relax(ref):
    ref.pool_size = ref.finished = 0
    ref.cum_travel_time = 0.0
    return ref


def _run_against_port(cfg, steps, every=1, hook=None):
    from cityflow_b200.capi import CEngine
    eng = CEngine(cfg)
    ora = H.PortOracle(cfg)
    for s in range(1, steps + 1):
        if hook:
            hook(eng, ora, s)
        eng.next_step()
        ora.next_step()
        if s % every == 0 or s == steps:
            bad = H.compare_states(_relax(ora.snapshot()), _gpu_state(eng, s))
            assert not bad, "step %d: %s" % (s, "; ".join(bad[:6]))
    assert eng.gpu_launches() >= steps
    return eng, ora


def test_single_intersection_vs_port(cfg_1x1):
    _run_against_port(cfg_1x1, 300)


def test_3x3_dense_vs_port(cfg_3x3_dense):
    _run_against_port(cfg_3x3_dense, 600)


def test_6x6_default_vs_port(cfg_6x6):
    _run_against_port(cfg_6x6, 400, every=5)


def test_6x6_dense_vs_port(cfg_6x6_dense):
    eng, ora = _run_against_port(cfg_6x6_dense, 1200, every=10)
    assert ora.tie_count() == 0
    # finished vehicles and travel time bookkeeping (engine.cpp:299-303, :682-691): exact
    assert ora.lib.cfo_finished_count(ora.h) > 1000
    assert eng.average_travel_time() == ora.average_travel_time()


def test_rl_phases_vs_port(cfg_6x6_rl):
    # virtual intersections have no phases: the C-ABI rejects them, the oracle ignores them
    from cityflow_b200.capi import CEngine
    eng = CEngine(cfg_6x6_rl)
    ora = H.PortOracle(cfg_6x6_rl)
    ph0 = np.zeros(ora.n_inter, np.int32)
    ora.lib.cfo_phases(ora.h, ph0.ctypes.data)
    real = np.nonzero(ph0 >= 0)[0]
    for s in range(1, 401):
        if s % 10 == 1:
            for i in real:
                ph = int((s // 10 + i) % 8)
                eng.set_tl_phase(int(i), ph)
                ora.set_tl_phase(int(i), ph)
        eng.next_step()
        ora.next_step()
        if s % 5 == 0:
            bad = H.compare_states(_relax(ora.snapshot()), _gpu_state(eng, s))
            assert not bad, "step %d: %s" % (s, "; ".join(bad[:6]))


@pytest.mark.skipif(not H.have_ref(), reason="compiled reference (oracle/_ref) not present")
def test_6x6_dense_vs_compiled_reference(cfg_6x6_dense):
    from cityflow_b200.capi import CEngine
    eng = CEngine(cfg_6x6_dense)
    steps, every = 800, 20
    ref = H.RefDump.run(cfg_6x6_dense, steps, 1, every, n_inter=eng.n_inter, n_drivables=eng.n_drivables)
    k = 0
    for s in range(1, steps + 1):
        eng.next_step()
        if s % every == 0 or s == steps:
            st = ref[k]
            k += 1
            assert st.step == s
            st.lane_queue = None
            st.phases = None
            st.order = None
            bad = H.compare_states(_relax(st), _gpu_state(eng, s))
            assert not bad, "step %d: %s" % (s, "; ".join(bad[:6]))


def test_reset_determinism(cfg_3x3_dense):
    """The reference's own Basic.reset test (tests/cpp/basic_test.cpp:37-53)."""
    from cityflow_b200.capi import CEngine
    eng = CEngine(cfg_3x3_dense)
    eng.next_step(200)
    a = (eng.vehicle_count(), eng.lane_vehicle_count().copy(), eng.debug_vehicles().copy())
    eng.reset(True)
    eng.next_step(200)
    b = (eng.vehicle_count(), eng.lane_vehicle_count(), eng.debug_vehicles())
    assert a[0] == b[0]
    assert np.array_equal(a[1], b[1])
    assert np.array_equal(np.sort(a[2], order=["flow", "cnt"]), np.sort(b[2], order=["flow", "cnt"]))


def test_30x30_dense_lane_counts_vs_port(scenario_dir):
    """BASELINE.json configs[2] shape (30x30, dense demand): per-lane counts bit-exact and all
    speeds bit-equal against the CPU restatement while the network fills up."""
    from cityflow_b200 import scenario
    from cityflow_b200.capi import CEngine
    cfg = scenario.make_grid_scenario(scenario_dir, 30, 30, name="g30d", dense=dict(frac=0.5, interval=10.0, seed=1))
    eng = CEngine(cfg)
    ora = H.PortOracle(cfg)
    for s in (100, 250, 400):
        eng.next_step(s - ora.steps)
        ora.next_step(s - ora.steps)
        assert np.array_equal(eng.lane_vehicle_count(), ora.lane_vehicle_count()), "lane counts differ at step %d" % s
        assert np.array_equal(eng.lane_waiting_count(), ora.lane_waiting_count())
        bad = H.compare_states(_relax(ora.snapshot()), _gpu_state(eng, s))
        assert not bad, "step %d: %s" % (s, "; ".join(bad[:6]))
    assert ora.vehicle_count() > 50000


def _archive_record(eng, n):
    for _ in range(n):
        eng.next_step()
    return eng.get_lane_vehicle_count(), eng.get_average_travel_time(), eng.get_vehicle_speed()


def test_archive_snapshot_load_like_reference_tests(cfg_3x3_dense, tmp_path):
    """The reference's own result-pinning tests (tests/python/test_archive.py:16-23): run, snapshot,
    run 100 -> record, load, run 100 -> the record must be equal; also via dump / load_from_file and
    into a second engine built from the same config."""
    import cityflow
    eng = cityflow.Engine(cfg_3x3_dense, thread_num=1)
    for _ in range(150):
        eng.next_step()
    arc = eng.snapshot()
    rec1 = _archive_record(eng, 100)
    eng.load(arc)
    assert eng.get_current_time() == 150.0
    rec2 = _archive_record(eng, 100)
    assert rec1 == rec2
    # multiple loads of the same archive, and Archive(engine) constructor
    eng.load(arc)
    arc2 = cityflow.Archive(eng)
    assert _archive_record(eng, 100) == rec1
    eng.load(arc2)
    assert _archive_record(eng, 100) == rec1
    # file round trip into a fresh engine
    path = str(tmp_path / "save.bin")
    arc.dump(path)
    eng2 = cityflow.Engine(cfg_3x3_dense, thread_num=1)
    eng2.load_from_file(path)
    assert _archive_record(eng2, 100) == rec1


def test_vehicle_api_info_speed_route(cfg_3x3_dense):
    """SURVEY.md §8f-3 rows: get_vehicle_info / set_vehicle_speed / set_vehicle_route / get_leader."""
    import cityflow
    eng = cityflow.Engine(cfg_3x3_dense, thread_num=1)
    for _ in range(120):
        eng.next_step()
    speeds = eng.get_vehicle_speed()
    dist = eng.get_vehicle_distance()
    vid = next(k for k, v in speeds.items() if v > 3.0)
    info = eng.get_vehicle_info(vid)
    assert info["running"] == "1"
    assert float(info["speed"]) == pytest.approx(speeds[vid], abs=1e-6)
    assert float(info["distance"]) == pytest.approx(dist[vid], abs=1e-6)
    assert info["route"].endswith(" ") and "drivable" in info
    with pytest.raises(RuntimeError, match="not found"):
        eng.get_vehicle_info("flow_999999_0")
    with pytest.raises(RuntimeError, match="not found"):
        eng.set_vehicle_speed("nope", 1.0)
    # custom speed caps the next step's speed (Vehicle::getCarFollowSpeed, vehicle.cpp:214-221) for one step
    eng.set_vehicle_speed(vid, 0.5)
    eng.next_step()
    after = eng.get_vehicle_speed()
    if vid in after:
        assert after[vid] <= max(0.5, speeds[vid] - 4.5) + 1e-9
    leader = eng.get_leader(vid) if vid in after else ""
    assert isinstance(leader, str)
    # waiting vehicles are known but not running
    allv = eng.get_vehicles(include_waiting=True)
    run = set(eng.get_vehicles())
    assert run <= set(allv) and len(run) == eng.get_vehicle_count()
    lanes = eng.get_lane_vehicles()
    assert sum(len(v) for v in lanes.values()) == sum(eng.get_lane_vehicle_count().values())
    # re-routing: an unknown road or a vehicle on a laneLink is refused, a vehicle on a lane may keep its road
    assert eng.set_vehicle_route(vid, ["no_such_road"]) is False
    assert eng.set_vehicle_route("flow_999999_0", []) is False
    ok_any = False
    for cand, inf in ((k, eng.get_vehicle_info(k)) for k in list(after)[:200]):
        if "road" in inf:
            roads = inf["route"].split()
            if len(roads) >= 2:
                ok_any = eng.set_vehicle_route(cand, roads[1:2]) or ok_any
                break
    assert ok_any
    for _ in range(50):
        eng.next_step()
    assert eng.get_vehicle_count() > 0


def test_heterogeneous_vehicles_half_second_step_vs_port(cfg_hetero_halfstep):
    eng, ora = _run_against_port(cfg_hetero_halfstep, 1500, every=10)
    assert ora.vehicle_count() > 300


def test_push_vehicle_rng_interleaving_vs_port(cfg_3x3_dense):
    """push_vehicle draws its priority from the engine RNG at call time, i.e. between the flow
    draws of two steps (engine.cpp:693-717): the whole future then depends on the interleaving."""
    import json
    import os
    import cityflow
    cfgj = json.load(open(cfg_3x3_dense))
    flows = json.load(open(os.path.join(cfgj["dir"], cfgj["flowFile"])))
    route = flows[0]["route"][:3]
    eng = cityflow.Engine(cfg_3x3_dense, thread_num=1)
    ora = H.PortOracle(cfg_3x3_dense)
    for s in range(1, 301):
        if s % 7 == 0:
            info = {"speed": 0.0, "length": 6.0, "maxSpeed": 12.0} if s % 14 == 0 else {}
            eng.push_vehicle(info, route)
            ora.push_vehicle(info, route)
        eng.next_step()
        ora.next_step()
        if s % 25 == 0:
            assert eng.get_vehicle_count() == ora.vehicle_count()
            assert sum(eng.get_lane_vehicle_count().values()) == int(ora.lane_vehicle_count().sum())
            ov = ora.vehicles()
            sp = eng.get_vehicle_speed()
            names = ["flow_%d_%d" % (f, c) if f >= 0 else "manually_pushed_%d" % c for f, c in zip(ov["flow"], ov["cnt"])]
            assert set(names) == set(sp.keys())
            assert all(sp[n] == v for n, v in zip(names, ov["speed"]))
            assert eng.get_average_travel_time() == ora.average_travel_time()
    assert any(k.startswith("manually_pushed_") for k in sp)


@pytest.mark.parametrize("world", [2, 3])
def test_sharded_loopback_equals_unsharded(cfg_6x6_dense, world):
    """SURVEY.md §8e exactness requirement: the network cut into `world` column strips (ranks on one
    GPU, seam exchanges by device copies) evolves bit-identically to the unsharded engine: every vehicle's
    every field, every drivable's list order (both engines list vehicles drivable by drivable in list order),
    lane and waiting counts, and the ranks' summed counters, every step for 100 steps and every 20 after."""
    from cityflow_b200.capi import CEngine, CShardGroup
    ref = CEngine(cfg_6x6_dense)
    grp = CShardGroup(cfg_6x6_dense, world)
    for s in range(1, 801):
        ref.next_step()
        grp.next_step()
        if s > 100 and s % 20:
            continue
        assert grp.vehicle_count() == ref.vehicle_count(), "step %d" % s
        assert np.array_equal(grp.lane_counts(ref.n_lanes), ref.lane_vehicle_count()), "lane counts differ at step %d" % s
        assert np.array_equal(grp.lane_counts(ref.n_lanes, True), ref.lane_waiting_count()), "waiting counts, step %d" % s
        assert grp.counters() == (ref.vehicle_steps(), ref.tie_count()), "counters, step %d" % s
        va, vb = ref.debug_vehicles(), grp.debug_vehicles()
        a, b = np.sort(va, order=["flow", "cnt"]), np.sort(vb, order=["flow", "cnt"])
        assert len(a) == len(b), "step %d" % s
        for f in ("flow", "cnt", "priority", "drivable", "dis", "speed", "leader_flow", "leader_cnt", "blocker_flow",
                  "blocker_cnt", "gap", "enter_ll_time"):
            assert np.array_equal(a[f], b[f]), (s, f)
        la, lb = (v[np.argsort(v["drivable"], kind="stable")] for v in (va, vb))
        for f in ("drivable", "flow", "cnt"):
            assert np.array_equal(la[f], lb[f]), "list order, step %d" % s
    assert ref.vehicle_count() > 3000


def test_priority_collisions_after_reseed_vs_port(cfg_3x3_dense):
    """Re-seeding the engine RNG mid-run makes it re-issue the priorities it drew at the start:
    draws collide with vehicles that are still alive (redraw, vehicle.cpp:45) and re-use the
    priorities of vehicles that already left (legal).  Exercises Engine::checkPriority
    (engine.cpp:601) against the host's lazily drained bookkeeping."""
    import cityflow
    eng = cityflow.Engine(cfg_3x3_dense, thread_num=1)
    ora = H.PortOracle(cfg_3x3_dense)
    for s in range(1, 701):
        if s in (250, 400, 401, 550):
            eng.set_random_seed(0)
            ora.set_random_seed(0)
        eng.next_step()
        ora.next_step()
        if s % 50 == 0 or s in (251, 252, 402):
            assert eng.get_vehicle_count() == ora.vehicle_count(), s
            ov = ora.vehicles()
            sp = eng.get_vehicle_speed()
            names = ["flow_%d_%d" % (f, c) for f, c in zip(ov["flow"], ov["cnt"])]
            assert set(names) == set(sp.keys()), s
            assert all(sp[n] == v for n, v in zip(names, ov["speed"])), s
    assert eng.get_average_travel_time() == ora.average_travel_time()


def test_irregular_roadnet_vs_port(cfg_irregular):
    _run_against_port(cfg_irregular, 600, every=10)


def test_device_resident_lane_observations(cfg_6x6_dense):
    """SURVEY.md §8f-3 zero-copy observations: the torch CUDA tensors alias the engine's buffers and
    carry exactly what the host getters report, refreshed without a host synchronisation."""
    import torch
    import cityflow
    import cityflow_b200
    eng = cityflow.Engine(cfg_6x6_dense, thread_num=1)
    side = torch.cuda.Stream()
    for rounds in range(3):
        for _ in range(100):
            eng.next_step()
        with torch.cuda.stream(side if rounds == 1 else torch.cuda.current_stream()):
            ids, cnt, wait, ssum = cityflow_b200.lane_observation_tensors(eng)
            total = cnt.sum()                               # consumer work on the ordered stream
            cnt_h, wait_h, ssum_h = cnt.cpu(), wait.cpu(), ssum.cpu()
        assert cnt.is_cuda and cnt.dtype == torch.int32 and ssum.dtype == torch.float64
        counts = eng.get_lane_vehicle_count()
        waiting = eng.get_lane_waiting_vehicle_count()
        assert ids == eng.lane_ids() and set(ids) == set(counts)
        assert cnt_h.tolist() == [counts[i] for i in ids]
        assert wait_h.tolist() == [waiting[i] for i in ids]
        assert int(total) == sum(counts.values())
        speeds = eng.get_vehicle_speed()
        per_lane = {i: 0.0 for i in ids}
        for lane, vs in eng.get_lane_vehicles().items():
            per_lane[lane] = sum(speeds[v] for v in vs)
        np.testing.assert_allclose(ssum_h.numpy(), np.array([per_lane[i] for i in ids]), rtol=0, atol=1e-9)
    assert sum(counts.values()) > 500
    # same storage every call (zero-copy): the next refresh shows through the old tensor
    old_ptr = cnt.data_ptr()
    eng.next_steps(50)
    ids2, cnt2, _, _ = cityflow_b200.lane_observation_tensors(eng)
    assert cnt2.data_ptr() == old_ptr
    assert cnt.tolist() == [eng.get_lane_vehicle_count()[i] for i in ids]
    # the persistent form: tensors made once, refresh() only re-computes their content
    obs = cityflow_b200.LaneObservations(eng)
    eng.next_steps(25)
    before = obs.vehicle_count.clone()
    assert obs.refresh() is obs and obs.vehicle_count.data_ptr() == old_ptr
    now = eng.get_lane_vehicle_count()
    assert obs.vehicle_count.tolist() == [now[i] for i in obs.lane_ids]
    assert not torch.equal(before, obs.vehicle_count)


def test_rl_actions_and_observations_on_device_vs_port(cfg_6x6_rl):
    """The RL loop with nothing crossing to the host: actions come from a torch tensor
    (cfb_set_tl_phases_device), observations are torch tensors; the oracle gets the same actions
    through its host API and must see the same lane counts every step."""
    import torch
    import cityflow
    import cityflow_b200
    eng = cityflow.Engine(cfg_6x6_rl, thread_num=1)
    ora = H.PortOracle(cfg_6x6_rl)
    ph0 = np.zeros(ora.n_inter, np.int32)
    ora.lib.cfo_phases(ora.h, ph0.ctypes.data)
    real = np.nonzero(ph0 >= 0)[0]
    assert eng.num_intersections() == ora.n_inter
    idx = torch.arange(ora.n_inter, device="cuda", dtype=torch.int32)
    for s in range(1, 301):
        if s % 10 == 1:
            act = ((s // 10 + idx) % 8).to(torch.int32)       # computed on the GPU, never copied down
            cityflow_b200.set_tl_phases_tensor(eng, act)
            del act
            for i in real:
                ora.set_tl_phase(int(i), int((s // 10 + i) % 8))
        eng.next_step()
        ora.next_step()
        if s % 5 == 0:
            ids, cnt, wait, _ = cityflow_b200.lane_observation_tensors(eng)
            snap = ora.snapshot()
            assert cnt.cpu().numpy().tolist() == list(snap.lane_count)
            assert wait.cpu().numpy().tolist() == list(snap.lane_waiting)
    assert int(cnt.sum()) > 300
    # host-side set_tl_phase after a device-side one starts from the device's phases
    some = eng.intersection_ids()[int(real[0])]
    eng.set_tl_phase(some, 3)
    ora.set_tl_phase(int(real[0]), 3)
    for _ in range(40):
        eng.next_step()
        ora.next_step()
    counts = eng.get_lane_vehicle_count()
    assert [counts[i] for i in ids] == list(ora.snapshot().lane_count)
    # an out-of-range action is reported (the reference would throw from phases.at())
    bad = torch.full((ora.n_inter,), 99, device="cuda", dtype=torch.int32)
    cityflow_b200.set_tl_phases_tensor(eng, bad)
    eng.next_step()
    with pytest.raises(RuntimeError, match="out of range"):
        for _ in range(300):          # surfaced by the next bookkeeping drain at the latest
            eng.next_step()
        eng.get_average_travel_time()


def test_replay_files_written_by_the_engine(cfg_replay):
    """SURVEY.md §8f-4: with saveReplay the engine writes the reference's two log files.  The step
    lines must be exactly what the stand-alone formatter makes of the ORACLE's states (so: device
    positions, priority order and light states all agree); tests/test_cpu.py pins that formatter
    against the files the compiled reference writes."""
    import json
    import os
    import cityflow
    from cityflow_b200.capi import CReplay, REPLAY_DTYPE
    c = json.load(open(cfg_replay))
    log, netlog, log2 = c["dir"] + c["replayLogFile"], c["dir"] + c["roadnetLogFile"], c["dir"] + "replay_second.txt"
    for f in (log, netlog, log2):
        if os.path.exists(f):
            os.remove(f)
    flows = json.load(open(c["dir"] + c["flowFile"]))
    eng = cityflow.Engine(cfg_replay, thread_num=1)
    ora = H.PortOracle(cfg_replay)
    rp = CReplay(c["dir"] + c["roadnetFile"])
    assert open(netlog).read() == rp.roadnet_json()
    expect = []
    for s in range(1, 201):
        if s == 151:
            eng.set_save_replay(False)          # engine.cpp:736-742: steps 151..160 leave no line
        if s == 161:
            eng.set_save_replay(True)
            eng.set_replay_file("replay_second.txt")   # engine.cpp:727-734: relative to "dir"
        eng.next_step()
        ora.next_step()
        st = ora.snapshot()
        v = np.zeros(len(st.vehicles), REPLAY_DTYPE)
        v["drivable"], v["distance"] = st.vehicles["drivable"], st.vehicles["dis"]
        v["flow"], v["index"] = st.vehicles["flow"], st.vehicles["cnt"]
        v["length"] = [flows[f]["vehicle"]["length"] for f in st.vehicles["flow"]]
        v["width"] = [flows[f]["vehicle"]["width"] for f in st.vehicles["flow"]]
        expect.append(rp.format_step(v, np.where(st.phases < 0, 0, st.phases)))
    del eng                                      # closes the log like ~Engine (engine.cpp:763)
    first = open(log).read().split("\n")
    second = open(log2).read().split("\n")
    assert first[-1] == "" and second[-1] == ""
    assert first[:-1] == expect[:150]
    assert second[:-1] == expect[160:]
    assert len(expect[-1].split(",")) > 100


def _lc_gpu_states(eng, steps):
    """Per-step LC_DTYPE records of the GPU engine (every running vehicle including shadows) as StepState objects."""
    import ctypes
    lib = eng.lib
    lib.cfb_debug_lc_vehicles.restype = ctypes.c_int64
    lib.cfb_debug_lc_vehicles.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int64]
    lib.cfb_finished_vehicle_count.restype = ctypes.c_int64
    lib.cfb_finished_vehicle_count.argtypes = [ctypes.c_void_p]
    out = []
    for _ in range(steps):
        eng.next_step()
        n = int(lib.cfb_debug_lc_vehicles(eng.h, None, 0))
        got = np.zeros(n, H.LC_DTYPE)
        if n:
            lib.cfb_debug_lc_vehicles(eng.h, got.ctypes.data, n)
        st = H.StepState()
        st.vehicles = got
        st.finished = int(lib.cfb_finished_vehicle_count(eng.h))
        out.append(st)
    return out


def test_lane_change_statistics_vs_unmodified_reference(tmp_path):
    """laneChange=true against the UNMODIFIED reference.  Its lane-change schedule follows heap addresses (the order of
    a std::set<Vehicle*>), so only aggregates can agree: vehicles that finished, lane changes started, mean speed, running
    vehicles -- same tolerances as the restatement's own comparison (tests/test_cpu.py)."""
    if not H.have_ref():
        pytest.skip("oracle/_ref was not built")
    from cityflow_b200 import scenario
    from cityflow_b200.capi import CEngine
    cfg = scenario.make_grid_scenario(str(tmp_path), 5, 5, dense=dict(frac=1.0, interval=2.0, seed=11), name="lcstat", lane_change=True)
    eng = CEngine(cfg)
    ref = H.RefDump.runlc(cfg, 800, 1, n_inter=eng.n_inter, n_drivables=eng.n_drivables, patched=False)

    def summary(states):
        started, seen, speed = 0, set(), []
        for st in states:
            sh = st.vehicles["priority"][st.vehicles["partner_type"] == 2]
            started += len(set(sh.tolist()) - seen)
            seen |= set(sh.tolist())
            speed.append(float(st.vehicles["speed"].mean()))
        return dict(finished=states[-1].finished, started=started, speed=float(np.mean(speed[200:])), vehicles=len(states[-1].vehicles))

    a, b = summary(ref), summary(_lc_gpu_states(eng, 800))
    assert a["started"] > 200 and b["started"] > 200, (a, b)
    for k, tol in (("finished", 0.03), ("started", 0.15), ("speed", 0.03), ("vehicles", 0.03)):
        assert abs(a[k] - b[k]) <= tol * a[k], (k, a, b)


def test_lane_change_vs_restatement(tmp_path):
    """laneChange=true on the GPU against the restatement (pinned to oracle/_ref/refdump_lcorder, the reference with its
    worker sets ordered by priority): every running vehicle including shadows, every field, every step."""
    import ctypes
    from cityflow_b200 import scenario
    from cityflow_b200.capi import CEngine
    cfg = scenario.make_grid_scenario(str(tmp_path), 4, 4, dense=dict(frac=1.0, interval=3.0, seed=2), name="lc", lane_change=True)
    eng, ora = CEngine(cfg), H.PortOracle(cfg)
    lib = eng.lib
    lib.cfb_debug_lc_vehicles.restype = ctypes.c_int64
    lib.cfb_debug_lc_vehicles.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int64]
    shadows = 0
    for s in range(1, 401):
        eng.next_step()
        ora.next_step()
        want = ora.lc_snapshot()
        n = int(lib.cfb_debug_lc_vehicles(eng.h, None, 0))
        got = np.zeros(n, H.LC_DTYPE)
        if n:
            lib.cfb_debug_lc_vehicles(eng.h, got.ctypes.data, n)
        assert eng.vehicle_count() == want.vehicle_count, "step %d" % s
        assert np.array_equal(eng.lane_vehicle_count(), want.lane_count), "lane counts, step %d" % s
        assert len(got) == len(want.vehicles), "step %d" % s
        for f in H.LC_DTYPE.names:
            assert np.array_equal(got[f], want.vehicles[f]), "step %d field %s" % (s, f)
        shadows += int((want.vehicles["partner_type"] == 2).sum())
    assert shadows > 300


# ------------------------------------------------------------------------------------------
# Irregular networks (tests/randnet.py): missing streets, 1-3 lanes, bent roads, sparse laneLink sets -- including first
# lanes that cannot continue the route two roads ahead, where Vehicle::getNextSpeed's `if (laneChange)` block
# (vehicle.cpp:323-329, it tests the LaneChange OBJECT and so runs with laneChange=false too) parks the vehicle at the end
# of the lane.  Full state every step against the restatement (which is pinned to the compiled reference on the same
# generator, tests/test_cpu.py::test_random_network_loader_and_oracle_vs_reference).
@pytest.mark.parametrize("seed", [1, 2, 3, 5, 8, 11])
def test_fuzzed_irregular_networks_vs_port(seed, tmp_path):
    import randnet
    from cityflow_b200 import scenario
    net = randnet.random_roadnet(seed, rows=2 + seed % 3, cols=3 + seed % 2)
    flows = randnet.random_flows(net, seed + 100, n_flows=40 + seed % 50)
    cfg = scenario.write_scenario(str(tmp_path), net, flows, seed=seed, interval=[1.0, 0.5, 2.0, 1.0][seed % 4], name="g%d" % seed)
    _run_against_port(cfg, 500)


def test_fuzzed_network_vs_compiled_reference(tmp_path):
    """The same kind of network straight against the UNMODIFIED reference (oracle/_ref/refdump): the restatement shares the
    product's loader, the compiled reference does not -- a loader / routing bug cannot hide behind it here."""
    if not H.have_ref():
        pytest.skip("oracle/_ref was not built")
    import randnet
    from cityflow_b200 import scenario
    from cityflow_b200.capi import CEngine
    net = randnet.random_roadnet(4, rows=3, cols=4)
    flows = randnet.random_flows(net, 104, n_flows=70)
    cfg = scenario.write_scenario(str(tmp_path), net, flows, seed=4, interval=1.0, name="gref")
    eng = CEngine(cfg)
    ref = H.RefDump.run(cfg, 500, threads=2, every=10, n_inter=eng.n_inter, n_drivables=eng.n_drivables)
    done = 0
    for st in ref:
        eng.next_step(st.step - done)
        done = st.step
        bad = H.compare_states(_relax(st), _gpu_state(eng, st.step), check_order=False)
        assert not bad, "step %d: %s" % (st.step, "; ".join(bad[:6]))
    assert eng.tie_count() == 0


def test_vehicle_setters_step_by_step_vs_port(tmp_path):
    """set_vehicle_speed / set_vehicle_route (engine.cpp:827-866) applied identically to the GPU engine and to the
    restatement (itself pinned to the reference's Python module): every speed of every vehicle after every step."""
    import json
    import os
    import cityflow
    from cityflow_b200 import scenario
    cfg = scenario.make_grid_scenario(str(tmp_path), 4, 4, dense=dict(frac=1.0, interval=3.0, seed=2), name="api")
    flows = json.load(open(os.path.join(str(tmp_path), "flow_api.json")))
    eng, ora = cityflow.Engine(cfg, thread_num=1), H.PortOracle(cfg)

    def vid(f, k):
        return "manually_pushed_%d" % k if f == -2 else "flow_%d_%d" % (f, k)

    for s in range(1, 401):
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
                assert eng.set_vehicle_route(vid(f, k), target) == ora.set_vehicle_route(f, k, target), (s, vid(f, k))
        eng.next_step()
        ora.next_step()
        v = ora.vehicles()
        mine = eng.get_vehicle_speed()
        theirs = {vid(f, k): sp for f, k, sp in zip(v["flow"], v["cnt"], v["speed"])}
        assert mine == theirs, "step %d: %s" % (s, [(k, mine.get(k), theirs[k]) for k in theirs if mine.get(k) != theirs[k]][:3])


def test_30x30_through_the_bench_window_vs_compiled_reference(scenario_dir):
    """The bench operating point itself: BASELINE.json configs[2] (30x30, ~1.3e5 vehicles, gridlock) against the UNMODIFIED
    reference -- vehicle count after every step, per-lane counts, per-lane waiting counts (speed < 0.1) and per-lane speed
    sums (within 1e-6 per vehicle) every 50 steps and at steps 1200, 1210, 1220, 1230 (the vehicle count at every step of
    the window 1200..1230)."""
    if not H.have_ref():
        pytest.skip("oracle/_ref was not built")
    import os
    from cityflow_b200 import scenario
    from cityflow_b200.capi import CEngine
    cfg = scenario.make_grid_scenario(scenario_dir, 30, 30, name="g30w", dense=dict(frac=0.5, interval=10.0, seed=1, fleet_spread=0.02))
    ref = H.RefDump.counts(cfg, 1230, os.cpu_count() or 8, 10)
    eng = CEngine(cfg)
    for s in range(1, 1231):
        eng.next_step()
        if s >= 1200 or s % 5 == 0:
            assert eng.vehicle_count() == int(ref["vehicle_count"][s - 1]), s
        if s % 10 or (s % 50 and s < 1200):
            continue
        rc, rw, rs = ref["dumps"][s]
        assert eng.vehicle_count() == int(ref["vehicle_count"][s - 1]), s
        mc, mw = eng.lane_vehicle_count(), eng.lane_waiting_count()
        assert np.array_equal(mc, rc), "step %d: %d lane counts differ" % (s, int((mc != rc).sum()))
        assert np.array_equal(mw, rw), "step %d: %d lane waiting counts differ" % (s, int((mw != rw).sum()))
    # per-vehicle speeds at the end, through the per-lane speed sums (bar: 1e-6 per vehicle; the sums differ by summation order only)
    v = eng.debug_vehicles()
    on = v[v["drivable"] < eng.n_lanes]
    mine = np.bincount(on["drivable"], weights=on["speed"], minlength=eng.n_lanes)
    assert np.all(np.abs(mine - rs) <= 1e-6 * np.maximum(mc, 1)), "per-lane speed sums differ"
    assert eng.vehicle_count() > 120000
    assert eng.tie_count() == 0   # (the bench fleet: no entrant tie, so the reference's result is defined -- bench.py FLEET_SPREAD)


def test_6x6_3600_steps_vs_port(cfg_6x6):
    """BASELINE.json configs[1] length: the generator's default 6x6 scenario for the full 3600 steps, full state every 100."""
    _run_against_port(cfg_6x6, 3600, every=100)


# ------------------------------------------------------------------------------------------
# Edge shapes (tests/edgenet.py): buckets of 3+ warp chunks filled beyond 2.5 m spacing, laneLinks with more than 32
# vehicles and more than 64 crosses (three mask words and more), vehicles crossing 3+ drivables per step.  The restatement
# is pinned to the compiled reference on the same shapes (tests/test_cpu.py::test_edge_network_loader_and_restatement_vs_reference).
def _edge_static(cfg):
    import edgenet
    return edgenet.loader_tables(cfg)


@pytest.mark.parametrize("shape,steps", [("long_queue", 700), ("star", 400), ("short_hops", 500)])
def test_edge_networks_vs_port(shape, steps, tmp_path):
    import edgenet
    cfg = edgenet.write(shape, str(tmp_path))
    static = _edge_static(cfg)
    reach = edgenet.Reach(static)
    eng, ora = _run_against_port(cfg, steps, hook=lambda eng, ora, s: reach.add(eng.debug_vehicles()))
    print("%s: %s; highest refused cross index %d" % (shape, reach, ora.max_refused_cross_index()))
    assert ora.tie_count() == 0 and eng.average_travel_time() == ora.average_travel_time()
    if shape == "long_queue":
        assert reach.lane_occ > 96 and reach.link_occ > 32
    if shape == "star":
        assert max(static["link_cross_count"]) > 64 and ora.max_refused_cross_index() >= 32
    if shape == "short_hops":
        assert reach.hops >= 3


def test_edge_long_queue_lane_change_vs_restatement(tmp_path):
    """Lane change over buckets of 3+ warp chunks (shadow inserts into long buckets, segment scans): every running
    vehicle including shadows, every field, every step."""
    import ctypes
    import edgenet
    from cityflow_b200.capi import CEngine
    cfg = edgenet.write("long_queue", str(tmp_path), lane_change=True)
    eng, ora = CEngine(cfg), H.PortOracle(cfg)
    lib = eng.lib
    lib.cfb_debug_lc_vehicles.restype = ctypes.c_int64
    lib.cfb_debug_lc_vehicles.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int64]
    reach = edgenet.Reach(_edge_static(cfg))
    shadows = 0
    for s in range(1, 701):
        eng.next_step()
        ora.next_step()
        want = ora.lc_snapshot()
        n = int(lib.cfb_debug_lc_vehicles(eng.h, None, 0))
        got = np.zeros(n, H.LC_DTYPE)
        if n:
            lib.cfb_debug_lc_vehicles(eng.h, got.ctypes.data, n)
        assert eng.vehicle_count() == want.vehicle_count, "step %d" % s
        assert np.array_equal(eng.lane_vehicle_count(), want.lane_count), "lane counts, step %d" % s
        assert len(got) == len(want.vehicles), "step %d" % s
        for f in H.LC_DTYPE.names:
            assert np.array_equal(got[f], want.vehicles[f]), "step %d field %s" % (s, f)
        shadows += int((want.vehicles["partner_type"] == 2).sum())
        reach.add(got[got["partner_type"] != 2])
    print("long_queue with lane change: %s; %d shadow states" % (reach, shadows))
    assert shadows > 100 and reach.lane_occ > 96 and reach.link_occ > 32


def test_edge_star_vs_compiled_reference(tmp_path):
    """laneLinks with hundreds of crosses straight against the UNMODIFIED reference: the cross order of the product's
    loader cannot hide behind the restatement, which shares it."""
    if not H.have_ref():
        pytest.skip("oracle/_ref was not built")
    import edgenet
    from cityflow_b200.capi import CEngine
    cfg = edgenet.write("star", str(tmp_path))
    eng = CEngine(cfg)
    ref = H.RefDump.run(cfg, 400, threads=1, every=1, n_inter=eng.n_inter, n_drivables=eng.n_drivables)
    for st in ref:
        eng.next_step()
        bad = H.compare_states(_relax(st), _gpu_state(eng, st.step), check_order=False)
        assert not bad, "step %d: %s" % (st.step, "; ".join(bad[:6]))
    assert eng.tie_count() == 0 and ref[-1].vehicle_count > 1000


def test_edge_long_queue_lane_observations(tmp_path):
    """LaneObservations (per-lane warp loops over buckets of more than 64 vehicles) against the host getters."""
    import cityflow
    import cityflow_b200
    import edgenet
    cfg = edgenet.write("long_queue", str(tmp_path))
    eng = cityflow.Engine(cfg, thread_num=1)
    obs = cityflow_b200.LaneObservations(eng)
    most = 0
    for _ in range(7):
        eng.next_steps(100)
        obs.refresh()
        counts, waiting = eng.get_lane_vehicle_count(), eng.get_lane_waiting_vehicle_count()
        assert obs.vehicle_count.tolist() == [counts[i] for i in obs.lane_ids]
        assert obs.waiting_count.tolist() == [waiting[i] for i in obs.lane_ids]
        speeds = eng.get_vehicle_speed()
        per_lane = {i: 0.0 for i in obs.lane_ids}
        for lane, vs in eng.get_lane_vehicles().items():
            per_lane[lane] = sum(speeds[v] for v in vs)
        np.testing.assert_allclose(obs.speed_sum.cpu().numpy(), np.array([per_lane[i] for i in obs.lane_ids]), rtol=0, atol=1e-9)
        most = max(most, max(counts.values()))
    print("long_queue: most vehicles on one lane %d" % most)
    assert most > 96


# ------------------------------------------------------------------------------------------
# The tie rule (tests/edgenet.py merge_ties): 2, 3 and 4 vehicles enter one lane in the same step at the same distance.
# k_move ranks them by ascending priority whatever order they were staged in (atomics: nondeterministic).  The
# restatement's tie order is pinned to the priority-ordered reference on this shape
# (tests/test_cpu.py::test_tie_rule_restatement_vs_priority_ordered_reference).  The GPU's state has no list positions:
# list order shows in leader, gap and blocker, which differ for a swapped pair.
TIE_STEPS = 600


def test_tie_network_vs_port_twice(tmp_path):
    """Two runs on the GPU, each equal to the restatement every step, tie counts included: a tie order that followed
    the staging order would differ between runs or from the restatement."""
    import edgenet
    cfg = edgenet.write("merge_ties", str(tmp_path))
    for run in range(2):
        counts = []
        eng, ora = _run_against_port(cfg, TIE_STEPS, hook=lambda eng, ora, s: counts.append((s, eng.tie_count(), ora.tie_count())))
        assert eng.tie_count() == ora.tie_count()
        assert all(a == b for _, a, b in counts), [c for c in counts if c[1] != c[2]][:3]
        assert eng.average_travel_time() == ora.average_travel_time()
        print("merge_ties run %d: %d tied pairs" % (run, ora.tie_count()))
        assert ora.tie_count() >= 50


def test_tie_network_lane_change_vs_restatement(tmp_path):
    """merge_ties with lane change: tied pairs in both lanes of I -> J, neighbours at bit-equal distances, every
    running vehicle including shadows, every field, every step."""
    import ctypes
    import edgenet
    from cityflow_b200.capi import CEngine
    cfg = edgenet.write("merge_ties", str(tmp_path), lane_change=True)
    eng, ora = CEngine(cfg), H.PortOracle(cfg)
    lib = eng.lib
    lib.cfb_debug_lc_vehicles.restype = ctypes.c_int64
    lib.cfb_debug_lc_vehicles.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int64]
    shadows = 0
    for s in range(1, TIE_STEPS + 1):
        eng.next_step()
        ora.next_step()
        want = ora.lc_snapshot()
        n = int(lib.cfb_debug_lc_vehicles(eng.h, None, 0))
        got = np.zeros(n, H.LC_DTYPE)
        if n:
            lib.cfb_debug_lc_vehicles(eng.h, got.ctypes.data, n)
        assert eng.vehicle_count() == want.vehicle_count, "step %d" % s
        assert np.array_equal(eng.lane_vehicle_count(), want.lane_count), "lane counts, step %d" % s
        assert len(got) == len(want.vehicles), "step %d" % s
        for f in H.LC_DTYPE.names:
            assert np.array_equal(got[f], want.vehicles[f]), "step %d field %s" % (s, f)
        assert eng.tie_count() == ora.tie_count(), "step %d" % s
        shadows += int((want.vehicles["partner_type"] == 2).sum())
    reach = ora.tie_reach()
    print("merge_ties with lane change: %s; %d shadow states" % (reach, shadows))
    assert reach["ties"] >= 50 and reach["lc_equal_schedules"] >= 1 and shadows > 0


def test_tie_network_sharded_loopback_vs_restatement(tmp_path):
    """merge_ties on two ranks of one GPU: I on rank 0, J on rank 1, so I -> J is a seam lane and the tied entrants
    reach its owner through the mover mailbox.  Every vehicle equal to the restatement every step."""
    import edgenet
    from cityflow_b200.capi import CShardGroup
    cfg = edgenet.write("merge_ties", str(tmp_path))
    grp, ora = CShardGroup(cfg, 2), H.PortOracle(cfg)
    for s in range(1, TIE_STEPS + 1):
        grp.next_step()
        ora.next_step()
        st = ora.snapshot()
        assert grp.vehicle_count() == st.vehicle_count, "step %d" % s
        assert np.array_equal(grp.lane_counts(ora.n_lanes), st.lane_count), "lane counts, step %d" % s
        a, b = np.sort(grp.debug_vehicles(), order=["flow", "cnt"]), np.sort(st.vehicles, order=["flow", "cnt"])
        assert len(a) == len(b), "step %d" % s
        for f in ("flow", "cnt", "priority", "drivable", "dis", "speed", "leader_flow", "leader_cnt", "blocker_flow", "blocker_cnt", "gap",
                  "enter_ll_time"):
            assert np.array_equal(a[f], b[f]), "step %d field %s" % (s, f)
    assert ora.tie_count() >= 50


def test_tie_network_binary_snapshot_with_a_tied_pair(tmp_path):
    """A binary snapshot taken while a tied pair shares a lane at one distance, loaded into a fresh engine and run on
    for 100 steps against the restatement: the image codec has to keep the pair's list order."""
    import edgenet
    from cityflow_b200.capi import CEngine
    cfg = edgenet.write("merge_ties", str(tmp_path))
    eng, ora = CEngine(cfg), H.PortOracle(cfg)
    for s in range(1, 400):
        eng.next_step()
        ora.next_step()
        v = ora.vehicles()
        if s > 100 and len({(int(d), float(x)) for d, x in zip(v["drivable"], v["dis"])}) < len(v):
            break
    else:
        pytest.fail("no two vehicles shared a drivable and a distance")
    path = str(tmp_path / "tied.bin")
    eng.dump(path)
    fresh = CEngine(cfg)
    fresh.load_from_file(path)
    bad = H.compare_states(_relax(ora.snapshot()), _gpu_state(fresh, s))
    assert not bad, "after load at step %d: %s" % (s, "; ".join(bad[:6]))
    for k in range(1, 101):
        fresh.next_step()
        ora.next_step()
        bad = H.compare_states(_relax(ora.snapshot()), _gpu_state(fresh, s + k))
        assert not bad, "step %d after a load at step %d: %s" % (s + k, s, "; ".join(bad[:6]))
    assert ora.tie_count() > 0
