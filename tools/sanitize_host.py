"""Host-side sanitizer tour (no GPU): builds the TEST library of the C-ABI (csrc/host_engine.cpp & co. over
tests/device_sim_emu.cpp -- the kernel bodies on an emulated warp) with one of the compiler's sanitizers and drives it
through the paths the GPU tests drive: the host engine with pushes / re-seeding / reset (both spawner modes), lane
change, a three-rank loop-back group, fuzzed irregular networks, both archive forms, damaged archives.

    python tools/sanitize_host.py undefined      # -fsanitize=undefined,bounds + libstdc++ assertions, -O2
    python tools/sanitize_host.py address        # -fsanitize=address (LD_PRELOADs libasan into the child python)
    python tools/sanitize_host.py thread         # -fsanitize=thread, kernel-free spawner mode only (four-thread creation, collisions)

A report aborts the child (non-recoverable); the script prints "clean" when every stage ran.  The GPU-side twin is
tools/sanitize_run.py (compute-sanitizer on the GPU).  TEST INFRASTRUCTURE: the emulated device is not a CPU path of the
product (it refuses to start without CFB_EMULATED_DEVICE_FOR_TESTS=1 and nothing in cityflow_b200/ can load it)."""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "oracle", "_build")
CSRC = os.path.join(ROOT, "cityflow_b200", "csrc")

FLAGS = {
    "undefined": ["-O2", "-fsanitize=undefined,bounds", "-fno-sanitize-recover=undefined", "-D_GLIBCXX_ASSERTIONS"],
    "address": ["-O1", "-fsanitize=address", "-fno-omit-frame-pointer"],
    "thread": ["-O1", "-fsanitize=thread"],
}
RUNTIME = {"undefined": "libubsan.so", "address": "libasan.so", "thread": "libtsan.so"}

DRIVER = r'''
import ctypes, json, os, sys
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
from cityflow_b200 import capi, scenario
lib = capi.bind(ctypes.CDLL(LIB))
class E(capi.CEngine):
    def _library(self): return lib
d = TMP
if MODE == "thread":
    cfg = scenario.make_grid_scenario(d, 30, 12, name="t", dense=dict(frac=0.5, interval=10.0, seed=1, fleet_spread=0.02))
    e = E(cfg, 0); e.next_step(40); e.set_random_seed(0); e.next_step(40); e.set_random_seed(0); e.next_step(20)
    print("parallel creation with collisions ok"); sys.exit(0)
import randnet, archive_checks
cfg = scenario.make_grid_scenario(d, 3, 3, dense=dict(frac=1.0, interval=3.0, seed=3), name="h")
route = json.load(open(os.path.join(d, "flow_h.json")))[2]["route"]
e = E(cfg, 0)
for s in range(1, 231):
    if s in (30, 31, 90): e.push_vehicle({"speed": 2.0, "length": 6.0} if s != 31 else {}, route)
    if s == 120: e.set_random_seed(5)
    if s == 150: e.set_random_seed(0)
    if s == 200: e.reset(True)
    e.next_step(); e.vehicle_count(); e.lane_vehicle_count(); e.debug_vehicles()
e.dump(d + "/a.json"); e.dump(d + "/a.bin"); e.load_from_file(d + "/a.json"); e.next_step(3); e.load_from_file(d + "/a.bin"); e.next_step(3)
print("host engine + archives ok")
cfg = scenario.make_grid_scenario(d, 3, 3, dense=dict(frac=1.0, interval=3.0, seed=3), name="lc", lane_change=True)
e = E(cfg, 0); e.next_step(200); e.dump(d + "/lc.bin"); e.load_from_file(d + "/lc.bin"); e.next_step(10)
print("lane change ok")
cfg = scenario.make_grid_scenario(d, 3, 6, dense=dict(frac=1.0, interval=3.0, seed=4), name="seam")
g = lib.cfb_shard_group_create(cfg.encode(), 3, 0); assert g
assert lib.cfb_shard_group_step(g, 200) == 0
lib.cfb_shard_group_destroy(g)
print("three-rank loop-back group ok")
for seed, lc in ((2, False), (11, False), (7, True)):
    net = randnet.random_roadnet(seed, rows=2 + seed % 3, cols=3 + seed % 2)
    flows = randnet.random_flows(net, seed + 100, n_flows=40 + seed % 50)
    cfg = scenario.write_scenario(d, net, flows, seed=seed, interval=[1.0, 0.5, 2.0, 1.0][seed % 4], lane_change=lc, name="fz%d" % seed)
    e = E(cfg, 0); e.next_step(300); e.close()
print("fuzzed networks ok")
if MODE == "undefined":   # (C++ exceptions thrown under a preloaded ASan trip its interceptor in a python host)
    cfg = scenario.make_grid_scenario(d, 2, 2, dense=dict(frac=1.0, interval=3.0, seed=3), name="fj")
    print("damaged archives refused:", archive_checks.check_damaged_json_is_refused(lambda c: E(c, 0), cfg, d, rounds=300))
'''


def main():
    mode = sys.argv[1] if len(sys.argv) > 1 else "undefined"
    if mode not in FLAGS:
        sys.exit(__doc__)
    os.makedirs(OUT, exist_ok=True)
    lib = os.path.join(OUT, "libcfb_hostcheck_%s.so" % mode)
    srcs = [os.path.join(ROOT, "tests", "device_sim_emu.cpp")] + [os.path.join(CSRC, f) for f in
            ("host_engine.cpp", "roadnet.cpp", "flows.cpp", "partition.cpp", "shard.cpp", "replay.cpp", "json_write.cpp")]
    subprocess.check_call(["g++", "-std=c++17", "-g", "-fPIC", "-shared", "-ffp-contract=off"] + FLAGS[mode] +
                          ["-I/usr/local/cuda/include", "-I" + CSRC, "-I" + os.path.join(ROOT, "include")] + srcs +
                          ["-L/usr/local/cuda/lib64", "-lcudart", "-ldl", "-o", lib])
    import tempfile
    runtime = subprocess.check_output(["g++", "-print-file-name=" + RUNTIME[mode]], text=True).strip()
    with tempfile.TemporaryDirectory() as tmp:
        env = dict(os.environ, CFB_EMULATED_DEVICE_FOR_TESTS="1", LD_PRELOAD=runtime,
                   ASAN_OPTIONS="detect_leaks=0:detect_stack_use_after_return=0")
        if mode == "thread":
            env.update(CFB_EMU_HOST_ONLY="50000", CITYFLOW_B200_PARALLEL_SPAWN_MIN="2")
        head = "ROOT=%r\nLIB=%r\nTMP=%r\nMODE=%r\n" % (ROOT, lib, tmp, mode)
        out = subprocess.run([sys.executable, "-c", head + DRIVER], env=env, capture_output=True, text=True)
    sys.stdout.write(out.stdout)
    reports = [l for l in out.stderr.splitlines() if "runtime error" in l or "ERROR: AddressSanitizer" in l or "WARNING: ThreadSanitizer" in l]
    if out.returncode != 0 or reports:
        sys.stderr.write(out.stderr[-4000:])
        sys.exit("NOT clean (%s): exit %d, %d report lines" % (mode, out.returncode, len(reports)))
    print("clean (%s)" % mode)


if __name__ == "__main__":
    main()
