"""Developer tool (TEST INFRASTRUCTURE): run the LOGIC of the `-m gpu` tests without a GPU.

    PYTHONPATH=tests python -m pytest tests/test_gpu_parity.py tests/test_gpu_zarchive.py tests/test_gpu_zz_python_api.py \
        -p emulated_device_plugin -m gpu -k "not 30x30 and not device_resident and not on_device"

With this plugin loaded, `cityflow_b200.capi.CEngine` opens the TEST build of the C-ABI (csrc/host_engine.cpp over
tests/device_sim_emu.cpp: the kernel bodies on an emulated warp) and `import cityflow` resolves to csrc/pymodule.cpp linked
against it, so everything above the kernels' launch configuration -- the host engine, the C-ABI, the pybind11 module and
the test code itself -- is exercised exactly as on the GPU box, about a thousand times slower.  It is how tests added
after a round's last GPU session are checked before the driver runs them on hardware (33 of the 37 single-GPU tests
fit: not the 30x30 ones (capacity of the emulated device) and not the device-resident observation / action tests).

It is NOT a way to run the product on a CPU: nothing in cityflow_b200/ can load these libraries, the emulated device
refuses to start without CFB_EMULATED_DEVICE_FOR_TESTS=1 (set here), and a run with this plugin says nothing about
kernels on hardware -- the driver's `pytest -m gpu` on an H100 does not load it."""
import ctypes
import os
import sys

os.environ["CFB_EMULATED_DEVICE_FOR_TESTS"] = "1"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)


def pytest_configure(config):
    import test_cpu
    sys.path.insert(0, test_cpu._pyemu_dir())
    import cityflow   # the emulated build first: the real extension then cannot register its types and the package falls back
    assert "pyemu" in cityflow.__file__
    from cityflow_b200 import capi
    lib = capi.bind(ctypes.CDLL(test_cpu._hostcheck_lib()))
    capi.CEngine._library = lambda self: lib
    capi.load_library = lambda: lib
