"""cityflow_b200 -- H100-native step engine behind the ``cityflow.Engine`` Python surface.

``Engine`` is the pybind11 class built from ``csrc/pymodule.cpp`` over the C-ABI in
``include/cityflow_b200.h`` (``libcityflow_b200.so``: host loader + sm_90a kernels).  There is no
CPU fallback: importing works anywhere (so the package can be built and inspected on a CPU box),
but constructing an ``Engine`` without a CUDA device raises ``RuntimeError``.
"""
import os as _os

_HERE = _os.path.dirname(_os.path.abspath(__file__))
LIB_PATH = _os.path.join(_HERE, "libcityflow_b200.so")

try:
    from ._cityflow_b200 import Archive, Engine, __version__, nccl_unique_id  # noqa: F401
except ImportError as _e:  # extension not built: fail loudly at use, not silently
    _IMPORT_ERROR = _e

    class Engine:  # type: ignore
        def __init__(self, *a, **k):
            raise RuntimeError(
                "cityflow_b200: the CUDA extension is not built (%s). Run "
                "`python -c 'import __graft_entry__ as g; g.build()'` in the repo root." % (_IMPORT_ERROR,))

    __version__ = "unbuilt"

    class Archive:  # type: ignore
        def __init__(self, *a, **k):
            raise RuntimeError("cityflow_b200: the CUDA extension is not built")


class _DeviceArray:
    """A device array of the engine exposed through ``__cuda_array_interface__`` (keeps the engine alive)."""

    def __init__(self, owner, ptr, n, typestr):
        self._owner = owner
        self.__cuda_array_interface__ = {"shape": (n,), "typestr": typestr, "data": (ptr, False),
                                         "version": 2, "strides": None}


class LaneObservations:
    """Zero-copy per-lane observations as torch CUDA tensors (SURVEY 8f-3).

    ``vehicle_count`` (int32) and ``waiting_count`` (int32) are the arrays
    ``get_lane_vehicle_count`` / ``get_lane_waiting_vehicle_count`` report (engine.cpp:628-648),
    ``speed_sum`` (float64) the per-lane sum of speeds, all in ``lane_ids`` (= ``engine.lane_ids()``)
    order and living on the engine's GPU.  The tensors alias the engine's buffers and are created
    once; ``refresh()`` re-computes their content on the engine's stream, ordered against ``stream``
    (default: torch's current stream on that device) in both directions -- nothing is copied to the
    host and the host does not wait.  ``clone()`` what must survive the next refresh.
    """

    def __init__(self, engine, stream=None):
        import torch
        self.engine = engine
        self.lane_ids = engine.lane_ids()
        self._device = engine.device()
        o = engine.observe_device(self._stream(stream))
        n = o["n_lanes"]
        dev = torch.device("cuda", o["device"])
        self._ptrs = (o["lane_vehicle_count"], o["lane_waiting_count"], o["lane_speed_sum"])
        mk = lambda ptr, ts: torch.as_tensor(_DeviceArray(engine, ptr, n, ts), device=dev)  # noqa: E731
        self.vehicle_count = mk(self._ptrs[0], "<i4")
        self.waiting_count = mk(self._ptrs[1], "<i4")
        self.speed_sum = mk(self._ptrs[2], "<f8")

    def _stream(self, stream):
        if stream is None:
            import torch
            return torch.cuda.current_stream(self._device).cuda_stream
        return int(getattr(stream, "cuda_stream", stream))

    def refresh(self, stream=None):
        o = self.engine.observe_device(self._stream(stream))
        assert (o["lane_vehicle_count"], o["lane_waiting_count"], o["lane_speed_sum"]) == self._ptrs
        return self


def lane_observation_tensors(engine, stream=None):
    """One-shot form of :class:`LaneObservations`:
    ``(lane_ids, vehicle_count, waiting_count, speed_sum)``, freshly computed."""
    o = LaneObservations(engine, stream)
    return o.lane_ids, o.vehicle_count, o.waiting_count, o.speed_sum


def set_tl_phases_tensor(engine, phases, stream=None):
    """``set_tl_phase`` for every traffic light at once from a torch CUDA tensor (no host copy).

    ``phases``: int32, contiguous, one entry per intersection in ``engine.intersection_ids()`` order
    (virtual intersections included, their entries ignored), on the engine's GPU, produced on
    ``stream`` (default: torch's current stream there).  Needs ``"rlTrafficLight": true``.
    """
    import torch
    if not (phases.is_cuda and phases.dtype == torch.int32 and phases.is_contiguous()
            and phases.device.index == engine.device() and phases.numel() == engine.num_intersections()):
        raise ValueError("phases must be a contiguous int32 CUDA tensor on the engine's device, one entry per intersection")
    if stream is None:
        stream = torch.cuda.current_stream(engine.device()).cuda_stream
    engine.set_tl_phases_device(phases.data_ptr(), int(stream))
