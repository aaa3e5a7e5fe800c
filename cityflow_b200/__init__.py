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


class VehicleObservations:
    """Zero-copy table of every running vehicle as torch CUDA tensors, for a policy on the engine's GPU.

    Rows are drivable-major: lanes in ``engine.lane_ids()`` order, then the laneLinks (``drivable_ids``
    holds the ids of both); the rows of drivable ``d`` are ``drivable_begin[d]:drivable_begin[d + 1]``, in
    list order, front first -- for a lane the order ``get_lane_vehicles()`` reports.  Columns: ``slot``,
    ``priority`` and ``drivable`` (int32), ``distance`` and ``speed`` (float64, bit-equal to
    ``get_vehicle_distance()`` / ``get_vehicle_speed()``), ``shadow`` (uint8, 1 for a lane-change shadow).
    ``count`` (int32, one element) is the number of rows in use (= ``get_vehicle_count()``); the rows from
    ``count`` to the tensors' length are padding with ``slot == -1``, so a policy of fixed shape can mask them.
    Waiting vehicles are not rows.

    ``(slot, priority)`` is a row's vehicle handle: :func:`set_vehicle_speeds_tensor` takes it, and
    ``vehicle_ids(slots)`` turns slots into the reference's ids.  ``refresh()`` re-computes the table on the
    engine's stream, ordered against ``stream`` (default: torch's current stream on that device) in both
    directions, without a host copy or wait; the tensors alias the engine's buffers and keep their storage
    across refreshes.  ``clone()`` what must survive the next refresh.  Single-GPU engines only.

    With ``context=True`` every refresh also fills, from the same state, what lies ahead of each row (capacity
    length, aligned with the rows):

    * ``leader`` (int32): the row of the vehicle's leader as the last step found it (``get_leader``), which may
      be on the next lane or on an overlapping laneLink; -1 none.
    * ``gap`` (float64): the gap to that leader, bit-equal to the reference's; ``+inf`` without a leader.
    * ``next_drivable`` (int32): the drivable the vehicle takes next, in ``drivable_ids`` numbering -- for a lane
      row the laneLink it will take, for a laneLink row its end lane; -1 on the route's last road, -2 on a lane
      that cannot continue the route.
    * ``signal`` (int8): for a lane row heading for a laneLink, 1 if that movement is green in its
      intersection's current phase (including ``set_tl_phase`` calls made since the last step), else 0; -1 on
      every other row.

    Padding rows hold leader -1, gap ``+inf``, next_drivable -1 and signal -1.  A lane-change shadow's row holds
    the shadow's own leader, gap and next drivable, while ``get_leader`` of a shadow answers for its car.  Static
    columns, aliases of the engine's tables: ``drivable_length`` and ``drivable_max_speed`` (float64, per
    drivable; a laneLink's max speed is the reference's placeholder 10000) and ``link_road_link`` (int32, per
    laneLink: the movement index of :class:`IntersectionObservations`).  ``n_lanes`` is where the laneLinks'
    drivable numbers start.
    """

    _COLUMNS = (("slot", "<i4"), ("priority", "<i4"), ("drivable", "<i4"), ("distance", "<f8"), ("speed", "<f8"),
                ("shadow", "|u1"))
    _CONTEXT = (("leader", "<i4"), ("gap", "<f8"), ("next_drivable", "<i4"), ("signal", "|i1"))

    def __init__(self, engine, stream=None, context=False):
        self.engine = engine
        self._device = engine.device()
        self._ptrs = None
        self._context = context
        self.drivable_ids = engine.drivable_ids()
        self.refresh(stream)

    def _stream(self, stream):
        if stream is None:
            import torch
            return torch.cuda.current_stream(self._device).cuda_stream
        return int(getattr(stream, "cuda_stream", stream))

    def refresh(self, stream=None):
        if self._context:
            o = self.engine.observe_vehicle_context_device(self._stream(stream))
            columns = self._COLUMNS + self._CONTEXT
        else:
            o = self.engine.observe_vehicles_device(self._stream(stream))
            columns = self._COLUMNS
        ptrs = tuple(o[k] for k, _ in columns) + (o["drivable_begin"], o["count"], o["capacity"])
        if ptrs != self._ptrs:   # first call, or the engine re-allocated its buffers
            import torch
            dev = torch.device("cuda", o["device"])
            mk = lambda ptr, n, ts: torch.as_tensor(_DeviceArray(self.engine, ptr, n, ts), device=dev)  # noqa: E731
            for k, ts in columns:
                setattr(self, k, mk(o[k], o["capacity"], ts))
            self.drivable_begin = mk(o["drivable_begin"], o["n_drivables"] + 1, "<i4")
            self.count = mk(o["count"], 1, "<i4")
            if self._context:
                self.drivable_length = mk(o["drivable_length"], o["n_drivables"], "<f8")
                self.drivable_max_speed = mk(o["drivable_max_speed"], o["n_drivables"], "<f8")
                self.link_road_link = mk(o["link_road_link"], o["n_links"], "<i4")
                self.n_lanes = o["n_lanes"]
            self._ptrs = ptrs
        return self

    def vehicle_ids(self, slots):
        """The reference's ids of the vehicles in ``slots`` (a tensor, array or list; host side: it waits for the
        device), ``None`` where a slot holds no vehicle.  A shadow still changing lanes is ``"<id>_shadow"``."""
        if hasattr(slots, "tolist"):
            slots = slots.tolist()
        return self.engine.vehicle_ids([int(s) for s in slots])


class IntersectionObservations:
    """Zero-copy traffic-light observations as torch CUDA tensors: every light's phase and every movement's queue and
    pressure, for a signal controller on the engine's GPU (MaxPressure, PressLight).

    A movement is a roadLink; ``road_links`` (``engine.road_links()``) names them in the order of the movement
    columns: intersections in ``engine.intersection_ids()`` order, each one's ``"roadLinks"`` in file order.
    ``in_lanes(r)`` / ``out_lanes(r)`` are the distinct start / end lanes of r's laneLinks, ``in_lanes(i)`` /
    ``out_lanes(i)`` their union over intersection i; ``count`` / ``waiting`` are ``get_lane_vehicle_count()`` /
    ``get_lane_waiting_vehicle_count()``.  Per intersection (``[n_intersections]``): ``phase`` (int32, the index
    ``set_tl_phase`` takes, -1 for a virtual intersection), ``phase_remaining`` (float64, remainDuration as
    ``Archive.dump("x.json")`` writes it), ``pressure`` (int32, count over in_lanes(i) minus over out_lanes(i)),
    ``queue`` (int32, waiting over in_lanes(i)).  Per movement (``[n_road_links]``, int32): ``movement_in``,
    ``movement_in_waiting``, ``movement_out``, ``movement_inside`` (vehicles on its laneLinks) and
    ``movement_pressure`` (in - out).  ``phase_pressure`` (int32 ``[n_intersections, max_phases]``): the sum of
    movement_pressure over the movements available in each phase, ``INT32_MIN`` past ``phase_count[i]``, so
    ``phase_pressure.argmax(1).to(torch.int32)`` is the MaxPressure action for :func:`set_tl_phases_tensor`.
    Static: ``movement_begin`` ``[n_intersections + 1]``, ``movement_intersection``, ``phase_count`` and
    ``phase_movements`` (uint8 ``[n_intersections, max_phases, max_movements]``).

    ``refresh()`` re-computes the dynamic columns on the engine's stream after every ``set_tl_phase`` made before it,
    ordered against ``stream`` (default: torch's current stream on that device) in both directions, without a host
    copy or wait; the tensors alias the engine's buffers and keep their storage across refreshes.  ``clone()`` what
    must survive the next refresh.  Single-GPU engines only.
    """

    _FLAT = (("phase", "<i4", "n_intersections"), ("phase_remaining", "<f8", "n_intersections"),
             ("pressure", "<i4", "n_intersections"), ("queue", "<i4", "n_intersections"),
             ("movement_in", "<i4", "n_road_links"), ("movement_in_waiting", "<i4", "n_road_links"),
             ("movement_out", "<i4", "n_road_links"), ("movement_inside", "<i4", "n_road_links"),
             ("movement_pressure", "<i4", "n_road_links"), ("movement_intersection", "<i4", "n_road_links"),
             ("phase_count", "<i4", "n_intersections"))

    def __init__(self, engine, stream=None):
        import torch
        self.engine = engine
        self._device = engine.device()
        self.road_links = engine.road_links()
        o = engine.observe_intersections_device(self._stream(stream))
        dev = torch.device("cuda", o["device"])
        mk = lambda k, n, ts: torch.as_tensor(_DeviceArray(engine, o[k], n, ts), device=dev)  # noqa: E731
        for k, ts, n in self._FLAT:
            setattr(self, k, mk(k, o[n], ts))
        nI, mP, mM = o["n_intersections"], o["max_phases"], o["max_movements"]
        self.movement_begin = mk("movement_begin", nI + 1, "<i4")
        self.phase_pressure = mk("phase_pressure", nI * mP, "<i4").view(nI, mP)
        self.phase_movements = mk("phase_movements", nI * mP * mM, "|u1").view(nI, mP, mM)
        self._ptrs = tuple(o[k] for k in sorted(o))

    def _stream(self, stream):
        if stream is None:
            import torch
            return torch.cuda.current_stream(self._device).cuda_stream
        return int(getattr(stream, "cuda_stream", stream))

    def refresh(self, stream=None):
        o = self.engine.observe_intersections_device(self._stream(stream))
        assert tuple(o[k] for k in sorted(o)) == self._ptrs
        return self


def set_vehicle_speeds_tensor(engine, slot, priority, speed, stream=None):
    """``set_vehicle_speed`` for many vehicles at once from torch CUDA tensors (no host copy, no host wait).

    ``slot`` / ``priority`` (int32) and ``speed`` (float64): contiguous, the same length, on the engine's GPU,
    produced on ``stream`` (default: torch's current stream there).  Entry ``i`` sets a one-shot custom speed
    for the coming step on the vehicle whose :class:`VehicleObservations` handle is ``(slot[i], priority[i])``;
    entries with ``slot < 0`` are skipped, so the padded columns of a table can be passed as they are.  A handle
    that no longer names a running vehicle, or a slot given twice, raises ``RuntimeError`` at the engine's next
    synchronising call (``get_vehicle_count()``, the getters).  Single-GPU engines only.
    """
    import torch
    n = slot.numel()
    for t, dt in ((slot, torch.int32), (priority, torch.int32), (speed, torch.float64)):
        if not (t.is_cuda and t.dtype == dt and t.is_contiguous() and t.device.index == engine.device() and t.numel() == n):
            raise ValueError("slot / priority must be contiguous int32 and speed contiguous float64 CUDA tensors of one "
                             "length on the engine's device")
    if stream is None:
        stream = torch.cuda.current_stream(engine.device()).cuda_stream
    engine.set_vehicle_speeds_device(slot.data_ptr(), priority.data_ptr(), speed.data_ptr(), n, int(stream))


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
