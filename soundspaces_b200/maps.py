"""AV-WaN's geometric, acoustic and action maps on the device, built from map-update records the env workers send.

In the reference (``ss_baselines/av_wan``) every env worker keeps a numpy ``Mapper`` and, after every step,
``Planner.add_maps_to_observation`` (planner.py:76-83) crops the ``(MAP_SIZE, MAP_SIZE, 2)`` geometric map, the
``(20, 20, 1)`` acoustic map and the ``(9, 9, 1)`` action map out of rotated float64 copies of its internal maps; the
trainer's ``batch_obs`` stacks them on the host and copies them to the GPU.  With :func:`patch_planner` the worker's
``Mapper`` keeps running (the planner's graph needs what ``Mapper.update`` returns), but the observation carries a
:class:`MapDescriptor` per map instead of an array: the env's token, its pose, the last sequence number and the
geometry, plus -- on the first descriptor pickled after them -- the records that changed the maps since the last
pickled observation: one per ``Mapper.reset``, one per completed ``Mapper.update`` with the post-update pose, the ego
map thresholded at 0.5 and bit-packed, ``float64(intensity)`` and ``0.5 * intensity`` as the reference evaluates it --
or, when the worker's ``Intensity`` sensor defers its value to the trainer (:class:`~soundspaces_b200.remote.
IntensityRequest`), the request in their place; the trainer then computes every such intensity of the step on the
device and applies the records with ``ssb_map_update_device_intensity_batch``.
``sensors.batch_obs`` in the trainer replays a step's records into per-env device maps (:class:`DeviceMaps`, one
``ssb_map_update_batch`` launch) and writes the three egocentric maps with one ``ssb_map_observe_batch`` launch.

Workers import only this module's numpy half: nothing here touches CUDA until :class:`DeviceMaps` is used.
"""
from __future__ import annotations

import uuid
import warnings
from typing import Dict, List, NamedTuple, Optional, Sequence

import numpy as np

from .remote import IntensityRequest

MAP_KINDS = ("gm", "am", "action_map")
ENCODINGS = {"intensity": 0, "average_intensity": 1}
RESET, UPDATE = 0, 1
MAX_SLOTS, MAX_INTERNAL, MAX_EGO = 65535, 4096, 255
AM_CROP = 20                # get_egocentric_acoustic_map()'s default crop, whatever ACOUSTIC_MAP.MAP_SIZE says


class MapGeometry(NamedTuple):
    """What the device maps of one env need to know (``ssb_map_geometry`` without the slot count)."""
    internal_size: int      # GEOMETRIC_MAP.INTERNAL_MAP_SIZE
    stride: int             # Mapper._stride = int(ACTION_MAP.MAP_RESOLUTION / GEOMETRIC_MAP.MAP_RESOLUTION)
    map_size: int           # GEOMETRIC_MAP.MAP_SIZE
    action_size: int        # ACTION_MAP.MAP_SIZE
    ego_size: int           # TASK.EGOMAP_SENSOR.MAP_SIZE
    encoding: int           # ENCODINGS[ACOUSTIC_MAP.ENCODING]
    acoustic: int           # use_acoustic_map

    @property
    def acoustic_size(self) -> int:
        return self.internal_size // self.stride

    def refusal(self) -> Optional[str]:
        """Why the device path cannot take this geometry, or None."""
        if self.map_size % 2:
            return f"odd MAP_SIZE {self.map_size}"
        if self.action_size % 2 == 0:
            return f"even ACTION_MAP.MAP_SIZE {self.action_size}"
        if not (1 <= self.internal_size <= MAX_INTERNAL and 2 <= self.map_size <= MAX_INTERNAL
                and 1 <= self.stride <= self.internal_size and 1 <= self.action_size <= MAX_EGO
                and 1 <= self.ego_size <= min(MAX_EGO, self.internal_size)):
            return (f"shape past the limits (internal {self.internal_size} <= {MAX_INTERNAL}, MAP_SIZE {self.map_size} "
                    f"<= {MAX_INTERNAL}, stride {self.stride}, action map {self.action_size} <= {MAX_EGO}, ego map "
                    f"{self.ego_size} <= {MAX_EGO})")
        return None


def navigable_tables(g: MapGeometry) -> np.ndarray:
    """``Mapper.compute_navigable_xys`` restated for the pose every Mapper starts from: int32 ``[4][2][L]``, for each
    quarter turn k the sorted rotated xs (``_rotated_xs[90 k]``), then ys."""
    n, s = g.internal_size, g.stride
    x0 = int(n / 2)
    xs = [x0 + i * s for i in range(int(-x0 / s), int((n - x0) / s))]
    out = np.empty((4, 2, len(xs)), dtype=np.int32)
    for k in range(4):
        pairs = [_rot_xy(k, n, a, b) for a, b in zip(xs, xs)]
        out[k, 0] = sorted(c for c, _ in pairs)
        out[k, 1] = sorted(d for _, d in pairs)
    return out


def _rot_xy(k: int, n: int, x: int, y: int):
    """mapper.transform_coordinates(x, y, 90 k, n, n)."""
    return ((x, y), (y, n - 1 - x), (n - 1 - x, n - 1 - y), (n - 1 - y, x))[k]


class MapLog:
    """One env's map-update records with consecutive sequence numbers.  Records are tuples
    ``(seq, kind, x, y, orientation, intensity, half, ego_bits)``; ``ego_bits`` is ``np.packbits(ego_map > 0.5)``
    as bytes; ``intensity`` may be an :class:`IntensityRequest` (``half`` is None then).  ``pending`` holds the
    records not yet pickled (remote) or not yet applied (in process)."""

    def __init__(self, geometry: MapGeometry):
        self.token = uuid.uuid4().hex
        self.geometry = geometry
        self.seq = -1
        self.pending: List[tuple] = []

    def reset(self):
        self.seq += 1
        self.pending.append((self.seq, RESET, 0, 0, 0, 0.0, 0.0, b""))

    def update(self, mapper, ego_map, intensity):
        e = np.asarray(ego_map)
        E = self.geometry.ego_size
        if e.shape != (E, E, 2):
            raise ValueError(f"the device maps of this planner take ({E}, {E}, 2) ego maps "
                             f"(TASK.EGOMAP_SENSOR.MAP_SIZE); got {e.shape}")
        if self.geometry.acoustic and isinstance(intensity, IntensityRequest):
            value, half = intensity, None                                                    # computed by the trainer
        elif self.geometry.acoustic:
            value, half = float(np.float64(intensity)), float(np.float64(0.5 * intensity))   # mapper.py:127-134
        else:
            value = half = 0.0
        self.seq += 1
        self.pending.append((self.seq, UPDATE, int(mapper._x), int(mapper._y), int(mapper._orientation), value, half,
                             np.packbits(e > 0.5).tobytes()))

    def drain(self) -> List[tuple]:
        out, self.pending = self.pending, []
        return out

    def trim(self, seq: int):
        """Drop the records up to ``seq`` (in process: the trainer has applied them)."""
        self.pending = [r for r in self.pending if r[0] > seq]


# receiving side: token -> records that arrived through pickled descriptors and are not applied yet
_RECEIVED: Dict[str, List[tuple]] = {}


class MapDescriptor:
    """One env's ``gm`` / ``am`` / ``action_map`` observation as the patched planner returns it.  In process it refers
    to the env's :class:`MapLog`; pickled, it carries the log's pending records (drained at pickling time, so records
    of an observation a vector env built and dropped still travel with the next one), and unpickling files them in
    this process.  ``np.asarray(descriptor)`` resolves this one env on the default CUDA device."""

    __slots__ = ("kind", "token", "pose", "seq", "geometry", "log")

    def __init__(self, kind: str, token: str, pose: tuple, seq: int, geometry: MapGeometry, log: Optional[MapLog]):
        self.kind, self.token, self.pose, self.seq, self.geometry, self.log = kind, token, pose, seq, geometry, log

    def __reduce__(self):
        records = self.log.drain() if self.log is not None else []
        return (_unpickle_descriptor, (self.kind, self.token, self.pose, self.seq, tuple(self.geometry), records))

    def pending(self) -> List[tuple]:
        return self.log.pending if self.log is not None else _RECEIVED.get(self.token, [])

    def trim(self, seq: int):
        if self.log is not None:
            self.log.trim(seq)
        elif self.token in _RECEIVED:
            _RECEIVED[self.token] = [r for r in _RECEIVED[self.token] if r[0] > seq]

    def __array__(self, dtype=None, copy=None):
        a = DeviceMaps.get(geometry=self.geometry).resolve({self.kind: [self]})[self.kind][0].cpu().numpy()
        return a.astype(dtype) if dtype is not None and a.dtype != dtype else a


def contiguous_records(d: MapDescriptor, applied: int) -> List[tuple]:
    """The records after ``applied`` up to ``d.seq``; a gap in their sequence numbers is a ``RuntimeError`` naming
    the env, never a silent skip."""
    recs = [r for r in d.pending() if applied < r[0] <= d.seq]
    if [r[0] for r in recs] != list(range(applied + 1, d.seq + 1)):
        have = {r[0] for r in recs}
        missing = next(q for q in range(applied + 1, d.seq + 1) if q not in have)
        raise RuntimeError(f"map records of env {d.token} are not contiguous: applied up to {applied}, the observation "
                           f"needs {d.seq}, record {missing} never reached this process")
    return recs


def _unpickle_descriptor(kind, token, pose, seq, geometry, records):
    if records:
        have = _RECEIVED.setdefault(token, [])
        last = have[-1][0] if have else -1
        have.extend(r for r in records if r[0] > last)
    return MapDescriptor(kind, token, tuple(pose), seq, MapGeometry(*geometry), None)


def planner_geometry(planner, task_config):
    """``(MapGeometry, None)`` for a constructed reference ``Planner``, or ``(None, reason)``."""
    m = planner.mapper
    ratio = m._action_map_res / m._gm_res
    if ratio != int(ratio):
        return None, f"non-integer stride ACTION_MAP.MAP_RESOLUTION / GEOMETRIC_MAP.MAP_RESOLUTION = {ratio!r}"
    acoustic = bool(m._use_acoustic_map)
    if acoustic and m._am_encoding not in ENCODINGS:
        return None, f"unknown acoustic map encoding {m._am_encoding!r}"
    try:
        ego = task_config.TASK.EGOMAP_SENSOR.MAP_SIZE
    except AttributeError:
        return None, "no ego map size in TASK.EGOMAP_SENSOR.MAP_SIZE"
    if isinstance(ego, (tuple, list)):
        if len(ego) != 2 or ego[0] != ego[1]:
            return None, f"non-square ego map {tuple(ego)}"
        ego = ego[0]
    g = MapGeometry(int(m._internal_gm_size), int(m._stride), int(m._gm_size), int(planner._action_map_size),
                    int(ego), ENCODINGS.get(m._am_encoding, 0) if acoustic else 0, int(acoustic))
    why = g.refusal()
    return (None, why) if why else (g, None)


def patch_planner(Planner) -> bool:
    """Patch AV-WaN's ``Planner`` class in place: its mapper logs map-update records, and ``add_maps_to_observation``
    puts :class:`MapDescriptor` s in ``gm`` / ``am`` / ``action_map``.  A planner whose geometry the device path does
    not take (odd MAP_SIZE, non-square ego map, non-integer stride, unknown encoding, shapes past the limits) stays
    unpatched with a warning that says why, as does a class without the reference's methods (returns False then).

    An :class:`IntensityRequest` reaching ``Mapper.update`` (``patch_simulator(..., remote_intensity=True)``) is logged
    in the record and the reference's update runs with a placeholder intensity of 0.0: the worker's host acoustic map
    then holds placeholders, and only the trainer's device map is right.  A planner that kept its host maps cannot take
    one when it uses an acoustic map: ``Mapper.update`` raises ``RuntimeError`` naming why the maps were refused."""
    if getattr(Planner, "_b200_maps", False):
        return True
    missing = [n for n in ("add_maps_to_observation", "update_map_and_graph", "reset") if not hasattr(Planner, n)]
    if missing:
        warnings.warn(f"patch_planner: {Planner.__name__} has no {', '.join(missing)}; left unpatched")
        return False
    orig_init, orig_add = Planner.__init__, Planner.add_maps_to_observation

    def __init__(self, *args, **kwargs):
        orig_init(self, *args, **kwargs)
        task_config = kwargs["task_config"] if "task_config" in kwargs else (args[0] if args else None)
        geometry, why = planner_geometry(self, task_config)
        if geometry is None:
            warnings.warn(f"patch_planner: {why}; this planner keeps the reference's host maps")
            _refuse_deferred(self.mapper, why)
            return
        _attach(self.mapper, geometry)

    def add_maps_to_observation(self, observation):
        log = getattr(self.mapper, "_b200_map_log", None)
        if log is None or ("am" in observation and not log.geometry.acoustic):
            return orig_add(self, observation)
        m = self.mapper
        pose = (int(m._x), int(m._y), int(m._orientation))
        for kind in MAP_KINDS:
            if kind in observation:
                observation[kind] = MapDescriptor(kind, log.token, pose, log.seq, log.geometry, log)

    Planner.__init__ = __init__
    Planner.add_maps_to_observation = add_maps_to_observation
    Planner._b200_maps = True
    return True


def _attach(mapper, geometry: MapGeometry):
    """Log the mapper's resets and completed updates.  The log starts with one reset record: the mapper is freshly
    reset by ``Mapper.__init__`` and ``Planner.__init__``."""
    log = MapLog(geometry)
    log.reset()
    reset, update = mapper.reset, mapper.update

    def logged_reset():
        reset()
        log.reset()

    def logged_update(prev_action, ego_map, intensity):
        out = update(prev_action, ego_map, 0.0 if isinstance(intensity, IntensityRequest) else intensity)
        log.update(mapper, ego_map, intensity)
        return out

    object.__setattr__(mapper, "reset", logged_reset)
    object.__setattr__(mapper, "update", logged_update)
    object.__setattr__(mapper, "_b200_map_log", log)


def _refuse_deferred(mapper, why: str):
    """A planner that keeps the reference's host maps: a deferred intensity has no value in this process, so its
    acoustic map cannot take one; without an acoustic map the reference ignores the intensity."""
    update = mapper.update

    def checked_update(prev_action, ego_map, intensity):
        if isinstance(intensity, IntensityRequest):
            if mapper._use_acoustic_map:
                raise RuntimeError(f"this planner keeps the reference's host maps ({why}); its acoustic map needs the "
                                   "intensity inside the env worker, which remote_intensity=True leaves to the trainer")
            intensity = 0.0
        return update(prev_action, ego_map, intensity)

    object.__setattr__(mapper, "update", checked_update)


# numpy mirror of ssb_map_record (include/ssb200.h)
RECORD_DTYPE = np.dtype([("slot", "<i4"), ("kind", "<i4"), ("x", "<i4"), ("y", "<i4"), ("orientation", "<i4"),
                         ("reserved", "<i4"), ("intensity", "<f8"), ("half", "<f8"), ("ego_offset", "<i8")])
assert RECORD_DTYPE.itemsize == 48


class DeviceMaps:
    """Per-env geometric (uint8, two bits per cell) and acoustic (float64) maps on one device, in slots of one
    geometry (:meth:`get` keeps one per device and geometry).  Tokens get slots on first sight; :meth:`forget` frees a
    slot for reuse."""

    _instances: dict = {}

    def __init__(self, device="cuda:0"):
        import torch
        from .renderer import WaveformOps
        self.ops = WaveformOps.get(device)
        self.device = self.ops.device
        self.geometry: Optional[MapGeometry] = None
        self.slots: Dict[str, int] = {}
        self.applied: Dict[str, int] = {}
        self.free: List[int] = []
        self.capacity = 0
        self._torch = torch

    @classmethod
    def get(cls, device=None, geometry: Optional[MapGeometry] = None) -> "DeviceMaps":
        """The process's maps for ``geometry`` on ``device`` (a CUDA device; None or a CPU device: the current one)."""
        import torch
        dev = torch.device(device) if device is not None else None
        index = dev.index if dev is not None and dev.type == "cuda" and dev.index is not None \
            else torch.cuda.current_device()
        key = (index, geometry)
        if key not in cls._instances:
            cls._instances[key] = cls(torch.device("cuda", index))
        return cls._instances[key]

    def forget(self, token: str):
        """Free ``token``'s slot (its env is gone); records still pending for it are dropped."""
        slot = self.slots.pop(token, None)
        self.applied.pop(token, None)
        _RECEIVED.pop(token, None)
        if slot is not None:
            self.free.append(slot)

    def _c_geometry(self):
        from ._lib import MapGeometry as CGeometry
        return CGeometry(*self.geometry, self.capacity)

    def _slot(self, token: str, geometry: MapGeometry) -> int:
        if self.geometry is None:
            why = geometry.refusal()
            if why:
                raise ValueError(f"DeviceMaps: {why}")
            self.geometry = geometry
            self.tables = navigable_tables(geometry)
        elif geometry != self.geometry:
            raise ValueError(f"DeviceMaps holds maps of geometry {self.geometry}; env {token} has {geometry}")
        slot = self.slots.get(token)
        if slot is None:
            if self.free:
                slot = self.free.pop()
            else:
                slot = len(self.slots)
                if slot >= MAX_SLOTS:
                    raise ValueError(f"DeviceMaps: more than {MAX_SLOTS} envs")
                self._grow(slot + 1)
            self.slots[token] = slot
            self.applied[token] = -1
        return slot

    def _grow(self, need: int):
        if need <= self.capacity:
            return
        torch, g = self._torch, self.geometry
        cap = min(max(need, 2 * self.capacity, 16), MAX_SLOTS)
        pitch = (g.internal_size * g.internal_size + 15) & ~15
        m = g.acoustic_size
        gmap = torch.zeros((cap, pitch), dtype=torch.uint8, device=self.device)
        amap = torch.zeros((cap, m, m), dtype=torch.float64, device=self.device)
        if self.capacity:
            gmap[:self.capacity].copy_(self.gmap)
            amap[:self.capacity].copy_(self.amap)
        self.gmap, self.amap, self.capacity = gmap, amap, cap

    def update(self, descs: Sequence[MapDescriptor], intensities: Sequence[IntensityRequest] = ()):
        """Apply every env's records up to its descriptor's sequence number in ONE ``ssb_map_update_batch`` launch.
        A missing record (a sequence gap) is an error naming the env; nothing is launched then.  Records whose
        intensity is an :class:`IntensityRequest` are resolved first (``RemoteObservations.intensities``: the step's
        waveforms rendered and reduced on the device) and applied by ONE ``ssb_map_update_device_intensity_batch``
        launch; no intensity is read on the host.  ``intensities``: the step's other requests (the ``intensity``
        sensor's), resolved in the same render.  One step's requests must name one service, and cannot be mixed with
        host intensities (``ValueError``)."""
        if len({d.token for d in descs}) != len(descs):
            raise ValueError("one step's map descriptors must name each env once")
        todo = []
        for d in descs:
            slot = self._slot(d.token, d.geometry)
            todo.append((d, slot, contiguous_records(d, self.applied[d.token])))
        n = sum(len(r) for _, _, r in todo)
        rec = np.zeros(n, dtype=RECORD_DTYPE)
        ego = bytearray()
        deferred, host_values = [], 0
        i = 0
        for d, slot, recs in todo:
            for seq, kind, x, y, o, value, half, bits in recs:
                if isinstance(value, IntensityRequest):
                    rec[i] = (slot, kind, x, y, o, len(deferred), 0.0, 0.0, len(ego))
                    deferred.append(value)
                else:
                    rec[i] = (slot, kind, x, y, o, 0, value, half, len(ego))
                    host_values += kind == UPDATE
                ego += bits
                i += 1
        ego = np.frombuffer(bytes(ego), dtype=np.uint8)
        if deferred and host_values and self.geometry.acoustic:
            raise ValueError("one step's map records mix intensities computed by env workers with intensities "
                             "deferred to the trainer")
        ids = {id(q) for q in deferred}                # the sensor holds the last record's request itself
        requests = deferred + [q for q in intensities if q.value is None and id(q) not in ids]
        if requests:
            if any(q.request.service != requests[0].request.service for q in requests):
                raise ValueError("one step's deferred intensities must name one service")
            from .batching import RemoteObservations
            values = RemoteObservations.of(requests[0].request).intensities(requests)
        if deferred:
            if values.device != self.device:
                raise ValueError(f"the deferred intensities are computed on {values.device}; these maps live on "
                                 f"{self.device}")
            self.ops.map_update_device_intensity(self._c_geometry(), self.gmap, self.amap, rec, ego, values)
        else:
            self.ops.map_update(self._c_geometry(), self.gmap, self.amap, rec, ego)
        for d, _, _ in todo:
            self.applied[d.token] = d.seq
            d.trim(d.seq)

    def observe(self, descs: Sequence[MapDescriptor], kinds: Sequence[str], out: Optional[dict] = None) -> dict:
        """``{kind: (B, ...) float32 CUDA tensor}`` for the envs' current poses in ONE ``ssb_map_observe_batch``
        launch; ``out[kind]``, when given, is a ``(B, ...)`` float32 tensor on this device with contiguous rows
        (e.g. a rollout-storage slot) and receives the maps."""
        torch, g = self._torch, self.geometry
        B = len(descs)
        shapes = {"gm": (g.map_size, g.map_size, 2), "am": (AM_CROP, AM_CROP, 1),
                  "action_map": (g.action_size, g.action_size, 1)}
        res = {}
        for kind in kinds:
            t = (out or {}).get(kind)
            shape = (B,) + shapes[kind]
            if t is None:
                t = torch.empty(shape, dtype=torch.float32, device=self.device)
            elif not (t.device == self.device and t.dtype == torch.float32 and tuple(t.shape) == shape
                      and (B == 0 or t[0].is_contiguous())):
                raise ValueError(f"out[{kind!r}] must be a float32 {shape} tensor on {self.device} with contiguous rows")
            res[kind] = t
        poses = np.array([(self.slots[d.token],) + tuple(d.pose) for d in descs], dtype=np.int32).reshape(B, 4)
        self.ops.map_observe(self._c_geometry(), self.gmap, self.amap, poses, self.tables, res.get("gm"), res.get("am"),
                             res.get("action_map"))
        return res

    def resolve(self, by_kind: Dict[str, List[MapDescriptor]], out: Optional[dict] = None,
                intensities: Sequence[IntensityRequest] = ()) -> dict:
        """One step of the map sensors: ``by_kind`` maps ``gm`` / ``am`` / ``action_map`` to the envs' descriptors
        (the same envs, in the same order, for every kind).  Two launches whatever B: the update, then the crops.
        ``intensities``: as for :meth:`update`."""
        kinds = list(by_kind)
        descs = by_kind[kinds[0]]
        for k in kinds[1:]:
            if [d.token for d in by_kind[k]] != [d.token for d in descs]:
                raise ValueError("the map sensors of one step must list the same envs in the same order")
        bad = [d.kind for k in kinds for d in by_kind[k] if d.kind != k]
        if bad:
            raise ValueError(f"a {bad[0]!r} map descriptor sits under another sensor")
        self.update(descs, intensities)
        return self.observe(descs, kinds, out)
