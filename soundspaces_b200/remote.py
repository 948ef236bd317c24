"""Remote deferred mode: the audio observation of multiprocess vector-env workers, rendered once per step in the trainer.

habitat's default topology (``USE_VECENV=True``, ``USE_SYNC_VECENV=False``) runs one worker process per env and pickles
every observation back through a pipe.  With ``patch_simulator(cls, ..., deferred="remote")`` a worker never touches
CUDA: ``get_current_spectrogram_observation`` / ``get_current_audiogoal_observation`` return a
:class:`RemoteAudioRequest`, a small picklable description of the request (RIR keys, clip identity, sample offset, silent
flag, inline RIRs), and ``sensors.batch_obs`` in the trainer resolves the whole step's descriptors with ONE render
through the trainer's ``AudioRenderService`` (``batching.RemoteObservations``).

With ``remote_frames=True`` the discrete simulator's RGB and depth observations cross the pipe as :class:`FrameArray`
too: a frame's data once per worker, its key afterwards, gathered on the device by ``batch_obs``.

This module is imported by the workers: it uses numpy only.
"""
from __future__ import annotations

import hashlib
import uuid
from dataclasses import dataclass, replace
from typing import Dict, Optional

import numpy as np

SPECTROGRAM, WAVEFORM = "spectrogram", "waveform"


class ClipRef:
    """A source clip as it crosses the pipe: ``(name, length, digest)`` always, the float32 samples only the first time
    this process pickles the clip.  Deciding at pickling time, not when the descriptor is built, matters: a vector env
    with ``auto_reset_done`` builds the terminal step's observation and drops it unsent.  Unpickling one that carries
    samples registers them in this process, so the trainer keys clips by identity and workers playing the same sound
    share one device copy and one window-spectra set."""

    __slots__ = ("name", "length", "digest", "samples")

    def __init__(self, name, length: int, digest: str, samples: Optional[np.ndarray] = None):
        self.name, self.length, self.digest, self.samples = name, int(length), digest, samples

    @property
    def key(self) -> tuple:
        return (self.name, self.length, self.digest)

    def __getstate__(self):
        ship = self.samples is not None and self.key not in _SHIPPED
        if ship:
            _SHIPPED.add(self.key)
        return (self.name, self.length, self.digest, self.samples if ship else None)

    def __setstate__(self, state):
        self.name, self.length, self.digest, self.samples = state
        if self.samples is not None:
            _CLIPS.setdefault(self.key, self.samples)


_CLIPS: Dict[tuple, np.ndarray] = {}        # receiving side: identity -> the one array every worker's clip resolves to
_SHIPPED: set = set()                       # sending side: identities whose samples this process has pickled
_IDENTITY: Dict[int, tuple] = {}            # sending side: id(clip array) -> (array, identity, float32 samples)


def clip_ref(name, samples) -> ClipRef:
    hit = _IDENTITY.get(id(samples))
    if hit is None:                                  # the array is kept alive in the entry, so its id stays unique
        a = np.ascontiguousarray(np.asarray(samples, dtype=np.float32).reshape(-1))
        key = (name, int(a.shape[0]), hashlib.blake2b(a.tobytes(), digest_size=16).hexdigest())
        hit = _IDENTITY[id(samples)] = (samples, key, a)
    _, key, a = hit
    return ClipRef(*key, samples=a)


def clip_samples(clip) -> tuple:
    """``(name, samples)`` of a clip as ``AudioRenderService.source`` takes it; ``clip`` is that pair already (in-process)
    or a :class:`ClipRef` (trainer side of remote mode)."""
    if not isinstance(clip, ClipRef):
        return clip
    if clip.samples is not None:
        return clip.name, _CLIPS.setdefault(clip.key, clip.samples)
    a = _CLIPS.get(clip.key)
    if a is None:
        raise RuntimeError(f"clip {clip.name!r} ({clip.length} samples) has not reached this process: its samples travel "
                           "with the first pickled observation that uses it, which this process never received")
    return clip.name, a


class FrameArray(np.ndarray):
    """A visual observation a worker's discrete simulator took from its ``_frame_cache`` (remote deferred mode with
    ``remote_frames=True``): the same data as the sensor's array, plus ``frame_key`` = ``(scene observation file,
    receiver index, rotation angle, sensor uuid)``.  Being an ndarray, it serves every consumer in the worker as the
    plain array would (``EgoMap``'s ``asnumpy`` included).  Pickling sends a :class:`FrameRef`: key, dtype and shape
    always, the data only the first time this process pickles the key -- decided at pickling time, like
    :class:`ClipRef`, because a vector env with ``auto_reset_done`` builds the terminal step's observation and drops it
    unsent.  Views and results of operations carry no key: they pickle as plain arrays."""

    def __new__(cls, a: np.ndarray, key: tuple):
        obj = np.asarray(a).view(cls)
        obj.frame_key = key
        return obj

    def __array_finalize__(self, obj):
        self.frame_key = None

    def __reduce_ex__(self, protocol):
        a = np.asarray(self)
        if self.frame_key is None:
            return a.__reduce_ex__(protocol)
        ship = self.frame_key not in _FRAMES_SHIPPED
        if ship:
            _FRAMES_SHIPPED.add(self.frame_key)
        return (_received_frame, (self.frame_key, a.dtype.str, a.shape, np.ascontiguousarray(a) if ship else None))

    def __reduce__(self):
        return self.__reduce_ex__(2)


class FrameRef:
    """A :class:`FrameArray` as the trainer receives it: ``key``, ``dtype``, ``shape``, and ``data`` when this pickle
    carried the frame (it is then also in this process's frame dict).  ``sensors.batch_obs`` gathers a step's frames on
    the device (``soundspaces_b200.frames``); ``np.asarray(ref)`` gives the host frame."""

    __slots__ = ("key", "dtype", "shape", "data")

    def __init__(self, key: tuple, dtype, shape, data: Optional[np.ndarray] = None):
        self.key, self.dtype, self.shape, self.data = key, np.dtype(dtype), tuple(shape), data

    def __reduce__(self):
        return (_received_frame, (self.key, self.dtype.str, self.shape, self.data))

    def __array__(self, dtype=None, copy=None):
        a = frame_data(self)
        return a.astype(dtype) if dtype is not None and a.dtype != dtype else a


def _received_frame(key, dtype, shape, data):
    if data is not None:
        data = _FRAMES.setdefault(key, data)
    return FrameRef(key, dtype, shape, data)


_FRAMES: Dict[tuple, np.ndarray] = {}       # receiving side: key -> the frame, every frame this process has received
_FRAMES_SHIPPED: set = set()                # sending side: keys whose data this process has pickled


def frame_data(ref: FrameRef) -> np.ndarray:
    """The host frame of a :class:`FrameRef` (trainer side); ``RuntimeError`` naming the key when it never arrived."""
    if ref.data is not None:
        return ref.data
    a = _FRAMES.get(ref.key)
    if a is None:
        raise RuntimeError(f"frame {ref.key!r} has not reached this process: its data travels with the first pickled "
                           "observation that uses it, which this process never received")
    return a


@dataclass(slots=True)
class RemoteAudioRequest:
    """One env's audio request, as built by a simulator's ``_b200_keys`` without touching a bank, and -- in remote mode
    -- as it crosses the pipe.  ``rir_key`` is ``(binaural_rir_dir, azimuth, receiver, source_index)`` as
    ``AudioRenderService.rir`` takes it; ``rir_array`` / ``prev_rir`` are inline ``(L, 2)`` RIRs (the discrete
    simulator without rendered observations, the continuous simulator and its cross-fade); ``prefetch`` the read-ahead
    keys.  A memo hit is a reference: ``hit`` with ``(env, generation, memo_id)`` of the original.  It carries no sample
    data once the clip has crossed the pipe, but it keeps the original's request keys (RIR key, offset, silent flag,
    inline RIR) without the read-ahead keys, so the trainer can still render it when the original never reached it.
    That happens when a vector env with ``auto_reset_done`` drops a terminal step's observation.

    ``np.asarray(descriptor)`` in the trainer renders it (flushing the step) and copies its row to the host."""

    kind: str = SPECTROGRAM                 # or WAVEFORM: the (2, sr) waveform of AudioGoalSensor
    service: tuple = ()                     # (sr, device, pad_mode) of the trainer's AudioRenderService
    env: str = ""                           # env token (one per simulator object and memo dict kind)
    generation: int = 0                     # bumped whenever the reference replaces the memo dict
    memo_id: int = -1                       # -1: not memoised
    hit: bool = False
    silent: bool = False
    rir_key: Optional[tuple] = None
    rir_array: Optional[np.ndarray] = None
    clip: object = None                     # (name, samples) in process, ClipRef across the pipe
    offset: int = 0
    out_samples: Optional[int] = None
    wrap: bool = False
    distractor_key: Optional[tuple] = None
    distractor_clip: object = None
    prev_rir: Optional[np.ndarray] = None
    prev_wrap: bool = False
    prefetch: tuple = ()

    def __reduce__(self):                   # positional fields: no field names on the pipe
        return (RemoteAudioRequest, tuple(getattr(self, f) for f in self.__slots__))

    def reference(self) -> "RemoteAudioRequest":
        return replace(self, hit=True, prefetch=())

    def __array__(self, dtype=None, copy=None):
        from .batching import RemoteObservations
        a = RemoteObservations.of(self).numpy(self)
        return a.astype(dtype) if dtype is not None and a.dtype != dtype else a


class IntensityRequest:
    """AV-WaN's ``Intensity`` observation in remote deferred mode (``patch_simulator(..., deferred="remote",
    remote_intensity=True)``): the ``WAVEFORM`` :class:`RemoteAudioRequest` of ``get_current_audiogoal_observation``,
    whose intensity the trainer computes on the device.  It reaches ``Mapper.update`` as is (the reference's
    ``to_array`` only converts tensors) and travels in the map records; ``batch_obs`` resolves the ``intensity`` sensor.

    The process that built it has no value to give: ``float(d)`` / ``np.asarray(d)`` there raise ``RuntimeError``
    instead of rendering (a worker on a GPU machine would otherwise open a CUDA context of its own).  In the trainer,
    which receives it pickled, they resolve it.  ``value`` is the trainer's ``(1,)`` CUDA float32 result once resolved:
    one step resolves a waveform once, whether a map record or the sensor asks first."""

    __slots__ = ("request", "received", "value")

    def __init__(self, request: RemoteAudioRequest, received: bool = False):
        self.request, self.received, self.value = request, received, None

    def __reduce__(self):
        return (_received_intensity, (self.request,))

    def resolve(self):
        """The ``(1,)`` CUDA float32 intensity (trainer only)."""
        if not self.received:
            raise RuntimeError("this intensity is computed by the trainer from the waveform request it wraps; the env "
                               "worker that built it has no value (remote deferred mode with remote_intensity=True "
                               "sends it to batch_obs, and device maps take it from the map records)")
        if self.value is None:
            from .batching import RemoteObservations
            RemoteObservations.of(self.request).intensities([self])
        return self.value

    def __float__(self):
        return float(self.resolve()[0])

    def __array__(self, dtype=None, copy=None):
        a = self.resolve().cpu().numpy()[0]
        return np.asarray(a, dtype=dtype) if dtype is not None else np.asarray(a)


def _received_intensity(request):
    return IntensityRequest(request, received=True)


def _rir32(rir):
    # the conversion AudioRenderer._inline_rirs applies to inline RIRs, done before the pipe: same bits, half the bytes
    return None if rir is None else np.ascontiguousarray(np.asarray(rir, dtype=np.float32))


def package(k: RemoteAudioRequest, kind: str, service: tuple, memo=None) -> RemoteAudioRequest:
    """Make a request built by ``_b200_keys`` ready for the pipe (in place): clips become :class:`ClipRef`, inline RIRs
    float32.  ``memo``: ``(env, generation, memo_id)`` when the worker memoises the descriptor."""
    k.kind, k.service = kind, service
    if memo is not None:
        k.env, k.generation, k.memo_id = memo
    if k.clip is not None:
        k.clip = clip_ref(*k.clip)
    if k.distractor_clip is not None:
        k.distractor_clip = clip_ref(*k.distractor_clip)
    k.rir_array, k.prev_rir = _rir32(k.rir_array), _rir32(k.prev_rir)
    return k


def memo_slot(sim, kind: str, memo: dict) -> tuple:
    """``(env, generation, memo_id)`` for the next descriptor stored in ``memo``, one of the reference's memo dicts.
    The reference resets a memo by REPLACING the dict (simulator.py:395-397); a new dict object starts a new
    generation, so a reference can never resolve to another scene's observation."""
    st = getattr(sim, "_b200_remote_memo", None)
    if st is None:
        st = sim._b200_remote_memo = {"token": uuid.uuid4().hex}
    cur = st.get(kind)
    if cur is None or cur[0] is not memo:
        cur = st[kind] = [memo, cur[1] + 1 if cur else 0, 0]
    cur[2] += 1
    return f"{st['token']}/{kind}", cur[1], cur[2] - 1
