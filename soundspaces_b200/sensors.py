"""Habitat sensor plugins for the audio observation + the batch boundary.

Mirrors ``soundspaces/tasks/nav.py:37-105`` (``AudioGoalSensor``, ``SpectrogramSensor``: same
class names, uuids ``"audiogoal"`` / ``"spectrogram"``, ``SensorTypes.PATH``, ``spaces.Box`` of
float32 whose shape is obtained by running ``compute_spectrogram`` on ``np.ones((2, sr))``) and
``ss_baselines/common/utils.py:117-153`` (``to_tensor`` / ``batch_obs``).

With a simulator in deferred mode (``patch_simulator(..., deferred=True)``) ``SpectrogramSensor.get_observation``
returns a :class:`~soundspaces_b200.batching.DeferredObservation` handle instead of a host array and
:func:`batch_obs` turns the step's handles into the ``(N, 65, T', 2)`` CUDA batch with ONE render
(SURVEY.md 8(b) "Return/ownership").  With the simulators in remote deferred mode (envs in worker processes), both
``SpectrogramSensor`` and ``AudioGoalSensor`` return :class:`~soundspaces_b200.remote.RemoteAudioRequest` descriptors,
and :func:`batch_obs` in the trainer renders a step's descriptors with ONE flush (or ONE ``convolve`` for waveforms).

When habitat-lab is importable the classes subclass ``habitat.core.simulator.Sensor`` and are
registered with ``@registry.register_sensor``; otherwise a minimal stand-in base with the same
protocol is used (habitat is not installable in the build image).
"""
from __future__ import annotations

import contextlib
from typing import Any, Dict, List, Optional

import numpy as np
import torch

from .batching import DeferredObservation, RemoteObservations
from .frames import gather as gather_frames
from .maps import DeviceMaps, MapDescriptor
from .remote import WAVEFORM, FrameRef, IntensityRequest, RemoteAudioRequest
from .renderer import BatchedAudioRenderer, WaveformOps, spectrogram_shape
from .simulator import INTENSITY_REMOTE_ERROR, REMOTE, SPECTROGRAM_NATIVE_ATTR

try:  # pragma: no cover - habitat is absent in the build image
    from habitat.core.registry import registry
    from habitat.core.simulator import Sensor, SensorTypes
    from gym import spaces
    HAVE_HABITAT = True
except Exception:  # noqa: BLE001
    HAVE_HABITAT = False

    class _Registry:
        def __init__(self):
            self.sensors = {}

        def register_sensor(self, cls=None, *, name=None):
            def wrap(c):
                self.sensors[name or c.__name__] = c
                return c
            return wrap(cls) if cls is not None else wrap

        def get_sensor(self, name):
            return self.sensors.get(name)

    registry = _Registry()

    class SensorTypes:
        PATH = "PATH"

    class _Box:
        def __init__(self, low, high, shape, dtype):
            self.low, self.high, self.shape, self.dtype = low, high, tuple(shape), dtype

    class spaces:  # noqa: N801
        Box = _Box

    class Sensor:
        """Protocol of habitat.core.simulator.Sensor (v0.2.2)."""

        def __init__(self, *args: Any, **kwargs: Any) -> None:
            self.config = kwargs["config"] if "config" in kwargs else None
            self.uuid = self._get_uuid(*args, **kwargs)
            self.sensor_type = self._get_sensor_type(*args, **kwargs)
            self.observation_space = self._get_observation_space(*args, **kwargs)


def _device_spectrogram(audio_data, pad_mode="reflect", device="cuda:0"):
    """compute_spectrogram on the GPU for a host (2, n) array; result on the host."""
    a = np.asarray(audio_data)
    if a.ndim != 2 or a.shape[0] != 2:
        raise ValueError(f"audio_data must be (2, n), got {a.shape}")
    ops = WaveformOps.get(device)
    wave = torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).to(ops.device)
    out = ops.spectrogram(wave[None], pad_mode=pad_mode)[0].cpu().numpy()
    return out.astype(a.dtype) if a.dtype == np.float64 else out


@registry.register_sensor
class AudioGoalSensor(Sensor):
    def __init__(self, *args: Any, sim, config, **kwargs: Any):
        self._sim = sim
        super().__init__(config=config)

    def _get_uuid(self, *args: Any, **kwargs: Any):
        return "audiogoal"

    def _get_sensor_type(self, *args: Any, **kwargs: Any):
        return SensorTypes.PATH

    def _get_observation_space(self, *args: Any, **kwargs: Any):
        sensor_shape = (2, self._sim.config.AUDIO.RIR_SAMPLING_RATE)
        return spaces.Box(low=np.finfo(np.float32).min, high=np.finfo(np.float32).max,
                          shape=sensor_shape, dtype=np.float32)

    def get_observation(self, *args: Any, observations=None, episode=None, **kwargs: Any):
        return self._sim.get_current_audiogoal_observation()


@registry.register_sensor
class SpectrogramSensor(Sensor):
    cls_uuid: str = "spectrogram"
    pad_mode: str = "reflect"
    device: str = "cuda:0"

    def __init__(self, *args: Any, sim, config, **kwargs: Any):
        self._sim = sim
        super().__init__(config=config)

    def _get_uuid(self, *args: Any, **kwargs: Any):
        return "spectrogram"

    def _get_sensor_type(self, *args: Any, **kwargs: Any):
        return SensorTypes.PATH

    def _get_observation_space(self, *args: Any, **kwargs: Any):
        # nav.py:77 runs compute_spectrogram on ones((2, sr)) only for its shape
        shape = spectrogram_shape(self._sim.config.AUDIO.RIR_SAMPLING_RATE)
        return spaces.Box(low=np.finfo(np.float32).min, high=np.finfo(np.float32).max,
                          shape=shape, dtype=np.float32)

    @staticmethod
    def compute_spectrogram(audio_data):
        """nav.py:86-100 on the GPU: host (2, n) in, host (65, T', 2) out.  Imported by
        savi/ppo/ppo_trainer.py:52 and belief_predictor.py:15, so it keeps working on host arrays."""
        return _device_spectrogram(audio_data, SpectrogramSensor.pad_mode, SpectrogramSensor.device)

    def get_observation(self, *args: Any, observations=None, episode=None, **kwargs: Any):
        # host ndarray (compat) or, with the simulator in deferred mode, a DeferredObservation handle
        return self._sim.get_current_spectrogram_observation(self.compute_spectrogram)


setattr(SpectrogramSensor.compute_spectrogram, SPECTROGRAM_NATIVE_ATTR, True)


@registry.register_sensor(name="Intensity")
class Intensity(Sensor):
    """AV-WaN ``Intensity`` sensor (ss_baselines/av_wan/avwan_sensors.py:69-100): mean square of the 150
    samples after the onset of the current waveform, reduced on the device.  With the simulator mixin the
    waveform never visits the host: only the resulting scalar is read back.  In remote deferred mode with
    ``remote_intensity`` (see ``patch_simulator``) it returns ``[IntensityRequest]`` and the trainer computes the
    value."""

    def __init__(self, sim, config, *args: Any, **kwargs: Any):
        self._sim = sim
        super().__init__(config=config)

    def _get_uuid(self, *args: Any, **kwargs: Any):
        return "intensity"

    def _get_sensor_type(self, *args: Any, **kwargs: Any):
        return getattr(SensorTypes, "COLOR", "COLOR")

    def _get_observation_space(self, *args: Any, **kwargs: Any):
        return spaces.Box(low=0, high=1, shape=(1,), dtype=bool)

    def get_observation(self, *args: Any, observations=None, episode=None, **kwargs: Any):
        if getattr(self._sim, "b200_deferred", False) == REMOTE:                 # discrete and continuous alike
            if not getattr(self._sim, "b200_remote_intensity", False):
                raise RuntimeError(INTENSITY_REMOTE_ERROR)
            # the reference's getter (avwan_sensors.py:91): its memo and _audio_index advance; the trainer reduces
            return [IntensityRequest(self._sim.get_current_audiogoal_observation())]
        dev_getter = getattr(self._sim, "get_current_audiogoal_device", None)
        if dev_getter is not None:
            wave = dev_getter()                                    # CUDA (2, sr): no host round trip
            ops = WaveformOps.get(wave.device)
        else:                                                      # a simulator without the mixin: host array in
            ops = WaveformOps.get(getattr(self._sim, "b200_device", "cuda:0"))
            audiogoal = np.asarray(self._sim.get_current_audiogoal_observation())
            wave = torch.from_numpy(np.ascontiguousarray(audiogoal, dtype=np.float32))
        return [float(ops.intensity(wave[None])[0])]


def to_tensor(v):
    """ss_baselines/common/utils.py:117-123, plus: a deferred handle resolves to its device row."""
    if isinstance(v, DeferredObservation):
        return v.resolve()
    if isinstance(v, FrameRef):
        return torch.from_numpy(np.asarray(v))
    if torch.is_tensor(v):
        return v
    if isinstance(v, np.ndarray):
        return torch.from_numpy(v)
    return torch.tensor(v, dtype=torch.float)


def batch_obs(observations: List[Dict], device: Optional[torch.device] = None, skip_list=(),
              out: Optional[Dict[str, torch.Tensor]] = None) -> Dict[str, torch.Tensor]:
    """Replacement of ``ss_baselines/common/utils.py:126-153`` (same signature and result: a dict of
    ``(N, ...)`` float tensors on ``device``), with the batch boundary moved onto the GPU:

    * a sensor whose values are :class:`DeferredObservation` handles is resolved by its batcher -- ONE render for
      the whole step, and the ``(N, 65, T', 2)`` result is a view of the renderer's ring (no stack, no H2D copy);
    * ``out[sensor]`` (optional) names the tensor the batch must land in, e.g. the rollout-storage slot
      ``rollouts.observations["spectrogram"][step + 1]`` (rollout_storage.py:88-91): pending handles are rendered
      straight into it;
    * the step's AV-WaN map descriptors (``soundspaces_b200.maps``, sensors ``gm`` / ``am`` / ``action_map``) are
      resolved together when the first of them comes up: every env's unapplied records in ONE update launch, then the
      egocentric maps of all of them in ONE crop launch, into ``out[sensor]`` when given;
    * AV-WaN's ``intensity`` as remote workers with ``remote_intensity`` send it (one-element lists of
      :class:`~soundspaces_b200.remote.IntensityRequest`) becomes an ``(N, 1)`` CUDA float32 batch computed on the
      device; values the step's map records already computed are not computed again;
    * the RGB / depth frames remote workers send with ``remote_frames`` (a sensor whose values are all
      :class:`~soundspaces_b200.remote.FrameRef`) are gathered from the device frame banks, every visual sensor of the
      step in ONE launch, into float32 ``(N, H, W, C)`` CUDA tensors or ``out[sensor]``; a sensor whose values mix
      them with plain arrays, or a batch that is not on a CUDA device, takes the reference's path (same values);
    * values that already are tensors on ``device`` are stacked there; host values take the reference's path.
    """
    keys: Dict[str, list] = {}
    for obs in observations:
        for sensor in obs:
            if sensor in skip_list:
                continue
            keys.setdefault(sensor, []).append(obs[sensor])
    batch: Dict[str, torch.Tensor] = {}
    maps: Optional[Dict[str, torch.Tensor]] = None
    frames: Optional[Dict[str, torch.Tensor]] = None
    # the maps first: they resolve the step's intensity requests, their records' and the intensity sensor's, in one
    # render
    with _arriving(keys):
        for sensor in sorted(keys, key=lambda s: 0 if _is_maps(keys[s]) else 1 if _is_intensity(keys[s]) else 2):
            vals = keys[sensor]
            dst = out.get(sensor) if out else None
            if vals and all(isinstance(v, RemoteAudioRequest) for v in vals):
                t = _resolve_remote(vals, dst)
            elif _is_maps(vals):
                if maps is None:                                   # the step's map sensors: update + crops, 2 launches
                    by_kind = {s: v for s, v in keys.items() if _is_maps(v)}
                    intensity = [v[0] for vs in keys.values() if _is_intensity(vs) for v in vs]
                    maps = DeviceMaps.get(_map_device(device, out), vals[0].geometry).resolve(
                        by_kind, {s: out[s] for s in by_kind if out and out.get(s) is not None}, intensity)
                t = maps[sensor]
            elif _is_frames(vals) and _map_device(device, out) is not None:
                if frames is None:                                 # the step's visual sensors: one gather launch
                    frames = gather_frames({s: v for s, v in keys.items() if _is_frames(v)}, _map_device(device, out),
                                           out={s: out[s] for s in keys if out and out.get(s) is not None})
                t = frames[sensor]
            elif _is_intensity(vals):
                t = _resolve_intensity([v[0] for v in vals], dst)
            elif vals and all(isinstance(v, DeferredObservation) for v in vals):
                batcher = vals[0]._batcher
                if all(v._batcher is batcher for v in vals):
                    t = batcher.gather(vals, out=dst)
                else:                                              # several devices / sample rates in one suite
                    t = torch.stack([v.resolve() for v in vals], dim=0)
                    t = t if dst is None else dst.copy_(t)
            else:
                t = torch.stack([to_tensor(v).float() for v in vals], dim=0)
                t = t if dst is None else dst.copy_(t)
            batch[sensor] = t.to(device=device, dtype=torch.float)
    return {s: batch[s] for s in keys}


def _is_maps(vals) -> bool:
    return bool(vals) and all(isinstance(v, MapDescriptor) for v in vals)


def _is_frames(vals) -> bool:
    return bool(vals) and all(isinstance(v, FrameRef) for v in vals)


def _is_intensity(vals) -> bool:
    """AV-WaN's ``Intensity`` in remote mode with ``remote_intensity``: ``[IntensityRequest]`` per env."""
    return bool(vals) and all(isinstance(v, list) and len(v) == 1 and isinstance(v[0], IntensityRequest) for v in vals)


@contextlib.contextmanager
def _arriving(keys):
    """Tell the remote tables which memo originals this step carries in its waveform sensors, so that a reference
    resolved before its original (a map record of a pose the audiogoal sensor saw first) is not counted as unseen."""
    tables = {}
    for vals in keys.values():
        if vals and all(isinstance(v, RemoteAudioRequest) for v in vals):
            for d in vals:
                if not d.hit and d.memo_id >= 0:
                    tables.setdefault(d.service, (d, set()))[1].add((d.env, d.generation, d.memo_id))
    remotes = [(RemoteObservations.of(d), arriving) for d, arriving in tables.values()]
    for r, arriving in remotes:
        r.arriving = arriving
    try:
        yield
    finally:
        for r, _ in remotes:
            r.arriving = set()


def _resolve_intensity(descs: List[IntensityRequest], dst: Optional[torch.Tensor]) -> torch.Tensor:
    """The ``intensity`` sensor's deferred requests -> ``(N, 1)`` CUDA float32 batch, without a host read; the values
    this step's map records already computed are reused."""
    d0 = descs[0].request
    if any(q.request.service != d0.service for q in descs):
        raise ValueError("one sensor's remote descriptors must name one service and one kind")
    t = RemoteObservations.of(d0).intensities(descs).view(len(descs), 1)
    return t if dst is None else dst.copy_(t)


def _map_device(device, out) -> Optional[torch.device]:
    """The CUDA device the step's map sensors resolve on: that of the first ``out`` tensor, else ``device``."""
    for t in (out or {}).values():
        if t is not None and t.is_cuda:
            return t.device
    return torch.device(device) if device is not None and torch.device(device).type == "cuda" else None


def _resolve_remote(descs: List[RemoteAudioRequest], dst: Optional[torch.Tensor]) -> torch.Tensor:
    """One sensor's worker descriptors -> ``(N, ...)`` CUDA batch: ONE flush (spectrograms, into ``dst`` when given)
    or ONE convolve (waveforms) for the whole step in the trainer's service."""
    d0 = descs[0]
    if any(d.service != d0.service or d.kind != d0.kind for d in descs):
        raise ValueError("one sensor's remote descriptors must name one service and one kind")
    remote = RemoteObservations.of(d0)
    if d0.kind == WAVEFORM:
        t = remote.waveforms(descs)
        return t if dst is None else dst.copy_(t)
    return remote.service.batcher.gather([remote.spectrogram(d) for d in descs], out=dst)


class VectorAudioObservations:
    """Batch the audio observation of many in-process envs into ONE render call without going through the sensor
    objects: ``collect(sims)`` builds one request per cache-missing env through the same attribute reads as the
    reference's per-env getter and returns the ``(n_envs, 65, T', 2)`` CUDA tensor the policy consumes -- the
    place where the reference does N separate CPU renders, N pickles and one ``batch_obs`` H2D copy.

    The memo is each simulator's OWN ``_spectrogram_cache`` dict, keyed ``(source, receiver, azimuth)`` exactly as
    simulator.py:696-699.  The reference replaces that dict whenever the scene or the sound changes
    (simulator.py:395-397), so a cached row can never be served to another scene's identical node indices;
    multi-second clips keep the reference's quirk that a memo hit does not advance ``_audio_index``
    (simulator.py:683-686).  Cached values are handles whose rows are detached (private 36 KB copies) before
    their ring slot is reused, so the memo pins no batch tensors."""

    def __init__(self, sr: int, device="cuda:0", pad_mode="reflect"):
        from .simulator import AudioRenderService
        self.service = AudioRenderService.get(sr, device, pad_mode=pad_mode)
        self.renderer: BatchedAudioRenderer = self.service.renderer
        self.batcher = self.service.batcher

    def collect(self, sims, out: Optional[torch.Tensor] = None) -> torch.Tensor:
        handles = []
        for sim in sims:
            sim._b200_svc = self.service
            handles.append(sim._b200_deferred_spectrogram())
        return self.batcher.gather(handles, out=out)
