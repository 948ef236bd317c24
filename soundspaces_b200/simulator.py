"""Drop-in audio slice for the SoundSpaces simulators.

Mirrors, method for method, the audio part of the reference simulator wrappers:

* ``SoundSpacesSim._compute_audiogoal``                 soundspaces/simulator.py:608-666
* ``SoundSpacesSim.get_current_audiogoal_observation``  soundspaces/simulator.py:678-688
* ``SoundSpacesSim.get_current_spectrogram_observation`` soundspaces/simulator.py:690-701
* ``ContinuousSoundSpacesSim._compute_audiogoal`` / ``_convolve_with_rir`` / getters
                                                        soundspaces/continuous_simulator.py:413-462

``B200AudioMixin`` / ``B200ContinuousAudioMixin`` read exactly the attributes the
reference methods read (``config.AUDIO.*``, ``_receiver_position_index``,
``azimuth_angle``, ``_audio_index`` ... see SURVEY.md App. D) and keep the
reference's memoisation and ``_audio_index`` quirks, but run the arithmetic on
the GPU through :class:`AudioRenderService`.  Use either

    class SoundSpacesSim(B200AudioMixin, Simulator): ...        # in the reference
    patch_simulator(SoundSpacesSim)                             # or monkey-patch

Three return modes for ``get_current_spectrogram_observation``:

* compat (default): one render per call, host ``ndarray`` back -- exactly the reference's contract;
* deferred (``b200_deferred = True`` / ``patch_simulator(..., deferred=True)``): the call only ENQUEUES the
  request and returns a :class:`~soundspaces_b200.batching.DeferredObservation` handle; all envs of a step are
  rendered by ONE launch when ``sensors.batch_obs`` (or anything else) resolves a handle (SURVEY.md 7 "Batching
  across a per-env API", 8(b) "Return/ownership");
* remote deferred (``patch_simulator(..., deferred="remote")``, envs in worker processes): the call returns a
  picklable :class:`~soundspaces_b200.remote.RemoteAudioRequest` and never touches CUDA; the trainer's ``batch_obs``
  renders the step's descriptors with ONE launch chain (``get_current_audiogoal_observation`` likewise).

There is no CPU fallback: without a CUDA device / libssb200.so these raise.
"""
from __future__ import annotations

import logging
import os
from concurrent.futures import ThreadPoolExecutor
from typing import Callable, Dict, Optional

import numpy as np
import torch

from .remote import SPECTROGRAM, WAVEFORM, FrameArray, RemoteAudioRequest, clip_samples, memo_slot, package
from .renderer import AudioRequest, BatchedAudioRenderer

REMOTE = "remote"
INTENSITY_REMOTE_ERROR = (
    "remote deferred mode renders the audio in the trainer, but AV-WaN's Intensity needs the waveform's value inside "
    "the env worker (MapNavEnv.step feeds it to the planner); run AV-WaN with an acoustic map on in-process envs "
    "(USE_SYNC_VECENV with patch_simulator(..., deferred=True) or the default compat mode), or let the trainer "
    "compute it with patch_simulator(..., deferred=\"remote\", remote_intensity=True) and patched device maps")

_MISSING = object()


def _read_rir_file(path: str, speculative: bool = False):
    """``wavfile.read`` exactly like soundspaces/simulator.py:615-624: unreadable -> warning + zero RIR,
    empty -> zero RIR (both reported as ``None``); otherwise float32 ``(L, 2)``.  ``speculative`` (prefetch): a
    file that does not exist is reported as ``_MISSING`` without a warning and is not registered -- the step that
    really asks for it takes the reference's path, warning included."""
    from scipy.io import wavfile
    if speculative and not os.path.exists(path):
        return _MISSING
    try:
        _, rir = wavfile.read(path)
    except (ValueError, OSError):
        logging.warning("{} file is not readable".format(path))
        return None
    if len(rir) == 0:
        logging.debug("Empty RIR file at {}".format(path))
        return None
    if rir.dtype != np.float32:
        rir = rir.astype(np.float32)
    return rir


class AudioRenderService:
    """Per-(device, sr) owner of the renderer, the RIR-file bank and the clip bank (SURVEY.md N1).

    RIR files are read with ``scipy.io.wavfile.read`` exactly like soundspaces/simulator.py:615-624 and stay
    resident on the device.  What the reference does synchronously every step (one wav read per env,
    ``simulator.py:303-305,615-624``) happens here at most once per file and normally OFF the step's critical
    path: :meth:`prefetch` hands the files the agent can reach next (its graph neighbours / the two adjacent
    headings) to a small reader pool, :meth:`poll` uploads whatever has arrived in one batched copy, and a step
    only blocks on a file that is neither resident nor already in flight (a *miss*; counted in :attr:`stats`).
    When the bank outgrows ``max_bank_bytes`` the RIRs not touched recently are dropped and the rest compacted
    (generation GC) instead of re-reading the whole working set."""

    _instances: Dict[tuple, "AudioRenderService"] = {}

    def __init__(self, sr: int, device="cuda:0", max_taps: Optional[int] = None, pad_mode: str = "reflect",
                 n_terms: int = 2, log2n: int = 0, max_bank_bytes: int = 16 << 30, prefetch_workers: int = 4,
                 renderer=None):
        self.sr = sr
        self.max_bank_bytes = int(max_bank_bytes)
        # 1-s clips only ever use the first sr taps; multi-second clips need the whole RIR
        self.max_taps = int(max_taps) if max_taps else 4 * sr
        # ``renderer``: an already constructed renderer (the host-logic tests inject a stand-in without CUDA)
        self.renderer = renderer if renderer is not None else BatchedAudioRenderer(
            sr, self.max_taps, device=device, n_terms=n_terms, log2n=log2n, pad_mode=pad_mode)
        self._kwargs = dict(max_taps=self.max_taps, n_terms=n_terms, log2n=log2n, max_bank_bytes=self.max_bank_bytes)
        self._rir_ids: Dict[object, int] = {}        # key (path or (dir, az, r, s)) -> bank id
        self._touched: Dict[object, int] = {}        # key -> step of last use (sorted only when the bank is compacted)
        self._src_ids: Dict[tuple, tuple] = {}
        self._step = 0
        self._clock = 0                               # use counter behind the LRU order
        self._pool = ThreadPoolExecutor(max_workers=prefetch_workers, thread_name_prefix="ssb-rir") if prefetch_workers else None
        self._inflight: Dict[object, object] = {}    # key -> Future of _read_rir_file
        self._batcher = None
        self._remote = None
        self.stats = {"hits": 0, "misses": 0, "prefetched": 0, "waited": 0, "compactions": 0}

    @classmethod
    def get(cls, sr: int, device="cuda:0", **kw) -> "AudioRenderService":
        key = (int(sr), str(torch.device(device)), kw.get("pad_mode", "reflect"))
        inst = cls._instances.get(key)
        if inst is None:
            inst = cls._instances[key] = cls(sr, device=device, **kw)
        else:
            for k, v in kw.items():                   # a silently ignored kwarg would be a wrong-size plan later
                if k in inst._kwargs and v is not None and int(v) != int(inst._kwargs[k]) and not (k == "max_taps" and int(v) <= inst.max_taps):
                    raise ValueError(f"AudioRenderService for {key} already exists with {k}={inst._kwargs[k]}, asked for {v}")
        return inst

    @property
    def batcher(self):
        """The per-service queue behind the deferred sensor path (one render per step for all envs)."""
        if self._batcher is None:
            from .batching import AudioObservationBatcher
            self._batcher = AudioObservationBatcher(self)
        return self._batcher

    @property
    def remote(self):
        """The trainer side of remote deferred mode: resolves worker descriptors and keeps their memo table."""
        if self._remote is None:
            from .batching import RemoteObservations
            self._remote = RemoteObservations(self)
        return self._remote

    def requests(self, k: RemoteAudioRequest):
        """Bank resolution of a request description built by a simulator's ``_b200_keys`` -- in process, or in the
        trainer for a worker's descriptor: RIR files are looked up (read on a miss) and read ahead here, clips
        registered.  Returns the request and, with a cross-fade, the request of the previous RIR."""
        if k.silent:
            return AudioRequest(rir=-1, source=0, silent=True), None
        rid = -1
        if k.rir_key is not None:
            rid = self.rir(k.rir_key)
            self.prefetch(k.prefetch)
        req = AudioRequest(rir=rid, source=self.source(*clip_samples(k.clip)), offset=k.offset,
                           out_samples=k.out_samples, wrap=k.wrap, rir_array=k.rir_array)
        if k.distractor_key is not None:
            req.distractor_source = self.source(*clip_samples(k.distractor_clip))
            req.distractor_rir = self.rir(k.distractor_key)
        prev = None
        if k.prev_rir is not None:
            prev = AudioRequest(rir=-1, rir_array=k.prev_rir, source=req.source, offset=k.offset,
                                out_samples=k.out_samples, wrap=k.prev_wrap)
        return req, prev

    # -- banks ---------------------------------------------------------------
    @staticmethod
    def _path_of(key) -> str:
        if isinstance(key, str):
            return key
        d, az, r, s = key
        return os.path.join(d, str(az), "{}_{}.wav".format(r, s))      # simulator.py:615-616

    def maybe_trim(self):
        """Call between steps (never while requests are being built).  Advances the LRU clock, lands finished
        prefetches, and when the resident bank exceeds its budget drops the least recently used half (the full
        dataset is 867 GB; a scene's working set is what has to stay resident)."""
        self._step += 1
        self.poll()
        r = self.renderer
        if self._batcher is not None and self._batcher._pending:
            return                                    # queued requests already hold bank ids: compact after their flush
        if r.bank_bytes > self.max_bank_bytes:
            keep, kept_bytes = [], 0
            for key in sorted(self._touched, key=self._touched.get, reverse=True):      # most recently used first
                rid = self._rir_ids.get(key)
                if rid is None:
                    continue
                b = r._rir_len[rid] * 8
                if kept_bytes + b > self.max_bank_bytes // 2:
                    break
                keep.append(key)
                kept_bytes += b
            keep.reverse()
            new_ids = r.compact_bank([self._rir_ids[k] for k in keep])
            self._rir_ids = {k: i for k, i in zip(keep, new_ids)}
            self._touched = {k: self._touched[k] for k in keep}
            self.stats["compactions"] += 1

    def prefetch(self, keys):
        """Start reading the given RIR files (keys as for :meth:`rir`) unless resident or already in flight."""
        if self._pool is None:
            return
        for key in keys:
            if key in self._rir_ids or key in self._inflight:
                continue
            self._inflight[key] = self._pool.submit(_read_rir_file, self._path_of(key), True)

    def poll(self, wait_for=None):
        """Upload every finished prefetch in ONE batched host->device copy (main thread: the bank's index lists
        are not shared with the reader threads).  ``wait_for``: a key that must be resident on return."""
        if not self._inflight:
            return
        done = [k for k, f in self._inflight.items() if f.done() or k == wait_for]
        if not done:
            return
        rirs = [self._inflight.pop(k).result() for k in done]
        done = [k for k, r in zip(done, rirs) if r is not _MISSING]
        rirs = [r for r in rirs if r is not _MISSING]
        if not done:
            return
        ids = self.renderer.add_rirs(rirs)
        for k, i in zip(done, ids):
            self._rir_ids[k] = i
            self._touched.setdefault(k, 0)            # prefetched, not used yet: first to go
        self.stats["prefetched"] += len(done)

    def rir(self, key) -> int:
        """Bank id of an RIR file; ``key`` is the path, or ``(binaural_rir_dir, azimuth, receiver, source)``
        (formatted into the reference's path only when the file has to be opened)."""
        rid = self._rir_ids.get(key)
        if rid is not None:                           # the per-env hot path: two dict operations
            self.stats["hits"] += 1
            self._clock += 1
            self._touched[key] = self._clock
            return rid
        if key in self._inflight:
            self.stats["waited"] += 1
            self.poll(wait_for=key)
            rid = self._rir_ids.get(key)
            if rid is None:                           # the speculative read found no file: the reference's path
                rid = self._rir_ids[key] = self.renderer.add_rirs([_read_rir_file(self._path_of(key))])[0]
        else:
            self.stats["misses"] += 1
            rid = self.renderer.add_rirs([_read_rir_file(self._path_of(key))])[0]
            self._rir_ids[key] = rid
        self._clock += 1
        self._touched[key] = self._clock
        return rid

    rir_from_file = rir

    @property
    def miss_rate(self) -> float:
        n = self.stats["hits"] + self.stats["misses"] + self.stats["waited"]
        return (self.stats["misses"] + self.stats["waited"]) / n if n else 0.0

    def source(self, key, samples) -> int:
        """Device copy of a decoded clip, memoised per array object (the reference memoises the
        decoded clip per sound name in ``_source_sound_dict``, simulator.py:595-600; keying on the
        array keeps two simulators with different clips under one name apart)."""
        k = (key, len(samples), id(samples))
        hit = self._src_ids.get(k)
        if hit is None:
            hit = (self.renderer.add_source(np.asarray(samples, dtype=np.float32)), samples)  # keep the array alive
            self._src_ids[k] = hit
        return hit[0]


SPECTROGRAM_NATIVE_ATTR = "_b200_native_spectrogram"


def _is_native_spectrogram(fn: Callable) -> bool:
    return bool(getattr(fn, SPECTROGRAM_NATIVE_ATTR, False))


def _check_remote_callable(fn: Callable):
    # any other callable wants the host waveform inside the worker, which remote mode never renders
    if not _is_native_spectrogram(fn):
        raise RuntimeError("remote deferred mode serves SpectrogramSensor.compute_spectrogram only; another "
                           "audiogoal2spectrogram callable needs the waveform in the worker (use compat mode)")


class B200AudioMixin:
    """Audio slice of ``SoundSpacesSim`` (discrete, SoundSpaces 1.0)."""

    b200_device = "cuda:0"
    b200_pad_mode = "reflect"          # librosa < 0.10 behaviour (published checkpoints); see SURVEY.md #5
    b200_deferred = False              # True: get_current_spectrogram_observation returns a handle (see module doc)
    b200_remote_intensity = False      # remote mode: Intensity returns the waveform request (patch_simulator)
    b200_remote_frames = False         # remote mode: reset / step return FrameArray visual entries (patch_simulator)
    b200_prefetch = True               # read the RIRs reachable by the next action ahead of time (SURVEY.md N1)

    # -- plumbing --------------------------------------------------------------
    def _b200_service(self) -> AudioRenderService:
        svc = getattr(self, "_b200_svc", None)
        if svc is None:
            svc = AudioRenderService.get(self.config.AUDIO.RIR_SAMPLING_RATE, self.b200_device,
                                         pad_mode=self.b200_pad_mode)
            self._b200_svc = svc
        return svc

    def _b200_rir_path(self, source_index) -> str:
        # simulator.py:303-305 + :615-616 (azimuth_angle: :568-573)
        return os.path.join(self.binaural_rir_dir, str(self.azimuth_angle),
                            "{}_{}.wav".format(self._receiver_position_index, source_index))

    def _b200_prefetch_keys(self, rir_dir, az, receiver, source_index) -> tuple:
        """Files the NEXT action can ask for (simulator.py:496-516): MOVE_FORWARD lands on a graph neighbour with
        the same heading, TURN_LEFT / TURN_RIGHT keep the node and change the azimuth by 90 degrees."""
        keys = [(rir_dir, (az + 90) % 360, receiver, source_index), (rir_dir, (az - 90) % 360, receiver, source_index)]
        graph = getattr(self, "graph", None)
        if graph is not None:
            try:
                keys.extend((rir_dir, az, nb, source_index) for nb in graph[receiver])
            except Exception:          # noqa: BLE001 - a graph without this node: nothing to prefetch
                pass
        return tuple(keys)

    def _b200_keys(self, az=None) -> RemoteAudioRequest:
        """What one call of ``_compute_audiogoal`` (simulator.py:608-666) asks for, without touching a bank: the RIR
        key or the inline RIR, the clip, the sample offset -- with the ``_audio_index`` advance at :635 --, the
        distractor and the read-ahead keys.  ``az``: the azimuth when the caller has already read it."""
        cfg = self.config
        sr = cfg.AUDIO.RIR_SAMPLING_RATE
        if self._episode_step_count > self._duration:
            return RemoteAudioRequest(silent=True)
        k = RemoteAudioRequest()
        if not cfg.USE_RENDERED_OBSERVATIONS:
            # simulator.py:626: RIR rendered by habitat-sim for this step -> transient, supplied inline
            k.rir_array = np.transpose(np.array(self._sim.get_sensor_observations()["audio_sensor"]))
        else:
            rir_dir, recv = self.binaural_rir_dir, self._receiver_position_index
            if az is None:
                az = self.azimuth_angle
            k.rir_key = (rir_dir, az, recv, self._source_position_index)
            if self.b200_prefetch:
                k.prefetch = self._b200_prefetch_keys(rir_dir, az, recv, self._source_position_index)
        clip = self.current_source_sound
        k.clip = (self._current_sound, clip)
        if clip.shape[0] != sr:
            index = self._audio_index
            self._audio_index = (self._audio_index + 1) % self._audio_length
            k.offset = index * sr
        if cfg.AUDIO.HAS_DISTRACTOR_SOUND:
            k.distractor_clip = (self._current_distractor_sound, self._source_sound_dict[self._current_distractor_sound])
            k.distractor_key = (self.binaural_rir_dir, self.azimuth_angle, self._receiver_position_index,
                                self._distractor_position_index)
        return k

    def _b200_request(self, az=None) -> AudioRequest:
        """The request equivalent to one call of ``_compute_audiogoal`` (simulator.py:608-666), resolved against the
        service's banks.  ``az``: the azimuth when the caller has already read it."""
        svc = getattr(self, "_b200_svc", None) or self._b200_service()
        return svc.requests(self._b200_keys(az))[0]

    def _b200_remote_observation(self, kind: str) -> RemoteAudioRequest:
        """Remote mode: the descriptor of this step's spectrogram or waveform.  The memo is the reference's own
        ``_spectrogram_cache`` / ``_audiogoal_cache`` (simulator.py:678-701): a miss stores the descriptor there, a hit
        returns a payload-free reference to it (and, as in the reference, does not advance ``_audio_index``)."""
        service = (self.config.AUDIO.RIR_SAMPLING_RATE, str(self.b200_device), self.b200_pad_mode)
        if self.config.AUDIO.HAS_DISTRACTOR_SOUND:
            return package(self._b200_keys(), kind, service)
        memo = self._spectrogram_cache if kind == SPECTROGRAM else self._audiogoal_cache
        az = self.azimuth_angle
        joint_index = (self._source_position_index, self._receiver_position_index, az)
        d = memo.get(joint_index)
        if d is not None:
            return d.reference()
        slot = memo_slot(self, kind, memo)
        d = memo[joint_index] = package(self._b200_keys(az), kind, service, slot)
        return d

    # -- reference API ---------------------------------------------------------
    def _compute_audiogoal(self):
        sr = self.config.AUDIO.RIR_SAMPLING_RATE
        self._b200_service().maybe_trim()
        req = self._b200_request()
        if req.silent:
            logging.debug('Step count is greater than duration. Empty spectrogram.')
            return np.zeros((2, sr))                       # float64, as simulator.py:612
        wave = self._b200_service().renderer.convolve([req])
        return wave[0].cpu().numpy()

    def get_current_audiogoal_observation(self):
        if self.b200_deferred == REMOTE:
            return self._b200_remote_observation(WAVEFORM)
        if self.config.AUDIO.HAS_DISTRACTOR_SOUND:
            audiogoal = self._compute_audiogoal()
        else:
            joint_index = (self._source_position_index, self._receiver_position_index, self.azimuth_angle)
            if joint_index not in self._audiogoal_cache:
                self._audiogoal_cache[joint_index] = self._compute_audiogoal()
            audiogoal = self._audiogoal_cache[joint_index]
        return audiogoal

    def get_current_audiogoal_device(self) -> torch.Tensor:
        """The current ``(2, sr)`` waveform as a CUDA tensor, for on-device side consumers (AV-WaN ``Intensity``,
        avwan_sensors.py:91-100).  Follows the memo of ``get_current_audiogoal_observation``: a waveform already
        cached on the host is uploaded once, a cache miss renders on the device and never visits the host."""
        if self.b200_deferred == REMOTE:
            raise RuntimeError(INTENSITY_REMOTE_ERROR)
        r = self._b200_service().renderer
        sr = r.sr
        cacheable = not self.config.AUDIO.HAS_DISTRACTOR_SOUND
        joint_index = (self._source_position_index, self._receiver_position_index, self.azimuth_angle)
        dev = getattr(self, "_b200_dev_waves", None)
        if dev is None or dev[0] is not self._audiogoal_cache:        # the reference resets the memo by REPLACING the dict
            dev = self._b200_dev_waves = (self._audiogoal_cache, {})
        if cacheable and joint_index in dev[1]:
            return dev[1][joint_index]
        if cacheable and joint_index in self._audiogoal_cache:
            wave = torch.from_numpy(np.ascontiguousarray(self._audiogoal_cache[joint_index], dtype=np.float32)).to(r.device)
        else:
            self._b200_service().maybe_trim()
            req = self._b200_request()
            wave = torch.zeros((2, sr), device=r.device) if req.silent else r.convolve([req])[0].clone()
        if cacheable:
            dev[1][joint_index] = wave
        return wave

    def _b200_spectrogram(self, audiogoal2spectrogram):
        """One cache-missing spectrogram.  The fused device path is taken when the callable is this
        package's ``SpectrogramSensor.compute_spectrogram``; any other callable receives the host
        waveform exactly as in the reference."""
        if not _is_native_spectrogram(audiogoal2spectrogram):
            return audiogoal2spectrogram(self.get_current_audiogoal_observation())
        joint_index = (self._source_position_index, self._receiver_position_index, self.azimuth_angle)
        use_cache = not self.config.AUDIO.HAS_DISTRACTOR_SOUND
        r = self._b200_service().renderer
        if use_cache and joint_index in self._audiogoal_cache:
            wave = self._audiogoal_cache[joint_index]
            if not np.any(wave):
                return np.zeros(r.spec_shape)              # float64 zeros, as the reference on silence
            spec = r.spectrogram(torch.from_numpy(np.asarray(wave, dtype=np.float32)).to(r.device))
            return spec[0].cpu().numpy()
        self._b200_service().maybe_trim()
        req = self._b200_request()
        if req.silent:
            if use_cache:
                self._audiogoal_cache[joint_index] = np.zeros((2, r.sr))
            return np.zeros(r.spec_shape)
        spec, wave = r.render([req], want_wave=True)
        if use_cache:
            self._audiogoal_cache[joint_index] = wave[0].cpu().numpy()
        return spec[0].cpu().numpy()

    def _b200_deferred_spectrogram(self):
        """Deferred mode: enqueue, return the handle.  The memo is the reference's own ``_spectrogram_cache`` dict
        (keyed ``(source, receiver, azimuth)``, simulator.py:696-699), which the reference REPLACES on every scene
        or sound change (simulator.py:395-397) -- so a handle can never outlive its scene."""
        svc = getattr(self, "_b200_svc", None) or self._b200_service()
        if self.config.AUDIO.HAS_DISTRACTOR_SOUND:
            return svc.batcher.enqueue(self._b200_request())
        az = self.azimuth_angle
        joint_index = (self._source_position_index, self._receiver_position_index, az)
        handle = self._spectrogram_cache.get(joint_index)
        if handle is None:
            handle = self._spectrogram_cache[joint_index] = svc.batcher.enqueue(self._b200_request(az))
        return handle

    def get_current_spectrogram_observation(self, audiogoal2spectrogram):
        if self.b200_deferred == REMOTE:
            _check_remote_callable(audiogoal2spectrogram)
            return self._b200_remote_observation(SPECTROGRAM)
        if self.b200_deferred and _is_native_spectrogram(audiogoal2spectrogram):
            return self._b200_deferred_spectrogram()
        if self.config.AUDIO.HAS_DISTRACTOR_SOUND:
            spectrogram = self._b200_spectrogram(audiogoal2spectrogram)
        else:
            joint_index = (self._source_position_index, self._receiver_position_index, self.azimuth_angle)
            if joint_index not in self._spectrogram_cache:
                self._spectrogram_cache[joint_index] = self._b200_spectrogram(audiogoal2spectrogram)
            spectrogram = self._spectrogram_cache[joint_index]
        return spectrogram


class B200ContinuousAudioMixin:
    """Audio slice of ``ContinuousSoundSpacesSim`` (SoundSpaces 2.0)."""

    b200_device = "cuda:0"
    b200_pad_mode = "reflect"
    b200_deferred = False
    b200_remote_intensity = False

    def _b200_service(self) -> AudioRenderService:
        svc = getattr(self, "_b200_svc", None)
        if svc is None:
            svc = AudioRenderService.get(self.config.AUDIO.RIR_SAMPLING_RATE, self.b200_device,
                                         pad_mode=self.b200_pad_mode)
            self._b200_svc = svc
        return svc

    def _b200_keys(self) -> RemoteAudioRequest:
        """What one step's ``_compute_audiogoal`` (continuous_simulator.py:413-456) asks for: the current RIR, the
        previous one when CROSSFADE applies, the clip and the sample window."""
        sr = self.config.AUDIO.RIR_SAMPLING_RATE
        index = int(self._current_sample_index)
        # continuous_simulator.py:433-445: the clip wraps around only in the steady-state branch (index >= len(rir));
        # the early branch convolves source[:index + num_sample] and therefore sees zeros past the end of the clip.
        cur = np.asarray(np.transpose(np.array(self._prev_sim_obs["audio_sensor"])))
        k = RemoteAudioRequest(rir_array=cur, clip=(self._current_sound, self.current_source_sound), offset=index,
                               out_samples=int(sr * self.config.STEP_TIME), wrap=bool(index - cur.shape[0] >= 0))
        if self.config.AUDIO.CROSSFADE and self._last_rir is not None:
            k.prev_rir = np.asarray(self._last_rir)
            k.prev_wrap = bool(index - k.prev_rir.shape[0] >= 0)
        return k

    def _b200_requests(self):
        return self._b200_service().requests(self._b200_keys())

    def _b200_remote_observation(self, kind: str) -> RemoteAudioRequest:
        """Remote mode: the descriptor of this step's spectrogram or waveform (the continuous simulator has no memo)."""
        service = (self.config.AUDIO.RIR_SAMPLING_RATE, str(self.b200_device), self.b200_pad_mode)
        if self._episode_step_count > self._duration:
            return package(RemoteAudioRequest(silent=True), kind, service)
        return package(self._b200_keys(), kind, service)

    def _compute_audiogoal(self):
        sr = self.config.AUDIO.RIR_SAMPLING_RATE
        if self._episode_step_count > self._duration:
            logging.debug('Step count is greater than duration. Empty spectrogram.')
            return np.zeros((2, sr))
        r = self._b200_service().renderer
        cur, prev = self._b200_requests()
        with r.transient_windows():                    # a new sample index every step: do not let the pool fill up
            if prev is None:
                return r.convolve([cur])[0].cpu().numpy()
            _, wave = r.render_crossfade([cur], [prev], want_wave=True)
            return wave[0].cpu().numpy()

    def get_current_audiogoal_observation(self):
        if self.b200_deferred == REMOTE:
            return self._b200_remote_observation(WAVEFORM)
        return self._compute_audiogoal()

    def get_current_spectrogram_observation(self, audiogoal2spectrogram):
        if self.b200_deferred == REMOTE:
            _check_remote_callable(audiogoal2spectrogram)
            return self._b200_remote_observation(SPECTROGRAM)
        if not _is_native_spectrogram(audiogoal2spectrogram):
            return audiogoal2spectrogram(self.get_current_audiogoal_observation())
        r = self._b200_service().renderer
        silent = self._episode_step_count > self._duration
        if self.b200_deferred:
            batcher = self._b200_service().batcher
            if silent:
                return batcher.enqueue(AudioRequest(rir=-1, source=0, silent=True))
            cur, prev = self._b200_requests()
            return batcher.enqueue(cur, crossfade_from=prev)
        if silent:
            return np.zeros(r.spec_shape)
        cur, prev = self._b200_requests()
        with r.transient_windows():
            spec = r.render([cur]) if prev is None else r.render_crossfade([cur], [prev])
            return spec[0].cpu().numpy()


FRAME_DTYPES = (np.dtype(np.uint8), np.dtype(np.float32))


def frame_observations(sim, observations):
    """Remote mode with ``remote_frames``: each entry of ``observations`` (what the reference's ``reset`` / ``step``
    returned) that a sim sensor produced from the frame the reference took from ``_frame_cache`` -- its uuid is in
    that frame dict, its value a plain uint8 or float32 ndarray -- becomes a :class:`~soundspaces_b200.remote.
    FrameArray` keyed ``(current_scene_observation_file, receiver index, rotation angle, uuid)``.  Without
    ``USE_RENDERED_OBSERVATIONS``, or when the frame is not the ``_frame_cache`` entry of the current pose, nothing
    changes and the plain arrays cross the pipe."""
    if not getattr(sim, "b200_remote_frames", False) or not sim.config.USE_RENDERED_OBSERVATIONS or not observations:
        return observations
    recv, rot = sim._receiver_position_index, sim._rotation_angle
    frame = sim._frame_cache.get((recv, rot))
    if frame is None or frame is not sim._prev_sim_obs:
        return observations
    scene = sim.current_scene_observation_file
    for uuid in list(observations.keys()):
        v = observations[uuid]
        if uuid in frame and type(v) is np.ndarray and v.dtype in FRAME_DTYPES:
            observations[uuid] = FrameArray(v, (scene, recv, rot, uuid))
    return observations


def _frames_wrapper(fn):
    def wrapper(self, *args, **kwargs):
        return frame_observations(self, fn(self, *args, **kwargs))
    wrapper.__name__, wrapper.__qualname__, wrapper.__doc__ = fn.__name__, fn.__qualname__, fn.__doc__
    wrapper.__wrapped__ = fn
    wrapper._b200_frames = True
    return wrapper


def _patch_frames(sim_cls, on: bool):
    """Wrap (``on``) or unwrap the class's own ``reset`` and ``step`` with :func:`frame_observations`; the reference's
    methods run unchanged inside the wrappers.  Patching twice wraps once."""
    for name in ("reset", "step"):
        fn = getattr(sim_cls, name, None)
        if fn is None:
            if on:
                raise ValueError(f"remote_frames wraps the simulator's reset and step; {sim_cls.__name__} has no {name}")
            continue
        wrapped = getattr(fn, "_b200_frames", False)
        if on and not wrapped:
            setattr(sim_cls, name, _frames_wrapper(fn))
        elif not on and wrapped and name in vars(sim_cls):
            setattr(sim_cls, name, fn.__wrapped__)


_DISCRETE = ("_compute_audiogoal", "get_current_audiogoal_observation", "get_current_spectrogram_observation")
_DISCRETE_HELPERS = ("_b200_service", "_b200_rir_path", "_b200_keys", "_b200_request", "_b200_spectrogram",
                     "_b200_prefetch_keys", "_b200_deferred_spectrogram", "_b200_remote_observation",
                     "get_current_audiogoal_device")
_CONTINUOUS = ("_compute_audiogoal", "get_current_audiogoal_observation", "get_current_spectrogram_observation")
_CONTINUOUS_HELPERS = ("_b200_service", "_b200_keys", "_b200_requests", "_b200_remote_observation")

# attributes of the reference object that the patched methods read (checked against the real classes by
# tests/test_host_logic.py::test_patch_simulator_on_reference_classes)
DISCRETE_READS = ("config", "_episode_step_count", "_duration", "_sim", "binaural_rir_dir", "azimuth_angle",
                  "_receiver_position_index", "_source_position_index", "current_source_sound", "_current_sound",
                  "_audio_index", "_audio_length", "_source_sound_dict", "_current_distractor_sound",
                  "_distractor_position_index", "_audiogoal_cache", "_spectrogram_cache", "graph")
CONTINUOUS_READS = ("config", "_episode_step_count", "_duration", "current_source_sound", "_current_sound",
                    "_current_sample_index", "_prev_sim_obs", "_last_rir")


def patch_simulator(sim_cls, continuous: bool = False, device: str = "cuda:0", pad_mode: str = "reflect",
                    deferred=False, remote_intensity: bool = False, remote_frames: bool = False):
    """Replace the audio methods of an existing (reference) simulator class in place: exactly the three methods
    of the reference's audio slice are overridden, the ``_b200_*`` helpers are added next to them.

    ``deferred``: False (compat: host arrays), True (handles rendered once per step in this process) or ``"remote"``
    (multiprocess vector-env workers: the simulator returns :class:`~soundspaces_b200.remote.RemoteAudioRequest`
    descriptors, never touches CUDA, and the trainer's ``batch_obs`` renders the step).

    ``remote_intensity`` (remote mode only): AV-WaN's ``Intensity`` sensor returns ``[IntensityRequest]`` -- the
    waveform request, whose intensity the trainer computes on the device for the ``intensity`` batch and for the device
    acoustic map (``maps.patch_planner``) -- instead of refusing remote mode.  The worker's host acoustic map then holds
    placeholders.

    ``remote_frames`` (remote mode only): the discrete simulator's ``reset`` and ``step`` are wrapped so that the RGB /
    depth entries taken from ``_frame_cache`` (``USE_RENDERED_OBSERVATIONS``) cross the pipe as
    :class:`~soundspaces_b200.remote.FrameArray` -- a frame's data once per worker, its key afterwards -- and the
    trainer's ``batch_obs`` gathers them on the device (``soundspaces_b200.frames``).  The continuous simulator's frames
    are rendered live and have no key: with ``continuous=True`` its observations stay plain arrays."""
    if deferred != REMOTE and not isinstance(deferred, bool):
        raise ValueError(f"deferred must be False, True or {REMOTE!r}, got {deferred!r}")
    if remote_intensity and deferred != REMOTE:
        raise ValueError(f"remote_intensity needs deferred={REMOTE!r}")
    if remote_frames and deferred != REMOTE:
        raise ValueError(f"remote_frames needs deferred={REMOTE!r}")
    mixin = B200ContinuousAudioMixin if continuous else B200AudioMixin
    for name in (_CONTINUOUS + _CONTINUOUS_HELPERS if continuous else _DISCRETE + _DISCRETE_HELPERS):
        setattr(sim_cls, name, getattr(mixin, name))
    sim_cls.b200_device = device
    sim_cls.b200_pad_mode = pad_mode
    sim_cls.b200_deferred = deferred
    sim_cls.b200_remote_intensity = bool(remote_intensity)
    if not continuous:
        sim_cls.b200_prefetch = True
        sim_cls.b200_remote_frames = bool(remote_frames)
        _patch_frames(sim_cls, bool(remote_frames))
    return sim_cls
