"""Trace-replay environment for BASELINE.json config 5 (DD-PPO rollout with the audio observation fused into the
step), used where habitat-lab / habitat-sim are not installed (SURVEY.md 8(d): "a fake env that replays recorded
(rir_id, action) traces").

What is real here is everything ON the audio path, driven exactly as the reference drives it:

* :class:`ReplaySim` is a simulator object with the attributes and the ``step`` semantics of the discrete
  ``SoundSpacesSim`` (grid graph, MOVE_FORWARD / TURN_LEFT / TURN_RIGHT / STOP, soundspaces/simulator.py:478-566,
  azimuth rule :568-573, memo dicts replaced on scene / sound change :395-397) with the audio slice supplied by
  :class:`~soundspaces_b200.simulator.B200AudioMixin`;
* observations come from this package's ``SpectrogramSensor`` (deferred handles) through ``batch_obs`` into the
  ``RolloutStorage`` slot ``observations["spectrogram"][step + 1]`` (ss_baselines/common/rollout_storage.py:27-35,88-91);
* the consumer is an ``AudioCNN``-shaped encoder (ss_baselines/av_nav/models/audio_cnn.py:31-89: three convolutions,
  flatten, linear) with a 4-way policy head -- ordinary PyTorch policy code, not part of this library's kernels.

:class:`ReplayVectorEnv` steps the envs in process (``SyncVectorEnv``); :class:`ProcessReplayVectorEnv` is the stand-in
for ``habitat.VectorEnv`` -- one worker process per env, observations pickled back -- used with the simulators in
remote deferred mode (or in compat mode: one CUDA context per worker).

What is replayed instead of simulated: the visual sensors, rewards and episode logic (none of which touch audio).
Visual observations are off by default; with ``frames=`` (a scene-observation pickle, :func:`write_scene_observations`)
the sim returns the ``rgb`` / ``depth`` observations of the frame ``_frame_cache[(node, rotation)]`` from ``reset`` and
``step`` as the reference's ``SoundSpacesSim`` does with ``USE_RENDERED_OBSERVATIONS`` (soundspaces/simulator.py:448-
566), and :class:`FrameReplaySim` is that sim patched as ``patch_simulator(..., remote_frames=True)`` patches the
reference's.
"""
from __future__ import annotations

import os
import time
from types import SimpleNamespace
from typing import Dict, List, Optional, Sequence

import numpy as np
import torch
import torch.nn as nn

from .simulator import REMOTE, AudioRenderService, B200AudioMixin, _patch_frames

STOP, MOVE_FORWARD, TURN_LEFT, TURN_RIGHT = 0, 1, 2, 3          # HabitatSimActions


class ReplayScene:
    """A navigation graph on a square grid (node = row * side + col, 1 m spacing in the X-Z plane) and the bank ids
    of its binaural RIRs keyed like the reference's wav tree ``<dir>/<azimuth>/<receiver>_<source>.wav``."""

    def __init__(self, name: str, side: int, rir_root: str = "/replay", dataset: str = "replica"):
        import networkx as nx
        self.name, self.side = name, int(side)
        self.rir_dir = os.path.join(rir_root, dataset, name)
        g = nx.Graph()
        for r in range(side):
            for c in range(side):
                g.add_node(r * side + c, point=(float(c), 0.0, float(r)))
        for r in range(side):
            for c in range(side):
                if c + 1 < side:
                    g.add_edge(r * side + c, r * side + c + 1)
                if r + 1 < side:
                    g.add_edge(r * side + c, (r + 1) * side + c)
        self.graph = g

    @property
    def n_nodes(self) -> int:
        return self.side * self.side

    def register_rirs(self, service: AudioRenderService, source: int, rirs, azimuths=(0, 90, 180, 270)):
        """Make the scene's RIRs device-resident: ``rirs[az_index][receiver]`` -> one batched upload; afterwards
        ``service.rir((rir_dir, az, receiver, source))`` is a hit, as after the reference's first visit + N1 prefetch."""
        flat, keys = [], []
        for ai, az in enumerate(azimuths):
            for recv in range(self.n_nodes):
                flat.append(rirs[ai][recv])
                keys.append((self.rir_dir, az, recv, source))
        ids = service.renderer.add_rirs(flat)
        for k, i in zip(keys, ids):
            service._rir_ids[k] = i
            service._touched.setdefault(k, 0)
        return ids


MIN_DEPTH, MAX_DEPTH = 0.0, 10.0                  # habitat's DEPTH_SENSOR defaults, NORMALIZE_DEPTH on


def scene_observations(n_nodes: int, height: int, width: int, seed: int = 0, rotations=(0, 90, 180, 270)) -> dict:
    """A seeded stand-in for a scene-observation pickle's contents (scripts/cache_observations.py): ``{(node, rotation):
    {"rgb": (H, W, 4) uint8 RGBA, "depth": (H, W) float32 metres}}``.  The depth spans 0 to beyond ``MAX_DEPTH``."""
    rng = np.random.default_rng(seed)
    cache = {}
    for node in range(n_nodes):
        for rot in rotations:
            rgb = rng.integers(0, 256, size=(height, width, 4), dtype=np.uint8)
            depth = (rng.random((height, width), dtype=np.float32) * np.float32(1.2 * MAX_DEPTH)).astype(np.float32)
            depth[0, 0] = 0.0
            cache[(node, rot)] = {"rgb": rgb, "depth": depth}
    return cache


def write_scene_observations(path: str, cache: dict) -> str:
    """Pickle ``cache`` where ``SoundSpacesSim`` reads it (``<dir>/<dataset>/<scene>.pkl``, simulator.py:143-146)."""
    import pickle
    os.makedirs(os.path.dirname(path), exist_ok=True)
    with open(path, "wb") as f:
        pickle.dump(cache, f, protocol=pickle.HIGHEST_PROTOCOL)
    return path


def visual_observations(sim_obs: dict) -> dict:
    """habitat's RGB and depth sensors on a cached frame (habitat/sims/habitat_simulator/habitat_simulator.py:
    HabitatSimRGBSensor / HabitatSimDepthSensor.get_observation): RGB without alpha, depth clipped, given a channel
    axis and normalised."""
    depth = np.clip(sim_obs["depth"], MIN_DEPTH, MAX_DEPTH)
    depth = (np.expand_dims(depth, axis=2) - MIN_DEPTH) / (MAX_DEPTH - MIN_DEPTH)
    return {"rgb": sim_obs["rgb"][:, :, :3], "depth": depth.astype(np.float32, copy=False)}


class ReplaySim(B200AudioMixin):
    """The audio-relevant state machine of ``SoundSpacesSim`` driven by actions (see module docstring).  ``frames``: a
    scene-observation pickle; ``reset`` and ``step`` then return the visual observations of the current pose (an
    empty dict without it)."""

    def __init__(self, service: Optional[AudioRenderService], scene: ReplayScene, sound: str, clip: np.ndarray,
                 source_node: int, start_node: int = 0, start_rotation: int = 0, deferred=True, duration: int = 500,
                 sr: Optional[int] = None, frames: Optional[str] = None):
        # service None (a worker process): ``sr`` names the rate; compat mode then builds the worker's own service
        sr = service.sr if service is not None else int(sr)
        self._b200_svc = service
        self.b200_deferred = deferred
        self.config = SimpleNamespace(
            USE_RENDERED_OBSERVATIONS=True, SCENE_DATASET="replica",
            AUDIO=SimpleNamespace(RIR_SAMPLING_RATE=sr, HAS_DISTRACTOR_SOUND=False, EVERLASTING=True))
        self._source_sound_dict: Dict[str, np.ndarray] = {}
        self._current_sound = None
        self._current_scene = None
        self._audiogoal_cache, self._spectrogram_cache = dict(), dict()
        self._duration = duration
        self._frames_file, self._frame_cache, self._prev_sim_obs = frames, {}, None
        if frames is not None:
            import pickle
            with open(frames, "rb") as f:
                self._frame_cache = pickle.load(f)
        self.reconfigure(scene, sound, clip, source_node, start_node, start_rotation)

    @property
    def current_scene_observation_file(self):
        return self._frames_file

    def _observations(self) -> dict:
        """simulator.py:448-458 and the sim sensors' observations of the frame (empty without ``frames``)."""
        if not self._frame_cache:
            return {}
        self._prev_sim_obs = self._frame_cache[(self._receiver_position_index, self._rotation_angle)]
        return visual_observations(self._prev_sim_obs)

    # -- what the reference's reconfigure() does to the audio state (simulator.py:340-397) ------------------------
    def reconfigure(self, scene: ReplayScene, sound: str, clip: np.ndarray, source_node: int, start_node: int,
                    start_rotation: int):
        sr = self.config.AUDIO.RIR_SAMPLING_RATE
        self._audio_index = 0
        same_sound = sound == self._current_sound
        if not same_sound:
            self._current_sound = sound
            self._source_sound_dict.setdefault(sound, clip)
        self._audio_length = self._source_sound_dict[self._current_sound].shape[0] // sr
        same_scene = scene is self._current_scene
        if not same_scene:
            self._current_scene = scene
            self.graph = scene.graph
        if not same_scene or not same_sound:
            self._audiogoal_cache = dict()
            self._spectrogram_cache = dict()
        self._episode_step_count = 0
        self._start = (int(start_node), int(start_rotation))
        self._receiver_position_index = int(start_node)
        self._source_position_index = int(source_node)
        self._rotation_angle = int(start_rotation) % 360
        self._is_episode_active = True

    def reset(self):
        """A new episode from the start pose, same scene and sound: the memo dicts are kept (simulator.py:395-397)."""
        self.reconfigure(self._current_scene, self._current_sound, self.current_source_sound,
                         self._source_position_index, *self._start)
        return self._observations()

    @property
    def binaural_rir_dir(self):
        return self._current_scene.rir_dir

    @property
    def current_source_sound(self):
        return self._source_sound_dict[self._current_sound]

    @property
    def azimuth_angle(self):
        return -(self._rotation_angle + 0) % 360            # simulator.py:568-573

    @property
    def is_silent(self):
        return self._episode_step_count > self._duration

    def get_orientation(self):
        return (270 - self._rotation_angle) % 360            # simulator.py:563-565

    def step(self, action: int):
        """simulator.py:496-516."""
        if action == STOP:
            self._is_episode_active = False
        elif action == MOVE_FORWARD:
            here = self.graph.nodes[self._receiver_position_index]["point"]
            for nb in self.graph[self._receiver_position_index]:
                p2 = self.graph.nodes[nb]["point"]
                direction = int(np.around(np.rad2deg(np.arctan2(p2[2] - here[2], p2[0] - here[0])))) % 360
                if direction == self.get_orientation():
                    self._receiver_position_index = nb
                    break
        elif action == TURN_LEFT:
            self._rotation_angle = (self._rotation_angle + 90) % 360
        elif action == TURN_RIGHT:
            self._rotation_angle = (self._rotation_angle - 90) % 360
        self._episode_step_count += 1
        return self._observations()


class FrameReplaySim(ReplaySim):
    """:class:`ReplaySim` with ``reset`` / ``step`` wrapped as ``patch_simulator(..., deferred="remote",
    remote_frames=True)`` wraps the reference's: the visual entries become ``FrameArray`` s."""

    b200_remote_frames = True


_patch_frames(FrameReplaySim, True)


class ReplayVectorEnv:
    """``n`` in-process envs stepped like ``SyncVectorEnv`` (ss_baselines/common/sync_vector_env.py:186-199): every
    env's sensor suite is asked for its observation once per step; the spectrogram sensors return handles.

    ``episode_steps``: auto-reset as the trainers' vector envs do (``auto_reset_done=True``,
    sync_vector_env.py:82-85): when an episode reaches this many steps, the terminal step's observation is built and
    dropped, and the env returns the observation of a new episode from its start pose (:meth:`ReplaySim.reset`)."""

    def __init__(self, sims: Sequence[ReplaySim], audiogoal: bool = False, episode_steps: Optional[int] = None):
        from .sensors import AudioGoalSensor, SpectrogramSensor
        self.sims = list(sims)
        kinds = {"spectrogram": SpectrogramSensor, **({"audiogoal": AudioGoalSensor} if audiogoal else {})}
        self.sensors = [{uuid: cls(sim=s, config=None) for uuid, cls in kinds.items()} for s in self.sims]
        self.num_envs = len(self.sims)
        self.episode_steps = episode_steps
        # the sim's own observations of the current pose (visual, with ``frames``), as its last reset / step returned
        self._sim_obs = [s.reset() if getattr(s, "_frame_cache", None) else {} for s in self.sims]

    def observe(self) -> List[dict]:
        return [self._observe(suite, sim_obs) for suite, sim_obs in zip(self.sensors, self._sim_obs)]

    @staticmethod
    def _observe(suite, sim_obs=None) -> dict:
        obs = dict(sim_obs) if sim_obs else {}
        obs.update({uuid: sensor.get_observation(observations=None, episode=None) for uuid, sensor in suite.items()})
        return obs

    def step(self, actions: Sequence[int]):
        for i, (sim, a) in enumerate(zip(self.sims, actions)):
            if a == STOP or not sim._is_episode_active:       # episode over: a new one starts where it stands
                sim._is_episode_active, sim._episode_step_count = True, 0
            else:
                self._sim_obs[i] = sim.step(int(a))
        obs = self.observe()
        if self.episode_steps:
            for i, sim in enumerate(self.sims):
                if sim._episode_step_count >= self.episode_steps:
                    self._sim_obs[i] = sim.reset()
                    obs[i] = self._observe(self.sensors[i], self._sim_obs[i])
        return obs


def replay_sim(sr: int, scene: str, side: int, rir_root: str, sound: str, clip: np.ndarray, source_node: int,
               start_node: int = 0, start_rotation: int = 0, deferred=REMOTE, duration: int = 500,
               frames: Optional[str] = None, remote_frames: bool = False) -> ReplaySim:
    """A :class:`ReplaySim` whose RIRs are the wav tree ``<rir_root>/replica/<scene>/<az>/<recv>_<source>.wav`` and
    which has no service of its own: the factory :class:`ProcessReplayVectorEnv` calls in each worker.  ``frames``:
    its scene-observation pickle; ``remote_frames``: a :class:`FrameReplaySim` (remote mode)."""
    if remote_frames and deferred != REMOTE:
        raise ValueError(f"remote_frames needs deferred={REMOTE!r}")
    cls = FrameReplaySim if remote_frames else ReplaySim
    return cls(None, ReplayScene(scene, side, rir_root=rir_root), sound, clip, source_node, start_node,
               start_rotation, deferred=deferred, duration=duration, sr=sr, frames=frames)


def worker_report(sim) -> dict:
    """What a worker process has loaded: whether torch has initialised CUDA and whether libssb200 is mapped."""
    with open("/proc/self/maps") as f:
        lib = any("libssb200" in line for line in f)
    return {"pid": os.getpid(), "cuda_initialized": torch.cuda.is_initialized(), "libssb200_loaded": lib}


class _WorkerError:
    def __init__(self, text: str):
        self.text = text


def _replay_worker(conn, make_sim, args, audiogoal, episode_steps):
    """One env of :class:`ProcessReplayVectorEnv`: build the simulator, then answer commands until ``close``."""
    import pickle
    import traceback
    try:
        try:
            env = ReplayVectorEnv([make_sim(*args)], audiogoal=audiogoal, episode_steps=episode_steps)
            conn.send_bytes(pickle.dumps(None))
        except Exception:                             # noqa: BLE001 - reported to the parent, which raises
            conn.send_bytes(pickle.dumps(_WorkerError(traceback.format_exc())))
            return
        while True:
            cmd, arg = conn.recv()
            if cmd == "close":
                return
            try:
                if cmd == "observe":
                    res = env.observe()[0]
                elif cmd == "step":
                    res = env.step([arg])[0]
                else:                                 # "call": arg = (fn, args), fn(sim, *args)
                    res = arg[0](env.sims[0], *arg[1])
                payload = pickle.dumps(res, protocol=pickle.HIGHEST_PROTOCOL)
            except Exception:                         # noqa: BLE001
                payload = pickle.dumps(_WorkerError(traceback.format_exc()))
            conn.send_bytes(payload)
    except (EOFError, KeyboardInterrupt):              # parent gone
        pass
    finally:
        conn.close()


class ProcessReplayVectorEnv:
    """The multiprocess counterpart of :class:`ReplayVectorEnv`, shaped like ``habitat.VectorEnv`` (the trainers'
    default, ``USE_VECENV`` without ``USE_SYNC_VECENV``): one worker process per env started by ``forkserver`` or
    ``spawn``, commands and observations through pipes, every observation pickled back.  ``make_sim(*args)`` builds
    the worker's simulator (:func:`replay_sim`); ``episode_steps`` auto-resets as in :class:`ReplayVectorEnv`, inside
    the worker, so a terminal step's observation never crosses the pipe.  ``bytes_received`` counts the pickled
    observation bytes.

    :meth:`close` (also on ``with`` exit) joins every worker; none outlives it."""

    def __init__(self, make_sim, args_list: Sequence[tuple], start_method: str = "forkserver", audiogoal: bool = False,
                 episode_steps: Optional[int] = None):
        import multiprocessing as mp
        ctx = mp.get_context(start_method)
        self._conns, self._procs = [], []
        self.num_envs = len(args_list)
        self.bytes_received = 0
        try:
            for args in args_list:
                parent, child = ctx.Pipe()
                p = ctx.Process(target=_replay_worker, args=(child, make_sim, tuple(args), audiogoal, episode_steps),
                                daemon=True)
                p.start()
                child.close()
                self._conns.append(parent)
                self._procs.append(p)
            for c in self._conns:
                self._recv(c)
        except BaseException:
            self.close()
            raise

    def _recv(self, conn):
        import pickle
        data = conn.recv_bytes()
        self.bytes_received += len(data)
        res = pickle.loads(data)
        if isinstance(res, _WorkerError):
            raise RuntimeError("replay worker failed:\n" + res.text)
        return res

    def _all(self, msgs) -> list:
        for c, m in zip(self._conns, msgs):
            c.send(m)
        return [self._recv(c) for c in self._conns]

    def observe(self) -> List[dict]:
        return self._all([("observe", None)] * self.num_envs)

    def step(self, actions: Sequence[int]) -> List[dict]:
        return self._all([("step", int(a)) for a in actions])

    def call(self, fn, *args) -> list:
        """``fn(sim, *args)`` in every worker (``fn`` picklable by reference), results in env order."""
        return self._all([("call", (fn, args))] * self.num_envs)

    def close(self):
        for c in self._conns:
            try:
                c.send(("close", None))
            except (OSError, ValueError):             # worker already gone
                pass
        for p in self._procs:
            p.join(timeout=30)
            if p.is_alive():
                p.terminate()
                p.join()
        for c in self._conns:
            c.close()
        self._conns, self._procs = [], []

    @property
    def processes(self) -> list:
        return list(self._procs)

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()


class AudioPolicy(nn.Module):
    """``AudioCNN`` (audio_cnn.py:31-89: Conv 8x8/4 -> 4x4/2 -> 3x3/1, or the 5/3/3 variant for small inputs, flatten,
    linear, ReLU) feeding a 4-action categorical head and a value head.  ``channels_first``: the observation already
    is (N, 2, 65, T') -- what the reference obtains with ``permute(0, 3, 1, 2)`` (audio_cnn.py:86)."""

    def __init__(self, spec_shape, hidden: int = 512, channels_first: bool = False):
        super().__init__()
        h, w, c = spec_shape
        if h < 30 or w < 30:
            ks, st = [(5, 5), (3, 3), (3, 3)], [(2, 2), (2, 2), (1, 1)]
        else:
            ks, st = [(8, 8), (4, 4), (3, 3)], [(4, 4), (2, 2), (1, 1)]
        dims = [h, w]
        for k, s in zip(ks, st):
            dims = [int(np.floor((d - (kk - 1) - 1) / ss + 1)) for d, kk, ss in zip(dims, k, s)]
        self.channels_first = channels_first
        self.cnn = nn.Sequential(
            nn.Conv2d(c, 32, ks[0], st[0]), nn.ReLU(True), nn.Conv2d(32, 64, ks[1], st[1]), nn.ReLU(True),
            nn.Conv2d(64, 64, ks[2], st[2]), nn.Flatten(), nn.Linear(64 * dims[0] * dims[1], hidden), nn.ReLU(True))
        self.actor, self.critic = nn.Linear(hidden, 4), nn.Linear(hidden, 1)

    def forward(self, spectrogram: torch.Tensor):
        x = spectrogram if self.channels_first else spectrogram.permute(0, 3, 1, 2)
        f = self.cnn(x)
        return self.actor(f), self.critic(f)

    @torch.no_grad()
    def forward_fused(self, spectrogram: torch.Tensor):
        """Rollout-time forward with the first layer fused (SURVEY.md N2): permute + Conv2d + ReLU of ``cnn[0:2]``
        run as ONE kernel straight from the (N, 65, T', 2) observation (``WaveformOps.audio_conv1``)."""
        from .renderer import WaveformOps
        if self.channels_first or not spectrogram.is_cuda:
            return self.forward(spectrogram)
        f = self.cnn[2:](WaveformOps.get(spectrogram.device).audio_conv1(spectrogram.contiguous(), self.cnn[0], relu=True))
        return self.actor(f), self.critic(f)

    @torch.no_grad()
    def act(self, spectrogram: torch.Tensor, fused: bool = False):
        logits, value = self.forward_fused(spectrogram) if fused else self.forward(spectrogram)
        dist = torch.distributions.Categorical(logits=logits)
        actions = dist.sample()
        return value, actions, dist.log_prob(actions)


def collect_rollout(envs: ReplayVectorEnv, policy: AudioPolicy, storage: torch.Tensor, num_steps: int,
                    forced_actions: Optional[np.ndarray] = None, fused: bool = False):
    """One rollout of ``num_steps`` env steps with the reference's timers (ppo_trainer.py:125-194): ``pth_time`` =
    action sampling + observation batching / insertion, ``env_time`` = ``envs.step``.  ``storage``: the
    ``(num_steps + 1, num_envs, 65, T', 2)`` tensor ``rollouts.observations["spectrogram"]``; the step's batch is
    rendered straight into ``storage[step + 1]`` by ``batch_obs`` (nothing for ``RolloutStorage.insert`` to copy).
    ``forced_actions`` (``(num_steps, num_envs)``): replay a recorded action trace instead of the sampled actions.
    ``fused``: run the policy's first layer with the fused permute + Conv2d + ReLU kernel (SURVEY.md N2)."""
    from .sensors import batch_obs
    dev = storage.device
    pth_time = env_time = 0.0
    batch_obs(envs.observe(), device=dev, out={"spectrogram": storage[0]})
    for step in range(num_steps):
        t0 = time.time()
        _, actions, _ = policy.act(storage[step], fused=fused)
        acts = actions.tolist() if forced_actions is None else forced_actions[step].tolist()
        pth_time += time.time() - t0
        t0 = time.time()
        observations = envs.step(acts)
        env_time += time.time() - t0
        t0 = time.time()
        batch_obs(observations, device=dev, out={"spectrogram": storage[step + 1]})
        pth_time += time.time() - t0
    torch.cuda.synchronize(dev) if dev.type == "cuda" else None
    return pth_time, env_time, num_steps * envs.num_envs
