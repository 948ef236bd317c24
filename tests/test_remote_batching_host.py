"""CPU tests of remote deferred mode (``patch_simulator(..., deferred="remote")``): simulators in worker processes
return picklable request descriptors and the trainer renders the whole step once.  The trainer side runs on the
stand-in renderer; the worker side runs in real worker processes (forkserver and spawn)."""
import contextlib
import os
import pickle

import numpy as np
import pytest
import torch

from oracle.ref_harness import write_rir
from stubs import StubRenderer
from synth import make_rir, make_source

from soundspaces_b200.remote import ClipRef, RemoteAudioRequest
from soundspaces_b200.replay import (ProcessReplayVectorEnv, ReplayScene, ReplaySim, ReplayVectorEnv, replay_sim,
                                     worker_report)
from soundspaces_b200.sensors import Intensity, batch_obs
from soundspaces_b200.simulator import INTENSITY_REMOTE_ERROR, AudioRenderService

SR = 16000


class WaveStub(StubRenderer):
    """StubRenderer plus the waveform entry: row ``i`` of ``convolve`` is ``1000 * rir + offset // sr``."""

    def __init__(self, sr=SR):
        super().__init__(sr)
        self.convolves = []

    def convolve(self, reqs):
        self.convolves.append(list(reqs))
        return torch.stack([torch.full((2, self.sr), float(1000 * q.rir + q.offset // self.sr)) for q in reqs])


@contextlib.contextmanager
def trainer_service(sr=SR):
    """The trainer's service for ``(sr, "cuda:0", "reflect")`` with the stand-in renderer, logging RIR keys."""
    svc = AudioRenderService(sr, renderer=WaveStub(sr), prefetch_workers=0)
    svc.rir_log, svc.prefetch_log = [], []
    rir, prefetch = svc.rir, svc.prefetch
    svc.rir = lambda key: (svc.rir_log.append(key), rir(key))[1]
    svc.prefetch = lambda keys: (svc.prefetch_log.append(tuple(keys)), prefetch(keys))[1]
    key = (sr, "cuda:0", "reflect")
    old = AudioRenderService._instances.get(key)
    AudioRenderService._instances[key] = svc
    try:
        yield svc
    finally:
        if old is None:
            AudioRenderService._instances.pop(key)
        else:
            AudioRenderService._instances[key] = old


def wav_tree(root, scenes=("apartment_0", "office_3"), side=2, source=3):
    """RIRs for every (azimuth, receiver) of each scene, except one missing file and one empty file."""
    for si, scene in enumerate(scenes):
        for ai, az in enumerate((0, 90, 180, 270)):
            for recv in range(side * side):
                if (si, az, recv) == (0, 90, 3):
                    continue                                              # missing: the zero-RIR fallback
                rir = np.zeros((0, 2), np.float32) if (si, az, recv) == (0, 180, 2) else \
                    make_rir(100 * si + 10 * ai + recv, 200 + 50 * recv + 13 * si)
                write_rir(root, "replica", scene, az, recv, source, SR, rir)
                if si == 1:                                               # the distractor's RIRs
                    write_rir(root, "replica", scene, az, recv, 1, SR, make_rir(500 + 10 * ai + recv, 120 + recv))


class InlineRirs:
    """``_sim.get_sensor_observations()`` of habitat-sim: a new RIR every call, the same sequence for twin sims."""

    def __init__(self, seed):
        self.n, self.seed = 0, seed

    def get_sensor_observations(self):
        self.n += 1
        return {"audio_sensor": make_rir(self.seed + self.n, 150 + self.n).T.astype(np.float64).tolist()}


def make_sims(svc, root, deferred):
    """Four envs covering a 1-s clip, a 3-s clip, a distractor, and a habitat-rendered (inline) RIR going silent."""
    scenes = [ReplayScene(n, 2, rir_root=root) for n in ("apartment_0", "office_3")]
    one, three, two = make_source(0, SR), make_source(1, 3 * SR), make_source(2, 2 * SR)
    kw = dict(deferred=deferred, sr=SR)
    sims = [ReplaySim(svc, scenes[0], "bell.wav", one, 3, 3, 270, **kw),                  # starts on the missing file
            ReplaySim(svc, scenes[0], "phone.wav", three, 3, 2, 180, duration=40, **kw),  # ... and on the empty one
            ReplaySim(svc, scenes[1], "bell.wav", one, 3, 2, 180, **kw),
            ReplaySim(svc, scenes[1], "radio.wav", two, 3, 3, 270, duration=20, **kw)]
    d = sims[2]
    d.config.AUDIO.HAS_DISTRACTOR_SOUND = True
    d._current_distractor_sound, d._distractor_position_index = "dog.wav", 1
    d._source_sound_dict["dog.wav"] = make_source(3, SR)
    sims[3].config.USE_RENDERED_OBSERVATIONS = False
    sims[3]._sim = InlineRirs(7)
    return sims, scenes


def request_view(svc, q):
    """A render request in bank-independent terms: RIR keys instead of bank ids."""
    inv = {v: k for k, v in svc._rir_ids.items()}
    return (q.silent, q.offset, q.out_samples, q.wrap, inv.get(q.rir, q.rir), inv.get(q.distractor_rir),
            None if q.rir_array is None else np.asarray(q.rir_array, np.float32).tobytes())


def test_descriptors_pickle_and_drop_payload_after_first_use(tmp_path):
    root = str(tmp_path)
    wav_tree(root)
    sims, _ = make_sims(None, root, "remote")
    sim = sims[1]
    spec = sims[1].get_current_spectrogram_observation(_native())
    first = pickle.loads(pickle.dumps(spec))
    assert isinstance(first, RemoteAudioRequest) and not first.hit and first.memo_id == 0
    assert first.rir_key == (sim.binaural_rir_dir, 180, 2, 3) and first.offset == 0 and sim._audio_index == 1
    assert isinstance(first.clip, ClipRef) and first.clip.length == 3 * SR
    assert set(first.prefetch) == {(sim.binaural_rir_dir, az, 2, 3) for az in (90, 270)} | \
        {(sim.binaural_rir_dir, 180, nb, 3) for nb in (0, 3)}
    # memo hit: a reference without sample data that still names its request, and (the reference's quirk) no
    # _audio_index advance
    hit = pickle.loads(pickle.dumps(sim.get_current_spectrogram_observation(_native())))
    assert hit.hit and (hit.env, hit.generation, hit.memo_id) == (first.env, first.generation, first.memo_id)
    assert hit.clip.samples is None and hit.rir_array is None and not hit.prefetch
    assert (hit.rir_key, hit.offset, hit.silent) == (first.rir_key, first.offset, first.silent)
    assert len(pickle.dumps(hit)) < 1000 and sim._audio_index == 1
    # a new node: the clip travels by identity only
    sim.step(1)
    sim.step(2)
    nxt = pickle.loads(pickle.dumps(sim.get_current_spectrogram_observation(_native())))
    assert not nxt.hit and nxt.clip.samples is None and nxt.clip.key == first.clip.key and nxt.offset == SR
    assert len(pickle.dumps(nxt)) < 2000
    # the waveform memo is the reference's _audiogoal_cache, a separate generation counter
    wave = sim.get_current_audiogoal_observation()
    assert wave.kind == "waveform" and wave.env != first.env and sim._audiogoal_cache


def test_trainer_renders_what_in_process_deferred_mode_enqueues(tmp_path):
    """A seeded 50-step trace through twin sims: in-process deferred on one service, remote (descriptors pickled) on
    the trainer's service.  Same RIR keys, read-ahead keys, offsets, _audio_index sequence, distractor terms, inline
    RIRs and silent flags; one flush per step; memo hits render nothing; a scene change never hits the memo."""
    root = str(tmp_path)
    wav_tree(root)
    local = AudioRenderService(SR, renderer=StubRenderer(SR), prefetch_workers=0)
    local.rir_log, local.prefetch_log = [], []
    rir, prefetch = local.rir, local.prefetch
    local.rir = lambda key: (local.rir_log.append(key), rir(key))[1]
    local.prefetch = lambda keys: (local.prefetch_log.append(tuple(keys)), prefetch(keys))[1]
    with trainer_service() as svc:
        sims_a, scenes = make_sims(local, root, True)
        sims_b, _ = make_sims(None, root, "remote")
        env_a, env_b = ReplayVectorEnv(sims_a), ReplayVectorEnv(sims_b)
        actions = np.random.default_rng(5).choice([1, 1, 2, 3], size=(50, 4))
        hits = silent = 0
        obs_a, obs_b = env_a.observe(), env_b.observe()
        for step in range(51):
            descs = pickle.loads(pickle.dumps([o["spectrogram"] for o in obs_b]))
            if step == 25:
                assert not descs[0].hit and descs[0].generation == 1
            f0, r0, n_a = svc.batcher.flushes, len(svc.renderer.renders), len(local.renderer.renders)
            got_a = batch_obs(obs_a)["spectrogram"]
            got_b = batch_obs([{"spectrogram": d} for d in descs])["spectrogram"]
            fresh = sum(not d.hit for d in descs)
            hits += len(descs) - fresh
            silent += sum(d.silent for d in descs)
            assert svc.batcher.flushes - f0 == (1 if fresh else 0)
            assert len(svc.renderer.renders) - r0 == len(local.renderer.renders) - n_a
            if fresh:
                assert len(svc.renderer.renders[-1]) == fresh
                assert [request_view(svc, q) for q in svc.renderer.renders[-1]] == \
                    [request_view(local, q) for q in local.renderer.renders[-1]]
            assert svc.rir_log == local.rir_log and svc.prefetch_log == local.prefetch_log
            assert [s._audio_index for s in sims_a] == [s._audio_index for s in sims_b]
            assert torch.equal(got_a, got_b)
            if step == 24:                                   # env 0 moves to the other scene at the same node indices
                for s in (sims_a[0], sims_b[0]):
                    s.reconfigure(scenes[1], "bell.wav", s.current_source_sound, 3, s._receiver_position_index,
                                  s._rotation_angle)
            if step < 50:
                obs_a, obs_b = env_a.step(actions[step]), env_b.step(actions[step])
        assert hits > 20 and silent > 0
        assert any(k[0].endswith("office_3") and k[3] == 1 for k in svc.rir_log)           # the distractor
        assert any(svc.renderer._rir_len[i] == 0 for i in svc._rir_ids.values())         # missing / empty files
        assert {g for g, _ in svc.remote._memo.values()} == {0, 1}                        # env 0's old scene dropped


def test_waveform_descriptors_one_convolve_and_memo(tmp_path):
    root = str(tmp_path)
    wav_tree(root)
    with trainer_service() as svc:
        sims, _ = make_sims(None, root, "remote")
        env = ReplayVectorEnv(sims[:3], audiogoal=True)
        obs = pickle.loads(pickle.dumps(env.observe()))
        batch = batch_obs(obs)
        assert batch["audiogoal"].shape == (3, 2, SR) and len(svc.renderer.convolves) == 1
        assert len(svc.renderer.convolves[0]) == 3 and svc.batcher.flushes == 1
        again = pickle.loads(pickle.dumps(env.observe()))
        assert all(o["audiogoal"].hit for o in again[:2]) and not again[2]["audiogoal"].hit    # 2: distractor, no memo
        b2 = batch_obs(again)
        assert len(svc.renderer.convolves) == 2 and len(svc.renderer.convolves[1]) == 1
        assert torch.equal(b2["audiogoal"][:2], batch["audiogoal"][:2])


def test_intensity_refuses_remote_mode(tmp_path):
    from remote_envs import continuous_sim
    sims, _ = make_sims(None, str(tmp_path), "remote")
    for sim in (sims[0], continuous_sim(SR, make_source(0, SR), 0, True)):
        with pytest.raises(RuntimeError, match="in-process envs") as e:
            Intensity(sim=sim, config=None).get_observation()
        assert str(e.value) == INTENSITY_REMOTE_ERROR
    assert not torch.cuda.is_initialized()


def test_clip_samples_travel_with_the_first_pickled_observation(tmp_path):
    """A descriptor built but never sent (the terminal step an auto-resetting vector env drops) does not count as
    having shipped its clip."""
    root = str(tmp_path)
    wav_tree(root)
    clip = make_source(11, SR)
    sim = ReplaySim(None, ReplayScene("apartment_0", 2, rir_root=root), "fresh.wav", clip, 3, 0, 0, deferred="remote",
                    sr=SR)
    dropped = sim.get_current_spectrogram_observation(_native())
    assert dropped.clip.samples is not None
    sim.step(2)
    sent = pickle.loads(pickle.dumps(sim.get_current_spectrogram_observation(_native())))
    assert sent.clip.samples is not None and np.array_equal(sent.clip.samples, clip)
    again = pickle.loads(pickle.dumps(sim.get_current_spectrogram_observation(_native())))
    assert again.hit and again.clip.samples is None


def test_auto_reset_drops_terminal_observations_and_revisits_render(tmp_path):
    """Workers that auto-reset (auto_reset_done=True in the trainers' vector envs) build the terminal step's
    observation, memoise it and drop it unsent.  A later episode that revisits the pose sends a memo reference whose
    original the trainer never saw: it is rendered from the keys it carries, as in-process deferred mode rendered the
    dropped handle."""
    root = str(tmp_path)
    wav_tree(root)
    clips = [make_source(0, SR), make_source(1, 3 * SR)]
    args = [(SR, "apartment_0", 2, root, f"c{e}.wav", clips[e % 2], 3, e, 90 * e) for e in range(3)]
    actions = np.random.default_rng(9).choice([1, 2, 3], size=(40, 3))
    local = AudioRenderService(SR, renderer=StubRenderer(SR), prefetch_workers=0)
    sims = [ReplaySim(local, ReplayScene("apartment_0", 2, rir_root=root), *a[4:9], deferred=True) for a in args]
    in_process = ReplayVectorEnv(sims, episode_steps=4)

    def rows(service, t):                                     # stub rows -> (RIR key, offset in seconds)
        inv = {v: k for k, v in service._rir_ids.items()}
        return [(inv[int(v) // 1000], int(v) % 1000) for v in t[:, 0, 0, 0].tolist()]

    with trainer_service() as svc:
        for s in (svc, local):
            s.renderer.add_rirs([None])                       # bank id 0 unused: a row value names its RIR
        with ProcessReplayVectorEnv(replay_sim, args, start_method="spawn", episode_steps=4) as envs:
            got = batch_obs(envs.observe())["spectrogram"]
            want = batch_obs(in_process.observe())["spectrogram"]
            assert rows(svc, got) == rows(local, want)
            for a in actions:
                got = batch_obs(envs.step(a))["spectrogram"]
                want = batch_obs(in_process.step(a))["spectrogram"]
                assert rows(svc, got) == rows(local, want)
        assert svc.remote.unseen_hits > 0


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the refusal in a process without CUDA")
def test_asarray_without_cuda_is_a_clear_error():
    d = RemoteAudioRequest(service=(8000, "cuda:0", "reflect"), silent=True)
    with pytest.raises(RuntimeError, match="no CUDA device"):
        np.asarray(d)


@pytest.mark.parametrize("start_method", ["forkserver", "spawn"])
def test_workers_never_touch_cuda_and_are_joined(tmp_path, start_method):
    root = str(tmp_path)
    wav_tree(root)
    clip = make_source(0, SR)
    args = [(SR, "apartment_0", 2, root, "bell.wav", clip, 3, i, 90 * i) for i in range(3)]
    with trainer_service() as svc:
        envs = ProcessReplayVectorEnv(replay_sim, args, start_method=start_method)
        procs = envs.processes
        with envs:
            assert len({p.pid for p in procs}) == 3 and os.getpid() not in {p.pid for p in procs}
            obs = envs.observe()
            assert all(isinstance(o["spectrogram"], RemoteAudioRequest) for o in obs)
            batch_obs(obs)
            for a in (2, 1, 3):
                obs = envs.step([a] * 3)
                batch_obs(obs)
            assert svc.batcher.flushes == 4 and envs.bytes_received > 0
            for report in envs.call(worker_report):
                assert report["cuda_initialized"] is False and report["libssb200_loaded"] is False
        assert all(p.exitcode is not None and not p.is_alive() for p in procs)


def _native():
    from soundspaces_b200.sensors import SpectrogramSensor
    return SpectrogramSensor.compute_spectrogram
