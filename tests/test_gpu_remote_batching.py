"""Remote deferred mode on the GPU: 16 envs in worker processes hand request descriptors to the trainer, whose
``batch_obs`` renders each step once.  The result must be bit-identical to in-process deferred mode on the same wav
trees and actions, within the suite's tolerance of the oracle, and the workers must never create a CUDA context."""
import numpy as np
import pytest
import torch

from oracle import audio_oracle as ao
from oracle.ref_harness import write_rir
from remote_envs import continuous_sim
from synth import make_rir, make_source

from soundspaces_b200.replay import (ProcessReplayVectorEnv, ReplayScene, ReplaySim, ReplayVectorEnv, replay_sim,
                                     worker_report)
from soundspaces_b200.sensors import batch_obs
from soundspaces_b200.simulator import AudioRenderService

pytestmark = pytest.mark.gpu

SR, N_ENVS, STEPS, SIDE = 16000, 16, 50, 3
AZ = (0, 90, 180, 270)


def _check_workers(envs):
    for report in envs.call(worker_report):
        assert report["cuda_initialized"] is False and report["libssb200_loaded"] is False


@pytest.mark.parametrize("episode_steps", [None, 12])
def test_discrete_remote_equals_in_process_and_oracle(tmp_path, episode_steps):
    """``episode_steps``: workers auto-reset, dropping each terminal step's observation; revisits of those poses
    reach the trainer as memo references it has never seen."""
    root = str(tmp_path)
    rirs = {(az, n): make_rir(50 * ai + n, 2000 + 150 * n) for ai, az in enumerate(AZ) for n in range(SIDE * SIDE)}
    for (az, n), rir in rirs.items():
        write_rir(root, "replica", "scene", az, n, 0, SR, rir)
    clips = [make_source(0, SR), make_source(1, 2 * SR)]
    args = [(SR, "scene", SIDE, root, f"s{e % 2}.wav", clips[e % 2], 0, e % (SIDE * SIDE), 90 * (e % 4), "remote", 30)
            for e in range(N_ENVS)]
    actions = np.random.default_rng(3).choice([1, 1, 2, 3], size=(STEPS, N_ENVS))
    svc = AudioRenderService.get(SR, "cuda:0")
    shape = svc.renderer.spec_shape
    storage = torch.full((STEPS + 1, N_ENVS) + shape, -1.0, device="cuda")
    waves = torch.empty((STEPS + 1, N_ENVS, 2, SR), device="cuda")

    unseen = svc.remote.unseen_hits
    with ProcessReplayVectorEnv(replay_sim, args, audiogoal=True, episode_steps=episode_steps) as envs:
        _check_workers(envs)
        obs = envs.observe()
        for step in range(STEPS + 1):
            f0, n0 = svc.batcher.flushes, svc.batcher._next
            fresh = sum(not o["spectrogram"].hit for o in obs)
            b = batch_obs(obs, device=torch.device("cuda"), out={"spectrogram": storage[step]})
            assert b["spectrogram"].data_ptr() == storage[step].data_ptr()          # landed in the rollout slot
            assert svc.batcher.flushes - f0 == (1 if fresh else 0) or svc.batcher._next < n0
            waves[step] = b["audiogoal"]
            if step < STEPS:
                obs = envs.step(actions[step])
        _check_workers(envs)
    assert (svc.remote.unseen_hits > unseen) == bool(episode_steps)

    # in-process deferred mode on the same trees and actions, through the same trainer service
    sims = [ReplaySim(svc, ReplayScene("scene", SIDE, rir_root=root), a[4], a[5], 0, a[7], a[8], deferred=True,
                      duration=30) for a in args]
    env = ReplayVectorEnv(sims, audiogoal=True, episode_steps=episode_steps)
    ref = torch.full_like(storage, -2.0)
    obs = env.observe()
    state = []
    for step in range(STEPS + 1):
        b = batch_obs(obs, device=torch.device("cuda"), out={"spectrogram": ref[step]})
        assert torch.equal(waves[step].cpu(), b["audiogoal"].cpu()), step
        state.append([(s._receiver_position_index, s.azimuth_angle, s._episode_step_count > s._duration) for s in sims])
        if step < STEPS:
            obs = env.step(actions[step])
    got, want = storage.cpu().numpy(), ref.cpu().numpy()
    assert np.array_equal(got, want)

    # the oracle, for the 1-s clip envs (offset 0): a row is the RIR at the env's node / heading, or an exact zero
    # when the step was a memo miss after DURATION
    silent_rows = 0
    for step in range(STEPS + 1):
        for e in range(0, N_ENVS, 2):
            recv, az, past = state[step][e]
            if past and not np.any(got[step, e]):
                silent_rows += 1
                continue
            oracle = ao.compute_spectrogram(ao.compute_audiogoal(clips[0], rirs[(az, recv)], SR).astype(np.float32))
            assert np.allclose(got[step, e], oracle, rtol=1e-4, atol=1e-5), (step, e)
    assert silent_rows > 0 or episode_steps                 # auto-reset episodes never reach DURATION


@pytest.mark.parametrize("crossfade", [False, True])
def test_continuous_remote_equals_in_process(crossfade):
    clip = make_source(7, SR)
    args = [(SR, clip, e, crossfade) for e in range(N_ENVS)]
    svc = AudioRenderService.get(SR, "cuda:0")
    shape = svc.renderer.spec_shape
    storage = torch.full((STEPS + 1, N_ENVS) + shape, -1.0, device="cuda")
    waves = torch.empty((STEPS + 1, N_ENVS, 2, SR), device="cuda")
    wrapped = 0
    with ProcessReplayVectorEnv(continuous_sim, args, start_method="spawn", audiogoal=True) as envs:
        obs = envs.observe()
        for step in range(STEPS + 1):
            wrapped += sum(o["spectrogram"].wrap and o["spectrogram"].offset + int(0.3 * SR) > SR for o in obs)
            f0, n0 = svc.batcher.flushes, svc.batcher._next
            b = batch_obs(obs, device=torch.device("cuda"), out={"spectrogram": storage[step]})
            # one flush, or two when the step's rows would have crossed the end of the ring (wrapped to slot 0)
            assert svc.batcher.flushes - f0 == 1 or svc.batcher._next < n0
            waves[step] = b["audiogoal"]
            if step < STEPS:
                obs = envs.step([1] * N_ENVS)
        _check_workers(envs)
    assert wrapped > 0

    sims = [continuous_sim(*a, deferred=True) for a in args]
    env = ReplayVectorEnv(sims, audiogoal=True)
    ref = torch.full_like(storage, -2.0)
    obs = env.observe()
    for step in range(STEPS + 1):
        batch_obs(obs, device=torch.device("cuda"), out={"spectrogram": ref[step]})
        want = np.stack([np.asarray(o["audiogoal"], dtype=np.float32) for o in obs])
        assert np.array_equal(waves[step].cpu().numpy(), want), step
        if step < STEPS:
            obs = env.step([1] * N_ENVS)
    got = storage.cpu().numpy()
    assert np.array_equal(got, ref.cpu().numpy())
    assert not np.any(got[-1]) and np.all(np.any(got[1].reshape(N_ENVS, -1), axis=1))   # silent after DURATION


def test_asarray_of_a_descriptor_in_the_trainer(tmp_path):
    root = str(tmp_path)
    rir = make_rir(9, 3000)
    for az in AZ:
        for n in range(4):
            write_rir(root, "replica", "scene", az, n, 0, SR, rir)
    clip = make_source(4, SR)
    with ProcessReplayVectorEnv(replay_sim, [(SR, "scene", 2, root, "c.wav", clip, 0, 1, 0)], audiogoal=True) as envs:
        obs = envs.observe()[0]
        spec, wave = np.asarray(obs["spectrogram"]), np.asarray(obs["audiogoal"])
    w_ref = ao.compute_audiogoal(clip, rir, SR)
    assert spec.shape == AudioRenderService.get(SR, "cuda:0").renderer.spec_shape and wave.shape == (2, SR)
    assert np.abs(wave - w_ref).max() <= 1e-4 * np.abs(w_ref).max()
    assert np.allclose(spec, ao.compute_spectrogram(w_ref.astype(np.float32)), rtol=1e-4, atol=1e-5)
