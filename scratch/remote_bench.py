"""Env-steps/s of a 16-env rollout on the trace-replay env (``soundspaces_b200.replay``) at 16 and 44.1 kHz, in three
process topologies, alternated in one run:
  remote      envs in worker processes (``ProcessReplayVectorEnv``, forkserver) in remote deferred mode: workers pickle
              request descriptors, the trainer renders each step once in ``batch_obs``
  compat-mp   the same workers in compat mode: one CUDA context per worker, host spectrograms pickled back
              (today's behaviour of habitat.VectorEnv with the patched simulators)
  inproc      in-process deferred mode (``ReplayVectorEnv``, one process)
The RIRs are a seeded wav tree (3 x 3 grid, 4 headings, 1-s RIRs) read by the services; the clips are 1 s (half the
envs) and 3 s.  Each mode runs --warmup steps, then --steps timed steps (host clock ending in a device synchronise)
with a fixed random action trace, the policy's first layer consuming every observation from the rollout slot.
Reports env-steps/s, the bytes pickled per step, the card name and power limit, and one JSON line.

    python scratch/remote_bench.py [--steps 200] [--warmup 20] [--reps 2]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

sys.path.insert(0, os.getcwd())
import numpy as np  # noqa: E402
import torch  # noqa: E402
from scipy.io import wavfile  # noqa: E402

from soundspaces_b200.replay import (AudioPolicy, ProcessReplayVectorEnv, ReplayScene, ReplaySim,  # noqa: E402
                                     ReplayVectorEnv, collect_rollout, replay_sim)
from soundspaces_b200.simulator import AudioRenderService  # noqa: E402

N_ENVS, SIDE = 16, 3


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name(0)


def wav_tree(root, sr, rng):
    for az in (0, 90, 180, 270):
        d = os.path.join(root, "replica", "scene", str(az))
        os.makedirs(d, exist_ok=True)
        for n in range(SIDE * SIDE):
            r = rng.standard_normal((sr, 2)) * np.exp(-np.arange(sr) / (sr / 8.0))[:, None]
            wavfile.write(os.path.join(d, f"{n}_0.wav"), sr, (0.5 * r / np.abs(r).max()).astype(np.float32))


def env_args(sr, root, mode, clips):
    return [(sr, "scene", SIDE, root, f"c{e % 2}.wav", clips[e % 2], 0, e % (SIDE * SIDE), 90 * (e % 4),
             "remote" if mode == "remote" else False, 10 ** 6) for e in range(N_ENVS)]


def run(mode, sr, root, clips, trace, warmup):
    svc = AudioRenderService.get(sr, "cuda:0")
    policy = AudioPolicy(svc.renderer.spec_shape).cuda()
    steps = trace.shape[0] - warmup
    storage = torch.zeros((trace.shape[0] + 1, N_ENVS) + svc.renderer.spec_shape, device="cuda")
    args = env_args(sr, root, mode, clips)
    if mode == "inproc":
        envs = ReplayVectorEnv([ReplaySim(svc, ReplayScene("scene", SIDE, rir_root=root), *a[4:9], deferred=True,
                                          duration=a[10]) for a in args])
    else:
        envs = ProcessReplayVectorEnv(replay_sim, args)
    try:
        collect_rollout(envs, policy, storage[: warmup + 1], warmup, trace[:warmup])
        b0 = getattr(envs, "bytes_received", 0)
        t0 = time.perf_counter()
        collect_rollout(envs, policy, storage[warmup:], steps, trace[warmup:])
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        pickled = (getattr(envs, "bytes_received", 0) - b0) / (steps + 1)
    finally:
        if mode != "inproc":
            envs.close()
    return steps * N_ENVS / dt, pickled


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--reps", type=int, default=2)
    a = ap.parse_args()
    print("card:", card())
    rng = np.random.default_rng(0)
    out = {"card": card(), "envs": N_ENVS, "steps": a.steps, "results": {}}
    with tempfile.TemporaryDirectory() as tmp:
        for sr in (16000, 44100):
            root = os.path.join(tmp, str(sr))
            wav_tree(root, sr, rng)
            clips = [(0.1 * rng.standard_normal(sr)).astype(np.float32),
                     (0.1 * rng.standard_normal(3 * sr)).astype(np.float32)]
            trace = rng.choice([1, 1, 2, 3], size=(a.warmup + a.steps, N_ENVS))
            res = {m: [] for m in ("remote", "compat-mp", "inproc")}
            for rep in range(a.reps):
                for m in res:
                    rate, pickled = run(m, sr, root, clips, trace, a.warmup)
                    res[m].append((rate, pickled))
                    print(f"sr={sr} rep={rep} {m:10s} {rate:9.1f} env-steps/s  {pickled / 1024:9.1f} KiB pickled/step",
                          flush=True)
            out["results"][sr] = {m: {"env_steps_per_s": [round(r, 1) for r, _ in v],
                                      "bytes_pickled_per_step": round(float(np.mean([p for _, p in v])))}
                                  for m, v in res.items()}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
