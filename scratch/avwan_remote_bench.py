"""High-level env-steps/s of AV-WaN's MapNav loop (tests/avwan_remote_envs.py: up to PREDICTION_INTERVAL = 10
low-level steps per step, Intensity sensor, acoustic map on, MAP_SIZE 200) with 5 and 16 envs at 16 and 44.1 kHz, in
three topologies:
  remote     worker processes (forkserver) in remote deferred mode with remote_intensity: workers send waveform
             requests in the map records, the trainer renders, reduces and applies them in batch_obs
  compat-mp  the same workers in compat mode: one CUDA context per worker, one waveform rendered and reduced per
             low-level step there, float intensities in the records
  inproc     in-process deferred mode (one process)
Each mode runs --warmup steps, then --steps timed steps (host clock ending in a device synchronise).  Also reported,
for the remote mode: the trainer's batch_obs time per step split into render, intensity, map update and crop (CUDA
events around each call, from a separate pass), and the bytes pickled per step.  The card name and power limit are
read in the same run.  Every worker process is joined before the script exits.

    python scratch/avwan_remote_bench.py [--steps 30] [--warmup 5]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

sys.path[:0] = [os.getcwd(), os.path.join(os.getcwd(), "tests")]
import numpy as np  # noqa: E402
import torch  # noqa: E402
from scipy.io import wavfile  # noqa: E402

from avwan_remote_envs import MapNavReplayEnv, ProcessMapNavEnvs  # noqa: E402
from soundspaces_b200.renderer import WaveformOps  # noqa: E402
from soundspaces_b200.sensors import batch_obs  # noqa: E402
from soundspaces_b200.simulator import AudioRenderService  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name(0)


def wav_tree(root, sr, rng):
    for az in (0, 90, 180, 270):
        d = os.path.join(root, "replica", "scene", str(az))
        os.makedirs(d, exist_ok=True)
        for n in range(9):
            r = rng.standard_normal((sr, 2)) * np.exp(-np.arange(sr) / (sr / 8.0))[:, None]
            wavfile.write(os.path.join(d, f"{n}_0.wav"), sr, (0.5 * r / np.abs(r).max()).astype(np.float32))


class InProcess:
    def __init__(self, args):
        self.envs = [MapNavReplayEnv(*a, **k) for a, k in args]

    def reset(self):
        return [e.reset() for e in self.envs]

    def step(self):
        return [e.step() for e in self.envs]

    def close(self):
        pass


class Timers:
    """CUDA event pairs around the renderer's and the maps' calls inside batch_obs."""

    def __init__(self, svc):
        self.ms, self.patched = {}, []
        r, ops = svc.renderer, WaveformOps.get("cuda:0")
        for obj, name, label in ((r, "convolve", "render"), (r, "render_crossfade", "render"),
                                 (r, "intensity", "intensity"), (ops, "map_update_device_intensity", "update"),
                                 (ops, "map_update", "update"), (ops, "map_observe", "crop")):
            setattr(obj, name, self._wrap(getattr(obj, name), label))
            self.patched.append((obj, name))
        self.pending = []

    def close(self):
        for obj, name in self.patched:
            delattr(obj, name)                                  # back to the class's method

    def _wrap(self, fn, label):
        def timed(*a, **k):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            out = fn(*a, **k)
            e1.record()
            self.pending.append((label, e0, e1))
            return out
        return timed

    def collect(self):
        torch.cuda.synchronize()
        for label, e0, e1 in self.pending:
            self.ms[label] = self.ms.get(label, 0.0) + e0.elapsed_time(e1)
        self.pending = []


def run(mode, n_envs, sr, root, clips, steps, warmup, timers=None):
    svc = AudioRenderService.get(sr, "cuda:0")
    deferred = {"remote": "remote", "compat-mp": False, "inproc": True}[mode]
    args = [(("discrete", sr, root, clips[e % 2], e, deferred),
             dict(encoding="average_intensity", service=svc if mode == "inproc" else None)) for e in range(n_envs)]
    envs = InProcess(args) if mode == "inproc" else ProcessMapNavEnvs(args)
    try:
        obs = envs.reset()
        batch_obs(obs, device=torch.device("cuda"))
        for _ in range(warmup):
            batch_obs(envs.step(), device=torch.device("cuda"))
        torch.cuda.synchronize()
        if timers is not None:
            timers.pending = []                                 # warm-up calls are not part of the split
        b0 = getattr(envs, "bytes_received", 0)
        t_obs = 0.0
        t0 = time.perf_counter()
        for _ in range(steps):
            obs = envs.step()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            batch_obs(obs, device=torch.device("cuda"))
            e1.record()
            if timers is not None:
                timers.collect()
            e1.synchronize()
            t_obs += e0.elapsed_time(e1)
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        pickled = (getattr(envs, "bytes_received", 0) - b0) / steps
    finally:
        envs.close()
    return {"env_steps_per_s": steps * n_envs / dt, "batch_obs_ms_per_step": t_obs / steps,
            "bytes_pickled_per_step": pickled}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    a = ap.parse_args()
    torch.cuda.init()
    result = {"card": card(), "runs": []}
    print("card:", result["card"])
    rng = np.random.default_rng(0)
    with tempfile.TemporaryDirectory() as root:
        for sr in (16000, 44100):
            wav_tree(os.path.join(root, str(sr)), sr, rng)
            clips = [rng.standard_normal(sr).astype(np.float32) * 0.1,
                     rng.standard_normal(3 * sr).astype(np.float32) * 0.1]
            for n_envs in (5, 16):
                for mode in ("remote", "compat-mp", "inproc"):
                    r = run(mode, n_envs, sr, os.path.join(root, str(sr)), clips, a.steps, a.warmup)
                    r.update(mode=mode, envs=n_envs, sr=sr)
                    result["runs"].append(r)
                    print(json.dumps(r), flush=True)
                timers = Timers(AudioRenderService.get(sr, "cuda:0"))     # split pass, remote mode
                try:
                    run("remote", n_envs, sr, os.path.join(root, str(sr)), clips, a.steps, a.warmup, timers)
                finally:
                    timers.close()
                split = {k: v / a.steps for k, v in timers.ms.items()}
                result["runs"].append({"mode": "remote-split", "envs": n_envs, "sr": sr, "ms_per_step": split})
                print(json.dumps(result["runs"][-1]), flush=True)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
