"""Env-steps/s of a 16-env rollout on the trace-replay env in remote deferred mode with 128 x 128 RGB-D observations,
with and without ``remote_frames``, alternated in one run:
  frames      workers send each rendered frame once, then its key; batch_obs gathers the step's RGB and depth from the
              device frame banks in one launch
  plain       workers pickle every step's rgb (uint8) and depth (float32) arrays; batch_obs stacks them on the host and
              copies them to the device (the reference's path)
Both modes run forkserver workers (``ProcessReplayVectorEnv``) on one seeded scene (a 3 x 3 grid, 4 headings, a
synthetic scene-observation pickle; the warm-up lets every worker send most of its 36 poses) with 1-s RIRs and 1-s
clips; every step's spectrogram, rgb and depth land in rollout slots.  Each mode runs --warmup steps, then --steps timed steps (host clock ending in a device synchronise) on
a fixed random action trace.  Also reports the bytes pickled per env and step over the timed steps, and the gather
kernel's device time (torch.profiler) for one 16-env RGB-D step served from the bank.  Prints the card name and
power limit and one JSON line.

    python scratch/frames_bench.py [--steps 400] [--warmup 400] [--reps 2]
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

from soundspaces_b200 import frames as fr  # noqa: E402
from soundspaces_b200.remote import FrameRef  # noqa: E402
from soundspaces_b200.replay import (ProcessReplayVectorEnv, replay_sim, scene_observations,  # noqa: E402
                                     write_scene_observations)
from soundspaces_b200.sensors import batch_obs  # noqa: E402
from soundspaces_b200.simulator import AudioRenderService  # noqa: E402

N_ENVS, SIDE, SR, H, W = 16, 3, 16000, 128, 128


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name(0)


def wav_tree(root, rng):
    for az in (0, 90, 180, 270):
        d = os.path.join(root, "replica", "scene", str(az))
        os.makedirs(d, exist_ok=True)
        for n in range(SIDE * SIDE):
            r = rng.standard_normal((SR, 2)) * np.exp(-np.arange(SR) / (SR / 8.0))[:, None]
            wavfile.write(os.path.join(d, f"{n}_0.wav"), SR, (0.5 * r / np.abs(r).max()).astype(np.float32))


def run(mode, root, path, clip, trace, warmup):
    svc = AudioRenderService.get(SR, "cuda:0")
    total = trace.shape[0]
    slots = {"spectrogram": torch.zeros((total + 1, N_ENVS) + svc.renderer.spec_shape, device="cuda"),
             "rgb": torch.zeros((total + 1, N_ENVS, H, W, 3), device="cuda"),
             "depth": torch.zeros((total + 1, N_ENVS, H, W, 1), device="cuda")}
    args = [(SR, "scene", SIDE, root, "c.wav", clip, 0, e % (SIDE * SIDE), 90 * (e % 4), "remote", 10 ** 6, path,
             mode == "frames") for e in range(N_ENVS)]
    with ProcessReplayVectorEnv(replay_sim, args) as envs:
        obs = envs.observe()
        batch_obs(obs, device=torch.device("cuda"), out={k: v[0] for k, v in slots.items()})
        t0, b0 = None, 0
        for step in range(total):
            if step == warmup:
                torch.cuda.synchronize()
                t0, b0 = time.perf_counter(), envs.bytes_received
            obs = envs.step(trace[step])
            batch_obs(obs, device=torch.device("cuda"), out={k: v[step + 1] for k, v in slots.items()})
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        per_env_step = (envs.bytes_received - b0) / ((total - warmup) * N_ENVS)
    assert mode != "frames" or isinstance(obs[0]["rgb"], FrameRef)
    return (total - warmup) * N_ENVS / dt, per_env_step, slots


def gather_time(path, iters=2000):
    """One 16-env RGB and depth gather from resident banks (no misses): CUDA-event time per ``frames.gather`` call and
    per back-to-back launch, and the kernel's device time."""
    import pickle
    from soundspaces_b200.remote import FrameArray
    from soundspaces_b200.replay import visual_observations
    with open(path, "rb") as f:
        cache = pickle.load(f)
    poses = list(cache)[:N_ENVS]
    refs = {u: [pickle.loads(pickle.dumps(FrameArray(visual_observations(cache[p])[u], ("bench",) + p + (u,))))
                for p in poses] for u in ("rgb", "depth")}
    out = {"rgb": torch.empty((N_ENVS, H, W, 3), device="cuda"), "depth": torch.empty((N_ENVS, H, W, 1), device="cuda")}
    for _ in range(20):
        fr.gather(refs, torch.device("cuda:0"), out=out)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(iters):
        fr.gather(refs, torch.device("cuda:0"), out=out)
    b.record()
    torch.cuda.synchronize()
    per_call_us = a.elapsed_time(b) * 1e3 / iters
    # the kernel alone: the same launch through the ops wrapper, host planning excluded
    from soundspaces_b200.renderer import WaveformOps
    ops = WaveformOps.get("cuda:0")
    jobs = []
    for u, t in (("rgb", out["rgb"]), ("depth", out["depth"])):
        store = fr.FrameStore.get("cuda:0", u, refs[u][0].dtype, refs[u][0].shape)
        jobs.append((store.bank, None, t.view(N_ENVS, -1), [store._rows[r.key] for r in refs[u]], []))
    a.record()
    for _ in range(iters):
        ops.frame_gather(N_ENVS, jobs)
    b.record()
    torch.cuda.synchronize()
    launch_us = a.elapsed_time(b) * 1e3 / iters                 # back to back: bounded by the host's submit rate
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(200):
            ops.frame_gather(N_ENVS, jobs)
        torch.cuda.synchronize()
    ev = [e for e in prof.key_averages() if "frame_gather_kernel" in e.key][0]
    kernel_us = getattr(ev, "device_time_total", None) or ev.cuda_time_total
    kernel_us /= ev.count
    bytes_moved = N_ENVS * H * W * (3 + 3 * 4 + 4 + 4)        # uint8 read + float32 write, float32 read + write
    return per_call_us, launch_us, kernel_us, bytes_moved


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=400)
    ap.add_argument("--warmup", type=int, default=400)
    ap.add_argument("--reps", type=int, default=2)
    a = ap.parse_args()
    name = card()
    print("card:", name)
    rng = np.random.default_rng(0)
    out = {"card": name, "envs": N_ENVS, "frame": [H, W], "steps": a.steps, "results": {}}
    with tempfile.TemporaryDirectory() as tmp:
        wav_tree(tmp, rng)
        path = write_scene_observations(os.path.join(tmp, "obs", "replica", "scene.pkl"),
                                        scene_observations(SIDE * SIDE, H, W, seed=1))
        clip = (0.1 * rng.standard_normal(SR)).astype(np.float32)
        trace = rng.choice([1, 1, 2, 3], size=(a.warmup + a.steps, N_ENVS))
        res = {m: [] for m in ("frames", "plain")}
        last = {}
        for rep in range(a.reps):
            for m in res:
                rate, per_env, slots = run(m, tmp, path, clip, trace, a.warmup)
                res[m].append((rate, per_env))
                last[m] = slots
                print(f"rep={rep} {m:7s} {rate:9.1f} env-steps/s  {per_env / 1024:9.2f} KiB pickled per env-step",
                      flush=True)
        for k in ("rgb", "depth", "spectrogram"):
            assert torch.equal(last["frames"][k], last["plain"][k]), k
        per_call_us, launch_us, kernel_us, moved = gather_time(path)
        print(f"gather: {per_call_us:.1f} us per frames.gather call, {launch_us:.1f} us per back-to-back launch, "
              f"kernel {kernel_us:.2f} us ({moved / kernel_us / 1e3:.0f} GB/s of {moved / 1e6:.2f} MB)")
        out["results"] = {m: {"env_steps_per_s": [round(r, 1) for r, _ in v],
                              "bytes_pickled_per_env_step": round(float(np.mean([p for _, p in v])))}
                          for m, v in res.items()}
        out["gather_us_per_call"] = round(per_call_us, 2)
        out["gather_launch_us"] = round(launch_us, 2)
        out["gather_kernel_us"] = round(kernel_us, 2)
        out["identical_rollout_slots"] = True
    print(json.dumps(out))


if __name__ == "__main__":
    main()
