"""Per-step cost of AV-WaN's map observations, reference path against the record path (soundspaces_b200.maps).

Reference path: each env's worker crops gm / am / action_map from its float64 maps (the numpy stand-in does what
Mapper's getters do: rot90 view, crop, astype(float32)), pickles and unpickles them, then batch_obs stacks them and
copies them to the device.  Record path: the worker logs the step's record, pickles and unpickles the descriptors,
then one update and one crop launch.  Host timings include a device synchronise; kernel times come from CUDA events.
Prints the card and its power limit with the results.

    python scratch/map_obs_bench.py [--steps 20]
"""
import argparse
import os
import pickle
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
from mapper_models import StandInPlanner, drive, task_config  # noqa: E402
from soundspaces_b200 import maps  # noqa: E402
from soundspaces_b200.sensors import batch_obs  # noqa: E402

KINDS = ("gm", "am", "action_map")


def envs(B, config, patched):
    class P(StandInPlanner):
        pass
    if patched:
        maps.patch_planner(P)
    ps = [P(task_config=task_config(config, "average_intensity"), use_acoustic_map=True) for _ in range(B)]
    gens = [drive(p, 1000 + i, 10 ** 6) for i, p in enumerate(ps)]
    return gens


def run(B, config, patched, steps, warmup):
    gens = envs(B, config, patched)
    dev = torch.device("cuda", 0)
    times = []
    for s in range(warmup + steps):
        t0 = time.perf_counter()
        obs = [pickle.loads(pickle.dumps({k: o[k] for k in KINDS})) for o in (next(g) for g in gens)]
        batch = batch_obs(obs, device=dev)
        torch.cuda.synchronize()
        if s >= warmup:
            times.append(time.perf_counter() - t0)
    return float(np.median(times)) * 1e3, batch


def kernel_ms(B, config, reps=50):
    gens = envs(B, config, True)
    obs = [next(g) for g in gens]
    dm = maps.DeviceMaps.get("cuda:0", obs[0]["gm"].geometry)
    batch_obs(obs, device=torch.device("cuda", 0))
    descs = {k: [o[k] for o in obs] for k in KINDS}
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        dm.observe(descs["gm"], KINDS)
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print("card:", card)
    print("config  B  reference_ms  record_ms  crop_kernel_ms")
    for config in ("avwan", "mp3d"):
        for B in (1, 16, 64, 128):
            ref_ms, rb = run(B, config, False, args.steps, args.warmup)
            rec_ms, _ = run(B, config, True, args.steps, args.warmup)
            print(f"{config:6s} {B:4d} {ref_ms:12.2f} {rec_ms:10.2f} {kernel_ms(B, config):14.3f}", flush=True)


if __name__ == "__main__":
    main()
