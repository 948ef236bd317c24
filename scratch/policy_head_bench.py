"""The policies' action and value heads (everything in ``Policy.act`` after ``self.net``), eager PyTorch against
``soundspaces_b200.policy.fused_head``, alternated in one process, at B in {16, 128, 512} for the three trainers'
shapes: AV-Nav H = 512, A = 4; SAVi H = 128, A = 4; AV-WaN H = 512, A = 81 with the action-map mask.  Both sides
sample (``deterministic=False``), the eager side with torch's default ``Distribution`` validation.

    python scratch/policy_head_bench.py

Per call: host time (perf_counter around 200 calls; each call ends in its own host sync on both sides, so this is
the time a rollout step spends on the head), wall time on the stream (CUDA events around each of those calls,
averaged), kernel launches and summed kernel time (device kernels ``torch.profiler`` records over 20 calls in a run of
their own, memcpy / memset counted apart) and host syncs (``torch.cuda.set_sync_debug_mode("warn")`` warnings, after
a warm-up call).  Prints the card's name and power limit and one JSON line per
case."""
import json
import os
import subprocess
import sys
import time
import warnings

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

import policy_head_models as phm  # noqa: E402
from soundspaces_b200 import policy as ph  # noqa: E402

CALLS, ROUNDS, PROF_CALLS = 200, 3, 20
DEV = torch.device("cuda", 0)
CASES = {"av_nav": ("av_nav", None), "savi": ("savi", None), "av_wan": ("av_wan", True)}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name(0)


def setup(name, N):
    trainer, masking = CASES[name]
    H, A = phm.SHAPES[trainer]
    policy = phm.make_policy(trainer, H, A, seed=1, gain=0.01, masking=bool(masking)).to(DEV).eval()
    features = torch.tanh(torch.randn((N, H), device=DEV))
    obs = {"action_map": phm.action_map(N, A, 1).to(DEV)} if trainer == "av_wan" else {}
    return policy, features, obs


def runners(policy, features, obs):
    return {"eager": lambda: policy._head(features, obs, False),
            "fused": lambda: ph.fused_head(policy, features, obs, False)}


def timed(fn):
    starts = [torch.cuda.Event(enable_timing=True) for _ in range(CALLS)]
    ends = [torch.cuda.Event(enable_timing=True) for _ in range(CALLS)]
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for i in range(CALLS):
        starts[i].record()
        fn()
        ends[i].record()
    torch.cuda.synchronize()
    host = (time.perf_counter() - t0) / CALLS * 1e6
    dev = sum(s.elapsed_time(e) for s, e in zip(starts, ends)) / CALLS * 1e3
    return host, dev


def launches(fn):
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(PROF_CALLS):
            fn()
        torch.cuda.synchronize()
    kinds = {"kernels": 0, "copies": 0, "kernel_us": 0.0}
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA:
            copy = "emcpy" in e.name or "emset" in e.name
            kinds["copies" if copy else "kernels"] += 1
            kinds["kernel_us"] += 0.0 if copy else e.time_range.elapsed_us()
    return {k: round(v / PROF_CALLS, 2) for k, v in kinds.items()}


def syncs(fn):
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        torch.cuda.set_sync_debug_mode("warn")
        try:
            fn()
        finally:
            torch.cuda.set_sync_debug_mode(0)
    return sum("synchroniz" in str(w.message) for w in caught)


def main():
    print("card:", card())
    with torch.no_grad():
        for name in CASES:
            for N in (16, 128, 512):
                policy, features, obs = setup(name, N)
                run = runners(policy, features, obs)
                for fn in run.values():
                    for _ in range(20):
                        fn()
                host = {k: [] for k in run}
                dev = {k: [] for k in run}
                for _ in range(ROUNDS):
                    for k, fn in run.items():
                        h, d = timed(fn)
                        host[k].append(h)
                        dev[k].append(d)
                res = {"case": name, "B": N}
                for k, fn in run.items():
                    res[k] = {"host_us": round(min(host[k]), 1), "stream_us": round(min(dev[k]), 1),
                              **launches(fn), "syncs": syncs(fn)}
                res["host_speedup"] = round(res["eager"]["host_us"] / res["fused"]["host_us"], 2)
                print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
