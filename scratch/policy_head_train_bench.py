"""Forward plus backward of the heads of ``evaluate_actions`` (actor Linear, log_probs, entropy, critic Linear) at the
three trainers' minibatch shapes (150 steps x the envs of one minibatch: AV-Nav 5, SAVi 8 / 2, AV-WaN 5), fused
(``PolicyHeadFunction``) against eager PyTorch with TF32 allowed and with TF32 off, the three alternating.

    python scratch/policy_head_train_bench.py [--iters 200] [--out results.json]

Reports wall time per call (host clock around ``iters`` calls that end in a device synchronise, median of 5
windows), then in a separate ``torch.profiler`` run the device time and kernel count per call, and the card's name
and power limit read in the same run."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import torch  # noqa: E402

import policy_head_models as phm  # noqa: E402
import policy_head_train_models as ptm  # noqa: E402
from soundspaces_b200.policy import patch_policy  # noqa: E402

# trainer: (H, A, rows)
SHAPES = {"av_nav": (512, 4, 750), "savi": (128, 4, 600), "av_wan": (512, 81, 750)}
MODES = ("fused", "eager_tf32", "eager_fp32")


def setup(trainer):
    H, A, B = SHAPES[trainer]
    cls = patch_policy(type("P", (ptm.POLICIES[trainer],), {}), training=True)
    fused = ptm.make_policy(trainer, H, A, 1, 1.0, True, classes={trainer: cls}).cuda()
    eager = ptm.make_policy(trainer, H, A, 1, 1.0, True).cuda()
    g = torch.Generator().manual_seed(2)
    features = torch.tanh(torch.randn((B, H), generator=g) * 2).cuda().requires_grad_(True)
    obs = {"features": features}
    if trainer == "av_wan":
        obs["action_map"] = phm.action_map(B, A, 3).cuda()
    actions = torch.randint(0, A, (B, 1), generator=g).cuda()
    args = ptm.evaluate_args(trainer, obs, actions)[0]
    return {"fused": fused, "eager_tf32": eager, "eager_fp32": eager}, args


def call(policy, args, mode):
    torch.backends.cuda.matmul.allow_tf32 = mode == "eager_tf32"
    v, lp, ent = policy.evaluate_actions(*args)[:3]
    (v.sum() + lp.sum() + ent).backward()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--out", default=None, help="also write the results as JSON to this file")
    a = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    res = {"card": card, "torch": torch.__version__, "shapes": {}}
    for trainer in SHAPES:
        policies, args = setup(trainer)
        walls = {m: [] for m in MODES}
        for m in MODES:                         # warm-up
            for _ in range(20):
                call(policies[m], args, m)
        torch.cuda.synchronize()
        for _ in range(5):
            for m in MODES:
                t0 = time.perf_counter()
                for _ in range(a.iters):
                    call(policies[m], args, m)
                torch.cuda.synchronize()
                walls[m].append((time.perf_counter() - t0) / a.iters * 1e6)
        row = {m: {"wall_us": statistics.median(walls[m]), "wall_us_all": walls[m]} for m in MODES}
        for m in MODES:                         # separate profiled run
            n = 50
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                for _ in range(n):
                    call(policies[m], args, m)
                torch.cuda.synchronize()
            ev = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
            kern = [e for e in ev if "memcpy" not in e.name.lower() and "memset" not in e.name.lower()]
            row[m]["device_us"] = sum(e.device_time for e in kern) / n
            row[m]["kernels"] = len(kern) / n
        H, A, B = SHAPES[trainer]
        res["shapes"][trainer] = {"H": H, "A": A, "rows": B, **row}
        print(trainer, json.dumps({m: {k: round(v, 1) for k, v in row[m].items() if k != "wall_us_all"}
                                   for m in MODES}), flush=True)
    torch.backends.cuda.matmul.allow_tf32 = False
    print("card:", card)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
