"""SAVi's visual encoder (SMTCNN, 128 x 128 RGB-D) in the PPO update: eager with cuDNN TF32 at its default and off,
against the patched module (patch_smt_cnn(..., training=True)), per call.

    python scratch/smt_cnn_train_bench.py [--calls 5] [--rounds 3] [--out results.json]

Per B in 150, 600 (4 envs x 150 steps, SAVi's minibatch) and 1200, two calls:
  train   every parameter trainable (stage 1): the forward plus the backward of sum(out * g)
  frozen  every parameter frozen under grad mode (stage 2, freeze_encoders): the forward
CUDA events around `calls` calls, the modes alternated `rounds` times (median reported); then, in a separate
torch.profiler run of 2 calls per mode, the summed device time of the kernels and the kernel launches per call; and
the peak memory of one call over what was allocated before it (torch.cuda.max_memory_allocated), beside the
library's workspace bytes.  Prints the card and its power limit as found (nothing is changed), one JSON line per
(B, call) and a table; `--out` also writes the whole result as JSON."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import torch  # noqa: E402

from smt_cnn_bench import ResizeCenterCropper, card  # noqa: E402
from smt_cnn_models import SMTCNN, observations, set_params  # noqa: E402
from soundspaces_b200.encoder import patch_smt_cnn, smt_cnn_params  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None, help="also write the result as JSON to this file")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a GPU")
    from soundspaces_b200.renderer import WaveformOps
    ops = WaveformOps.get("cuda:0")
    Patched = patch_smt_cnn(type("Patched", (SMTCNN,), {}), training=True)
    eager_m = set_params(SMTCNN({"rgb": 3, "depth": 1}, obs_transform=ResizeCenterCropper()), 1).cuda()
    fused_m = set_params(Patched({"rgb": 3, "depth": 1}, obs_transform=ResizeCenterCropper()), 1).cuda()
    tf32_default = torch.backends.cudnn.allow_tf32
    res = {"card": card(), "calls": a.calls, "rounds": a.rounds, "rows": []}
    print("card:", res["card"], flush=True)

    def call(m, tf32, obs, g, train):
        torch.backends.cudnn.allow_tf32 = tf32
        out = m(obs)
        if train:
            torch.autograd.backward(out, g)
            for p in m.parameters():
                p.grad = None
        return out

    for B in (150, 600, 1200):
        obs = {k: v.cuda() for k, v in observations(B, 128, 128, seed=B).items()}
        g = torch.randn((B, 128), generator=torch.Generator().manual_seed(B)).cuda()
        from soundspaces_b200.belief_nets import conv_norm_pairs
        eps = tuple(float(n.eps) for k in ("rgb", "depth") for _, n in conv_norm_pairs(getattr(fused_m, f"{k}_encoder")))
        _, table, n, _ = ops._smt_cnn_train_table(obs["rgb"], obs["depth"], smt_cnn_params(fused_m), eps, True)
        ws_bytes = int(ops.lib.ssb_smt_cnn_train_workspace_bytes(B, n, table))
        for train in (True, False):
            for m in (eager_m, fused_m):
                m.requires_grad_(train)
            modes = {"eager_tf32": lambda: call(eager_m, True, obs, g, train),
                     "eager_fp32": lambda: call(eager_m, False, obs, g, train),
                     "fused": lambda: call(fused_m, tf32_default, obs, g, train)}
            row = {"B": B, "call": "train" if train else "frozen", "workspace_bytes": ws_bytes if train else 0}
            for f in modes.values():               # warm-up: module loads, cuDNN algorithm choice
                f()
                f()
            torch.cuda.synchronize()
            times = {k: [] for k in modes}
            for _ in range(a.rounds):
                for k, f in modes.items():
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    for _ in range(a.calls):
                        f()
                    e1.record()
                    torch.cuda.synchronize()
                    times[k].append(e0.elapsed_time(e1) / a.calls)
            for k, f in modes.items():
                row[f"{k}_ms"] = sorted(times[k])[len(times[k]) // 2]
                torch.cuda.synchronize()
                base = torch.cuda.memory_allocated()
                torch.cuda.reset_peak_memory_stats()
                f()
                torch.cuda.synchronize()
                row[f"{k}_peak_bytes"] = torch.cuda.max_memory_allocated() - base
                from torch.profiler import ProfilerActivity, profile
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    for _ in range(2):
                        f()
                    torch.cuda.synchronize()
                evs = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
                kern = [e for e in evs if "memcpy" not in e.name.lower() and "memset" not in e.name.lower()]
                row[f"{k}_device_ms"] = sum(e.device_time for e in kern) / 2 / 1e3
                row[f"{k}_kernels"] = len(kern) / 2
            torch.backends.cudnn.allow_tf32 = tf32_default
            row["card"] = res["card"]
            res["rows"].append(row)
            print(json.dumps(row), flush=True)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)
    print("card:", res["card"])
    print("| B | call | wall ms TF32 / FP32 / fused | device ms TF32 / FP32 / fused | kernels TF32 / FP32 / fused "
          "| peak GB TF32 / FP32 / fused | workspace GB |")
    for r in res["rows"]:
        k = ("eager_tf32", "eager_fp32", "fused")
        print("| %d | %s | %s | %s | %s | %s | %.2f |" % (
            r["B"], r["call"], " / ".join("%.1f" % r[f"{m}_ms"] for m in k),
            " / ".join("%.1f" % r[f"{m}_device_ms"] for m in k), " / ".join("%.0f" % r[f"{m}_kernels"] for m in k),
            " / ".join("%.2f" % (r[f"{m}_peak_bytes"] / 1e9) for m in k), r["workspace_bytes"] / 1e9))


if __name__ == "__main__":
    main()
