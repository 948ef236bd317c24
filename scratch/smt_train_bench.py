"""SAVi's scene memory transformer in the PPO update at SAVi's minibatch (600 rows = 150 steps x 4 envs, 300 memory
slots with episode masks, D 276, pose index 272, d_model 256, 8 heads): eager ``single_forward`` with TF32 matmuls
allowed and in FP32, against the patched module (patch_smt_state_encoder(..., training=True)), per forward plus the
backward of sum(out * g):

    python scratch/smt_train_bench.py [--calls 10] [--rounds 3] [--out results.json]

CUDA events around `calls` calls, the modes alternated `rounds` times (median reported); the peak memory of one call
over what was allocated before it (torch.cuda.max_memory_allocated), beside the library's workspace bytes; then, in a
separate torch.profiler run of 2 calls per mode, the summed device time of the kernels and the launches per call.
Also the FLOPs of the valid-token computation (from shapes; forward and backward ~ 3x the forward), and the card's name
and power limit as found (nothing is changed).  One JSON line per mode."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.dirname(os.path.abspath(__file__))]

import torch  # noqa: E402

from smt_bench import card  # noqa: E402
from smt_models import SMTStandIn, episode_masks, make_inputs, make_smt  # noqa: E402
from soundspaces_b200.smt import patch_smt_state_encoder, smt_params  # noqa: E402

B, M, D, PI, d, H = 600, 300, 276, 272, 256, 8


def valid_flops(masks):
    """Forward FLOPs on valid tokens: fusion MLP, QKV, attention, out_proj + FF, the decoder K/V and its one-token
    decoder; the backward is counted as twice the forward."""
    n = masks.sum(1).double() + 1                   # valid tokens per row, the current one included
    F = PI + 16
    tok = n.sum().item()
    fwd = 2 * tok * (F * d + d * d + 3 * d * d + d * d + 2 * d * d + 2 * d * d) + 4 * (n * n).sum().item() * d
    fwd += B * 2 * (6 * d * d) + 4 * tok * d
    return fwd, 3 * fwd


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a GPU")
    from soundspaces_b200.renderer import WaveformOps
    ops = WaveformOps.get("cuda:0")
    res = {"card": card(), "B": B, "M": M}
    print("card:", res["card"], flush=True)
    P = patch_smt_state_encoder(type("Patched", (SMTStandIn,), {}), training=True)
    eager_m = make_smt(seed=1).cuda().train()
    fused_m = make_smt(seed=1)
    fused_m.__class__ = P
    fused_m = fused_m.cuda().train()
    x, mem, _, goal = (t.cuda() for t in make_inputs(B, M, seed=1))
    masks = episode_masks(B, M, 2 * M, 40, torch.Generator().manual_seed(1)).cuda()
    g = torch.randn(B, d, generator=torch.Generator().manual_seed(2)).cuda()
    res["valid_tokens_mean"] = masks.sum(1).mean().item() + 1
    res["flops_fwd"], res["flops_fwd_bwd"] = valid_flops(masks.cpu())
    res["workspace_bytes"] = int(ops.lib.ssb_smt_train_workspace_bytes(B, M, __import__("ctypes").byref(
        smt_params(fused_m, D))))
    tf32_default = torch.backends.cuda.matmul.allow_tf32

    def call(m, tf32):
        torch.backends.cuda.matmul.allow_tf32 = tf32
        out = m.single_forward(x, mem, masks, goal)
        torch.autograd.backward(out, g)
        for p in m.parameters():
            p.grad = None

    modes = {"eager_tf32": lambda: call(eager_m, True), "eager_fp32": lambda: call(eager_m, False),
             "fused": lambda: call(fused_m, tf32_default)}
    for f in modes.values():
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
            e1.synchronize()
            times[k].append(e0.elapsed_time(e1) / a.calls)
    peak = {}
    for k, f in modes.items():
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        f()
        torch.cuda.synchronize()
        peak[k] = torch.cuda.max_memory_allocated() - base
    from torch.profiler import ProfilerActivity, profile
    prof = {}
    for k, f in modes.items():
        with profile(activities=[ProfilerActivity.CUDA]) as p:
            f()
            f()
            torch.cuda.synchronize()
        ev = [e for e in p.events() if e.device_type == torch.autograd.DeviceType.CUDA]
        smt = [e for e in ev if e.name.startswith("smt_") or "smt_" in e.name[:40]]
        prof[k] = {"device_ms": sum(e.device_time for e in ev) / 2e3, "kernels": len(ev) / 2,
                   "smt_kernel_ms": {n: sum(e.device_time for e in smt if e.name.split("(")[0] == n) / 2e3
                                     for n in sorted({e.name.split("(")[0] for e in smt})}}
    torch.backends.cuda.matmul.allow_tf32 = tf32_default
    res["modes"] = {}
    for k in modes:
        ms = sorted(times[k])[len(times[k]) // 2]
        row = {"mode": k, "ms_per_call": round(ms, 3), "peak_bytes": peak[k], "device_ms": round(prof[k]["device_ms"], 3),
               "kernels_per_call": prof[k]["kernels"], "valid_tflops": round(res["flops_fwd_bwd"] / ms / 1e9, 2)}
        if k == "fused":
            row["smt_kernel_ms"] = {n: round(v, 3) for n, v in prof[k]["smt_kernel_ms"].items()}
        res["modes"][k] = row
        print(json.dumps(row), flush=True)
    print(json.dumps({kk: v for kk, v in res.items() if kk != "modes"}), flush=True)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
