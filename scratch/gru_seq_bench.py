"""``RNNStateEncoder.seq_forward`` + backward per PPO minibatch, at three trainers' shapes (Hd = 512): AV-Nav
(T 150, N 10, I 1024), AV-WaN (T 150, N 5, I 2048) and SAVi's ``rnn`` policy (T 150, N 4, I 1024), each env done
with probability 0.02 per step (seeded).  Three ways, alternated in rounds in one process: the eager stand-in of the
reference (tests/gru_seq_models.RNNStateEncoder) with cuDNN's default (TF32 allowed), the same with TF32 off, and
``patch_rnn_state_encoder(cls, sequence=True)``.

    python scratch/gru_seq_bench.py [--out DIR]

Per call: seq_forward, then backward of sum(out * g) + sum(h_last * g') with x, h0 and the GRU's parameters
requiring grad, ending in a device synchronise (host clock, CALLS calls per round, ROUNDS rounds, the median round
reported).  Then the device kernel time per call from ``torch.profiler`` (a run of its own, PROF_CALLS calls, CUDA
kernels only, memcpy / memset apart).  Prints the segment count of each shape's done pattern, errors of the fused
path against the TF32-off eager run, the card's name and power limit, and one JSON line per shape."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

import gru_seq_models as gm  # noqa: E402
from soundspaces_b200.rnn import patch_rnn_state_encoder  # noqa: E402

CALLS, ROUNDS, PROF_CALLS, WARMUP = 20, 5, 10, 5
DEV = torch.device("cuda", 0)
HD = 512
SHAPES = {"av_nav": (150, 10, 1024), "av_wan": (150, 5, 2048), "savi_rnn": (150, 4, 1024)}
DONE_P = 0.02
Fused = patch_rnn_state_encoder(type("FusedRNNStateEncoder", (gm.RNNStateEncoder,), {}), sequence=True)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name(0)


def setup(T, N, I, seed=0):
    g = torch.Generator().manual_seed(seed)
    masks = (torch.rand(T * N, 1, generator=g) >= DONE_P).float()
    data = [torch.randn(T * N, I, generator=g), torch.randn(1, N, HD, generator=g), masks,
            torch.randn(T * N, HD, generator=g), torch.randn(1, N, HD, generator=g)]
    x, h0, masks, g_out, g_h = (t.to(DEV) for t in data)
    torch.manual_seed(seed)
    eager = gm.RNNStateEncoder(I, HD).to(DEV)
    fused = Fused(I, HD).to(DEV)
    fused.load_state_dict(eager.state_dict())
    zero = (masks.view(T, N)[1:] == 0).any(dim=1)
    segments = 1 + int(zero.sum())
    return eager, fused, (x, h0, masks, g_out, g_h), segments


def call(enc, inputs):
    x, h0, masks, g_out, g_h = inputs
    x = x.detach().requires_grad_(True)
    h0 = h0.detach().requires_grad_(True)
    enc.zero_grad(set_to_none=True)
    out, h_last = enc(x, h0, masks)
    ((out * g_out).sum() + (h_last * g_h).sum()).backward()
    return out, h_last, [x.grad, h0.grad] + [p.grad for p in gm.gru_params(enc)]


def runners(eager, fused, inputs):
    def with_tf32(flag, enc):
        def run():
            torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = flag
            return call(enc, inputs)
        return run
    return {"eager_tf32": with_tf32(True, eager), "eager_fp32": with_tf32(False, eager),
            "fused": with_tf32(False, fused)}


def timed(fn):
    for _ in range(WARMUP):
        fn()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(CALLS):
        fn()
        torch.cuda.synchronize()
    return (time.perf_counter() - t0) / CALLS * 1e3


def profiled(fn, out_dir, tag):
    from torch.profiler import ProfilerActivity, profile
    for _ in range(WARMUP):
        fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(PROF_CALLS):
            fn()
        torch.cuda.synchronize()
    kern_us, n_kern, per_name = 0.0, 0, {}
    for e in prof.events():
        if e.device_type != torch.autograd.DeviceType.CUDA:
            continue
        name = e.name
        if "memcpy" in name.lower() or "memset" in name.lower():
            continue
        us = e.device_time if hasattr(e, "device_time") else e.cuda_time
        kern_us += us
        n_kern += 1
        per_name[name] = per_name.get(name, 0.0) + us
    if out_dir:
        top = sorted(per_name.items(), key=lambda kv: -kv[1])[:12]
        with open(os.path.join(out_dir, f"gru_seq_kernels_{tag}.json"), "w") as f:
            json.dump({k[:160]: v / PROF_CALLS for k, v in top}, f, indent=1)
    return kern_us / PROF_CALLS / 1e3, n_kern / PROF_CALLS


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    if args.out:
        os.makedirs(args.out, exist_ok=True)
    print("card:", card())
    results = []
    for name, (T, N, I) in SHAPES.items():
        eager, fused, inputs, segments = setup(T, N, I)
        run = runners(eager, fused, inputs)
        (o, hl, g), (o2, hl2, g2) = run["fused"](), run["eager_fp32"]()
        names = ("out", "h_last", "dx", "dh0", "dw_ih", "dw_hh", "db_ih", "db_hh")
        errs = {k: float((a - b).abs().max() / b.abs().max())
                for k, a, b in zip(names, [o.detach(), hl.detach()] + g, [o2.detach(), hl2.detach()] + g2)}
        rounds = {k: [] for k in run}
        for _ in range(ROUNDS):
            for k, fn in run.items():
                rounds[k].append(timed(fn))
        med = {k: statistics.median(v) for k, v in rounds.items()}
        spread = {k: (min(v), max(v)) for k, v in rounds.items()}
        dev = {k: profiled(fn, args.out, f"{name}_{k}") for k, fn in run.items()}
        r = dict(shape=name, T=T, N=N, I=I, Hd=HD, done_p=DONE_P, segments=segments,
                 ms_per_call={k: round(v, 3) for k, v in med.items()},
                 ms_min_max={k: [round(a, 3), round(b, 3)] for k, (a, b) in spread.items()},
                 device_ms_per_call={k: round(v[0], 3) for k, v in dev.items()},
                 kernels_per_call={k: v[1] for k, v in dev.items()},
                 fused_rel_err_vs_eager_fp32={k: float(f"{v:.3g}") for k, v in errs.items()})
        results.append(r)
        print(json.dumps(r))
    torch.backends.cudnn.allow_tf32 = True
    if args.out:
        with open(os.path.join(args.out, "gru_seq_bench.json"), "w") as f:
            json.dump(dict(card=card(), results=results), f, indent=1)


if __name__ == "__main__":
    main()
