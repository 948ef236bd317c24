"""The CNN encoders' forward + backward per PPO minibatch at the trainers' update shapes: AV-Nav (B = 1500 = T 150 x
N 10) ``VisualCNN`` RGB-D and depth at 128 x 128 and ``AudioCNN`` at 16 and 44.1 kHz; SAVi's ``AudioCNN`` with a
distractor sound (B = 600); AV-WaN's ``MapCNN`` on gm 200 and am 20 (B = 750).  Three ways, alternated in rounds in
one process: eager with cuDNN's default (TF32 allowed), eager with TF32 off, and the ``training=True`` patches
(``ConvStackFunction``).

    python scratch/conv_stack_bench.py [--out DIR]

Per call: the encoder's forward, then the backward of sum(out * g) with every parameter requiring grad, ending in a
device synchronise (host clock, CALLS calls per round, ROUNDS rounds, the median round reported).  Then the device
kernel time and kernel count per call from ``torch.profiler`` (a run of its own, PROF_CALLS calls, CUDA kernels
only).  Prints the largest gradient error of the fused path against eager with TF32 off (relative to each tensor's
largest value), the card's name and power limit, and one JSON line per shape."""
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

from avnav_models import VisualCNN, visual_obs  # noqa: E402
from map_cnn_models import MapCNN, map_obs  # noqa: E402
from test_encoder_host import reference_classes  # noqa: E402
from soundspaces_b200.encoder import patch_audio_cnn, patch_map_cnn, patch_visual_cnn  # noqa: E402

CALLS, ROUNDS, PROF_CALLS, WARMUP = 10, 5, 5, 3
DEV = torch.device("cuda", 0)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name(0)


def build(name):
    """(eager module, fused module with the same parameters, observations, hidden) of a named shape."""
    torch.manual_seed(0)
    AvNav, _, Savi = reference_classes()
    if name.startswith("visual"):
        n_rgb = 3 if name == "visual_rgbd" else 0
        make = lambda: VisualCNN(n_rgb, 1, 128, 128, 512)                       # noqa: E731
        obs, hidden, patch = visual_obs(1500, 128, 128, n_rgb, 1, 0), 512, patch_visual_cnn
    elif name.startswith("audio_avnav"):
        shape = (65, 26, 2) if name.endswith("16k") else (65, 69, 2)
        make = lambda: AvNav(shape, hidden=512)                                # noqa: E731
        obs, hidden = {"spectrogram": torch.rand((1500,) + shape) * 3}, 512
        patch = patch_audio_cnn
    elif name == "audio_savi_category":
        make = lambda: Savi((65, 26, 2), hidden=128, has_distractor_sound=True)  # noqa: E731
        obs = {"audiogoal": torch.rand((600, 65, 26, 2)) * 3,
               "category": torch.nn.functional.one_hot(torch.randint(0, 21, (600,)), 21).float()}
        hidden, patch = 128, lambda c, training: patch_audio_cnn(c, category=True, training=training)
    else:
        kind, H, C = ("gm", 200, 2) if name == "map_gm200" else ("am", 20, 1)
        make = lambda: MapCNN(H, H, C, 512, map_type=kind)                      # noqa: E731
        obs, hidden, patch = {kind: map_obs(750, H, H, C, 0, kind)}, 512, patch_map_cnn
    eager = make().to(DEV)
    fused_cls = type("Fused" + type(eager).__name__, (type(eager),), {})
    patch(fused_cls, training=True)
    fused = make()
    fused.__class__ = fused_cls
    fused.load_state_dict(eager.state_dict())
    return eager, fused.to(DEV), {k: v.to(DEV) for k, v in obs.items()}, hidden


def call(m, obs, g):
    m.zero_grad(set_to_none=True)
    out = m(obs)
    (out * g).sum().backward()


def timed(m, obs, g, tf32):
    torch.backends.cudnn.allow_tf32 = tf32
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(CALLS):
        call(m, obs, g)
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / CALLS * 1e3


def device_time(m, obs, g, tf32):
    torch.backends.cudnn.allow_tf32 = tf32
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(PROF_CALLS):
            call(m, obs, g)
        torch.cuda.synchronize()
    kern = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA
            and "memcpy" not in e.name.lower() and "memset" not in e.name.lower()]
    per = {}
    for e in kern:
        per[e.name] = per.get(e.name, 0.0) + e.device_time / PROF_CALLS / 1e3
    top = sorted(per.items(), key=lambda kv: -kv[1])[:8]
    return sum(e.device_time for e in kern) / PROF_CALLS / 1e3, len(kern) / PROF_CALLS, top


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--shapes", default="visual_rgbd,visual_depth,audio_avnav_16k,audio_avnav_44k,"
                                        "audio_savi_category,map_gm200,map_am20")
    args = ap.parse_args()
    print("card:", card())
    results = []
    for name in args.shapes.split(","):
        eager, fused, obs, hidden = build(name)
        B = next(iter(obs.values())).shape[0]
        g = torch.randn((B, hidden), device=DEV)
        ways = {"eager_tf32": (eager, True), "eager_fp32": (eager, False), "fused": (fused, False)}
        for m, tf32 in ways.values():
            torch.backends.cudnn.allow_tf32 = tf32
            for _ in range(WARMUP):
                call(m, obs, g)
        ms = {k: [] for k in ways}
        for _ in range(ROUNDS):
            for k, (m, tf32) in ways.items():
                ms[k].append(timed(m, obs, g, tf32))
        torch.backends.cudnn.allow_tf32 = False
        call(eager, obs, g)
        call(fused, obs, g)
        err = max(((p.grad - q.grad).abs().max() / q.grad.abs().max().clamp_min(1e-30)).item()
                  for p, q in zip(fused.parameters(), eager.parameters()))
        dev = {k: device_time(m, obs, g, tf32) for k, (m, tf32) in ways.items()}
        row = {"shape": name, "B": B, "max_rel_grad_err_vs_eager_fp32": err}
        for k in ways:
            row[k + "_ms"] = statistics.median(ms[k])
            row[k + "_ms_spread"] = [min(ms[k]), max(ms[k])]
            row[k + "_device_ms"], row[k + "_kernels"], top = dev[k]
            if k == "fused":
                row["fused_top_kernels_ms"] = [(n[:60], round(t, 3)) for n, t in top]
        print(json.dumps(row))
        results.append(row)
        del eager, fused, obs
        torch.cuda.empty_cache()
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "conv_stack_bench.json"), "w") as f:
            json.dump({"card": card(), "results": results}, f, indent=1)


if __name__ == "__main__":
    main()
