"""SAVi's scene memory transformer per call at SAVi's shape (D 276, pose index 272, d 256, 8 heads), eager
``single_forward`` against the library (``fused_single_forward``), at B in {8, 16} for the training memory (300 slots,
150 valid in a wrapped ring) and the eval memory (150 slots, half valid):

    python scratch/smt_bench.py              # wall clock per call (1000 calls + synchronise, 3 alternated rounds)
    python scratch/smt_bench.py --profile    # device time and kernel count per call from torch.profiler

Also prints the FLOPs of the valid-token computation (from shapes) and their share of the 67 TFLOP/s FP32 data-sheet
peak at the measured device time, the max error of both paths against float64, and the card's name and power limit.
The module is in training mode with dropout 0, as the trainer leaves it during rollouts."""
import argparse
import copy
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

from smt_models import make_inputs, make_smt, ring_masks  # noqa: E402
from soundspaces_b200.smt import fused_single_forward  # noqa: E402

D, PI, d, H, F = 276, 272, 256, 8, 272 + 16
PEAK = 67e12
CALLS, ROUNDS = 1000, 3


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name(0)


def case(B, M, fill):
    x, memory, _, goal = make_inputs(B, M, seed=B + M)
    masks = ring_masks(B, M, [fill] * B, start=[(37 * b + 11) % M for b in range(B)])
    return x.cuda(), memory.cuda(), masks.cuda(), goal.cuda(), masks


def flops(masks):
    total = 0
    for row in masks:
        n = int(((1 - row) <= 0).sum()) + 1
        total += 2 * n * (5 * 16 + F * d + d * d)            # pose encoder, fusion
        total += 2 * n * d * 3 * d                             # QKV
        total += 2 * 2 * n * n * d                             # scores + P.V
        total += 2 * n * 3 * d * d                             # out_proj, FF
        total += 2 * n * d * 2 * d                             # cross-attention K / V
        total += 2 * 6 * d * d + 2 * 2 * n * d                 # decoder (one target token)
    return total


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--profile", action="store_true")
    args = ap.parse_args()
    print("card:", card())
    m = make_smt(seed=0).cuda().train()
    m64 = copy.deepcopy(m).cpu().double()
    for B in (8, 16):
        for M, fill in ((300, 150), (150, 75)):
            x, memory, masks, goal, cpu_masks = case(B, M, fill)
            eager = lambda: m.single_forward(x, memory, masks, goal)  # noqa: E731
            fused = lambda: fused_single_forward(m, x, memory, masks, goal)  # noqa: E731
            with torch.no_grad():
                assert fused() is not None
                ref = m64.single_forward(x.cpu().double(), memory.cpu().double(), cpu_masks.double(), goal.cpu().double())
                err = {k: (f().double().cpu() - ref).abs().max().item() for k, f in (("eager", eager), ("fused", fused))}
                for f in (eager, fused):
                    for _ in range(50):
                        f()
                torch.cuda.synchronize()
                fl = flops(cpu_masks)
                tag = f"B={B} M={M} valid={fill}"
                if args.profile:
                    from torch.profiler import ProfilerActivity, profile
                    for name, f in (("eager", eager), ("fused", fused)):
                        with profile(activities=[ProfilerActivity.CUDA]) as prof:
                            for _ in range(100):
                                f()
                            torch.cuda.synchronize()
                        ev = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
                        dev_us = sum(e.device_time for e in ev) / 100
                        if name == "fused":
                            per = {}
                            for e in ev:
                                per[e.name] = per.get(e.name, 0.0) + e.device_time / 100
                            print("   ", ", ".join(f"{k.split('(')[0]} {v:.1f} us" for k, v in per.items()))
                        print(f"{tag} {name}: device {dev_us:.1f} us/call, {len(ev) / 100:.0f} kernels/call, "
                              f"{fl / 1e9:.3f} GFLOP valid-token work = {fl / (dev_us * 1e-6) / 1e12:.2f} TFLOP/s "
                              f"({100 * fl / (dev_us * 1e-6) / PEAK:.1f}% of the FP32 peak)")
                    continue
                times = {"eager": [], "fused": []}
                for _ in range(ROUNDS):
                    for name, f in (("eager", eager), ("fused", fused)):
                        torch.cuda.synchronize()
                        t0 = time.perf_counter()
                        for _ in range(CALLS):
                            f()
                        torch.cuda.synchronize()
                        times[name].append((time.perf_counter() - t0) / CALLS * 1e6)
                print(f"{tag}: eager {' '.join(f'{t:.1f}' for t in times['eager'])} us/call, fused "
                      f"{' '.join(f'{t:.1f}' for t in times['fused'])} us/call; max|err| vs float64 eager "
                      f"{err['eager']:.2e} fused {err['fused']:.2e}")


if __name__ == "__main__":
    main()
