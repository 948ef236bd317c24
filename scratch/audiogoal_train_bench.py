"""SAVi's audio-goal predictor pretraining step (audiogoal_trainer.py:69-124: AudioGoalPredictor's ResNet-18 in
train() mode, CrossEntropy + MSE, Adam) three ways alternated in one process: eager with cuDNN TF32 allowed (torch's
default), eager with TF32 off, and the library (patch_audiogoal_predictor).  Two timings per way: forward + backward
of the network and loss, and the whole trainer step (zero_grad, forward, loss, backward, Adam).  Wall time per call
ends in a synchronise (median of --reps after one warm-up per shape and way); device time is the sum of the CUDA
kernel times of one call in a separate torch.profiler run.  Prints the card and its power limit, and the counted
network FLOPs (forward + backward = 3x forward) over each way's forward + backward device time.

    python scratch/audiogoal_train_bench.py [--reps 10]
"""
import argparse
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

from audiogoal_train_models import reference_loss, set_params, tv_net       # noqa: E402
from soundspaces_b200.pretraining import patch_audiogoal_predictor           # noqa: E402


class Predictor(torch.nn.Module):
    """AudioGoalPredictor's forward (audiogoal_predictor.py:29-38) on tensors."""

    def __init__(self):
        super().__init__()
        self.input_shape_printed = True
        self.predictor = set_params(tv_net(23)).cuda()

    def forward(self, audio_feature):
        return self.predictor(audio_feature["spectrogram"].permute(0, 3, 1, 2))


class Fused(Predictor):
    pass


patch_audiogoal_predictor(Fused)


def flops(H, W):
    """Forward FLOPs of one row (2 per multiply-add), counted from the layer shapes."""
    h, w = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    total = 2 * 64 * 49 * h * w
    h, w, ic = (h - 1) // 2 + 1, (w - 1) // 2 + 1, 64
    for s, oc in enumerate((64, 128, 256, 512)):
        for blk in range(2):
            stride = 2 if s and blk == 0 else 1
            ho, wo = (h - 1) // stride + 1, (w - 1) // stride + 1
            total += 2 * ho * wo * oc * (ic * 9 + oc * 9 + (ic if stride == 2 else 0))
            h, w, ic = ho, wo, oc
    return total + 2 * 512 * 23


def fwd_bwd(m, obs, gts, opt):
    m.zero_grad(set_to_none=True)
    reference_loss(m(obs), gts).backward()


def step(m, obs, gts, opt):
    opt.zero_grad()
    reference_loss(m(obs), gts).backward()
    opt.step()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    a = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print("card:", card)
    print("| input | B | what | wall: eager TF32 / eager FP32 / fused (ms) | device: eager TF32 / eager FP32 / fused (ms)"
          " | counted TFLOP/s over device time (fwd+bwd): TF32 / FP32 / fused |")
    for H, W in ((65, 26), (65, 69)):
        for B in (1024, 256):
            g = torch.Generator().manual_seed(1)
            obs = {"spectrogram": (torch.rand((B, H, W, 2), generator=g) * 3).cuda()}
            gts = torch.cat([torch.randint(0, 21, (B, 1), generator=g).float(),
                             torch.randn((B, 2), generator=g) * 5], 1).cuda()
            ways = {"tf32": Predictor().train(), "fp32": Predictor().train(), "fused": Fused().train()}
            opts = {k: torch.optim.Adam(m.parameters()) for k, m in ways.items()}
            fl = 3 * flops(H, W) * B
            tflops = {}
            for what, fn in (("fwd+bwd", fwd_bwd), ("step", step)):
                times = {k: [] for k in ways}
                for rep in range(a.reps + 1):
                    for k, m in ways.items():
                        torch.backends.cudnn.allow_tf32 = k == "tf32"
                        torch.cuda.synchronize()
                        t0 = time.perf_counter()
                        fn(m, obs, gts, opts[k])
                        torch.cuda.synchronize()
                        if rep:
                            times[k].append((time.perf_counter() - t0) * 1e3)
                dev = {}
                for k, m in ways.items():
                    torch.backends.cudnn.allow_tf32 = k == "tf32"
                    torch.cuda.synchronize()
                    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                        fn(m, obs, gts, opts[k])
                        torch.cuda.synchronize()
                    dev[k] = sum(e.self_device_time_total for e in prof.key_averages()) / 1e3
                torch.backends.cudnn.allow_tf32 = True
                med = {k: sorted(v)[len(v) // 2] for k, v in times.items()}
                if what == "fwd+bwd":
                    tflops = {k: fl / dev[k] / 1e9 for k in ways}
                rate = " / ".join(f"{tflops[k]:.1f}" for k in ways) if what == "fwd+bwd" else ""
                print(f"| {H}x{W} | {B} | {what} | {med['tf32']:.2f} / {med['fp32']:.2f} / {med['fused']:.2f} | "
                      f"{dev['tf32']:.2f} / {dev['fp32']:.2f} / {dev['fused']:.2f} | {rate} |", flush=True)


if __name__ == "__main__":
    main()
