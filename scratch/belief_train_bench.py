"""train_belief_predictor's body (ppo_trainer.py:342-400) on SAVi's online location predictor: 5 epochs of the masked
MSE, backward and Adam (lr 1e-3) over one 1200-row minibatch, three ways alternated in one process: eager with cuDNN
TF32 allowed (torch's default), eager with TF32 off, and the library (patch_belief_predictor(..., training=True)).
Wall time per call ends in a synchronise.  Device time comes from a separate torch.profiler run of one call per way
(the sum of its CUDA kernel times: network, loss and Adam).  Prints the card and its power limit, and the counted
network FLOPs (forward + backward, 5 epochs, every row) over the fused call's device time.

    python scratch/belief_train_bench.py [--rows 1200] [--reps 5]
"""
import argparse
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

from belief_nets_models import smt_net                                  # noqa: E402
from soundspaces_b200.belief import patch_belief_predictor              # noqa: E402

HW = (65, 26)


class Predictor(torch.nn.Module):
    def __init__(self, n_labels):
        super().__init__()
        self.has_distractor_sound = bool(n_labels)
        self.predictor = smt_net(2 + n_labels, HW, 2, 0).cuda()

    def cnn_forward(self, observations):
        s = observations["spectrogram"].permute(0, 3, 1, 2)
        if self.has_distractor_sound:
            labels = observations["category"]
            s = torch.cat([s, labels.reshape(labels.shape + (1, 1)).expand(labels.shape + s.shape[-2:])], dim=1)
        return self.predictor(s)

    def update(self, observations, dones):
        raise NotImplementedError


class Fused(Predictor):
    pass


patch_belief_predictor(Fused, networks=True, training=True)


def macs(c_in):
    """Forward multiply-adds of one row, counted from the layer shapes."""
    h, w, total, ic = HW[0], HW[1], c_in * 16 * 49 * HW[0] * HW[1], 16
    for s, oc in enumerate((16, 32, 64, 128)):
        for blk in range(2):
            stride = 2 if s and blk == 0 else 1
            ho, wo = (h - 1) // stride + 1, (w - 1) // stride + 1
            total += ho * wo * oc * (ic * 9 + oc * 9 + (ic if stride == 2 else 0))
            h, w, ic = ho, wo, oc
    return total + 128 * h * w * 2


def one_call(m, mb, gts, opt):
    x = mb["spectrogram"]
    for _ in range(5):
        opt.zero_grad()
        pred = m.cnn_forward(mb)
        masks = (torch.sum(x.reshape(x.shape[0], -1), dim=1, keepdim=True) != 0).float()
        loss = torch.nn.functional.mse_loss(masks * pred, masks * gts)
        loss.backward()
        opt.step()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1200)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print("card:", card)
    B = a.rows
    print("| channels | silent | wall: eager TF32 / eager FP32 / fused (ms) | device: eager TF32 / eager FP32 / "
          "fused (ms) | fused counted TFLOP/s over device time |")
    for n_labels in (0, 21):
        for frac in (0.0, 0.5, 0.9):
            g = torch.Generator().manual_seed(1)
            x = torch.rand((B, HW[0], HW[1], 2), generator=g) * 3
            x[torch.rand(B, generator=g) < frac] = 0
            mb = {"spectrogram": x.cuda()}
            if n_labels:
                mb["category"] = torch.nn.functional.one_hot(torch.randint(0, 21, (B,), generator=g), 21).float().cuda()
            gts = torch.randn((B, 2), generator=g).cuda()
            ways = {"tf32": Predictor(n_labels), "fp32": Predictor(n_labels), "fused": Fused(n_labels)}
            opts = {k: torch.optim.Adam(m.predictor.parameters(), lr=1e-3) for k, m in ways.items()}
            times = {k: [] for k in ways}
            for rep in range(a.reps + 1):
                for k, m in ways.items():
                    torch.backends.cudnn.allow_tf32 = k == "tf32"
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    one_call(m, mb, gts, opts[k])
                    torch.cuda.synchronize()
                    if rep:
                        times[k].append((time.perf_counter() - t0) * 1e3)
            dev = {}
            for k, m in ways.items():
                torch.backends.cudnn.allow_tf32 = k == "tf32"
                torch.cuda.synchronize()
                with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                    one_call(m, mb, gts, opts[k])
                    torch.cuda.synchronize()
                dev[k] = sum(e.self_device_time_total for e in prof.key_averages()) / 1e3
            torch.backends.cudnn.allow_tf32 = True
            med = {k: sorted(v)[len(v) // 2] for k, v in times.items()}
            flop = 5 * 3 * 2 * macs(2 + n_labels) * B          # forward + backward ~ 3x forward, 5 epochs
            print(f"| {2 + n_labels} | {frac} | {med['tf32']:.1f} / {med['fp32']:.1f} / {med['fused']:.1f} | "
                  f"{dev['tf32']:.1f} / {dev['fp32']:.1f} / {dev['fused']:.1f} | {flop / dev['fused'] / 1e9:.1f} |")


if __name__ == "__main__":
    main()
