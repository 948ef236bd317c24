"""SAVi's visual encoder (SMTCNN, RGB-D at 128 x 128): eager forward with cuDNN TF32 off and at its default, against
the patched forward (ssb_smt_cnn_batch), per call.

    python scratch/smt_cnn_bench.py [--calls 200] [--rounds 3] [--out results.json]

Per B in 8, 16, 64, 128: CUDA events around `calls` calls, the three modes alternated `rounds` times (median
reported); then, in a separate torch.profiler run of 20 calls per mode, the summed device time of the kernels per call
and the number of kernel launches per call.  Prints the card and its power limit as found (nothing is changed), one
JSON line per B and a table; `--out` also writes the whole result as JSON."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

from smt_cnn_models import SMTCNN, observations, set_params  # noqa: E402
from soundspaces_b200.encoder import fused_smt_cnn_forward  # noqa: E402


class ResizeCenterCropper(torch.nn.Module):
    """The reference's eager ops (ss_baselines/common/utils.py:341-466): area interpolate, then a slice."""

    def __init__(self):
        super().__init__()
        self._size, self.channels_last = (64, 64), False

    def forward(self, x):
        h, w = x.shape[-2:]
        scale = 64 / min(h, w)
        h, w = int(h * scale), int(w * scale)
        x = F.interpolate(x.float(), size=(h, w), mode="area").to(dtype=x.dtype)
        sx, sy = w // 2 - 32, h // 2 - 32
        return x[..., sy:sy + 64, sx:sx + 64]


ResizeCenterCropper.__module__ = "ss_baselines.common.utils"


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None, help="also write the result as JSON to this file")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a GPU")
    model = set_params(SMTCNN({"rgb": 3, "depth": 1}, obs_transform=ResizeCenterCropper()), 1).cuda().eval()

    def eager(obs, tf32):
        torch.backends.cudnn.allow_tf32 = tf32
        return model(obs)

    def fused(obs):
        out = fused_smt_cnn_forward(model, obs)
        assert out is not None, "the fused path refused the call"
        return out

    modes = {"eager_fp32": lambda o: eager(o, False), "eager_tf32": lambda o: eager(o, True), "fused": fused}
    tf32_default = torch.backends.cudnn.allow_tf32
    res = {"card": card(), "calls": a.calls, "rounds": a.rounds, "rows": []}
    print("card:", res["card"], flush=True)
    for B in (8, 16, 64, 128):
        obs = {k: v.cuda() for k, v in observations(B, 128, 128, seed=B).items()}
        row = {"B": B}
        with torch.no_grad():
            want = modes["eager_fp32"](obs)
            got = fused(obs)
            row["max_rel_err_vs_fp32"] = ((got - want).abs().max() / want.abs().max()).item()
            times = {m: [] for m in modes}
            for m, f in modes.items():                 # warm-up: module loads, cuDNN algorithm choice
                for _ in range(10):
                    f(obs)
            torch.cuda.synchronize()
            for _ in range(a.rounds):
                for m, f in modes.items():
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    for _ in range(a.calls):
                        f(obs)
                    e1.record()
                    torch.cuda.synchronize()
                    times[m].append(e0.elapsed_time(e1) * 1e3 / a.calls)
            for m in modes:
                row[f"{m}_us"] = sorted(times[m])[len(times[m]) // 2]
            for m, f in modes.items():
                from torch.profiler import ProfilerActivity, profile
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    for _ in range(20):
                        f(obs)
                    torch.cuda.synchronize()
                evs = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
                kern = [e for e in evs if "memcpy" not in e.name.lower() and "memset" not in e.name.lower()]
                row[f"{m}_device_us"] = sum(e.device_time for e in kern) / 20
                row[f"{m}_kernels"] = len(kern) / 20
        torch.backends.cudnn.allow_tf32 = tf32_default
        res["rows"].append(row)
        print(json.dumps(row), flush=True)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)
    print("| B | eager FP32 us | eager TF32 us | fused us | device us FP32 / TF32 / fused | kernels FP32 / TF32 / fused |")
    for r in res["rows"]:
        print("| %d | %.0f | %.0f | %.0f | %.0f / %.0f / %.0f | %.0f / %.0f / %.0f |" % (
            r["B"], r["eager_fp32_us"], r["eager_tf32_us"], r["fused_us"], r["eager_fp32_device_us"],
            r["eager_tf32_device_us"], r["fused_device_us"], r["eager_fp32_kernels"], r["eager_tf32_kernels"],
            r["fused_kernels"]))


if __name__ == "__main__":
    main()
