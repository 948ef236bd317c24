"""Observation (N, 65, T', 2) -> AudioCNN embedding (N, hidden) three ways, alternated in one process:
  torch   permute + cnn (cuDNN, TF32 off)
  conv1   ssb_audio_conv1_batch + cnn[2:] (what AudioPolicy.forward_fused runs)
  fused   ssb_audio_encoder_batch (conv kernel + linear kernel)
  patched the AudioCNN.forward of patch_audio_cnn (its host checks, then the fused entry)
plus, with --alt-lib PATH [PATH ...], ssb_audio_encoder_batch of other builds of libssb200.so (design comparisons).
With --savi: SAVi's encoder with a distractor sound (16 kHz, conv1 Conv2d(23 -> 32), hidden 128) two ways,
  torch   permute + expand + cat of the one-hot category + cnn (savi/models/audio_cnn.py:135-150; cuDNN, TF32 off)
  fused   ssb_audio_encoder_category_batch (the category folded into conv1's bias; conv kernel + linear kernel)
  patched the AudioCNN.forward of patch_audio_cnn(cls, category=True)
CUDA events around --iters back-to-back calls after warm-up; --reps rounds.  Prints the card name and power limit.

The one-CTA-per-env numbers in DESIGN.md come from a build of csrc/ssb200.cu with two constants changed,
ENC_CL = 1 and ENC_TPB = 1024, compiled with _lib.NVCC_FLAGS (the build keeps the include paths of a copy of the tree):

    sed -e 's/^constexpr int ENC_CL = 8;.*/constexpr int ENC_CL = 1;/' \
        -e 's/^constexpr int ENC_TPB = 256;/constexpr int ENC_TPB = 1024;/' soundspaces_b200/csrc/ssb200.cu > COPY/soundspaces_b200/csrc/ssb200.cu
    nvcc -shared -Xcompiler -fPIC -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -o lib_cl1.so COPY/soundspaces_b200/csrc/ssb200.cu
    python scratch/encoder_bench.py [--iters 1000] [--reps 3] [--profile] [--alt-lib lib_cl1.so]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

sys.path.insert(0, os.getcwd())
sys.path.insert(0, os.path.join(os.getcwd(), "tests"))
import torch  # noqa: E402

from soundspaces_b200 import _lib  # noqa: E402
from soundspaces_b200.encoder import patch_audio_cnn  # noqa: E402
from soundspaces_b200.renderer import WaveformOps, spectrogram_shape  # noqa: E402
from test_encoder_host import reference_classes  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name(0)


class AltLib:
    """ssb_audio_encoder_batch of another build, with its own context."""

    def __init__(self, path):
        self.lib = C.CDLL(os.path.abspath(path))
        fn = self.lib.ssb_audio_encoder_batch
        fn.restype, fn.argtypes = _lib.EXPORTS["ssb_audio_encoder_batch"]
        self.lib.ssb_create.argtypes = [C.c_int, C.POINTER(C.c_void_p)]
        self.h = C.c_void_p()
        assert self.lib.ssb_create(0, C.byref(self.h)) == 0
        self.name = os.path.basename(path)

    def runner(self, x, cnn):
        n, H, W, _ = x.shape
        layers = (_lib.Conv2dLayer * 3)()
        for i, (c, relu) in enumerate(((cnn[0], 1), (cnn[2], 1), (cnn[4], 0))):
            layers[i] = _lib.Conv2dLayer(c.weight.data_ptr(), c.bias.data_ptr(), c.out_channels, *c.kernel_size,
                                         *c.stride, relu)
        lin = cnn[6]
        feats = torch.empty((n, lin.in_features), device="cuda")
        out = torch.empty((n, lin.out_features), device="cuda")
        st = C.c_void_p(torch.cuda.current_stream().cuda_stream)

        def run():
            rc = self.lib.ssb_audio_encoder_batch(self.h, n, x.data_ptr(), H, W, layers, lin.weight.data_ptr(),
                                                  lin.bias.data_ptr(), lin.out_features, 1, feats.data_ptr(),
                                                  out.data_ptr(), st)
            assert rc == 0
            return out
        return run


def time_ways(ways, args, sr, B):
    """Check every way against ways["torch"], then time them alternated: {way: [us per call per round]}."""
    with torch.no_grad():
        ref = ways["torch"]().clone()
        for name, fn in ways.items():
            err = (fn() - ref).abs().max().item()
            assert err <= 1e-3 * max(1.0, ref.abs().max().item()), (name, err)
        for fn in ways.values():                      # warm-up (cuDNN algorithm choice, module load)
            for _ in range(50):
                fn()
        torch.cuda.synchronize()
        times = {k: [] for k in ways}
        for _ in range(args.reps):
            for name, fn in ways.items():
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                for _ in range(args.iters):
                    fn()
                b.record()
                b.synchronize()
                times[name].append(a.elapsed_time(b) * 1000.0 / args.iters)
        if args.profile:                                  # per-kernel device time, in a pass of its own
            from torch.profiler import ProfilerActivity, profile
            for name, fn in ways.items():
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    for _ in range(100):
                        fn()
                    torch.cuda.synchronize()
                evs = [e for e in prof.key_averages() if e.device_time_total > 0]
                print(json.dumps({"sr": sr, "B": B, "way": name, "device_us_per_call":
                                  round(sum(e.device_time_total for e in evs) / 100, 2)}))
                print(json.dumps({"sr": sr, "B": B, "way": name, "kernel_us_per_launch":
                                  {e.key: round(e.device_time_total / e.count, 2) for e in evs}}))
    return times


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=1000)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--alt-lib", nargs="*", default=[])
    ap.add_argument("--profile", action="store_true", help="also print per-kernel device times (torch.profiler)")
    ap.add_argument("--savi", action="store_true",
                    help="SAVi with a distractor sound instead: 16 kHz, 23-channel conv1, hidden 128")
    args = ap.parse_args()
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.benchmark = True
    print("card:", card())
    ops = WaveformOps.get("cuda:0")
    alts = [AltLib(p) for p in args.alt_lib]
    AvNav, _, Savi = reference_classes()
    patch_audio_cnn(AvNav)
    patch_audio_cnn(Savi, category=True)
    results = []
    for sr in ((16000,) if args.savi else (16000, 44100)):
        shape = spectrogram_shape(sr)
        torch.manual_seed(0)
        if args.savi:
            model = Savi(shape, hidden=128, has_distractor_sound=True).cuda().eval()
        else:
            model = AvNav(shape, hidden=512).cuda().eval()
        cnn = model.cnn
        for B in (16, 128):
            x = torch.rand((B,) + shape, device="cuda") * 3.0
            if args.savi:
                lab = torch.nn.functional.one_hot(torch.randint(0, 21, (B,), device="cuda"), 21).float()

                def reference(x=x, lab=lab):          # savi/models/audio_cnn.py:135-150
                    a = x.permute(0, 3, 1, 2)
                    return cnn(torch.cat([a, lab.reshape(lab.shape + (1, 1)).expand(lab.shape + a.shape[-2:])], dim=1))
                ways = {"torch": reference, "fused": lambda x=x, lab=lab: ops.audio_encoder(x, cnn, category=lab),
                        "patched": lambda x=x, lab=lab: model({"audiogoal": x, "category": lab})}
            else:
                ways = {
                    "torch": lambda x=x: cnn(x.permute(0, 3, 1, 2)),
                    "conv1": lambda x=x: cnn[2:](ops.audio_conv1(x, cnn[0], relu=True)),
                    "fused": lambda x=x: ops.audio_encoder(x, cnn),
                    "patched": lambda x=x: model({"spectrogram": x}),
                }
                for a in alts:
                    ways["fused:" + a.name] = a.runner(x, cnn)
            times = time_ways(ways, args, sr, B)
            row = {"sr": sr, "B": B, "us_per_call": {k: [round(t, 2) for t in v] for k, v in times.items()}}
            if args.savi:
                row["mode"] = "savi_distractor"
            results.append(row)
            print(json.dumps(row))
    return results


if __name__ == "__main__":
    main()
