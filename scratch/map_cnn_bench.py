"""AV-WaN's map encoders and policy network, eager PyTorch / cuDNN against the library, alternated in one process, at
B in {1, 16, 64, 128}: ``MapCNN`` on the 200 x 200 x 2 and 400 x 400 x 2 geometric maps and the 20 x 20 x 1 acoustic
map (hidden 512), and a stand-in of av_wan's ``AudioNavBaselineNet.forward`` (65 x 26 audio, 200 x 200 gm, am, 128 x
128 depth visual, GRU) with every patch against none.

    python scratch/map_cnn_bench.py              # wall clock per call (CUDA events around 100 calls, 3 rounds)
    python scratch/map_cnn_bench.py --profile    # device time per kernel and per call from torch.profiler

TF32 is off for the eager path (cudnn.allow_tf32 = False), so both sides do FP32 arithmetic.  Prints the card's name
and power limit, and the max |fused - eager| / max |eager| of each case."""
import argparse
import copy
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

from avnav_models import RNNStateEncoder, VisualCNN  # noqa: E402
from map_cnn_models import AudioNavBaselineNet, MapCNN  # noqa: E402
from test_encoder_host import reference_classes  # noqa: E402
from soundspaces_b200.encoder import patch_audio_cnn, patch_map_cnn, patch_visual_cnn  # noqa: E402
from soundspaces_b200.rnn import patch_rnn_state_encoder  # noqa: E402

CALLS, ROUNDS = 100, 3


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name(0)


def patched(base, patch):
    cls = type(base.__name__ + "Fused", (base,), {})
    return patch(cls)


def make_cases(B):
    g = torch.Generator(device="cuda").manual_seed(B)
    maps = {"gm200": ("gm", (torch.rand((B, 200, 200, 2), device="cuda", generator=g) < 0.3).float()),
            "gm400": ("gm", (torch.rand((B, 400, 400, 2), device="cuda", generator=g) < 0.3).float()),
            "am20": ("am", torch.rand((B, 20, 20, 1), device="cuda", generator=g)
                     * (torch.rand((B, 20, 20, 1), device="cuda", generator=g) < 0.125).float())}
    cases = {}
    torch.manual_seed(0)
    for name, (map_type, x) in maps.items():
        eager = MapCNN(*x.shape[1:], 512, map_type).cuda().eval()
        fused = copy.deepcopy(eager)
        fused.__class__ = patched(MapCNN, patch_map_cnn)
        obs = {map_type: x}
        cases[f"map {name}"] = (lambda m=eager, o=obs: m(o), lambda m=fused, o=obs: m(o))
    spec = torch.rand((B, 65, 26, 2), device="cuda", generator=g) * 3
    depth = torch.rand((B, 128, 128, 1), device="cuda", generator=g)
    h = torch.randn(1, B, 512, device="cuda", generator=g)
    masks = (torch.arange(B, device="cuda") % 5 != 0).float()[:, None]
    AudioCNN = reference_classes()[1]
    net = AudioNavBaselineNet(AudioCNN((65, 26, 2), 512), MapCNN(200, 200, 2, 512, "gm"), MapCNN(20, 20, 1, 512, "am"),
                              VisualCNN(0, 1, 128, 128, 512, "av_wan")).cuda()
    net_f = copy.deepcopy(net)
    net_f.audio_encoder.__class__ = patched(AudioCNN, patch_audio_cnn)
    net_f.gm_encoder.__class__ = net_f.am_encoder.__class__ = patched(MapCNN, patch_map_cnn)
    net_f.visual_encoder.__class__ = patched(VisualCNN, patch_visual_cnn)
    net_f.state_encoder.__class__ = patched(RNNStateEncoder, patch_rnn_state_encoder)
    obs = {"spectrogram": spec, "gm": maps["gm200"][1], "am": maps["am20"][1], "depth": depth}
    cases["net forward (gm200)"] = (lambda: net(obs, h, masks)[0], lambda: net_f(obs, h, masks)[0])
    return cases


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--profile", action="store_true")
    args = ap.parse_args()
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    print("card:", card())
    for B in (1, 16, 64, 128):
        with torch.no_grad():
            for name, (eager, fused) in make_cases(B).items():
                want, got = eager(), fused()
                rel = ((got - want).abs().max() / want.abs().max()).item()
                for f in (eager, fused):
                    for _ in range(10):
                        f()
                torch.cuda.synchronize()
                tag = f"B={B} {name}"
                if args.profile:
                    from torch.profiler import ProfilerActivity, profile
                    for side, f in (("eager", eager), ("fused", fused)):
                        with profile(activities=[ProfilerActivity.CUDA]) as prof:
                            for _ in range(20):
                                f()
                            torch.cuda.synchronize()
                        ev = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
                        per = {}
                        for e in ev:
                            k = e.name.split("(")[0][:60]
                            per[k] = per.get(k, 0.0) + e.device_time / 20
                        print(f"{tag} {side}: device {sum(per.values()):.1f} us/call, {len(ev) / 20:.0f} kernels/call")
                        for k, v in sorted(per.items(), key=lambda kv: -kv[1]):
                            print(f"      {v:8.1f} us  {k}")
                    continue
                times = {"eager": [], "fused": []}
                for _ in range(ROUNDS):
                    for side, f in (("eager", eager), ("fused", fused)):
                        start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                        torch.cuda.synchronize()
                        start.record()
                        for _ in range(CALLS):
                            f()
                        end.record()
                        end.synchronize()
                        times[side].append(start.elapsed_time(end) / CALLS * 1e3)
                print(f"{tag}: eager {' '.join(f'{t:.1f}' for t in times['eager'])} us/call, fused "
                      f"{' '.join(f'{t:.1f}' for t in times['fused'])} us/call; max|fused-eager|/max|eager| {rel:.2e}",
                      flush=True)


if __name__ == "__main__":
    main()
