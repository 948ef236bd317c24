"""Wall time per SAVi ``BeliefPredictor.update`` call, the reference-shaped stand-in (tests/test_belief_host.py: per-env
host loops, as belief_predictor.py:136-202) against the same class patched by ``patch_belief_predictor`` ("patched")
and by ``patch_belief_predictor(networks=True)`` ("patched + networks"), alternated in one process, for
  offline    torchvision resnet18 (2-channel conv1, eval mode, randomised BatchNorm) with a 23-column location head and
             a 21-column label head: the networks of configs without online training
  online2    the SMT location predictor (tests/belief_nets_models.py, 2 input channels, fc 4608 -> 2) and the
             torchvision label classifier: savi.yaml without a distractor
  online23   the same with the 23-channel SMT predictor reading observations["category"]: with a distractor
  given      the networks return precomputed CUDA predictions (isolates the per-env part; no networks variant)
at B = 8 (the SAVi configs' envs per process) and 16, on 16 kHz observations (65, 26, 2) with silent rows and dones.
Per call: host clock around --iters back-to-back calls ending in a synchronise, after warm-up; --reps rounds.  Then,
in a separate torch.profiler run, the device time per network call: eager PyTorch (cuDNN, default TF32 settings)
against the library.  Prints the card name and power limit, and one JSON line.

    python scratch/belief_bench.py [--iters 1000] [--reps 3]
"""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.getcwd())
sys.path.insert(0, os.path.join(os.getcwd(), "tests"))
import torch  # noqa: E402

import belief_oracle as bo  # noqa: E402
from soundspaces_b200.belief import patch_belief_predictor  # noqa: E402
from belief_nets_models import make_net, network_input  # noqa: E402
from soundspaces_b200.renderer import WaveformOps  # noqa: E402
from test_belief_host import Fixed, make_reference_class  # noqa: E402

PAIRS = {"offline": ("tv23", "tv21"), "online2": ("smt2", "tv21"), "online23": ("smt23", "tv21")}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name(0)


def reference_class():
    """The stand-in with ``cnn_forward`` concatenating the category when ``has_distractor_sound``, as
    belief_predictor.py:123-134 does."""
    Base = make_reference_class()

    class BeliefPredictor(Base):
        has_distractor_sound = False

        def cnn_forward(self, observations):
            labels = observations["category"] if self.has_distractor_sound else None
            return self.predictor(network_input(observations["spectrogram"], labels))

    return BeliefPredictor


def device_us_per_call(fn, n=50):
    """Summed CUDA kernel time per call of ``fn`` from torch.profiler."""
    from torch.profiler import ProfilerActivity, profile
    for _ in range(5):
        fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(n):
            fn()
        torch.cuda.synchronize()
    total = sum(e.self_device_time_total for e in prof.key_averages() if e.device_type == torch.autograd.DeviceType.CUDA)
    return total / n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=1000)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    print("card:", card())
    torch.manual_seed(0)
    nets = {k: make_net(k, seed=i).cuda() for i, k in enumerate(("tv23", "tv21", "smt2", "smt23"))}
    shape, slots = (65, 26, 2), 16
    results = {}
    data = {}
    for B in (8, 16):
        seq = bo.make_sequence(B, slots, B, loc_cols=23)
        g = torch.Generator().manual_seed(B)
        obs = []
        for t in range(slots):
            obs.append({"spectrogram": torch.from_numpy(bo.make_spectrograms(seq["silent"][t], shape, t)).cuda(),
                        "pose": torch.from_numpy(seq["pose"][t]).cuda(), "location_belief": torch.zeros(B, 2, device="cuda"),
                        "category_belief": torch.zeros(B, 21, device="cuda"),
                        "category": torch.softmax(torch.randn(B, 21, generator=g), dim=1).cuda()})
        dones = [[bool(d) for d in seq["dones"][t]] for t in range(slots)]
        preds = [(torch.from_numpy(seq["loc_pred"][t]).cuda(), torch.from_numpy(seq["label_pred"][t]).cuda())
                 for t in range(slots)]
        data[B] = (obs, dones, preds)
    models = {}
    for B in (8, 16):
        for mode in list(PAIRS) + ["given"]:
            for way in ("reference", "patched", "patched + networks"):
                if mode == "given" and way == "patched + networks":
                    continue
                cls = reference_class()
                if way != "reference":
                    patch_belief_predictor(cls, networks=way == "patched + networks")
                if mode == "given":
                    m = cls(B, predictor=Fixed(), classifier=Fixed())
                else:
                    m = cls(B, predictor=nets[PAIRS[mode][0]], classifier=nets[PAIRS[mode][1]])
                    m.has_distractor_sound = mode == "online23"
                models[(B, mode, way)] = m

    def run(key, n):
        B, mode, _ = key
        obs, dones, preds = data[B]
        model = models[key]
        for i in range(n):
            t = i % slots
            if mode == "given":
                model.predictor.out, model.classifier.out = preds[t]
            model.update(obs[t], dones[t])

    for key in models:
        run(key, 50)
    torch.cuda.synchronize()
    times = {k: [] for k in models}
    for _ in range(args.reps):
        for key in models:                  # B = 8 and 16, every pair and variant, alternated in each round
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            run(key, args.iters)
            torch.cuda.synchronize()
            times[key].append((time.perf_counter() - t0) * 1e6 / args.iters)
    for (B, mode, way), ts in times.items():
        results[f"B{B}_{mode}_{way.replace(' + ', '_')}_us"] = [round(x, 1) for x in ts]
        print(f"B={B:3d} {mode:8s} {way:18s} us/call: " + " ".join(f"{x:8.1f}" for x in ts))
    # device time per network call (separate profiler run)
    ops = WaveformOps.get("cuda:0")
    for B in (8, 16):
        obs = data[B][0][1]
        x, labels = obs["spectrogram"], obs["category"]
        for kind, net in nets.items():
            lab = labels if kind == "smt23" else None
            inp = network_input(x, lab)
            with torch.no_grad():
                eager = device_us_per_call(lambda: net(inp))
                if kind.startswith("tv"):
                    fused = device_us_per_call(lambda: ops.resnet18(x, net))
                else:
                    fused = device_us_per_call(lambda: ops.smt_resnet18(x, net, lab))
            results[f"B{B}_{kind}_device_us"] = {"eager": round(eager, 1), "library": round(fused, 1)}
            print(f"B={B:3d} {kind:6s} device us/call: eager {eager:8.1f}  library {fused:8.1f}")
    print(json.dumps({"card": card(), **results}))


if __name__ == "__main__":
    main()
