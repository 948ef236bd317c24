"""Wall time per SAVi ``BeliefPredictor.update`` call, the reference-shaped stand-in (tests/test_belief_host.py: per-env
host loops, as belief_predictor.py:136-202) against the same class patched by ``patch_belief_predictor``, alternated in
one process:
  nets   the two networks run: torchvision resnet18 (weights=None, 2-channel conv1) with a 23-column location head and a
         21-column label head, eval mode
  given  the networks return precomputed CUDA predictions (isolates the per-env part)
at B = 8 (the SAVi configs' envs per process) and 16, on 16 kHz observations (65, 26, 2) with silent rows and dones.
Per call: host clock around --iters back-to-back calls ending in a synchronise, after warm-up; --reps rounds.  Prints
the card name and power limit, and one JSON line.

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
from test_belief_host import Fixed, make_reference_class  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name(0)


def resnet(n_out):
    import torchvision
    m = torchvision.models.resnet18(weights=None)
    m.conv1 = torch.nn.Conv2d(2, 64, kernel_size=7, stride=2, padding=3, bias=False)
    m.fc = torch.nn.Linear(512, n_out)
    return m.cuda().eval()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=1000)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    print("card:", card())
    torch.manual_seed(0)
    nets = (resnet(23), resnet(21))
    shape, slots = (65, 26, 2), 16
    results = {}
    for B in (8, 16):
        seq = bo.make_sequence(B, slots, B, loc_cols=23)
        obs = []
        for t in range(slots):
            obs.append({"spectrogram": torch.from_numpy(bo.make_spectrograms(seq["silent"][t], shape, t)).cuda(),
                        "pose": torch.from_numpy(seq["pose"][t]).cuda(), "location_belief": torch.zeros(B, 2, device="cuda"),
                        "category_belief": torch.zeros(B, 21, device="cuda")})
        dones = [[bool(d) for d in seq["dones"][t]] for t in range(slots)]
        preds = [(torch.from_numpy(seq["loc_pred"][t]).cuda(), torch.from_numpy(seq["label_pred"][t]).cuda())
                 for t in range(slots)]
        for mode in ("nets", "given"):
            models = {}
            for way in ("reference", "patched"):
                cls = make_reference_class()
                if way == "patched":
                    patch_belief_predictor(cls)
                if mode == "nets":
                    models[way] = cls(B, predictor=nets[0], classifier=nets[1])
                else:
                    models[way] = cls(B, predictor=Fixed(), classifier=Fixed())

            def run(model, n):
                for i in range(n):
                    t = i % slots
                    if mode == "given":
                        model.predictor.out, model.classifier.out = preds[t]
                    model.update(obs[t], dones[t])

            for m in models.values():
                run(m, 50)
            torch.cuda.synchronize()
            times = {w: [] for w in models}
            for _ in range(args.reps):
                for way, m in models.items():
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    run(m, args.iters)
                    torch.cuda.synchronize()
                    times[way].append((time.perf_counter() - t0) * 1e6 / args.iters)
            for way, ts in times.items():
                results[f"B{B}_{mode}_{way}_us"] = [round(x, 1) for x in ts]
                print(f"B={B:3d} {mode:5s} {way:9s} us/call: " + " ".join(f"{x:8.1f}" for x in ts))
    print(json.dumps({"card": card(), **results}))


if __name__ == "__main__":
    main()
