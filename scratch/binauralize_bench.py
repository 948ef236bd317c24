"""Ambisonic -> binaural conversion timings (DESIGN.md section 4, "Ambisonic trees").

  python scratch/binauralize_bench.py                 # on a GPU: decode per batch + tree conversion files/s
  python scratch/binauralize_bench.py --tool PATH     # the closed AmbisonicBinauralizer on the same synthetic tree
                                                        # (host CPUs, the script's 4 angles x scenes in parallel)

Decode: 64 inputs x 4 angles at L = 48000 (3 s at 16 kHz), K = 4, 9, 16; one multi-azimuth call that reads each input
once, against four one-azimuth calls (the input read once per angle, as a replicated batch would), and at K = 9
against ssb_sh_decode_batch on the input replicated 4x in memory.  Events around 20 calls after 3 warm-up calls,
three alternated rounds.  Tree: a seeded synthetic tree on local disk (4 scenes x 100 files, 9 channels, 4000-20000
samples) converted at 0/90/180/270.
"""
import argparse
import os
import shutil
import subprocess
import sys
import tempfile
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
from make_sh_orders_golden import write_wav  # noqa: E402

SCENES, FILES = 4, 100


def make_tree(root, seed=0):
    rng = np.random.default_rng(seed)
    n_bytes = 0
    for s in range(SCENES):
        d = os.path.join(root, f"scene{s}", "irs")
        os.makedirs(d)
        for f in range(FILES):
            L = int(rng.integers(4000, 20000))
            x = (rng.standard_normal((L, 9)) * np.exp(-np.arange(L) / (L / 5.0))[:, None] * 0.3).astype(np.float32)
            write_wav(os.path.join(d, f"{f}_{s}.wav"), x, 16000, "f32")
            n_bytes += x.nbytes
    return SCENES * FILES, n_bytes


def time_tool(tool):
    with tempfile.TemporaryDirectory() as d:
        amb, out = os.path.join(d, "amb"), os.path.join(d, "bin")
        n, nb = make_tree(amb)
        jobs = [(s, a) for s in sorted(os.listdir(amb)) for a in (0, 90, 180, 270)]

        def run(job):
            s, a = job
            subprocess.run([tool, "-i", os.path.join(amb, s, "irs"), "-o", os.path.join(out, s, str(a)), "-a", str(a)],
                           check=True, capture_output=True)
        t0 = time.perf_counter()
        with ThreadPoolExecutor(max_workers=160) as ex:
            list(ex.map(run, jobs))
        dt = time.perf_counter() - t0
    print(f"tool: {n} files x 4 angles ({nb / 1e6:.0f} MB in) in {dt:.2f} s = {n / dt:.1f} input files/s "
          f"on {os.cpu_count()} CPUs")


def time_gpu():
    import torch
    from soundspaces_b200 import BatchedAudioRenderer
    from soundspaces_b200.binauralize import binauralize_tree
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    print("gpu:", q)
    r = BatchedAudioRenderer(16000, 4096, device="cuda:0")
    L, n = 48000, 64
    angles = torch.tensor([0.0, 90.0, 180.0, 270.0])

    def timed(fn, steps=20, warm=3):
        for _ in range(warm):
            fn()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        a.record()
        for _ in range(steps):
            fn()
        b.record()
        b.synchronize()
        return a.elapsed_time(b) / steps

    for K in (4, 9, 16):
        amb = torch.randn((n, L, K), device="cuda:0") * 0.05
        arms = {"shared (1 call, A=4)": lambda: r.sh_decode_angles(amb, angles),
                "per angle (4 calls, A=1)": lambda: [r.sh_decode_angles(amb, angles[a:a + 1]) for a in range(4)]}
        if K == 9:
            rep = amb.repeat_interleave(4, dim=0).contiguous()
            az_rep = angles.repeat(n)
            arms["replicated (ssb_sh_decode_batch, B=256)"] = lambda: r.sh_decode(rep, az_rep)
        res = {k: [] for k in arms}
        for _ in range(3):
            for k, fn in arms.items():
                res[k].append(timed(fn))
        for k, v in res.items():
            print(f"K={K:2d} L={L} {n}x4: {k}: " + " / ".join(f"{x:.2f}" for x in v) + " ms per batch")
        del amb
        torch.cuda.empty_cache()
    with tempfile.TemporaryDirectory() as d:
        amb, out = os.path.join(d, "amb"), os.path.join(d, "bin")
        n_files, nb = make_tree(amb)
        for rnd in range(2):
            shutil.rmtree(out, ignore_errors=True)
            t0 = time.perf_counter()
            counts = binauralize_tree(amb, out, device="cuda:0")
            dt = time.perf_counter() - t0
            print(f"tree round {rnd}: {counts} ({nb / 1e6:.0f} MB in) in {dt:.2f} s = {n_files / dt:.1f} input files/s "
                  f"on {os.cpu_count()} CPUs")


if __name__ == "__main__":
    p = argparse.ArgumentParser()
    p.add_argument("--tool", default=None)
    args = p.parse_args()
    time_tool(args.tool) if args.tool else time_gpu()
