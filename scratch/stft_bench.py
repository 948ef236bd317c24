"""spectrogram_kernel alone on the bench workload's batch (C2: 128 envs x 44.1 kHz -> (65, 69, 2)), per library build.

    python scratch/stft_bench.py [lib_a.so lib_b.so ...]   # one subprocess per library (SSB200_LIB), alternated 3 times
    python scratch/stft_bench.py --child                   # measures the library named by SSB200_LIB (default: in-tree)

Per library:
  all   ssb_spectrogram_batch on the rendered waveforms: every env transformed (the entry has no requests);
        CUDA events around 1000 back-to-back launches after 100 warm-up launches.
  dead  the spectrogram launch inside ssb_render_batch with the bench's requests (5 % silent envs), one internal
        stream so nothing overlaps the kernel; the library's per-kernel events over 1000 renders.
  live  as dead with no silent env.
and a SHA-256 of the spectrograms of both render request sets, which every build must reproduce bit for bit."""
import hashlib, os, subprocess, sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def child():
    sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
    import numpy as np, torch
    import bench
    from soundspaces_b200 import AudioRequest, BatchedAudioRenderer, _lib
    from synth import make_source
    B, SR, TAPS, N = bench.ENVS_PER_GPU, bench.SR, bench.TAPS, 1000
    r = BatchedAudioRenderer(SR, TAPS, device="cuda:0")
    sid = r.add_source(make_source(7, SR))
    ids = r.set_dense_rir_bank(torch.from_numpy(bench.make_bank_host(B)).cuda())
    sil = bench.silent_mask(B)
    dead = r.prepare([AudioRequest(rir=ids[i], source=sid, silent=bool(sil[i])) for i in range(B)])
    live = r.prepare([AudioRequest(rir=ids[i], source=sid) for i in range(B)])
    h = hashlib.sha256()
    for b in (dead, live):
        h.update(r.execute(b).cpu().numpy().tobytes())
    spec, wave = r.execute(live, want_wave=True)
    wave = wave.clone()
    out = torch.empty_like(spec)
    st = r._stream()

    def all_envs():
        r.ctx.check(r.lib.ssb_spectrogram_batch(r.ctx.handle, B, wave.data_ptr(), SR, SR, r.pad_mode, out.data_ptr(), st),
                    "ssb_spectrogram_batch")
    for _ in range(100):
        all_envs()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(N):
        all_envs()
    e1.record()
    torch.cuda.synchronize()
    res = {"all": e0.elapsed_time(e1) / N}
    r.set_streams(1)
    for name, b in (("dead", dead), ("live", live)):
        for _ in range(100):
            r.execute(b, out=spec)
        r.ctx.set_kernel_timing(True)
        r.ctx.get_kernel_timing()
        for _ in range(N):
            r.execute(b, out=spec)
        ms, cnt = r.ctx.get_kernel_timing()["spectrogram_kernel"]
        r.ctx.set_kernel_timing(False)
        res[name] = ms / cnt
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()[0]
    print("STFT %-24s all %.4f ms  dead %.4f ms  live %.4f ms  silent %d/%d  sha256 %s  [%s]" % (
        os.path.basename(_lib.LIB_PATH), res["all"], res["dead"], res["live"], int(sil.sum()), B, h.hexdigest()[:16], gpu),
        flush=True)


def main():
    libs = sys.argv[1:] or [""]
    for _ in range(3 if len(libs) > 1 else 1):
        for lib in libs:
            env = dict(os.environ)
            if lib:
                env["SSB200_LIB"] = os.path.abspath(lib)
            subprocess.run([sys.executable, os.path.abspath(__file__), "--child"], env=env, check=True)


if __name__ == "__main__":
    child() if sys.argv[1:] == ["--child"] else main()
