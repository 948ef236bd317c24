"""The default partitioned schedule (``mac_ifft_cluster_kernel``) at the shapes where its host decisions change.

It runs the N = 4096 plan.  The host picks CL CTAs per env, the largest power of two <= min(8, n_blocks), and each CTA
takes ceil(n_blocks / CL) blocks in rounds of at most 3 receive buffers.  Every cluster size is run at n_blocks = CL - 1,
CL and CL + 1 (and 1), and at 24 blocks (3 per CTA: one round) and 25 (two rounds).
Requests mix both partition-sum paths (offset 0 with every window cached; offsets, wrap, > 8 partitions),
distractors, silent envs and short windows whose blocks end on different ranks.  Every waveform is checked against
the float64 direct formula (tests/conv_ref.py)."""
import numpy as np
import pytest

from conv_ref import direct
from oracle import audio_oracle as ao
from synth import make_rir, make_source
from test_gpu_parity import check_spec, check_wave

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")


@pytest.mark.parametrize("n_blocks", [1, 2, 3, 4, 5, 7, 8, 9, 24, 25])
def test_cluster_schedule_shapes(n_blocks):
    from soundspaces_b200 import AudioRequest, BatchedAudioRenderer
    log2n = 12
    P = (1 << log2n) // 2
    sr = max(n_blocks * P - 37, 600) if n_blocks > 1 else 1000      # a partial last block
    max_taps = min(9 * P + 1, 40000)
    r = BatchedAudioRenderer(sr, max_taps, device="cuda:0", n_terms=2, log2n=log2n, xpool_bytes=256 << 20)
    rng = np.random.default_rng(1000 * log2n + n_blocks)
    clips = [make_source(40 + n_blocks, 2 * sr + 11), make_source(41, 700)]
    lens = sorted({L for L in (1, P - 1, P + 1, 3 * P + 7, max_taps) if L <= max_taps})
    rirs = [make_rir(60 + i, L) for i, L in enumerate(lens)] + [None]
    outs = (sr, 1, min(P + 1, sr), max(1, sr - P - 3))
    specs = []
    for k in range(14):
        ri = int(rng.integers(len(rirs)))
        n = int(outs[k % len(outs)])
        if k < 6:                                   # offset 0, no wrap: the fast path when the RIR fits 8 partitions
            spec = (0, ri, 0, n, False, False, None)
        else:                                       # an offset inside the clip, as the reference draws them
            ci = int(rng.integers(2))
            spec = (ci, ri, int(rng.integers(0, len(clips[ci]))), n, bool(rng.integers(2)), k == 9, None)
        if k in (3, 8, 11):
            spec = spec[:6] + ((int(rng.integers(2)), int(rng.integers(len(rirs)))),)
        specs.append(spec)
    sids = [r.add_source(c) for c in clips]
    rids = r.add_rirs(rirs)
    reqs = []
    for ci, ri, off, n, wrap, silent, dis in specs:
        q = AudioRequest(rir=rids[ri], source=sids[ci], offset=off, out_samples=n, wrap=wrap, silent=silent)
        if dis is not None:
            q.distractor_source, q.distractor_rir = sids[dis[0]], rids[dis[1]]
        reqs.append(q)
    batch = r.prepare(reqs)
    assert batch.plan.log2n == log2n and batch.plan.n_blocks == n_blocks
    spec, wave = r.execute(batch, want_wave=True)
    torch.cuda.synchronize()
    spec, wave = spec.cpu().numpy(), wave.cpu().numpy()
    for i, (ci, ri, off, n, wrap, silent, dis) in enumerate(specs):
        ref = np.zeros((2, sr)) if silent else direct(clips[ci], rirs[ri], sr, off, n, wrap)
        if dis is not None and not silent:
            ref = ref + direct(clips[dis[0]], rirs[dis[1]], sr, 0, n, False)
        check_wave(wave[i], ref)
        check_spec(spec[i], ao.compute_spectrogram(wave[i]))
