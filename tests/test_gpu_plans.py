"""Both convolution plans on randomised requests at the rates and tap counts the golden cases do not reach, and the
stream / chunk splitting of the partitioned plan.

* single-block plan (``conv64k_kernel`` / ``src64k_kernel``): arbitrary offsets, wrap, short windows, clips shorter
  than the shift D = 65536 - sr, and effective tap counts on both sides of every 16384-tap step of phase A's RIR fold
  up to the eligibility limit 65536 - sr + 1; the same batch on the partitioned plan agrees to rounding;
* partitioned plan at 512 Hz ... 96 kHz (a partial last block, a single block shorter than P) with distractors;
* ``ssb_render_batch`` split over internal streams and chunks is bit-identical to one stream, one chunk.

Every waveform is checked against the float64 direct formula (tests/conv_ref.py)."""
import numpy as np
import pytest

from conv_ref import direct
from oracle import audio_oracle as ao
from synth import make_rir, make_source
from test_gpu_parity import check_spec, check_wave, renderer

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")


def _requests(r, sids, rids, specs):
    """specs: (clip, rir, offset, out_samples, wrap, silent, distractor (clip, rir) or None) -> AudioRequests."""
    from soundspaces_b200 import AudioRequest
    reqs = []
    for ci, ri, off, n, wrap, silent, dis in specs:
        q = AudioRequest(rir=rids[ri], source=sids[ci], offset=off, out_samples=n, wrap=wrap, silent=silent)
        if dis is not None:
            q.distractor_source, q.distractor_rir = sids[dis[0]], rids[dis[1]]
        reqs.append(q)
    return reqs


def _reference(clips, rirs, sr, spec):
    ci, ri, off, n, wrap, silent, dis = spec
    if silent:
        return np.zeros((2, sr))
    ref = direct(clips[ci], rirs[ri], sr, off, n, wrap)
    if dis is not None:                         # the whole distractor clip in full mode, cut to [:out_samples]
        ref = ref + direct(clips[dis[0]], rirs[dis[1]], sr, 0, n, False)
    return ref


# effective tap counts on both sides of each 16384-tap step of conv64k_kernel's phase A (nq2 = ceil(taps / 16384))
NQ2_TAPS = (1, 16384, 16385, 32768, 32769, 49152, 49153)


def single_block_requests(sr):
    """Clips, RIRs and request specs for the single-block plan at rate sr (see the test below)."""
    limit = 65536 - sr + 1
    D = 65536 - sr
    taps = sorted({t for t in NQ2_TAPS if t <= limit} | {limit})
    rng = np.random.default_rng(sr)
    S_long = limit + 2 * sr + 123
    clips = [make_source(500 + i, n) for i, n in enumerate((700, D - 1, sr, S_long))]
    lens = sorted(set(taps) | {2, 255, 4095, min(sr, limit)})
    rirs = [make_rir(600 + i, L, tau=L) for i, L in enumerate(lens)] + [None]     # slow decay: the last taps count
    longest = lens.index(limit)
    outs = (sr, 4000, 1, 777, sr - 1)
    specs = []
    for T in taps:
        # (a) an RIR of exactly T taps with a window reaching past it: all T taps are effective
        n = int(rng.choice(outs))
        off = int(rng.integers(max(0, T - n), S_long - n))
        specs.append((3, lens.index(T), off, n, bool(rng.integers(2)), False, None))
        # (b) the longest RIR cut to exactly T effective taps by offset + out_samples = T
        n = T if T <= sr else int(rng.choice(outs))
        specs.append((3, longest, T - n, n, bool(rng.integers(2)), False, None))
    for _ in range(40):
        ci, ri = int(rng.integers(len(clips))), int(rng.integers(len(rirs)))
        S = len(clips[ci])
        off = int(rng.integers(0, S)) if rng.random() < 0.8 else 0
        specs.append((ci, ri, off, int(rng.choice(outs)), bool(rng.integers(2)), rng.random() < 0.08, None))
    return clips, rirs, specs


@pytest.mark.parametrize("sr", [8000, 16000, 22050, 44100, 61440])
def test_randomised_requests_single_block(sr):
    """The RIRs decay slowly (tau = L), so the taps phase A folds in from the later 16384-tap quarters carry weight:
    dropping the last quarter moves the 8 and 16 kHz outputs by many times the tolerance."""
    limit = 65536 - sr + 1                      # the most effective taps the single-block plan takes at this rate
    clips, rirs, specs = single_block_requests(sr)
    refs = [_reference(clips, rirs, sr, s) for s in specs]

    waves = {}
    for log2n in (0, 13):                       # 0: prefers the single-block plan; 13: the partitioned plan
        r = renderer(sr, limit, log2n=log2n)
        sids = [r.add_source(c) for c in clips]
        rids = r.add_rirs(rirs)
        batch = r.prepare(_requests(r, sids, rids, specs))
        assert batch.plan.log2n == (16 if log2n == 0 else 13)
        spec, wave = r.execute(batch, want_wave=True)
        torch.cuda.synchronize()
        spec, wave = spec.cpu().numpy(), wave.cpu().numpy()
        for i, ref in enumerate(refs):
            check_wave(wave[i], ref)
            check_spec(spec[i], ao.compute_spectrogram(wave[i]))
        waves[log2n] = wave
    # two FFT factorisations of the same convolution agree to rounding
    assert np.abs(waves[0] - waves[13]).max() <= 3e-6 * np.abs(waves[0]).max()


_partitioned = {}


@pytest.mark.parametrize("conv_mode", [0, 1])
@pytest.mark.parametrize("log2n", [12, 13, 14])
@pytest.mark.parametrize("sr", [512, 8000, 22050, 96000])
def test_randomised_requests_partitioned_rates(sr, log2n, conv_mode):
    from soundspaces_b200 import BatchedAudioRenderer
    max_taps = 20000
    key = (sr, log2n)
    if key not in _partitioned:
        _partitioned.clear()                    # one renderer (and window-spectra pool) alive at a time
        _partitioned[key] = BatchedAudioRenderer(sr, max_taps, device="cuda:0", n_terms=2, log2n=log2n,
                                                 xpool_bytes=256 << 20)
    r = _partitioned[key]
    P = r.P
    rng = np.random.default_rng(sr + log2n)
    clips = [make_source(700 + i, n) for i, n in enumerate((sr, 2 * sr + 123, 5 * sr, 700))]
    lens = sorted({L for L in (1, 2, 255, P - 1, P, P + 1, sr - 1, sr, sr + 1, 12345, max_taps) if 1 <= L <= max_taps})
    rirs = [make_rir(800 + i, L) for i, L in enumerate(lens)] + [None]
    outs = (sr, min(4000, sr), 1, min(777, sr - 1), sr - 1)
    specs = []
    for _ in range(48):
        ci, ri = int(rng.integers(len(clips))), int(rng.integers(len(rirs)))
        S = len(clips[ci])
        wrap = bool(rng.integers(2))
        off = int(rng.integers(0, S)) if rng.random() < 0.8 else 0
        silent = rng.random() < 0.05
        dis = None
        if not silent and rng.random() < 0.3:
            dis = (int(rng.integers(len(clips))), int(rng.integers(len(rirs))))
        specs.append((ci, ri, off, int(rng.choice(outs)), wrap, silent, dis))
    sids = [r.add_source(c) for c in clips]
    rids = r.add_rirs(rirs)
    r.set_conv_mode(conv_mode)
    try:
        batch = r.prepare(_requests(r, sids, rids, specs))
        assert batch.plan.log2n == log2n
        spec, wave = r.execute(batch, want_wave=True)
        torch.cuda.synchronize()
    finally:
        r.set_conv_mode(0)
    spec, wave = spec.cpu().numpy(), wave.cpu().numpy()
    for i, s in enumerate(specs):
        check_wave(wave[i], _reference(clips, rirs, sr, s))
        check_spec(spec[i], ao.compute_spectrogram(wave[i]))


@pytest.mark.parametrize("conv_mode", [0, 1])
@pytest.mark.parametrize("log2n", [12, 13])
def test_streams_and_chunks_partitioned(log2n, conv_mode):
    """Sub-batches on 1..8 internal streams, each working through 1..4 chunks, on the partitioned plan (the one with
    per-sub-batch RIR-spectrum and partition-sum scratch): bit-identical to one stream and one chunk."""
    sr = 16000
    r = renderer(sr, 20000, log2n=log2n)
    rng = np.random.default_rng(log2n)
    clips = [make_source(900, sr), make_source(901, 3 * sr + 7)]
    lens = (1, 300, 2048, 4097, 8191, 12000, 16000, 20000)
    rirs = [make_rir(910 + i, L) for i, L in enumerate(lens)] + [None]
    specs = []
    for k in range(129):
        ci = k % 2
        off = 0 if ci == 0 else int(rng.integers(0, 2 * sr))
        specs.append((ci, int(rng.integers(len(rirs))), off, int(rng.choice((sr, 4000, 777))), bool(rng.integers(2)),
                      k % 17 == 5, None))
    sids = [r.add_source(c) for c in clips]
    rids = r.add_rirs(rirs)
    reqs = _requests(r, sids, rids, specs)
    r.set_conv_mode(conv_mode)
    try:
        for B in (64, 100, 129):
            batch = r.prepare(reqs[:B])
            assert batch.plan.log2n == log2n
            r.set_streams(1)
            r.set_chunks(1)
            spec, wave = r.execute(batch, want_wave=True)
            spec, wave = spec.cpu().numpy(), wave.cpu().numpy()
            for i in (0, 1, B // 2, B - 1):
                check_wave(wave[i], _reference(clips, rirs, sr, specs[i]))
                check_spec(spec[i], ao.compute_spectrogram(wave[i]))
            for streams in (1, 2, 3, 8):
                for chunks in (1, 2, 4):
                    r.set_streams(streams)
                    r.set_chunks(chunks)
                    spec2, wave2 = r.execute(batch, want_wave=True)
                    spec2, wave2 = spec2.cpu().numpy(), wave2.cpu().numpy()
                    assert np.array_equal(wave2, wave), (B, streams, chunks, np.abs(wave2 - wave).max())
                    assert np.array_equal(spec2, spec), (B, streams, chunks, np.abs(spec2 - spec).max())
    finally:
        r.set_streams(2)                        # the context defaults
        r.set_chunks(1)
        r.set_conv_mode(0)
