"""GPU parity: the CUDA path (through the C ABI) against the reference's golden
outputs and the CPU oracle.  Tolerances are SURVEY.md 8(c)'s:
waveform max|d| <= 1e-4 * max|ref| per env; spectrogram allclose(rtol=1e-4, atol=1e-5);
silent => exactly 0; PCM decode bit-exact."""
import importlib.util
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

from oracle import audio_oracle as ao  # noqa: E402
from synth import make_rir, make_source  # noqa: E402

_spec = importlib.util.spec_from_file_location(
    "make_golden", os.path.join(os.path.dirname(__file__), "golden", "make_golden.py"))
mg = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(mg)

WAVE_RTOL = 1e-4
SPEC_RTOL, SPEC_ATOL = 1e-4, 1e-5


def check_wave(got, ref, stride=1):
    got = np.asarray(got, dtype=np.float64)[:, ::stride]
    ref = np.asarray(ref, dtype=np.float64)
    assert got.shape == ref.shape
    peak = np.abs(ref).max()
    if peak == 0:
        assert not got.any()
    else:
        assert np.abs(got - ref).max() <= WAVE_RTOL * peak, (np.abs(got - ref).max(), peak)


def check_spec(got, ref):
    assert got.shape == ref.shape
    assert np.allclose(got, ref, rtol=SPEC_RTOL, atol=SPEC_ATOL), np.abs(got - ref).max()


_renderers = {}


def renderer(sr, max_taps, n_terms=1, log2n=0, pad_mode="reflect"):
    """log2n 12 / 13 / 14: the partitioned plan at that block size.  log2n 0 HERE: the renderer prefers the
    single-block plan (65536-point cluster kernel) for every batch that fits it and falls back to the partitioned
    default otherwise (prefer_block64=True; the library default prefers the partitioned plan, the faster one)."""
    from soundspaces_b200 import BatchedAudioRenderer
    key = (sr, max_taps, n_terms, log2n, pad_mode)
    if key not in _renderers:
        _renderers[key] = BatchedAudioRenderer(sr, max_taps, device="cuda:0", n_terms=n_terms, log2n=log2n,
                                               pad_mode=pad_mode, prefer_block64=(log2n == 0))
    return _renderers[key]


def golden_wave(golden, name):
    if f"{name}/wave" in golden:
        return golden[f"{name}/wave"], 1
    return golden[f"{name}/wave_stride5"], 5


@pytest.mark.parametrize("log2n", [13, 12, 14, 0])
@pytest.mark.parametrize("name", sorted(mg.DISCRETE_CASES))
def test_discrete_golden(golden, name, log2n):
    """log2n 12/13/14: the partitioned plan at that block size; 0: the default, i.e. the single-block 65536-point
    cluster kernel whenever the request fits it (one term, <= 65536 - sr + 1 effective taps), else partitioned."""
    from soundspaces_b200 import AudioRequest
    c = mg.DISCRETE_CASES[name]
    if log2n not in (0, 13) and name not in ("a2_16k", "a4_valid", "a5_distractor", "a2_44k"):
        pytest.skip("other FFT sizes are exercised on a subset")
    src, rir, dsrc, drir = mg.discrete_inputs(c)
    sr = c["sr"]
    for pad_mode in ("reflect", "constant"):
        r = renderer(sr, 48000, n_terms=2, log2n=log2n, pad_mode=pad_mode)
        sid = r.add_source(src)
        rid = r.add_rirs([rir])[0]
        req = AudioRequest(rir=rid, source=sid, silent=c.get("step_count", 0) > 500)
        if c["S"] != sr:
            req.offset = c.get("audio_index", 0) * sr          # simulator.py:634-647
        if dsrc is not None:
            req.distractor_source = r.add_source(dsrc)
            req.distractor_rir = r.add_rirs([drir])[0]
        batch = r.prepare([req])
        fits = dsrc is None and min(len(rir) if rir is not None else 0, req.offset + sr) <= 65536 - sr + 1
        if log2n == 0 and fits and not req.silent:
            assert batch.plan.log2n == 16, "eligible request must take the single-block plan"
        if log2n != 0 or not fits:
            assert batch.plan.log2n != 16
        spec, wave = r.execute(batch, want_wave=True)
        torch.cuda.synchronize()
        gw, stride = golden_wave(golden, name)
        check_wave(wave[0].cpu().numpy(), gw, stride)
        check_spec(spec[0].cpu().numpy(), golden[f"{name}/spec_{pad_mode}"])
        if req.silent:
            assert not spec.cpu().numpy().any() and not wave.cpu().numpy().any()


@pytest.mark.parametrize("name", sorted(mg.CONTINUOUS_CASES))
def test_continuous_golden(golden, name):
    from soundspaces_b200 import AudioRequest
    c = mg.CONTINUOUS_CASES[name]
    src, rir, last = mg.continuous_inputs(c)
    sr = c["sr"]
    r = renderer(sr, 48000, n_terms=2)
    sid = r.add_source(src)
    ids = r.add_rirs([rir] + ([last] if last is not None else []))
    kw = dict(source=sid, offset=c["sample_index"], out_samples=int(sr * 0.25), wrap=True,
              silent=c.get("step_count", 0) > 500)
    cur = AudioRequest(rir=ids[0], **kw)
    if last is not None:
        spec, wave = r.render_crossfade([cur], [AudioRequest(rir=ids[1], **kw)], want_wave=True)
    else:
        spec, wave = r.render([cur], want_wave=True)
    torch.cuda.synchronize()
    check_wave(wave[0].cpu().numpy(), golden[f"{name}/wave"])
    check_spec(spec[0].cpu().numpy(), golden[f"{name}/spec_reflect"])
    assert not wave[0, :, 4000:].cpu().numpy().any()


@pytest.mark.parametrize("sr", [16000, 44100, 48000])
@pytest.mark.parametrize("pad_mode", ["reflect", "constant"])
def test_spectrogram_only(golden, sr, pad_mode):
    r = renderer(sr, 4096, pad_mode=pad_mode)
    ones = torch.ones((1, 2, sr), dtype=torch.float32, device="cuda")
    check_spec(r.spectrogram(ones)[0].cpu().numpy(), golden[f"ones_{sr}/spec_{pad_mode}"].astype(np.float32))
    rng = np.random.default_rng(sr)
    w = (rng.standard_normal((3, 2, sr)) * np.array([1.0, 1e-3, 30.0])[:, None, None]).astype(np.float32)
    w[1, 1] = 0.0                                              # one silent ear
    got = r.spectrogram(torch.from_numpy(w).cuda()).cpu().numpy()
    for i in range(3):
        check_spec(got[i], ao.compute_spectrogram(w[i], pad_mode=pad_mode))
    # ears are packed into one complex FFT: a silent ear next to a live one sees only rounding
    # leakage (the exact-zero contract is for fully silent steps, simulator.py:610-612)
    assert np.abs(got[1, :, :, 1]).max() < 1e-7
    z = r.spectrogram(torch.zeros((2, 2, sr), dtype=torch.float32, device="cuda")).cpu().numpy()
    assert not z.any()


def test_singing_fixture(golden):
    from soundspaces_b200 import AudioRequest
    pcm = golden["singing/pcm16"]
    r = renderer(48000, 12000)
    sid = r.add_source_pcm16(pcm)
    dec = r._sources[sid]
    assert np.array_equal(dec.cpu().numpy(), ao.pcm16_to_float32(pcm))          # bit-exact decode
    assert np.array_equal(r.encode_pcm16(dec, "round").cpu().numpy(), pcm)      # bit-exact round trip
    x = ao.pcm16_to_float32(pcm) * np.float32(1.7)
    xd = torch.from_numpy(x).cuda()
    assert np.array_equal(r.encode_pcm16(xd, "demo").cpu().numpy(), ao.float32_to_pcm16_demo(x))
    assert np.array_equal(r.encode_pcm16(xd, "round").cpu().numpy(), ao.float32_to_pcm16_round(x))
    rid = r.add_rirs([make_rir(99, 12000)])[0]
    spec, wave = r.render([AudioRequest(rir=rid, source=sid)], want_wave=True)
    torch.cuda.synchronize()
    check_wave(wave[0].cpu().numpy(), golden["singing/wave_stride5"], 5)
    check_spec(spec[0].cpu().numpy(), golden["singing/spec_reflect"])


@pytest.mark.parametrize("log2n,conv_mode", [(13, 0), (13, 1), (0, 0)])
def test_ragged_batch_matches_oracle(log2n, conv_mode):
    """Mixed batch: ragged RIR lengths, zero-RIR fallback, silent envs, different offsets; the partitioned plan with
    both schedules (per-bin partition sums / fused into the inverse FFT) and the single-block plan (log2n 0:
    every request here fits it: 48000 taps <= 65536 - 16000 + 1)."""
    from soundspaces_b200 import AudioRequest
    sr = 16000
    r = renderer(sr, 48000, n_terms=2, log2n=log2n)
    r.set_conv_mode(conv_mode)
    clips = [make_source(40, sr), make_source(41, 5 * sr)]
    sids = [r.add_source(c) for c in clips]
    lens = [1, 17, 4095, 4096, 4097, 8192, 15999, 16000, 16001, 30011, 48000]
    rirs = [make_rir(100 + i, L) for i, L in enumerate(lens)] + [None, np.zeros((0, 2), np.float32)]
    rids = r.add_rirs(rirs)
    reqs, refs = [], []
    for i, rid in enumerate(rids):
        for (s, off) in ((0, 0), (1, 0), (1, sr), (1, 3 * sr), (1, 4 * sr)):
            silent = (i + off // sr) % 7 == 3
            reqs.append(AudioRequest(rir=rid, source=sids[s], offset=off, silent=silent))
            refs.append(ao.compute_audiogoal(clips[s], rirs[i], sr, silent=silent, audio_index=off // sr))
    batch = r.prepare(reqs)
    assert batch.plan.log2n == (16 if log2n == 0 else log2n)
    spec, wave = r.execute(batch, want_wave=True)
    torch.cuda.synchronize()
    spec, wave = spec.cpu().numpy(), wave.cpu().numpy()
    for i, ref in enumerate(refs):
        check_wave(wave[i], ref)
        check_spec(spec[i], ao.compute_spectrogram(ref.astype(np.float32)))
        if reqs[i].silent:
            assert not spec[i].any()
    r.set_conv_mode(0)


def test_full_size_c2_properties():
    """BASELINE config 2 at full size (128 envs, 44.1 kHz, 16384 taps): spot-check envs against the
    oracle and check size-independent properties: linearity in the RIR, batch-order independence
    (bit-identical), silence => exact zeros."""
    from soundspaces_b200 import AudioRequest
    sr, L, B = 44100, 16384, 128
    r = renderer(sr, L)
    src = make_source(7, sr)
    sid = r.add_source(src)
    rirs = np.stack([make_rir(i, L) for i in range(B)])
    rirs[5] = 0.0                                                   # zero-RIR fallback row
    rirs[64] = 2.0 * rirs[0] - 0.5 * rirs[1]                        # linear combination
    ids = r.add_rirs(list(rirs))
    reqs = [AudioRequest(rir=i, source=sid, silent=(k == 9)) for k, i in enumerate(ids)]
    assert r.prepare(reqs).plan.log2n == 16          # config 2 runs on the single-block cluster kernel
    try:
        _c2_properties(r, sr, L, B, src, rirs, reqs)
    finally:
        r.set_streams(2)                             # the context defaults
        r.set_chunks(1)


def _c2_properties(r, sr, L, B, src, rirs, reqs):
    from soundspaces_b200 import AudioRequest
    r.set_streams(1)                                 # the reference for the stream / chunk splits below
    r.set_chunks(1)
    spec, wave = r.render(reqs, want_wave=True)
    torch.cuda.synchronize()
    spec_h, wave_h = spec.cpu().numpy(), wave.cpu().numpy()
    assert spec_h.shape == (B, 65, 69, 2) and wave_h.shape == (B, 2, sr)
    # the partitioned plan on the same batch agrees to rounding (two different FFT factorizations)
    rp = renderer(sr, L, log2n=12)
    idp = rp.add_rirs(list(rirs))
    sidp = rp.add_source(src)
    wave_p = rp.render([AudioRequest(rir=i, source=sidp, silent=(k == 9)) for k, i in enumerate(idp)], want_wave=True)[1]
    torch.cuda.synchronize()
    dp = np.abs(wave_p.cpu().numpy() - wave_h).max(axis=(1, 2))
    assert (dp <= 3e-6 * np.abs(wave_h).max()).all()
    for i in (0, 1, 31, 127):
        w_ref, s_ref = ao.render_frame(src, rirs[i], sr)
        check_wave(wave_h[i], w_ref)
        check_spec(spec_h[i], s_ref)
    assert not wave_h[5].any() and not spec_h[5].any()
    assert not wave_h[9].any() and not spec_h[9].any()
    lin = 2.0 * wave_h[0].astype(np.float64) - 0.5 * wave_h[1]
    assert np.abs(wave_h[64] - lin).max() <= 1e-5 * np.abs(lin).max()
    perm = np.random.default_rng(0).permutation(B)
    spec2, wave2 = r.render([reqs[i] for i in perm], want_wave=True)
    torch.cuda.synchronize()
    assert np.array_equal(wave2.cpu().numpy(), wave_h[perm])
    assert np.array_equal(spec2.cpu().numpy(), spec_h[perm])
    # sub-batches on internal streams: bit-identical to the single-stream result
    for streams in (2, 3, 8):
        r.set_streams(streams)
        spec3, wave3 = r.render(reqs, want_wave=True)
        torch.cuda.synchronize()
        assert np.array_equal(wave3.cpu().numpy(), wave_h) and np.array_equal(spec3.cpu().numpy(), spec_h)
    # streams x chunks (each stream works through several smaller sub-batches in turn): bit-identical too
    for streams, chunks in ((2, 2), (2, 4), (3, 2), (4, 16)):
        r.set_streams(streams)
        r.set_chunks(chunks)
        spec4, wave4 = r.render(reqs, want_wave=True)
        torch.cuda.synchronize()
        assert np.array_equal(wave4.cpu().numpy(), wave_h) and np.array_equal(spec4.cpu().numpy(), spec_h)


@pytest.mark.parametrize("n_chunks", [1, 3, 4, 32])
def test_host_session_e2e(n_chunks):
    """Host-buffer entry, serial and pipelined (chunked H2D / kernels / D2H on separate streams)."""
    sr, L, B = 16000, 6000, 11
    r = renderer(sr, L)
    src = make_source(3, sr)
    sid = r.add_source(src)
    hs = r.make_host_session(B, L, want_wave=True, n_chunks=n_chunks)
    rirs = np.stack([make_rir(50 + i, L) for i in range(B)])
    taps = [L, L, 0, 1, 4097, L, L, 17, L, L, L]
    silent = [i == 4 for i in range(B)]
    for rep in range(3):                               # back-to-back steps reuse the staging buffers
        rirs = np.roll(rirs, 1, axis=0)
        hs.h_rir.numpy()[:] = rirs
        hs.set_requests(sid, silent=silent, taps=taps)
        hs.run()
    torch.cuda.synchronize()
    for i in range(B):
        w_ref, s_ref = ao.render_frame(src, rirs[i][:taps[i]], sr, silent=silent[i])
        check_wave(hs.h_wave[i].numpy(), w_ref)
        check_spec(hs.h_spec[i].numpy(), s_ref.astype(np.float32))


def test_error_reporting():
    from soundspaces_b200 import _lib
    r = renderer(16000, 6000)
    with pytest.raises(RuntimeError, match="log2n"):
        r.ctx.make_plan(16000, 100, 1, 11)
    with pytest.raises(ValueError):
        r.spectrogram(torch.zeros((1, 2, 100), device="cuda"))
    import ctypes
    rc = r.lib.ssb_spectrogram_batch(r.ctx.handle, 1, None, 100, 100, 0, None, None)
    assert rc == -1 and b"ssb_spectrogram_batch" in r.lib.ssb_last_error(r.ctx.handle)
    assert _lib.load_library().ssb_version() >= 100


def test_intensity_sensor_kernel():
    """N3: AV-WaN Intensity (avwan_sensors.py:91-100) on the device vs the oracle."""
    sr = 16000
    r = renderer(sr, 6000)
    rng = np.random.default_rng(4)
    waves = []
    for i in range(6):
        w = (rng.standard_normal((2, sr)) * np.exp(-np.arange(sr) / 3000.0)).astype(np.float32)
        w[:, : 500 * i] *= 1e-3                       # onset later and later
        waves.append(w)
    waves.append(np.zeros((2, sr), np.float32))       # silent: onset 0, mean square 0
    late = np.zeros((2, sr), np.float32); late[0, sr - 20] = 1.0     # window clipped at the end of the clip
    waves.append(late)
    neg = -np.abs(waves[0])                           # max <= 0: every sample of the max ear passes, onset per argmax rule
    waves.append(neg.astype(np.float32))
    w = np.stack(waves)
    got = r.intensity(torch.from_numpy(w).cuda()).cpu().numpy()
    for i in range(len(w)):
        ref = ao.intensity(w[i])
        assert np.isclose(got[i], ref, rtol=1e-5, atol=1e-12), (i, got[i], ref)


def test_savi_pretraining_dataset_quirk():
    """N4: the dataset's steady-state slice starts one sample earlier than the simulator's."""
    from soundspaces_b200.pretraining import BatchedAudioGoalDataset
    sr = 16000
    r = renderer(sr, 48000, n_terms=2)
    clips = [make_source(60, 5 * sr), make_source(61, 3 * sr)]
    sids = [r.add_source(c) for c in clips]
    rirs = [make_rir(70, 7001), make_rir(71, 20000), None]
    rids = r.add_rirs(rirs)
    files = [(rids[a], sids[b]) for a in range(3) for b in range(2)]
    ds = BatchedAudioGoalDataset(r, files)
    items, indices = [], []
    for item, (rid, sid) in enumerate(files):
        for index in range(ds.audio_length(sid) - 1):
            items.append(item); indices.append(index)
    spec, wave = ds.render(items, indices, want_wave=True)
    torch.cuda.synchronize()
    for k, (item, index) in enumerate(zip(items, indices)):
        a, b = divmod(item, 2)
        ref = ao.savi_dataset_audiogoal(clips[b], rirs[a], sr, index)
        check_wave(wave[k].cpu().numpy(), ref)
        check_spec(spec[k].cpu().numpy(), ao.compute_spectrogram(ref.astype(np.float32)))


@pytest.mark.parametrize("log2n", [0, 13])
def test_full_size_c3_head_and_valid(log2n):
    """(log2n 0: single-block cluster kernel, 13: partitioned plan.)  BASELINE config 3 at full size on one GPU's share and beyond: 16 kHz, 48000-tap RIRs (3 s reverb), 512 envs;
    "head" mode (1-s clip: only the first 16000 taps matter) and "valid" mode (4-s clip, steady state: all 48000
    taps).  Spot checks against the oracle + exact zeros for silent / zero-RIR envs."""
    from soundspaces_b200 import AudioRequest
    sr, L, B = 16000, 48000, 512
    r = renderer(sr, L, log2n=log2n)
    clip1, clip4 = make_source(80, sr), make_source(81, 4 * sr)
    s1, s4 = r.add_source(clip1), r.add_source(clip4)
    rng = np.random.default_rng(5)
    base = np.stack([make_rir(200 + i, L) for i in range(8)])
    mix = rng.standard_normal((B, 8)).astype(np.float32) / 3.0
    rirs = torch.from_numpy(np.einsum("bk,kle->ble", mix, base).astype(np.float32))
    rirs[7] = 0.0
    ids = r.set_dense_rir_bank(rirs.cuda())
    rirs_h = rirs.numpy()
    for mode, sid, clip, off in (("head", s1, clip1, 0), ("valid", s4, clip4, 3 * sr)):
        reqs = [AudioRequest(rir=i, source=sid, offset=off, silent=(k == 11)) for k, i in enumerate(ids)]
        assert r.prepare(reqs).plan.log2n == (16 if log2n == 0 else log2n)
        spec, wave = r.render(reqs, want_wave=True)
        torch.cuda.synchronize()
        assert spec.shape == (B, 65, 26, 2)
        spec_h, wave_h = spec.cpu().numpy(), wave.cpu().numpy()
        for i in (0, 1, 255, 511):
            ref = ao.compute_audiogoal(clip, rirs_h[i], sr, audio_index=off // sr)
            check_wave(wave_h[i], ref)
            check_spec(spec_h[i], ao.compute_spectrogram(ref.astype(np.float32)))
        assert not wave_h[7].any() and not spec_h[7].any() and not wave_h[11].any() and not spec_h[11].any()


def test_rollout_ingestion_in_place_and_channels_first():
    """N2: the observation is written straight into a rollout-storage slot (rollout_storage.py:27-35, :88-91), and
    optionally channels-first, the layout AudioCNN.forward permutes to (audio_cnn.py:86)."""
    from soundspaces_b200 import AudioRequest
    sr, n, T = 16000, 6, 3
    r = renderer(sr, 6000)
    src = make_source(8, sr)
    sid = r.add_source(src)
    rirs = [make_rir(300 + i, 2000 + 700 * i) for i in range(n)]
    ids = r.add_rirs(rirs)
    batch = r.prepare([AudioRequest(rir=i, source=sid) for i in ids])
    storage = torch.zeros((T + 1, n, 65, 26, 2), device="cuda")            # observations["spectrogram"]
    ret = r.execute(batch, out=storage[2])
    assert ret.data_ptr() == storage[2].data_ptr()
    ref = np.stack([ao.compute_spectrogram(ao.compute_audiogoal(src, rirs[i], sr)) for i in range(n)])
    torch.cuda.synchronize()
    check_spec(storage[2].cpu().numpy(), ref)
    assert not storage[1].any() and not storage[3].any()
    nchw = r.execute(batch, channels_first=True)
    assert nchw.shape == (n, 2, 65, 26) and nchw.is_contiguous()
    assert torch.equal(nchw.permute(0, 2, 3, 1), storage[2])               # bit-identical, reference-shaped view
    assert nchw.permute(0, 2, 3, 1).permute(0, 3, 1, 2).is_contiguous()    # what AudioCNN.forward feeds Conv2d


@pytest.mark.parametrize("log2n,conv_mode", [(12, 0), (13, 1), (14, 0)])
def test_randomised_requests(log2n, conv_mode):
    """160 random requests in one batch: arbitrary sample offsets (not block aligned), arbitrary window lengths,
    wrap-around, ragged RIRs, distractors, silence -- each checked against the oracle's direct formula
    out[m] = sum_k h[k] x_ext[offset + m - k] (tests/conv_ref.py)."""
    from conv_ref import direct as direct_ref
    from soundspaces_b200 import AudioRequest
    sr = 16000
    r = renderer(sr, 30000, n_terms=2, log2n=log2n)
    r.set_conv_mode(conv_mode)
    rng = np.random.default_rng(100 + log2n)
    clips = [make_source(90 + i, n) for i, n in enumerate((sr, 2 * sr + 123, 5 * sr, 700))]
    sids = [r.add_source(c) for c in clips]
    lens = [1, 2, 255, 2047, 2048, 2049, 4096, 8191, 12345, 16000, 16001, 29999, 30000]
    rirs = [make_rir(400 + i, L) for i, L in enumerate(lens)] + [None]
    rids = r.add_rirs(rirs)

    def direct(ci, ri, offset, out_samples, wrap):
        return direct_ref(clips[ci], rirs[ri], sr, offset, out_samples, wrap)

    reqs, refs = [], []
    for _ in range(160):
        ci, ri = int(rng.integers(len(clips))), int(rng.integers(len(rirs)))
        S = len(clips[ci])
        out_samples = int(rng.choice([sr, 4000, 1, 777, 15999]))
        wrap = bool(rng.integers(2))
        offset = int(rng.integers(0, S)) if rng.random() < 0.8 else 0
        if not wrap:
            offset = min(offset, max(0, S - 1))
        silent = rng.random() < 0.05
        req = AudioRequest(rir=rids[ri], source=sids[ci], offset=offset, out_samples=out_samples, wrap=wrap, silent=silent)
        ref = np.zeros((2, sr)) if silent else direct(ci, ri, offset, out_samples, wrap)
        if not silent and rng.random() < 0.3:
            dci, dri = int(rng.integers(len(clips))), int(rng.integers(len(rirs)))
            req.distractor_source, req.distractor_rir = sids[dci], rids[dri]
            ref = ref + direct(dci, dri, 0, out_samples, False)        # distractor: full conv of the whole clip, [:out]
        reqs.append(req)
        refs.append(ref)
    spec, wave = r.render(reqs, want_wave=True)
    torch.cuda.synchronize()
    spec, wave = spec.cpu().numpy(), wave.cpu().numpy()
    for i, ref in enumerate(refs):
        check_wave(wave[i], ref)
        check_spec(spec[i], ao.compute_spectrogram(wave[i]))          # spectrogram stage on the same waveform
    r.set_conv_mode(0)


@pytest.mark.parametrize("log2n", [12, 0])
def test_window_pool_recycling(log2n):
    """A tiny source-spectra pool is recycled mid-batch; prepare() restarts and results stay correct (partitioned
    plan: 64 windows; single-block plan: 8 spectra of 65536 points)."""
    from soundspaces_b200 import AudioRequest, BatchedAudioRenderer
    sr = 16000
    r = BatchedAudioRenderer(sr, 8192, device="cuda:0", xpool_bytes=1, log2n=log2n, prefer_block64=(log2n == 0))      # minimum pool
    clip = make_source(33, 6 * sr)
    sid = r.add_source(clip)
    rir = make_rir(34, 5000)
    rid = r.add_rirs([rir])[0]
    for rep in range(3):
        offs = [sr * k + 37 * rep for k in range(5)]
        reqs = [AudioRequest(rir=rid, source=sid, offset=o) for o in offs]
        wave = r.convolve(reqs)
        torch.cuda.synchronize()
        x = clip.astype(np.float64)
        from scipy.signal import fftconvolve
        for k, o in enumerate(offs):
            full = np.stack([fftconvolve(x[: o + sr], rir[:, ch].astype(np.float64)) for ch in range(2)])
            check_wave(wave[k].cpu().numpy(), full[:, o: o + sr])
