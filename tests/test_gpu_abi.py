"""The C ABI at the arguments the renderer never passes: row strides other than sr on every entry point that takes
one, and the small kernels (the fused first audio-encoder layer, PCM conversion, crossfade) at their limits."""
import ctypes as C

import numpy as np
import pytest

from conv_ref import direct
from oracle import audio_oracle as ao
from synth import make_rir, make_source
from test_gpu_parity import check_wave, renderer

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")


def _ops():
    from soundspaces_b200.renderer import WaveformOps
    return WaveformOps.get("cuda:0")


# ------------------------------------------------------------------------------------------------ row strides
SR, B_STRIDE = 16000, 72          # 72 envs: ssb_render_batch splits them over 2 internal streams (>= 32 envs each)


def _stride_setup():
    """Two renderers (single-block and partitioned plan) with the same 72 prepared requests."""
    from soundspaces_b200 import AudioRequest
    rng = np.random.default_rng(77)
    clips = [make_source(950, SR), make_source(951, 3 * SR + 5)]
    lens = (1, 700, 4096, 9000, 16001, 20000)
    rirs = [make_rir(960 + i, L) for i, L in enumerate(lens)] + [None]
    specs = []
    for k in range(B_STRIDE):
        ci = int(rng.integers(2))
        specs.append((ci, int(rng.integers(len(rirs))), int(rng.integers(0, len(clips[ci]))),
                      int(rng.choice((SR, 4000, 777))), bool(rng.integers(2)), k % 11 == 4))
    out = []
    for log2n in (0, 12):
        r = renderer(SR, 20001, log2n=log2n)
        sids = [r.add_source(c) for c in clips]
        rids = r.add_rirs(rirs)
        batch = r.prepare([AudioRequest(rir=rids[ri], source=sids[ci], offset=off, out_samples=n, wrap=w, silent=s)
                           for ci, ri, off, n, w, s in specs])
        assert batch.plan.log2n == (16 if log2n == 0 else 12)
        out.append((r, batch))
    return out, clips, rirs, specs


def _nan_rows(stride, rows=B_STRIDE):
    return torch.full((rows, 2, stride), float("nan"), dtype=torch.float32, device="cuda")


def _run_strided(setup, stride):
    """Every wave_stride-taking entry point at row stride `stride`.  Returns {name: device tensor}; waveform
    buffers are (B, 2, stride) with [sr, stride) initialised to NaN."""
    outs = {}
    for r, batch in setup:
        tag = "b64" if batch.plan.log2n == 16 else "part"
        lib, h, st, plan = r.lib, r.ctx.handle, r._stream(), C.byref(batch.plan)
        hs, _ = r._scratch(B_STRIDE, batch.plan)
        bank, xpool = r._bank.data_ptr(), r._xpool.data_ptr()
        spec_shape = (B_STRIDE,) + r.spec_shape
        w = _nan_rows(stride)
        r.ctx.check(lib.ssb_convolve_batch(h, plan, B_STRIDE, batch.reqs_dev.data_ptr(), bank, xpool, hs.data_ptr(),
                                           w.data_ptr(), stride, st), "ssb_convolve_batch")
        outs[f"conv_{tag}"] = w
        try:
            for streams in (1, 2):
                r.set_streams(streams)
                w = _nan_rows(stride)
                spec = torch.empty(spec_shape, dtype=torch.float32, device="cuda")
                r.ctx.check(lib.ssb_render_batch(h, plan, B_STRIDE, batch.reqs_dev.data_ptr(), bank, xpool, hs.data_ptr(),
                                                 w.data_ptr(), stride, r.pad_mode, spec.data_ptr(), st), "ssb_render_batch")
                outs[f"render_{tag}_s{streams}"], outs[f"render_{tag}_s{streams}_spec"] = w, spec
        finally:
            r.set_streams(2)
        h_reqs = torch.from_numpy(batch.reqs_host.view(np.uint8).copy()).pin_memory()
        h_rir = r._bank[: max(r._bank_used, 1)].cpu().pin_memory()
        d_rir = torch.empty_like(h_rir, device="cuda")
        d_reqs = torch.empty_like(h_reqs, device="cuda")
        for n_chunks in (1, 3):
            w = _nan_rows(stride)
            d_spec = torch.empty(spec_shape, dtype=torch.float32, device="cuda")
            h_spec = torch.empty(spec_shape, dtype=torch.float32).pin_memory()
            h_wave = torch.empty((B_STRIDE, 2, SR), dtype=torch.float32).pin_memory()
            r.ctx.check(lib.ssb_render_batch_host(h, plan, B_STRIDE, h_reqs.data_ptr(), h_rir.data_ptr(), h_rir.numel() * 4,
                                                  d_rir.data_ptr(), d_reqs.data_ptr(), xpool, hs.data_ptr(), w.data_ptr(),
                                                  stride, r.pad_mode, d_spec.data_ptr(), h_spec.data_ptr(),
                                                  h_wave.data_ptr(), n_chunks, st), "ssb_render_batch_host")
            torch.cuda.current_stream().synchronize()
            outs[f"host_{tag}_c{n_chunks}"] = w
            outs[f"host_{tag}_c{n_chunks}_hspec"] = h_spec.clone()
            outs[f"host_{tag}_c{n_chunks}_hwave"] = h_wave.clone()
    # the waveform consumers, on the partitioned plan's waveform re-laid at this stride
    ops = _ops()
    lib, h, st = ops.lib, ops.ctx.handle, ops._stream()
    wave = _nan_rows(stride)
    wave[:, :, :SR] = outs["conv_part"][:, :, :SR]
    prev = _nan_rows(stride)
    prev[:, :, :SR] = outs["conv_b64"][:, :, :SR].flip(0)
    cols = setup[0][0].spec_shape[1]
    for layout, shape in ((0, (B_STRIDE, 65, cols, 2)), (0x100, (B_STRIDE, 2, 65, cols))):
        for pad in (0, 1):
            spec = torch.empty(shape, dtype=torch.float32, device="cuda")
            ops.ctx.check(lib.ssb_spectrogram_batch(h, B_STRIDE, wave.data_ptr(), stride, SR, pad | layout,
                                                    spec.data_ptr(), st), "ssb_spectrogram_batch")
            outs[f"spec_{layout}_{pad}"] = spec
    mel = torch.empty((B_STRIDE, 64, 1 + SR // 160, 2), dtype=torch.float32, device="cuda")
    ops.ctx.check(lib.ssb_logmel_batch(h, B_STRIDE, wave.data_ptr(), stride, SR, 64, 2, 0, mel.data_ptr(), st),
                  "ssb_logmel_batch")
    outs["logmel"] = mel
    inten = torch.empty(B_STRIDE, dtype=torch.float32, device="cuda")
    ops.ctx.check(lib.ssb_intensity_batch(h, B_STRIDE, wave.data_ptr(), stride, SR, 150, inten.data_ptr(), st),
                  "ssb_intensity_batch")
    outs["intensity"] = inten
    enable = torch.from_numpy((np.arange(B_STRIDE) % 3 != 1).astype(np.uint8)).cuda()
    ops.ctx.check(lib.ssb_crossfade_batch(h, B_STRIDE, prev.data_ptr(), wave.data_ptr(), SR, stride, enable.data_ptr(), st),
                  "ssb_crossfade_batch")
    outs["crossfade"] = wave
    outs["crossfade_prev"] = prev
    torch.cuda.synchronize()
    return {k: v.cpu().numpy() for k, v in outs.items()}


_stride_base = {}


def _is_wave(v):
    return v.ndim == 3 and v.shape[:2] == (B_STRIDE, 2) and v.shape[2] >= SR and v.dtype == np.float32


@pytest.mark.parametrize("extra", [1, 37, 1024])
def test_row_stride(extra):
    """Every entry point at wave_stride = sr + extra, rows padded with NaN: the first sr samples of every row and every
    derived output are bit-identical to wave_stride = sr, all finite, and the padding is never written."""
    if not _stride_base:
        setup, clips, rirs, specs = _stride_setup()
        _stride_base.update(setup=setup, ref=_run_strided(setup, SR))
        conv = _stride_base["ref"]["conv_part"]
        for i in (0, 1, 4, B_STRIDE - 1):                      # the stride-sr reference itself against the oracle
            ci, ri, off, n, wrap, silent = specs[i]
            check_wave(conv[i], np.zeros((2, SR)) if silent else direct(clips[ci], rirs[ri], SR, off, n, wrap))
    base = _stride_base["ref"]
    got = _run_strided(_stride_base["setup"], SR + extra)
    assert set(got) == set(base)
    for k, v in got.items():
        if k.endswith("_hwave") or not _is_wave(v):
            assert np.array_equal(v, base[k]), k
            assert np.isfinite(v).all(), k
        else:
            assert v.shape[2] == SR + extra
            assert np.array_equal(v[:, :, :SR], base[k][:, :, :SR]), k
            assert np.isfinite(v[:, :, :SR]).all(), k
            assert np.isnan(v[:, :, SR:]).all(), k
    # the crossfade blended the enabled envs only
    keep = np.arange(B_STRIDE) % 3 == 1
    assert np.array_equal(got["crossfade"][keep, :, :SR], got["conv_part"][keep, :, :SR])
    assert not np.array_equal(got["crossfade"][~keep, :, :SR], got["conv_part"][~keep, :, :SR])


# ------------------------------------------------------------------------------------------------ audio_conv1
def _conv_case(sr, oc, k, s, bias, relu, seed):
    ops = _ops()
    rng = np.random.default_rng(seed)
    H, W = 65, -(-(1 + sr // 160) // 4)
    x = torch.from_numpy(rng.random((3, H, W, 2), dtype=np.float32) * 5.0).cuda()
    conv = torch.nn.Conv2d(2, oc, k, stride=s, bias=bias)
    with torch.no_grad():
        conv.weight.copy_(torch.from_numpy(rng.standard_normal(tuple(conv.weight.shape)).astype(np.float32)))
        if bias:
            conv.bias.copy_(torch.from_numpy(rng.standard_normal(oc).astype(np.float32)))
    got = ops.audio_conv1(x, conv.cuda(), relu=relu).cpu().numpy().astype(np.float64)
    x64 = x.cpu().double().permute(0, 3, 1, 2)
    w64, b64 = conv.weight.detach().cpu().double(), conv.bias.detach().cpu().double() if bias else None
    ref = torch.nn.functional.conv2d(x64, w64, b64, stride=s)
    bound = torch.nn.functional.conv2d(x64.abs(), w64.abs(), b64.abs() if bias else None, stride=s)   # sum |terms|
    if relu:
        ref = ref.clamp_min(0.0)
    ref, bound = ref.numpy(), bound.numpy()
    assert got.shape == ref.shape
    assert (np.abs(got - ref) <= 1e-5 * bound).all(), np.abs(got - ref).max()
    return got.shape


@pytest.mark.parametrize("sr,oc,k,s,bias,relu", [
    (16000, 32, (5, 5), (2, 2), True, True),          # AudioCNN's first layer for inputs under 30 columns
    (44100, 32, (8, 8), (4, 4), True, True),          # ... and for wider ones
    (48000, 32, (8, 8), (4, 4), False, False),
    (16000, 1, (3, 7), (1, 3), False, False),         # one output channel, non-square kernel and stride
    (44100, 7, (8, 2), (4, 1), True, False),
    (48000, 5, (65, 3), (1, 2), False, True),         # the whole height in one row of outputs
    (44100, 16, (3, 6), (1, 1), True, True),          # W1 * OC = 64 * 16 = 1024 threads, the block limit
    (48000, 20, (4, 73), (3, 1), True, False),        # 4 * 76 * 2 + 20 * 2 * 4 * 73 floats = exactly 48 KB staged
])
def test_audio_conv1_against_float64(sr, oc, k, s, bias, relu):
    _conv_case(sr, oc, k, s, bias, relu, seed=sr + oc)


@pytest.mark.parametrize("W,OC,KH,KW", [
    (69, 25, 1, 29),                                  # W1 * OC = 41 * 25 = 1025 > 1024
    (69, 20, 5, 58),                                  # 2 * 5 * (69 + 20 * 58) floats = 49160 bytes > 48 KB
])
def test_audio_conv1_refuses_oversized_layers(W, OC, KH, KW):
    ops = _ops()
    H = 65
    x = torch.zeros((1, H, W, 2), dtype=torch.float32, device="cuda")
    w = torch.zeros((OC, 2, KH, KW), dtype=torch.float32, device="cuda")
    out = torch.zeros((1, OC, H - KH + 1, W - KW + 1), dtype=torch.float32, device="cuda")
    rc = ops.lib.ssb_audio_conv1_batch(ops.ctx.handle, 1, x.data_ptr(), H, W, w.data_ptr(), None, OC, KH, KW, 1, 1, 0,
                                       out.data_ptr(), ops._stream())
    assert rc == -4                                   # SSB_E_SHAPE, decided on the host before any launch
    assert b"too large" in ops.lib.ssb_last_error(ops.ctx.handle)


# ------------------------------------------------------------------------------------------------ PCM
N_PCM = 1_000_003                 # more than 16 blocks x 256 threads per SM: the grid-stride loops run twice or more


def test_pcm16_decode_every_value():
    ops = _ops()
    pcm = np.resize(np.arange(-32768, 32768, dtype=np.int64).astype(np.int16), N_PCM)
    d_in = torch.from_numpy(pcm).cuda()
    out = torch.full((N_PCM,), float("nan"), dtype=torch.float32, device="cuda")
    ops.ctx.check(ops.lib.ssb_pcm16_decode(ops.ctx.handle, d_in.data_ptr(), N_PCM, out.data_ptr(), ops._stream()),
                  "ssb_pcm16_decode")
    assert np.array_equal(out.cpu().numpy(), ao.pcm16_to_float32(pcm))


def _encode_inputs():
    rng = np.random.default_rng(16)
    k = np.arange(-32768, 32768, dtype=np.float64)
    special = np.concatenate([
        (2 * k + 1) / 65536.0,                                   # x * 32768 = k + 1/2: ties of both signs
        k / 32768.0, k / 32767.0,
        [1.0, -1.0, 32767.5 / 32768, -32768.5 / 32768, 1.0 + 2 ** -23, -1.0 - 2 ** -23,
         1.5, -1.5, 2.0, -2.0, 1e4, -1e4, 1e30, -1e30, 0.0, -0.0, 1e-30, -1e-30],
    ]).astype(np.float32)
    x = rng.uniform(-1.25, 1.25, N_PCM).astype(np.float32)
    x[: special.size] = special
    return rng.permutation(x)


@pytest.mark.parametrize("mode", ["round", "demo"])
def test_pcm16_encode_against_oracle(mode):
    ops = _ops()
    x = _encode_inputs()
    d_in = torch.from_numpy(x).cuda()
    out = torch.zeros((N_PCM,), dtype=torch.int16, device="cuda")
    ops.ctx.check(ops.lib.ssb_pcm16_encode(ops.ctx.handle, d_in.data_ptr(), N_PCM, {"round": 0, "demo": 1}[mode],
                                           out.data_ptr(), ops._stream()), "ssb_pcm16_encode")
    ref = ao.float32_to_pcm16_round(x) if mode == "round" else ao.float32_to_pcm16_demo(x)
    assert np.array_equal(out.cpu().numpy(), ref)


# ------------------------------------------------------------------------------------------------ crossfade
@pytest.mark.parametrize("sr", [8000, 22050, 44100])
def test_crossfade_against_oracle(sr):
    ops = _ops()
    rng = np.random.default_rng(sr)
    B = 5
    prev = rng.standard_normal((B, 2, sr)).astype(np.float32)
    cur = (0.3 * rng.standard_normal((B, 2, sr))).astype(np.float32)
    enable = np.array([1, 0, 1, 1, 0], np.uint8)
    d_prev, d_cur = torch.from_numpy(prev).cuda(), torch.from_numpy(cur).cuda()
    d_en = torch.from_numpy(enable).cuda()
    ops.ctx.check(ops.lib.ssb_crossfade_batch(ops.ctx.handle, B, d_prev.data_ptr(), d_cur.data_ptr(), sr, sr,
                                              d_en.data_ptr(), ops._stream()), "ssb_crossfade_batch")
    got = d_cur.cpu().numpy()
    n = int(0.05 * sr)
    for i in range(B):
        if enable[i]:
            check_wave(got[i], ao.crossfade(prev[i].astype(np.float64), cur[i].astype(np.float64), sr))
            assert np.array_equal(got[i][:, n + 1:], cur[i][:, n + 1:])
        else:
            assert np.array_equal(got[i], cur[i])
