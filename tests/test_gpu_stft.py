"""The STFT front ends (``spectrogram_kernel``, ``logmel_kernel``) across the column geometry: rates whose last pooled
column holds 1, 2, 3 or 4 real frames, rates with no interior column (sr < 1344), the exact rate (1344) at which
column 1's branch-free path reads sample sr - 1, and rates that are not a multiple of the hop.  Signals are shaped
to hit the padding zones and the lone Nyquist row."""
import numpy as np
import pytest

from oracle import audio_oracle as ao
from test_gpu_parity import check_spec

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

# frames % 4 = 0 (512, 44100), 1 (1343, 1344, 11025, 16000, 96000), 2 (800, 16160, 22050), 3 (961, 16320, 24000)
RATES = [512, 800, 961, 1343, 1344, 11025, 16000, 16160, 16320, 22050, 24000, 44100, 96000]
NCHW = 0x100


def shaped_waves(sr):
    """(5, 2, sr) float32: noise; a quiet ear next to a 30x ear; unit impulses in and next to the padding zones;
    DC next to (-1)^n (all of its energy in the Nyquist bin, pooled row 64 on its own); silence."""
    rng = np.random.default_rng(sr)
    w = np.zeros((5, 2, sr), np.float32)
    w[0] = rng.standard_normal((2, sr))
    w[1, 0] = 0.1 * rng.standard_normal(sr)
    w[1, 1] = 3.0 * rng.standard_normal(sr)
    for n in (0, 255, 256, sr - 257, sr - 1):
        w[2, 0, n] = 1.0
    w[2, 1, sr // 2] = -1.0
    w[3, 0] = 1.0
    w[3, 1] = np.where(np.arange(sr) % 2 == 0, 1.0, -1.0)
    return w


def _ops():
    from soundspaces_b200.renderer import WaveformOps
    return WaveformOps.get("cuda:0")


def _spectrogram(ops, wave, pad, layout):
    n, _, sr = wave.shape
    cols = -(-(1 + sr // 160) // 4)
    shape = (n, 2, 65, cols) if layout else (n, 65, cols, 2)
    out = torch.empty(shape, dtype=torch.float32, device="cuda")
    ops.ctx.check(ops.lib.ssb_spectrogram_batch(ops.ctx.handle, n, wave.data_ptr(), sr, sr, pad | layout,
                                                out.data_ptr(), ops._stream()), "ssb_spectrogram_batch")
    return out


@pytest.mark.parametrize("pad_mode", ["reflect", "constant"])
@pytest.mark.parametrize("sr", RATES)
def test_spectrogram_geometry(sr, pad_mode):
    pad = {"reflect": 0, "constant": 1}[pad_mode]
    ops = _ops()
    w = shaped_waves(sr)
    wd = torch.from_numpy(w).cuda()
    nhwc = _spectrogram(ops, wd, pad, 0)
    nchw = _spectrogram(ops, wd, pad, NCHW)
    assert torch.equal(nchw.permute(0, 2, 3, 1), nhwc)          # the same numbers, channels first
    got = nhwc.cpu().numpy()
    for i in range(len(w)):
        check_spec(got[i], ao.compute_spectrogram(w[i], pad_mode=pad_mode))
    assert not got[4].any()


@pytest.mark.parametrize("pad_mode", ["reflect", "constant"])
@pytest.mark.parametrize("sr", RATES)
def test_logmel_geometry(sr, pad_mode):
    pad = {"reflect": 0, "constant": 1}[pad_mode]
    ops = _ops()
    w = shaped_waves(sr)
    wd = torch.from_numpy(w).cuda()
    frames = 1 + sr // 160
    for n_mels in (64, 13):
        for power in (1, 2):
            out = torch.empty((len(w), n_mels, frames, 2), dtype=torch.float32, device="cuda")
            ops.ctx.check(ops.lib.ssb_logmel_batch(ops.ctx.handle, len(w), wd.data_ptr(), sr, sr, n_mels, power, pad,
                                                   out.data_ptr(), ops._stream()), "ssb_logmel_batch")
            got = out.cpu().numpy()
            for i in range(len(w)):
                ref = ao.logmel(w[i], sr, n_mels=n_mels, power=power, pad_mode=pad_mode)
                assert np.allclose(got[i], ref, rtol=1e-4, atol=1e-5), (n_mels, power, i, np.abs(got[i] - ref).max())
            assert not got[4].any()


def test_spectrogram_refuses_misaligned_nhwc_output():
    """The (65, T', 2) layout is stored as ear pairs (8 bytes): an output pointer off by 4 bytes is refused.
    Channels-first stores single floats and takes it."""
    ops = _ops()
    sr = 16000
    w = torch.from_numpy(shaped_waves(sr)[:2].copy()).cuda()
    cols = -(-(1 + sr // 160) // 4)
    buf = torch.zeros(2 * 65 * cols * 2 + 2, dtype=torch.float32, device="cuda")
    rc = ops.lib.ssb_spectrogram_batch(ops.ctx.handle, 2, w.data_ptr(), sr, sr, 0, buf.data_ptr() + 4, ops._stream())
    assert rc == -1 and b"aligned" in ops.lib.ssb_last_error(ops.ctx.handle)
    torch.cuda.synchronize()
    assert not buf.any()                                          # nothing was launched
    rc = ops.lib.ssb_spectrogram_batch(ops.ctx.handle, 2, w.data_ptr(), sr, sr, NCHW, buf.data_ptr() + 4, ops._stream())
    assert rc == 0
    got = buf[1: 1 + 2 * 65 * cols * 2].view(2, 2, 65, cols)
    assert torch.equal(got, _spectrogram(ops, w, 0, NCHW))
    assert buf[0].item() == 0 and buf[-1].item() == 0

