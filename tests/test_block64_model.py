"""The index / twiddle algebra of the single-block 65536-point convolution kernel (tests/block64_model.py) against
the oracle: every phase's thread <-> element mapping, the cross-CTA combine and the alias-free shift."""
import numpy as np
import pytest

import block64_model as bm
from oracle import audio_oracle as ao
from synth import make_rir, make_source


def check(wave, ref, tol=2e-6):
    peak = np.abs(ref).max()
    assert np.abs(wave - ref).max() <= tol * peak


@pytest.mark.parametrize("sr,taps", [(44100, 16384), (44100, 21437), (44100, 5000), (16000, 16000)])
def test_head_mode(sr, taps):
    src, rir = make_source(1, sr), make_rir(taps, taps)
    SX = bm.source_spectrum(bm.source_segment(src, 0, False, sr))
    wave = bm.conv64k(rir, min(taps, sr), SX, sr, sr)
    check(wave, ao.compute_audiogoal(src, rir, sr))


def test_valid_mode_long_reverb():
    """C3: 16 kHz, 48000 taps, second 3 of a 4-s clip: all taps, previous seconds' reverb tail included."""
    sr, taps, index = 16000, 48000, 3
    src, rir = make_source(2, 4 * sr), make_rir(7, taps)
    SX = bm.source_spectrum(bm.source_segment(src, index * sr, False, sr))
    wave = bm.conv64k(rir, taps, SX, sr, sr)
    check(wave, ao.compute_audiogoal(src, rir, sr, audio_index=index))


def test_eligibility_limit_valid_mode():
    """16 kHz at the plan's limit 65536 - sr + 1 = 49537 taps, valid mode: all four 16384-tap quarters of phase A."""
    sr, taps, index = 16000, 49537, 4
    src, rir = make_source(5, 5 * sr), make_rir(11, taps)
    SX = bm.source_spectrum(bm.source_segment(src, index * sr, False, sr))
    wave = bm.conv64k(rir, taps, SX, sr, sr)
    check(wave, ao.compute_audiogoal(src, rir, sr, audio_index=index))


def test_eligibility_limit_low_rate_with_offset():
    """8 kHz at its limit of 57537 taps, window at an arbitrary sample offset."""
    from conv_ref import direct
    sr, taps, offset = 8000, 57537, 61234
    src, rir = make_source(6, 9 * sr), make_rir(12, taps)
    SX = bm.source_spectrum(bm.source_segment(src, offset, False, sr))
    wave = bm.conv64k(rir, taps, SX, sr, sr)
    check(wave, direct(src, rir, sr, offset, sr, False))


def test_largest_single_block_rate():
    """61440 Hz, the largest rate the plan takes: D = 4096, at most 4097 taps."""
    sr, taps = 61440, 4097
    src, rir = make_source(7, sr), make_rir(13, taps)
    SX = bm.source_spectrum(bm.source_segment(src, 0, False, sr))
    wave = bm.conv64k(rir, taps, SX, sr, sr)
    check(wave, ao.compute_audiogoal(src, rir, sr))


def test_continuous_window_with_wrap():
    sr, idx = 16000, 44000
    src, rir = make_source(3, 3 * sr), make_rir(9, 9000)
    SX = bm.source_spectrum(bm.source_segment(src, idx, True, sr))
    wave = bm.conv64k(rir, 9000, SX, sr, 4000)
    ref = ao.continuous_convolve_with_rir(src.astype(np.float64), rir.astype(np.float64), sr, 0.25, idx)
    check(wave, ref)
    assert not wave[:, 4000:].any()


def test_source_spectrum_layout():
    import fft_model as fm
    xs = bm.source_segment(make_source(4, 44100), 0, False, 44100)
    SX = bm.source_spectrum(xs)
    ref = np.fft.fft(xs.astype(np.float64))
    k1 = fm.freq_of_slot(12)                                   # [t, i]
    for r in (0, 5, 15):
        got = SX[r].reshape(16, 256).T
        assert np.abs(got - ref[16 * k1 + r]).max() <= 3e-6 * np.abs(ref).max()
