"""The shared float64 direct reference (tests/conv_ref.py) against the oracle's branch logic: every branch of
``compute_audiogoal`` (head, early, valid) and of ``continuous_convolve_with_rir`` (early, steady, wrap)."""
import numpy as np
import pytest

from conv_ref import direct
from oracle import audio_oracle as ao
from synth import make_rir, make_source


def close(got, ref):
    ref = np.asarray(ref, dtype=np.float64)
    assert got.shape == ref.shape
    assert np.abs(got - ref).max() <= 1e-12 * max(np.abs(ref).max(), 1e-300)


@pytest.mark.parametrize("S_mul,index,L", [
    (1, 0, 5000),          # head: 1-s clip
    (1, 0, 23000),         # head, RIR longer than the clip
    (4, 1, 23000),         # early: index * sr < L
    (4, 0, 7000),          # early at index 0 of a long clip
    (4, 2, 23000),         # valid: index * sr >= L
    (4, 3, 16000),         # valid at the boundary index * sr - L + 1 > 0
])
def test_direct_matches_compute_audiogoal(S_mul, index, L):
    sr = 8000
    x = make_source(5, S_mul * sr).astype(np.float64)
    h = make_rir(L, L).astype(np.float64)
    ref = ao.compute_audiogoal(x, h, sr, audio_index=index)
    close(direct(x, h, sr, index * sr if S_mul != 1 else 0, sr, False), ref)


def test_direct_zero_rir_is_zero():
    assert not direct(make_source(1, 800), None, 800, 0, 800, False).any()
    assert not direct(make_source(1, 800), np.zeros((0, 2)), 800, 10, 800, True).any()


@pytest.mark.parametrize("S,idx,L,wrap", [
    (30000, 3000, 9000, False),      # early: index < L, window inside the clip
    (30000, 3000, 9000, True),       # early: the flag is irrelevant while the window is inside the clip
    (30000, 12000, 9000, False),     # steady: index >= L, index + num < S
    (30000, 12000, 9000, True),
    (30000, 28000, 9000, True),      # wrap: index + num > S, the window continues at the clip start
    (15000, 14000, 14000, True),     # wrap with the RIR reaching back to the clip start
])
def test_direct_matches_continuous_convolve(S, idx, L, wrap):
    sr, step = 16000, 0.25
    x = make_source(7, S).astype(np.float64)
    h = make_rir(L, L).astype(np.float64)
    ref = ao.continuous_convolve_with_rir(x, h, sr, step, idx)
    close(direct(x, h, sr, idx, int(sr * step), wrap), ref)
