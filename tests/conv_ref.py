"""Float64 direct reference of one convolution request, shared by the GPU tests.

    out[ch, m] = sum_k h[k, ch] * x_ext[offset + m - k],   m < out_samples,

where x_ext is the clip, followed by one more copy of it when ``wrap`` (continuous_simulator.py:443-445) and by
zeros otherwise, with zeros before sample 0.  Samples m >= out_samples are zero.  ``tests/test_conv_ref.py`` pins it
to every branch of the oracle's ``compute_audiogoal`` and ``continuous_convolve_with_rir``."""
import numpy as np
from scipy.signal import fftconvolve


def direct(x, h, sr, offset, out_samples, wrap):
    """x: (S,) mono clip; h: (L, 2) RIR or None (zero RIR).  Returns the (2, sr) float64 waveform."""
    out = np.zeros((2, sr))
    if h is None or len(h) == 0:
        return out
    x = np.asarray(x, dtype=np.float64)
    S = len(x)
    ext = np.concatenate([x, x if wrap else np.zeros(S)])          # one wrap past the end, else zeros
    seg_end = offset + out_samples
    src = np.zeros(seg_end)
    m = min(seg_end, 2 * S)
    src[:m] = ext[:m]
    for ch in range(2):
        y = fftconvolve(src, np.asarray(h[:, ch], dtype=np.float64))
        out[ch, :out_samples] = y[offset: offset + out_samples]
    return out
