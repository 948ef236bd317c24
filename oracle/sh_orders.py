"""CPU oracle for the ambisonic -> binaural decode at orders 0 to 3 (1, 4, 9 or 16 channels, ACN order).

TEST INFRASTRUCTURE ONLY.  It generalises ``oracle/sh_oracle.py`` (second order) to every channel count the
reference's closed ``AmbisonicBinauralizer`` converts, as probed by ``tests/golden/make_sh_orders_golden.py``:

* one nested filter bank: a K-channel file uses the first K rows of the tool's 16 x 2 x 256 bank, behind the same
  128-sample bulk delay at every order;
* the rotation about the vertical axis adds the third-order pairs (11, 13) by az, (10, 14) by 2 az and (9, 15) by
  3 az to the second-order ones; the m = 0 channels 0, 2, 6 and 12 do not rotate.

At K = 9 both functions reproduce ``sh_oracle`` bit for bit.
"""
from __future__ import annotations

import numpy as np
from scipy.signal import fftconvolve

SH_ORDERS = {1: 0, 4: 1, 9: 2, 16: 3}        # channel count -> ambisonic order
SH_TAPS = 256
SH_DELAY = 128
# (m = -|m| channel, m = +|m| channel, |m|) in ACN order
PAIRS = ((1, 3, 1), (5, 7, 1), (4, 8, 2), (11, 13, 1), (10, 14, 2), (9, 15, 3))


def rotation_matrix(azimuth_deg, n_channels=9):
    """R such that the rotated signal is R @ a (ACN order, rotation about the vertical axis)."""
    if n_channels not in SH_ORDERS:
        raise ValueError(f"{n_channels} channels: 1, 4, 9 or 16")
    al = np.deg2rad(float(azimuth_deg))
    R = np.eye(n_channels)
    for i_neg, i_pos, m in PAIRS:
        if i_pos >= n_channels:
            continue
        c, s = np.cos(m * al), np.sin(m * al)
        R[i_pos, i_pos] = c
        R[i_pos, i_neg] = -s
        R[i_neg, i_pos] = s
        R[i_neg, i_neg] = c
    return R


def sh_decode(amb, azimuth_deg, hbank):
    """amb: (n, K); hbank: (>= K, 2, 256), of which the first K rows are used.  Returns (n, 2) float32."""
    amb = np.asarray(amb, dtype=np.float64)
    n, K = amb.shape
    rot = amb @ rotation_matrix(azimuth_deg, K).T
    out = np.zeros((n + SH_DELAY + SH_TAPS, 2))
    for k in range(K):
        for e in range(2):
            y = fftconvolve(rot[:, k], np.asarray(hbank[k, e], dtype=np.float64))
            out[SH_DELAY: SH_DELAY + y.shape[0], e] += y
    return out[:n].astype(np.float32)
