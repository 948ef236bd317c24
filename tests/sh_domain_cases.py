"""The cases of tests/test_gpu_sh_domain.py (the ambisonic -> binaural decode over the lengths, orders, azimuth counts,
banks and inputs its entries accept) as plain data, shared with tests/test_sh_domain_host.py, which checks through a
restatement of the host's rules that they reach every tile and block seam.  Needs numpy only.

A case is a dict: ``K`` channels, ``L`` samples, ``angles`` (degrees; one per input for the second-order entry), ``n``
inputs, ``form`` (``default``: the library's choice, the FFT form from 7424 samples; ``direct``: the direct form forced
through ``ssb_set_debug(ctx, 32)``), ``kind`` of input, ``bank`` (``packaged`` or ``random``) and ``entry`` (``multi``:
``ssb_sh_decode_multi_batch`` through ``sh_decode_angles``; ``batch``: ``ssb_sh_decode_batch`` through ``sh_decode``).
"""
import numpy as np

ORDERS_K = (1, 4, 9, 16)
SH_TAPS, SH_DELAY = 256, 128
SH_TILE = 1024                                  # direct form: outputs per CTA
SH_SPAN = SH_TILE + SH_DELAY + SH_TAPS - 1      # ... and the input samples staged for them (1407)
SHF_N = 4096                                    # FFT form: overlap-save block
SHF_F = SH_DELAY + SH_TAPS                      # ... of which the first 384 outputs are discarded
SHF_HOP = SHF_N - SHF_F                         # ... leaving 3712 valid ones
FFT_MIN_L = 2 * SHF_HOP                         # the FFT form starts at 7424 samples
SH_MAX_L = 1 << 30                              # SSB_SH_MAX_L

LONG_L = 300001
# the delay (128), the filter end (384), the direct tile (1024) and its staged span (1407), the overlap-save hop
# (3712: two blocks exactly at 7424, a third with one output at 7425, three blocks at 11136), and two long ones
LENGTHS = (1, 2, 127, 128, 129, 383, 384, 385, 1023, 1024, 1025, 1406, 1407, 1408, 2047, 2048, 3711, 3712, 3713, 7423,
           7424, 7425, 11135, 11136, 11137, 48000, LONG_L)
A_COUNTS = (1, 2, 3, 4, 5, 6, 7, 8, 9)
LARGE_A = 64
AZ_VALUES = (0.0, 90.0, 180.0, 270.0, 37.5, 359.999, -90.0, -37.5, 450.0, 720.5, -0.0)
AZ_DUPLICATE = (37.5, 200.0, 37.5)
AZ_DESCENDING = (300.0, 200.0, 90.0, 10.0, -45.0)
# any finite azimuth decodes: the kernel reduces it exactly before converting to radians
AZ_FAR = (36037.5, -36037.5, 1.0e6, -123456.78, 3.0e38)
# azimuths that decode alike: (angle, angle + 360 k)
AZ_ALIASES = ((90.0, 450.0), (0.5, 720.5), (-37.5, -397.5), (0.0, -0.0))
N_INPUTS = (1, 2, 17, 300)
BANKS = ("packaged", "random")
KINDS = ("flat", "decay", "zero_between", "one_channel", "impulse")
SCALES = (1e-6, 1e3)
DIRECT_L, FFT_L = 2500, 7425                    # three direct tiles (the last partial); three blocks, the last of 1


def angles_of(A):
    """A distinct azimuths in [-180, 540), multiples of 0.25 (exact in float32); a prefix of every longer list."""
    return tuple((37.5 + 83.25 * i) % 720.0 - 180.0 for i in range(A))


def case(name, K, L, angles, n=2, form="default", kind="flat", bank="packaged", entry="multi", seed=0, **extra):
    c = dict(name=f"K{K}_{name}", K=K, L=L, angles=tuple(float(a) for a in angles), n=n, form=form, kind=kind,
             bank=bank, entry=entry, seed=seed + 1000 * K, scale=1.0)
    c.update(extra)
    return c


def runs_fft(c):
    return c["form"] == "default" and c["L"] >= FFT_MIN_L


def tile_of(c):
    """Outputs per CTA of the form the case runs: the seams of its output lie at the multiples of this."""
    return SHF_HOP if runs_fft(c) else SH_TILE


def forms_at(L):
    return ("default", "direct") if L >= FFT_MIN_L else ("default",)


def length_cases(K):
    """Every length with one azimuth; from 7424 samples in both forms, and the FFT form also with three azimuths (its
    one-azimuth and grouped kernels are separate instances)."""
    out = []
    for i, L in enumerate(LENGTHS):
        n = 1 if L == LONG_L else 2
        for form in forms_at(L):
            out.append(case(f"L{L}_{form}", K, L, (37.5,), n=n, form=form, seed=i))
        if L >= FFT_MIN_L:
            out.append(case(f"L{L}_A3", K, L, (359.999, -90.0, 37.5), n=n, seed=i))
    return out


def batch_entry_cases():
    """The second-order entry (one azimuth per input) at every length, from 7424 samples in both forms."""
    return [case(f"batch_L{L}_{form}", 9, L, (200.0, 37.5)[:1 if L == LONG_L else 2], n=1 if L == LONG_L else 2,
                 form=form, entry="batch", seed=i) for i, L in enumerate(LENGTHS) for form in forms_at(L)]


def count_cases(K):
    """Azimuth counts 1 to 9 in both forms (the FFT form takes them in groups of four), and 64 at a short length."""
    out = [case(f"A{A}_L{L}", K, L, angles_of(A), seed=40) for L in (DIRECT_L, FFT_L) for A in A_COUNTS]
    out.append(case(f"A{LARGE_A}", K, 200, angles_of(LARGE_A), seed=41))
    return out


def azimuth_cases(K):
    lists = dict(values=AZ_VALUES, duplicate=AZ_DUPLICATE, descending=AZ_DESCENDING, far=AZ_FAR)
    return [case(f"az_{name}_L{L}", K, L, az, n=1, seed=50) for L in (DIRECT_L, FFT_L) for name, az in lists.items()]


def input_count_cases(K):
    """1, 2, 17 and 300 inputs per call (blockIdx.y past one wave of CTAs), each the first n of one pool."""
    return [case(f"n{n}_L{L}", K, L, angles_of(3), n=n, seed=60) for L in (1100, FFT_L) for n in N_INPUTS]


def bank_cases(K):
    """A bank whose ears are unrelated, in both forms (and the direct form forced at an FFT length), A = 1 and 5."""
    return [case(f"random_bank_A{A}_L{L}_{form}", K, L, angles_of(A), form=form, bank="random", seed=70)
            for L in (DIRECT_L, FFT_L) for form in forms_at(L) for A in (1, 5)]


def kind_cases(K):
    out = []
    for L in (DIRECT_L, 11137):
        for form in forms_at(L):
            t = f"L{L}_{form}"
            out.append(case(f"decay_{t}", K, L, angles_of(2), form=form, kind="decay", seed=80))
            out.append(case(f"zero_between_{t}", K, L, angles_of(2), n=3, form=form, kind="zero_between", seed=81))
            out.append(case(f"one_channel_{t}", K, L, angles_of(2), form=form, kind="one_channel", live=K - 1, seed=82))
            out += [case(f"scale{s:g}_{t}", K, L, angles_of(2), form=form, seed=83, scale=s) for s in SCALES]
    return out


def impulse_positions(L, tile):
    """Where a unit impulse goes: the ends of the input, the last position that still reaches an output (L - 129) and
    the first that does not, and for every seam s of the output the positions whose 256-sample response (outputs
    p + 128 ... p + 383) starts or ends on either side of s, plus the seam itself as an input position."""
    pos = {0, 1, L - 1, L - SH_DELAY - 1, L - SH_DELAY}
    for s in range(tile, L + 1, tile):
        pos |= {s - SHF_F, s - SHF_F + 1, s - SH_DELAY - 1, s - SH_DELAY, s - 1, s}
    return sorted(p for p in pos if 0 <= p < L)


def impulse_cases(K):
    """One input per (channel, position): n = K * len(impulse_positions)."""
    out = []
    for L in (DIRECT_L, FFT_L):
        for form in forms_at(L):
            tile = SHF_HOP if (form == "default" and L >= FFT_MIN_L) else SH_TILE
            P = impulse_positions(L, tile)
            out.append(case(f"impulse_L{L}_{form}", K, L, (37.5, 270.0), n=K * len(P), form=form, kind="impulse",
                            positions=tuple(P), seed=90))
    return out


def sweep():
    """Every accuracy case the GPU file runs."""
    out = batch_entry_cases()
    for K in ORDERS_K:
        out += (length_cases(K) + count_cases(K) + azimuth_cases(K) + input_count_cases(K) + bank_cases(K)
                + kind_cases(K) + impulse_cases(K))
    return out


# ---------------------------------------------------------------------------
# inputs, banks and references
# ---------------------------------------------------------------------------
def random_bank(K):
    """(K, 2, 256) float32 with independent ears: swapping them, or a wrong sign on one, changes every output."""
    return (np.random.default_rng(7000 + K).standard_normal((K, 2, SH_TAPS)) * 0.05).astype(np.float32)


def bank_of(c):
    if c["bank"] == "random":
        return random_bank(c["K"])
    from soundspaces_b200.renderer import sh_hrtf_bank
    return sh_hrtf_bank(c["K"])


def make_input(c):
    """(n, L, K) float32.  ``flat`` is noise with no envelope, so every tile and block holds full-scale content;
    ``decay`` is the RIR shape of the older tests."""
    n, L, K = c["n"], c["L"], c["K"]
    if c["kind"] == "impulse":
        P = c["positions"]
        x = np.zeros((n, L, K), np.float32)
        for k in range(K):
            for j, p in enumerate(P):
                x[k * len(P) + j, p, k] = 1.0
        return x
    x = np.random.default_rng(c["seed"]).standard_normal((n, L, K)) * 0.3
    if c["kind"] == "decay":
        x *= np.exp(-np.arange(L) / max(L / 5.0, 20.0))[None, :, None]
    elif c["kind"] == "zero_between":
        x[1] = 0.0
    elif c["kind"] == "one_channel":
        live = x[:, :, c["live"]].copy()
        x[:] = 0.0
        x[:, :, c["live"]] = live
    return (x * c["scale"]).astype(np.float32)


def ref_azimuth(az_deg):
    """The float32 azimuth the device receives, reduced to (-360, 360) in float64.  ``math.fmod`` is exact, so this is
    the same angle; without it ``deg2rad`` of a huge azimuth would carry the float64 rounding of ~1e36 rad."""
    import math
    return math.fmod(float(np.float32(az_deg)), 360.0)


def reference(x, az_deg, bank):
    """(L, K) input -> (L, 2): the float64 oracle at the azimuth the device receives."""
    from oracle import sh_orders as so
    return so.sh_decode(x, ref_azimuth(az_deg), bank)


def rotated_bank(az_deg, bank):
    """g[k] = sum_j R(az)[j][k] bank[j], float64 (K, 2, 256): the filters a unit impulse in channel k meets."""
    from oracle import sh_orders as so
    R = so.rotation_matrix(ref_azimuth(az_deg), bank.shape[0])
    return np.einsum("jk,jet->ket", R, np.asarray(bank, np.float64))


def impulse_response(K, k, p, L, az_deg, bank):
    """The decode of a unit impulse in channel k at sample p, in closed form (float64, (L, 2)):
    out[n][ear] = sum_j R[j][k] bank[j][ear][n - p - 128]."""
    out = np.zeros((L, 2))
    g = rotated_bank(az_deg, bank[:K])[k]                # (2, 256)
    lo = p + SH_DELAY
    hi = min(L, lo + SH_TAPS)
    if hi > lo:
        out[lo:hi] = g[:, : hi - lo].T
    return out


def segment_violations(got, ref, tile, rel=1e-4, window=64):
    """Seam-aware bound: split the output at every multiple of ``tile`` and require max|got - ref| <= rel * max|ref|
    inside each segment.  A segment shorter than ``window`` samples (a last block with one output) is weighed against
    the ``window`` samples that end with it, not against one value that may happen to be near zero.  Returns
    [(start, end, error, bound)] of the segments that fail; NaN fails."""
    ref = np.asarray(ref, np.float64)
    L = ref.shape[0]
    bad = []
    for s in range(0, L, tile):
        e = min(L, s + tile)
        bound = rel * np.abs(ref[max(0, min(s, e - window)):e]).max()
        err = np.abs(np.asarray(got[s:e], np.float64) - ref[s:e]).max()
        if not err <= bound:
            bad.append((s, e, float(err), float(bound)))
    return bad
