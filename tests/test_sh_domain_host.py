"""Host side of the ambisonic -> binaural decode sweep: the rules by which ``ssb_sh_decode_batch`` and
``ssb_sh_decode_multi_batch`` pick a form, a grid and a shared-memory size, restated; the case list of
tests/sh_domain_cases.py held against them, so that it reaches every tile and block seam; the closed form of the
decode of a unit impulse against the oracle; and a float32 model of ``sh_filters_kernel``'s angle arithmetic.  No GPU."""
import re
import os

import numpy as np
import pytest

import sh_domain_cases as dc
from oracle import sh_orders as so

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INT_MAX = 2 ** 31 - 1


# ---------------------------------------------------------------------------
# the host's rules, restated
# ---------------------------------------------------------------------------
def int32(v):
    """C ``int`` arithmetic: wraps modulo 2^32."""
    return (v + 2 ** 31) % 2 ** 32 - 2 ** 31


def takes_fft(L, debug=0):
    return L >= 2 * 3712 and not debug & 32


def direct_grid(L):
    return int32(L + 1024 - 1) // 1024


def fft_grid(L):
    return int32(L + 3712 - 1) // 3712


def az_groups(A):
    """(accumulators per group, groups, azimuths in the last group) of the FFT form."""
    if A == 1:
        return 1, 1, 1
    g = -(-A // 4)
    return 4, g, A - 4 * (g - 1)


def direct_smem(K):
    """Input tile [K][1407] (padded to an even float count) + one filter set [K][256] float2."""
    return (K * 1407 + 1) * 4 + K * 256 * 8


def last_tile(L, tile):
    t = -(-L // tile)
    return t, L - (t - 1) * tile


def test_rules_match_the_documented_figures():
    assert (dc.SH_TILE, dc.SH_SPAN, dc.SHF_HOP, dc.SHF_F, dc.FFT_MIN_L) == (1024, 1407, 3712, 384, 7424)
    assert not takes_fft(7423) and takes_fft(7424) and not takes_fft(7424, 32) and not takes_fft(10 ** 6, 32)
    assert [direct_grid(L) for L in (1, 1024, 1025, 7423)] == [1, 1, 2, 8]
    assert [fft_grid(L) for L in (7424, 7425, 11136, 11137)] == [2, 3, 3, 4]
    assert [az_groups(A) for A in (1, 2, 4, 5, 7, 8, 9)] == [(1, 1, 1), (4, 1, 2), (4, 1, 4), (4, 2, 1), (4, 2, 3),
                                                              (4, 2, 4), (4, 3, 1)]
    # DESIGN.md: 122 KB of shared memory at K = 16, 69 KB at K = 9, inside the 227 KB a CTA may opt in to
    assert direct_smem(16) // 1000 == 122 and direct_smem(9) // 1000 == 69 and direct_smem(16) <= 227 * 1024
    with open(os.path.join(ROOT, "DESIGN.md")) as f:
        design = f.read()
    assert "122 KB of shared memory at K = 16" in design and "69 KB at K = 9" in design


def test_length_limit_keeps_the_grids_inside_int():
    """At the largest accepted L neither ceil wraps, nor does the direct form's last output index n0 + 1023; at
    2^31 - 1 (refused) both grids wrap to a non-positive block count."""
    with open(os.path.join(ROOT, "include", "ssb200.h")) as f:
        m = re.search(r"#define SSB_SH_MAX_L \(1 << (\d+)\)", f.read())
    assert m and 1 << int(m.group(1)) == dc.SH_MAX_L
    L = dc.SH_MAX_L
    assert direct_grid(L) == -(-L // 1024) and fft_grid(L) == -(-L // 3712)
    assert (direct_grid(L) - 1) * 1024 + 1023 <= INT_MAX
    assert direct_grid(INT_MAX) <= 0 and fft_grid(INT_MAX) <= 0


# ---------------------------------------------------------------------------
# the sweep against the rules
# ---------------------------------------------------------------------------
def test_case_names_are_unique_and_inputs_have_the_listed_shape():
    cases = dc.sweep()
    names = [c["name"] for c in cases]
    assert len(names) == len(set(names))
    for c in cases:
        assert c["K"] in dc.ORDERS_K and c["form"] in ("default", "direct") and c["kind"] in dc.KINDS
        assert c["bank"] in dc.BANKS and c["n"] * len(c["angles"]) <= 65535 and 0 < c["L"] <= dc.SH_MAX_L
        if c["entry"] == "batch":
            assert c["K"] == 9 and len(c["angles"]) == c["n"]
        if c["kind"] == "impulse":
            assert c["n"] == c["K"] * len(c["positions"])
    c = next(c for c in cases if c["kind"] == "zero_between")
    x = dc.make_input(c)
    assert x.shape == (3, c["L"], c["K"]) and x.dtype == np.float32 and not x[1].any() and x[0].any() and x[2].any()
    c = next(c for c in cases if c["kind"] == "one_channel" and c["K"] == 16)
    x = dc.make_input(c)
    assert not x[:, :, :15].any() and x[:, :, 15].any()


def test_sweep_holds_every_listed_length_count_and_azimuth():
    """The values the sweep exists for, restated here so that deleting one from the case file fails."""
    lengths = {1, 2, 127, 128, 129, 383, 384, 385, 1023, 1024, 1025, 1406, 1407, 1408, 2048, 3711, 3712, 3713, 7423,
               7424, 7425, 11135, 11136, 11137, 48000}
    azimuths = {0.0, 90.0, 180.0, 270.0, 37.5, 359.999, -90.0, -37.5, 450.0, 720.5}
    cases = dc.sweep()
    for K in dc.ORDERS_K:
        mine = [c for c in cases if c["K"] == K and c["entry"] == "multi"]
        flat = [c for c in mine if c["kind"] == "flat" and c["scale"] == 1.0]
        for fft in (False, True):
            form = [c for c in flat if dc.runs_fft(c) == fft]
            seen = {c["L"] for c in form}
            want = {L for L in lengths if L >= 7424} if fft else lengths
            assert want <= seen, (K, fft, sorted(want - seen))
            assert any(L >= 200000 for L in seen), (K, fft)
            counts = {len(c["angles"]) for c in form}
            assert set(range(1, 10)) <= counts, (K, fft, counts)
            assert {c["n"] for c in form} >= {1, 2, 17} and max(c["n"] for c in form) >= 200, (K, fft)
            assert {c["bank"] for c in form} == {"packaged", "random"}, (K, fft)
            assert {c["kind"] for c in mine if dc.runs_fft(c) == fft} == set(dc.KINDS), (K, fft)
            assert {c["scale"] for c in mine if dc.runs_fft(c) == fft} >= {1e-6, 1.0, 1e3}, (K, fft)
            if K > 1:
                az = {a for c in form for a in c["angles"]}
                assert azimuths <= az and any(abs(a) > 1e5 for a in az), (K, fft, azimuths - az)
                assert any(str(a) == "-0.0" for c in form for a in c["angles"])
                assert any(len(set(c["angles"])) < len(c["angles"]) for c in form)                     # a duplicate
                assert any(list(c["angles"]) == sorted(c["angles"], reverse=True) and len(c["angles"]) > 2 for c in form)
        assert any(len(c["angles"]) >= 64 for c in flat), K
    batch = [c for c in cases if c["entry"] == "batch"]
    for fft in (False, True):
        seen = {c["L"] for c in batch if dc.runs_fft(c) == fft}
        assert ({L for L in lengths if L >= 7424} if fft else lengths) <= seen, (fft, seen)


def test_sweep_reaches_every_tile_edge():
    """Per K and form: one tile and several; a last tile or block with one output, with a full set and with one fewer;
    (direct form) lengths below, at and above the 128-sample delay and around the 1407-sample staged span; (FFT form)
    the first length that takes it, one azimuth and groups of four with every tail, A = 2 and 3 alone."""
    cases = [c for c in dc.sweep() if c["entry"] == "multi"]
    for K in dc.ORDERS_K:
        for fft in (False, True):
            seen = set()
            for c in cases:
                if c["K"] != K or dc.runs_fft(c) != fft:
                    continue
                assert takes_fft(c["L"], 32 if c["form"] == "direct" else 0) == fft
                tile = dc.tile_of(c)
                assert tile == (3712 if fft else 1024)
                tiles, last = last_tile(c["L"], tile)
                assert tiles == (fft_grid if fft else direct_grid)(c["L"])
                seen.add("one tile" if tiles == 1 else "several tiles")
                if tiles > 1:
                    seen.add("last 1" if last == 1 else "last full" if last == tile else
                             "last full - 1" if last == tile - 1 else "last partial")
                if not fft:
                    seen.add("below delay" if c["L"] < 128 else "at delay" if c["L"] == 128 else "above delay")
                    if c["L"] in (1406, 1407, 1408):
                        seen.add(f"span {c['L']}")
                ac, groups, tail = az_groups(len(c["angles"]))
                if fft:
                    seen.add("one azimuth" if ac == 1 else f"groups {min(groups, 2)} tail {tail % 4}")
            want = {"several tiles", "last 1", "last full", "last full - 1", "last partial"}
            if fft:
                want |= {"one azimuth", "groups 1 tail 2", "groups 1 tail 3", "groups 1 tail 0", "groups 2 tail 0",
                         "groups 2 tail 1", "groups 2 tail 2", "groups 2 tail 3"}
            else:
                want |= {"one tile", "below delay", "at delay", "above delay", "span 1406", "span 1407", "span 1408"}
            assert want <= seen, (K, fft, sorted(want - seen))


def test_impulse_positions_straddle_every_seam():
    for L, tile in ((dc.DIRECT_L, 1024), (dc.FFT_L, 3712), (11137, 3712)):
        P = dc.impulse_positions(L, tile)
        assert P == sorted(set(P)) and 0 <= P[0] and P[-1] == L - 1 and {0, 1} <= set(P)
        for s in range(tile, L + 1, tile):
            firsts = {p + 128 for p in P}              # first output of the response
            lasts = {p + 383 for p in P}               # last output of the response
            assert {s - 1, s} <= firsts and {s - 1, s} <= lasts, (L, s)
            assert {s - 1, s} & set(range(L)) <= set(P), (L, s)
        assert L - 129 in P and L - 128 in P           # the last input that reaches an output, the first that does not
    for K in dc.ORDERS_K:
        for c in dc.impulse_cases(K):
            assert c["positions"] == tuple(dc.impulse_positions(c["L"], dc.tile_of(c)))


# ---------------------------------------------------------------------------
# the closed form of an impulse's decode
# ---------------------------------------------------------------------------
@pytest.mark.parametrize("K", dc.ORDERS_K)
@pytest.mark.parametrize("bank_kind", dc.BANKS)
def test_impulse_closed_form_matches_the_oracle(K, bank_kind):
    """out[n] = sum_j R[j][k] bank[j][ear][n - p - 128]: the oracle (an FFT convolution, rounded to float32) agrees to
    1e-7 of the bank's peak for every channel, at positions at the start, inside, and cut off by the end."""
    L = 700
    bank = dc.bank_of(dict(bank=bank_kind, K=K))
    peak = np.abs(bank).max()
    for az in (0.0, 37.5, 270.0, -90.0, 720.5):
        for k in range(K):
            for p in (0, 1, 300, L - 384, L - 383, L - 130, L - 129, L - 128, L - 1):
                x = np.zeros((L, K), np.float32)
                x[p, k] = 1.0
                want = dc.impulse_response(K, k, p, L, az, bank)
                assert want.dtype == np.float64
                assert not want[: p + 128].any() and not want[p + 384:].any()
                assert np.abs(so.sh_decode(x, az, bank) - want).max() <= 1e-7 * peak, (az, k, p)
    # at az = 0 nothing rotates: the response is the bank's own row
    assert np.array_equal(dc.impulse_response(K, K - 1, 5, L, 0.0, bank)[133:389], bank[K - 1].T.astype(np.float64))


def test_reference_azimuth_is_reduced_exactly():
    assert dc.ref_azimuth(450.0) == 90.0 and dc.ref_azimuth(-90.0) == -90.0 and dc.ref_azimuth(720.5) == 0.5
    assert dc.ref_azimuth(36037.5) == 37.5 and abs(dc.ref_azimuth(3.0e38)) < 360.0
    x = np.random.default_rng(0).standard_normal((600, 16)).astype(np.float32)
    bank = dc.random_bank(16)
    assert np.array_equal(dc.reference(x, 36037.5, bank), dc.reference(x, 37.5, bank))


def test_segment_bound_sees_an_error_confined_to_the_last_block():
    """What the global bound of the older tests misses: an error of 1e-3 of the local level in the one output of a
    third block, under a decaying envelope."""
    rng = np.random.default_rng(1)
    ref = rng.standard_normal((7425, 2)) * np.exp(-np.arange(7425) / 1485.0)[:, None]
    got = ref.copy()
    got[7424] += 1e-3 * np.abs(ref[7361:]).max()
    assert np.abs(got - ref).max() <= 1e-4 * np.abs(ref).max()
    assert [v[:2] for v in dc.segment_violations(got, ref, 3712)] == [(7424, 7425)]
    assert dc.segment_violations(ref, ref, 3712) == [] and dc.segment_violations(ref, ref, 1024) == []
    got = ref.copy()
    got[100, 1] = np.nan
    assert [v[:2] for v in dc.segment_violations(got, ref, 1024)] == [(0, 1024)]
    zero = np.zeros((300, 2))
    assert dc.segment_violations(zero, zero, 1024) == [] and dc.segment_violations(zero + 1e-30, zero, 1024) != []


# ---------------------------------------------------------------------------
# sh_filters_kernel's angle arithmetic in float32
# ---------------------------------------------------------------------------
def angle_error(az, reduce):
    """Largest distance on the circle, over m = 1, 2, 3, between the angle the kernel hands to sincosf (float32:
    ``al = [fmodf(az, 360)] * (pi/180)``, then ``2 * al`` and ``3 * al``) and m times the float32 azimuth in float64.
    A model of the arithmetic, not a device measurement; sincosf's own error (about 1e-7) comes on top."""
    az32 = np.float32(az)
    if reduce:
        az32 = np.fmod(az32, np.float32(360.0))
    al = np.float32(az32 * np.float32(0.017453292519943295))
    exact = np.deg2rad(dc.ref_azimuth(az))
    worst = 0.0
    for m in (1.0, 2.0, 3.0):
        d = float(np.float32(np.float32(m) * al)) - m * exact
        worst = max(worst, abs(np.angle(np.exp(1j * d))))
    return worst


def test_float32_angle_model():
    """With the exact reduction the angle error stays below 2.5e-6 rad at every finite azimuth of the sweep, three
    orders below what the 1e-4 accuracy bound needs; without it the error grows with |az| (2e-5 rad at 36037.5,
    above 1e-3 rad at 1e6), which is why the kernel reduces first."""
    listed = set(dc.AZ_VALUES + dc.AZ_DUPLICATE + dc.AZ_DESCENDING + dc.AZ_FAR + dc.angles_of(dc.LARGE_A))
    listed |= {a for pair in dc.AZ_ALIASES for a in pair}
    grid = np.concatenate([np.linspace(-360.0, 360.0, 28801), np.random.default_rng(2).uniform(-1e7, 1e7, 2000)])
    worst = max(angle_error(a, True) for a in list(listed) + list(grid))
    assert worst <= 2.5e-6, worst
    assert max(angle_error(a, False) for a in np.linspace(-360.0, 360.0, 28801)) <= 2.5e-6
    assert angle_error(36037.5, False) > 1e-5 and angle_error(1.0e6, False) > 1e-3
    for a, b in dc.AZ_ALIASES:                           # fmodf maps both to the same float32 angle (or to +-0)
        ra, rb = np.fmod(np.float32(a), np.float32(360.0)), np.fmod(np.float32(b), np.float32(360.0))
        assert ra == rb, (a, b)
