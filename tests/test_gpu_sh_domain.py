"""The ambisonic -> binaural decode on the H100 over the inputs its entries accept (``ssb_sh_decode_batch``,
``ssb_sh_decode_multi_batch``, ``sh_decode``, ``sh_decode_angles``, ``soundspaces_b200.binauralize``): every case of
tests/sh_domain_cases.py against float64 (``oracle/sh_orders.py``, or the closed form of an impulse's decode), with a
bound per tile or block for full-scale inputs; bit identity across azimuth counts, batch sizes, positions and entries;
back-to-back calls; the refusals of the C entries; and a tree of files at the seam lengths.
tests/test_sh_domain_host.py checks that the case list reaches every seam."""
import os
import struct

import numpy as np
import pytest

import sh_domain_cases as dc

pytestmark = pytest.mark.gpu
DIRECT = 32                     # ssb_set_debug flag: force the direct form
SSB_E_INVALID_ARG = -1          # include/ssb200.h


@pytest.fixture(scope="module")
def r():
    from soundspaces_b200 import BatchedAudioRenderer
    return BatchedAudioRenderer(16000, 4096, device="cuda:0")


def run(r, x, angles, form="default", bank=None, entry="multi"):
    """(n, A, L, 2) from ``sh_decode_angles``; (n, L, 2) from ``sh_decode`` (``angles`` then holds one per input)."""
    import torch
    r.lib.ssb_set_debug(r.ctx.handle, DIRECT if form == "direct" else 0)
    try:
        f = r.sh_decode if entry == "batch" else r.sh_decode_angles
        out = f(torch.from_numpy(x), angles if isinstance(angles, torch.Tensor) else list(angles), hbank=bank)
        torch.cuda.synchronize()
        return out.cpu().numpy()
    finally:
        r.lib.ssb_set_debug(r.ctx.handle, 0)


def run_case(r, c, x=None):
    x = dc.make_input(c) if x is None else x
    return x, run(r, x, c["angles"], c["form"], dc.random_bank(c["K"]) if c["bank"] == "random" else None, c["entry"])


def accuracy(c, x, out, inputs=None):
    """Failures of one case against the oracle as strings.  Decaying inputs keep the global bound
    max|d| <= 1e-4 max|ref|; every other kind is full scale everywhere and is held to it inside each tile or block."""
    bank = dc.bank_of(c)
    bad = []
    for i in range(c["n"]) if inputs is None else inputs:
        for a, az in enumerate(c["angles"]):
            if c["entry"] == "batch":
                if a != i:
                    continue
                got = out[i]
            else:
                got = out[i, a]
            ref = dc.reference(x[i], az, bank)
            if c["kind"] == "decay":
                err, bound = np.abs(got.astype(np.float64) - ref).max(), 1e-4 * np.abs(ref).max()
                if not err <= bound:
                    bad.append(f"{c['name']} input {i} az {az}: {err:.3g} > {bound:.3g}")
            else:
                for s, e, err, bound in dc.segment_violations(got, ref, dc.tile_of(c)):
                    bad.append(f"{c['name']} input {i} az {az} outputs [{s}, {e}): {err:.3g} > {bound:.3g}")
    return bad


def report(bad):
    assert not bad, f"{len(bad)} failures, the first: " + "; ".join(bad[:8])


# ---------------------------------------------------------------------------
# accuracy
# ---------------------------------------------------------------------------
@pytest.mark.parametrize("K", dc.ORDERS_K)
def test_every_length_in_both_forms(r, K):
    """Each output tile (direct form) or overlap-save block (FFT form) within 1e-4 of its own peak; nothing but zeros
    up to the 128-sample delay; and the two forms within 1e-5 of the peak of each other from 7424 samples on."""
    bad, outs = [], {}
    for c in dc.length_cases(K):
        x, out = run_case(r, c)
        assert out.shape == (c["n"], len(c["angles"]), c["L"], 2)
        bad += accuracy(c, x, out)
        if not dc.runs_fft(c) and out[:, :, :dc.SH_DELAY].any():
            bad.append(f"{c['name']}: non-zero output before the delay")
        if len(c["angles"]) == 1:
            outs[c["L"], c["form"]] = out
    for (L, form), out in outs.items():
        if form == "direct":
            peak = np.abs(out).max()
            if not np.abs(outs[L, "default"].astype(np.float64) - out).max() <= 1e-5 * peak:
                bad.append(f"K{K} L{L}: the FFT and direct forms differ by more than 1e-5 of the peak")
    assert sum(1 for k in outs if k[1] == "direct") == sum(1 for L in dc.LENGTHS if L >= dc.FFT_MIN_L)
    report(bad)


def test_second_order_entry_at_every_length(r):
    """``ssb_sh_decode_batch`` against the oracle, and row for row bit-identical to the multi entry at K = 9."""
    bad = []
    for c in dc.batch_entry_cases():
        x, out = run_case(r, c)
        assert out.shape == (c["n"], c["L"], 2)
        bad += accuracy(c, x, out)
        for i, az in enumerate(c["angles"]):
            if not np.array_equal(out[i], run(r, x[i:i + 1], [az], c["form"])[0, 0]):
                bad.append(f"{c['name']} input {i}: differs from the multi entry")
    report(bad)


@pytest.mark.parametrize("K", dc.ORDERS_K)
def test_azimuth_counts(r, K):
    """A = 1 ... 9 and 64: every row against the oracle and bit-identical to the A = 1 decode at its azimuth (the FFT
    form takes the azimuths in groups of four; a partial last group must neither drop nor disturb a row)."""
    bad, single = [], {}
    for c in dc.count_cases(K):
        x, out = run_case(r, c)
        assert out.shape == (2, len(c["angles"]), c["L"], 2)
        bad += accuracy(c, x, out)
        for a, az in enumerate(c["angles"]):
            key = (c["L"], az)
            if key not in single:
                single[key] = run(r, x, [az], c["form"])[:, 0]
            if not np.array_equal(out[:, a], single[key]):
                bad.append(f"{c['name']} row {a}: differs from the A = 1 decode")
    report(bad)


@pytest.mark.parametrize("K", (4, 9, 16))
def test_azimuth_values(r, K):
    """Negative angles, angles of 360 and more, -0.0, duplicates, a descending list and azimuths up to 3e38 meet the
    bound (the kernel reduces the angle exactly); a duplicate gives identical rows; az and az + 360 k decode alike."""
    bad = []
    for c in dc.azimuth_cases(K):
        x, out = run_case(r, c)
        bad += accuracy(c, x, out)
        for a, az in enumerate(c["angles"]):
            first = c["angles"].index(az)
            if first != a and not np.array_equal(out[:, a], out[:, first]):
                bad.append(f"{c['name']}: rows {first} and {a} of the same azimuth differ")
    flat = [a for pair in dc.AZ_ALIASES for a in pair]
    for L in (dc.DIRECT_L, dc.FFT_L):
        x = dc.make_input(dc.case("alias", K, L, flat, n=1, seed=51))
        out = run(r, x, flat)
        for j, pair in enumerate(dc.AZ_ALIASES):
            if not np.array_equal(out[:, 2 * j], out[:, 2 * j + 1]):
                bad.append(f"K{K} L{L}: azimuths {pair} decode differently")
    report(bad)


@pytest.mark.parametrize("K", dc.ORDERS_K)
def test_non_finite_azimuths(r, K):
    """Given on the host they are refused before anything is launched.  In a device tensor they are not read back:
    their rows are NaN (at K = 1 nothing rotates and the azimuth is unused) and the other rows of the same call,
    including those of the same group of four, are unaffected bit for bit."""
    import torch
    x = dc.make_input(dc.case("nan", K, 100, (0.0,), seed=52))
    before = r.ctx.launch_count
    for az in ([0.0, float("nan")], [float("inf"), 0.0], [0.0, float("-inf")]):
        with pytest.raises(ValueError, match="finite"):
            r.sh_decode_angles(torch.from_numpy(x), az)
        with pytest.raises(ValueError, match="finite"):
            r.sh_decode(torch.from_numpy(x), az)
    assert r.ctx.launch_count == before
    az = [37.5, float("nan"), 90.0, float("inf"), float("-inf"), 200.0]
    finite = [0, 2, 5]
    for L in (dc.DIRECT_L, dc.FFT_L):
        x = dc.make_input(dc.case("nan", K, L, (0.0,), seed=53))
        out = run(r, x, torch.tensor(az, dtype=torch.float32, device=r.device))
        want = run(r, x, [az[a] for a in finite])
        assert np.array_equal(out[:, finite], want), (K, L)
        if K > 1:
            assert np.isnan(out[:, [1, 3, 4]]).all(), (K, L)
        else:
            assert np.array_equal(out[:, [1, 3, 4]], want), (K, L)


@pytest.mark.parametrize("K", dc.ORDERS_K)
def test_input_counts_and_positions(r, K):
    """An input's rows do not depend on how many inputs the call holds, on its position, or on its neighbours: the
    decodes of the first 1, 2 and 17 inputs of a pool of 300 are slices of the decode of all 300, and a permuted
    batch gives the permuted rows, bit for bit.  Accuracy at the first, middle and last input of each call."""
    bad = []
    for L in (1100, dc.FFT_L):
        cases = [c for c in dc.input_count_cases(K) if c["L"] == L]
        pool = dc.make_input(cases[-1])
        assert pool.shape[0] == 300
        _, full = run_case(r, cases[-1], pool)
        for c in cases:
            _, out = run_case(r, c, pool[:c["n"]])
            bad += accuracy(c, pool, out, sorted({0, c["n"] // 2, c["n"] - 1}))
            if not np.array_equal(out, full[:c["n"]]):
                bad.append(f"{c['name']}: differs from the same inputs in the call of 300")
        perm = np.random.default_rng(61).permutation(300)
        _, out = run_case(r, cases[-1], np.ascontiguousarray(pool[perm]))
        if not np.array_equal(out, full[perm]):
            bad.append(f"K{K} L{L}: a permuted batch does not give the permuted rows")
    report(bad)


@pytest.mark.parametrize("K", dc.ORDERS_K)
def test_random_bank_and_bank_lifetime(r, K):
    """A bank whose ears are unrelated (the packaged bank's ears are mirror images, so a swap of the ears is invisible
    at its sign + channels).  A bank passed to a call serves that call only: the next call without one decodes with
    the packaged bank again."""
    bad = []
    for c in dc.bank_cases(K):
        x, out = run_case(r, c)
        bad += accuracy(c, x, out)
        packaged = dict(c, bank="packaged", name=c["name"] + "_then_packaged")
        _, out = run_case(r, packaged, x)
        bad += accuracy(packaged, x, out)
    report(bad)
    c = dc.bank_cases(K)[0]
    x = dc.make_input(c)
    via_batch = run(r, x, c["angles"] * c["n"], bank=dc.random_bank(K), entry="batch")       # sh_decode takes one too
    assert not dc.segment_violations(via_batch[0], dc.reference(x[0], c["angles"][0], dc.random_bank(K)), dc.SH_TILE)
    again = run(r, x, c["angles"] * c["n"], entry="batch")
    assert not dc.segment_violations(again[0], dc.reference(x[0], c["angles"][0], dc.bank_of(dict(c, bank="packaged"))),
                                     dc.SH_TILE)


@pytest.mark.parametrize("K", dc.ORDERS_K)
def test_input_kinds(r, K):
    """The decaying RIR shape (global bound), inputs scaled by 1e-6 and 1e3 (the relative bound holds), one live
    channel, and a zero input between two live ones, whose rows are exactly zero in both forms."""
    bad = []
    for c in dc.kind_cases(K):
        x, out = run_case(r, c)
        bad += accuracy(c, x, out)
        if c["kind"] == "zero_between" and (out[1].any() or not out[0].any() or not out[2].any()):
            bad.append(f"{c['name']}: the zero input's rows are not exactly zero beside live ones")
    for L in (dc.DIRECT_L, dc.FFT_L):
        for form in dc.forms_at(L):
            if run(r, np.zeros((2, L, K), np.float32), dc.angles_of(5), form).any():
                bad.append(f"K{K} L{L} {form}: silence does not decode to exact zeros")
    report(bad)


@pytest.mark.parametrize("K", dc.ORDERS_K)
def test_impulses(r, K):
    """A unit impulse in channel k at sample p decodes to column k of the rotated bank behind p + 128, for every k
    and every p at the ends of the input and on both sides of every tile and block seam: within 2e-6 of the bank's
    peak in the direct form, with exact zeros outside the 256 taps, and within 1e-5 in the FFT form.  An index off by
    one at a seam is an error of the order of the bank itself."""
    bad = []
    for c in dc.impulse_cases(K):
        x, out = run_case(r, c)
        bank = dc.bank_of(c)
        peak = float(np.abs(bank).max())
        tol = (1e-5 if dc.runs_fft(c) else 2e-6) * peak
        P = c["positions"]
        for a, az in enumerate(c["angles"]):
            for k in range(K):
                for j, p in enumerate(P):
                    got = out[k * len(P) + j, a]
                    want = dc.impulse_response(K, k, p, c["L"], az, bank)
                    err = np.abs(got - want).max()
                    if not err <= tol:
                        bad.append(f"{c['name']} az {az} channel {k} at {p}: {err:.3g} > {tol:.3g} "
                                   f"(first bad output {int(np.argmax(~(np.abs(got - want).max(1) <= tol)))})")
                    elif not dc.runs_fft(c) and (got[:p + 128].any() or got[p + 384:].any()):
                        bad.append(f"{c['name']} az {az} channel {k} at {p}: non-zero output outside the taps")
    report(bad)


# ---------------------------------------------------------------------------
# calls in a row
# ---------------------------------------------------------------------------
def test_back_to_back_calls_share_the_filter_spectra_safely(r):
    """Two FFT-form calls with different azimuths on one stream with no synchronise between them (both write the
    context's filter-spectrum scratch), a call that makes that scratch grow, and the first call again: each equals
    its result when run alone."""
    import torch
    K, L = 16, dc.FFT_L
    x = torch.from_numpy(dc.make_input(dc.case("b2b", K, L, (0.0,), n=3, seed=95))).to(r.device)
    first, second, many = [10.0, 200.0, 37.5], [300.0, -45.0, 90.0, 0.5, 123.0], list(dc.angles_of(200))
    alone = []
    for az in (first, second, many):
        alone.append(r.sh_decode_angles(x, az).cpu())
        torch.cuda.synchronize()
    outs = [r.sh_decode_angles(x, first), r.sh_decode_angles(x, second)]
    outs.append(r.sh_decode_angles(x, list(dc.angles_of(300))))             # more azimuths than any call before
    outs += [r.sh_decode_angles(x, many), r.sh_decode_angles(x, first)]
    torch.cuda.synchronize()
    alone.append(r.sh_decode_angles(x, list(dc.angles_of(300))).cpu())
    for i, (got, want) in enumerate(zip(outs, (alone[0], alone[1], alone[3], alone[2], alone[0]))):
        assert torch.equal(got.cpu(), want), i
    c = dc.case("b2b", K, L, many[:2], n=3, seed=95)
    report(accuracy(c, x.cpu().numpy(), outs[3][:, :2].cpu().numpy(), [1]))


# ---------------------------------------------------------------------------
# refusals of ssb_sh_decode_batch (tests/test_gpu_sh_orders.py holds the multi entry's)
# ---------------------------------------------------------------------------
def test_second_order_entry_refusals_launch_nothing(r):
    import torch
    dev = r.device
    B, L = 2, 8000
    amb = torch.zeros((B, L, 9), device=dev)
    az = torch.zeros(B, device=dev)
    hb = torch.zeros((9, 2, 256), device=dev)
    filt = torch.zeros((B, 9, 256, 2), device=dev)
    out = torch.zeros((B, L, 2), device=dev)
    st = r._stream()

    def call(b=B, length=L, a=amb.data_ptr(), pz=az.data_ptr(), ph=hb.data_ptr(), pf=filt.data_ptr(), po=out.data_ptr()):
        return r.lib.ssb_sh_decode_batch(r.ctx.handle, b, a, length, pz, ph, pf, po, st)

    # L = 2^31 - 1 and no other large L: there both grid computations would wrap to a launch CUDA rejects, so even
    # without the limit no kernel would run over these small buffers
    bad = [dict(b=-1), dict(b=65536), dict(length=0), dict(length=-5), dict(length=2 ** 31 - 1), dict(a=None),
           dict(pz=None), dict(ph=None), dict(pf=None), dict(po=None), dict(a=amb.data_ptr() + 2),
           dict(pz=az.data_ptr() + 1), dict(ph=hb.data_ptr() + 2), dict(pf=filt.data_ptr() + 4), dict(po=out.data_ptr() + 4)]
    before = r.ctx.launch_count
    for kw in bad:
        assert call(**kw) == SSB_E_INVALID_ARG, kw
        assert b"ssb_sh_decode_batch" in r.lib.ssb_last_error(r.ctx.handle), kw
    assert r.ctx.launch_count == before
    assert call(b=0) == 0 and call(b=0, a=None) == 0 and r.ctx.launch_count == before
    r.lib.ssb_set_debug(r.ctx.handle, DIRECT)
    try:
        assert call() == 0 and r.ctx.launch_count == before + 2                     # filters + direct form
    finally:
        r.lib.ssb_set_debug(r.ctx.handle, 0)
    assert call() == 0 and r.ctx.launch_count == before + 5                         # filters + spectra + blocks
    big = 65535                                                                     # the largest batch runs
    amb, az = torch.zeros((big, 100, 9), device=dev), torch.zeros(big, device=dev)
    filt = torch.empty((big, 9, 256, 2), device=dev)
    out = torch.empty((big, 100, 2), device=dev)
    assert call(b=big, length=100, a=amb.data_ptr(), pz=az.data_ptr(), pf=filt.data_ptr(), po=out.data_ptr()) == 0
    torch.cuda.synchronize()
    assert not out.any()


# ---------------------------------------------------------------------------
# files
# ---------------------------------------------------------------------------
TREE_LENGTHS = (1, 129, 1023, 1025, 3713, 7424, 7425, 11137)
TREE_ANGLES = (-90, 0, 37.5, 450)


def write_wav(path, x, sr):
    """float32 data -> tag 3, int16 data -> tag 1 (PCM16), with a plain 16-byte ``fmt `` chunk."""
    n, ch = x.shape
    bits = 8 * x.dtype.itemsize
    fmt = struct.pack("<HHIIHH", 1 if x.dtype.kind == "i" else 3, ch, sr, sr * ch * bits // 8, ch * bits // 8, bits)
    payload = np.ascontiguousarray(x).tobytes()
    with open(path, "wb") as f:
        f.write(b"RIFF" + struct.pack("<I", 36 + len(payload)) + b"WAVE" + b"fmt " + struct.pack("<I", 16) + fmt
                + b"data" + struct.pack("<I", len(payload)) + payload)


def test_tree_at_the_seam_lengths(tmp_path):
    """``binauralize_tree`` on float32 and PCM16 files of every order at the seam lengths, at angles below 0 and above
    360: each output keeps its input's length and is held to the bound inside every tile or block of the padded batch
    it was decoded in; the directories are named as ``angle_dir_name`` names them."""
    from soundspaces_b200 import binauralize as bz
    from soundspaces_b200.renderer import sh_hrtf_bank
    rng = np.random.default_rng(96)
    files = {}
    for s, K in enumerate(dc.ORDERS_K):
        irs = tmp_path / "amb" / f"scene{K}" / "irs"
        irs.mkdir(parents=True)
        for i, L in enumerate(TREE_LENGTHS):
            x = (rng.standard_normal((L, K)) * 0.3).astype(np.float32)
            if (i + s) % 2:
                x = np.round(x * 8000.0).astype("<i2")
            write_wav(str(irs / f"{i}_{L}.wav"), x, 16000 + K)
            files[f"scene{K}", f"{i}_{L}.wav"] = (K, L)
    counts = bz.binauralize_tree(str(tmp_path / "amb"), str(tmp_path / "bin"), TREE_ANGLES, device="cuda:0")
    assert counts == {"converted": len(files), "written": 4 * len(files), "refused": 0, "skipped_dirs": 0}
    assert [bz.angle_dir_name(a) for a in TREE_ANGLES] == ["-90", "0", "37.5", "450"]
    bad = []
    for (scene, name), (K, L) in files.items():
        assert sorted(os.listdir(tmp_path / "bin" / scene)) == sorted(bz.angle_dir_name(a) for a in TREE_ANGLES)
        sr, x = bz.read_ambisonic_wav(str(tmp_path / "amb" / scene / "irs" / name))
        tile = dc.SHF_HOP if bz.length_bucket(L) >= dc.FFT_MIN_L else dc.SH_TILE
        for a in TREE_ANGLES:
            raw = (tmp_path / "bin" / scene / bz.angle_dir_name(a) / name).read_bytes()
            assert raw[:44] == bz.wav_header(L, 16000 + K) and len(raw) == 44 + 8 * L, (scene, name, a)
            got = np.frombuffer(raw[44:], "<f4").reshape(-1, 2)
            for s, e, err, bound in dc.segment_violations(got, dc.reference(x, a, sh_hrtf_bank(K)), tile):
                bad.append(f"{scene}/{a}/{name} outputs [{s}, {e}): {err:.3g} > {bound:.3g}")
    report(bad)
