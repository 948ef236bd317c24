"""Ambisonic -> binaural decode at orders 0 to 3 on the host: the generalised oracle against the outputs recorded from
the reference's closed AmbisonicBinauralizer (tests/golden/sh_orders_golden.npz, made by make_sh_orders_golden.py),
the packaged 16-row bank, and the file handling of soundspaces_b200.binauralize (formats, refusals, skip rule,
length buckets)."""
import importlib.util
import os
import struct

import numpy as np
import pytest

from oracle import sh_oracle
from oracle import sh_orders as so
from soundspaces_b200 import binauralize as bz

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_spec = importlib.util.spec_from_file_location(
    "make_sh_orders_golden", os.path.join(ROOT, "tests", "golden", "make_sh_orders_golden.py"))
mog = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(mog)
_spec = importlib.util.spec_from_file_location("make_sh_golden", os.path.join(ROOT, "tests", "golden", "make_sh_golden.py"))
msg = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(msg)


@pytest.fixture(scope="module")
def g():
    with np.load(os.path.join(ROOT, "tests", "golden", "sh_orders_golden.npz")) as z:
        return {k: z[k] for k in z.files}


@pytest.fixture(scope="module")
def g9():
    with np.load(os.path.join(ROOT, "tests", "golden", "sh_golden.npz")) as z:
        return {k: z[k] for k in z.files}


def test_bank16_packaged_and_nested(g):
    from soundspaces_b200.renderer import sh_hrtf_bank
    bank9 = np.load(os.path.join(ROOT, "soundspaces_b200", "data", "sh_hrtf_bank.npy"))
    assert np.array_equal(g["bank"][:9], bank9)              # the tool's 16-row bank nests the 9-row one, bit for bit
    for K in (1, 4, 9, 16):
        bank = sh_hrtf_bank(K)
        assert bank.dtype == np.float32 and bank.shape == (K, 2, 256) and bank.flags.c_contiguous
        assert np.array_equal(bank, g["bank"][:K])           # the text rows 9-15 round-trip exactly
    for K in (0, 2, 5, 25):
        with pytest.raises(ValueError):
            sh_hrtf_bank(K)


def test_rotation_matrix_third_order():
    for az in (0.0, 37.5, 90.0, 200.0):
        for K in (1, 4, 9, 16):
            R = so.rotation_matrix(az, K)
            assert R.shape == (K, K) and np.allclose(R @ R.T, np.eye(K), atol=1e-12)
        R = so.rotation_matrix(az, 16)
        for i_neg, i_pos, m in ((11, 13, 1), (10, 14, 2), (9, 15, 3)):
            assert R[i_pos, i_pos] == pytest.approx(np.cos(np.deg2rad(m * az)))
            assert R[i_neg, i_pos] == pytest.approx(np.sin(np.deg2rad(m * az)))
        assert R[12, 12] == R[6, 6] == R[2, 2] == R[0, 0] == 1.0
        assert np.array_equal(R[:9, :9], sh_oracle.rotation_matrix(az))
    for K in (2, 3, 5, 25):
        with pytest.raises(ValueError):
            so.rotation_matrix(0.0, K)


def test_oracle_unchanged_at_second_order(g9):
    for name, (az, seed) in msg.CASES.items():
        amb = msg.make_amb(seed)
        assert np.array_equal(so.sh_decode(amb, az, g9["bank"]), sh_oracle.sh_decode(amb, az, g9["bank"]))
        assert np.abs(so.sh_decode(amb, az, g9["bank"]) - g9[f"{name}/out"]).max() <= 5e-3 * np.abs(g9[f"{name}/out"]).max()


@pytest.mark.parametrize("K", mog.ORDERS_K)
@pytest.mark.parametrize("az", mog.AZIMUTHS)
def test_oracle_vs_tool_rir_shaped(g, K, az):
    ref = g[f"K{K}/az{az:g}"]
    got = so.sh_decode(mog.make_amb(mog.seed_of(K, az), K), az, g["bank"])
    assert got.shape == ref.shape == (mog.N, 2)
    assert np.abs(got - ref).max() <= 5e-3 * np.abs(ref).max()


@pytest.mark.parametrize("az", mog.IMPULSE_AZ)
def test_oracle_exact_on_third_order_impulses(g, az):
    for k in range(9, 16):
        got = so.sh_decode(mog.impulse(16, k), az, g["bank"])
        assert np.abs(got - g[f"imp/k{k}/az{az:g}"]).max() <= 1e-6


def test_recorded_tree_against_oracle(g, tmp_path):
    """Every recorded output of the tree, from the file as the reader decodes it (PCM16 at 1/32767)."""
    mog.write_tree(str(tmp_path))
    for scene, files in mog.TREE.items():
        for name, K, n, sr, kind, seed in files:
            path = tmp_path / scene / "irs" / name
            if kind in ("text", "extensible"):
                assert f"{name}" not in g[f"tree/{scene}/0/files"]
                continue
            got_sr, x = bz.read_ambisonic_wav(str(path))
            assert got_sr == sr and x.shape == (n, K)
            for angle in mog.ANGLES:
                ref = g[f"tree/{scene}/{angle}/{name}/out"]
                lti = so.sh_decode(x, angle, g["bank"])
                assert ref.shape == lti.shape
                assert np.abs(lti - ref).max() <= 5e-3 * np.abs(ref).max()


def test_reader_formats_and_refusals(tmp_path):
    x = mog.make_amb(1, 4, 500)
    mog.write_wav(str(tmp_path / "f.wav"), x, 16000, "f32")
    sr, y = bz.read_ambisonic_wav(str(tmp_path / "f.wav"))
    assert sr == 16000 and y.dtype == np.float32 and np.array_equal(y, x)
    q = (np.arange(-32768, 32768, 7, dtype=np.int64)[:4000].reshape(1000, 4)).astype("<i2")
    mog.write_wav(str(tmp_path / "p.wav"), q, 44100, "pcm16")
    sr, y = bz.read_ambisonic_wav(str(tmp_path / "p.wav"))
    assert sr == 44100 and np.array_equal(y, q.astype(np.float32) / np.float32(32767))     # the tool's scale
    assert y.min() < -1.0                                                                     # -32768 / 32767
    mog.write_wav(str(tmp_path / "e.wav"), x, 16000, "extensible")
    mog.write_wav(str(tmp_path / "c5.wav"), mog.make_amb(1, 5, 100), 16000, "f32")
    mog.write_wav(str(tmp_path / "c25.wav"), mog.make_amb(1, 25, 100), 16000, "f32")
    mog.write_wav(str(tmp_path / "i32.wav"), (x * 1e6).astype("<i4"), 16000, "pcm16")
    (tmp_path / "t.wav").write_text("not a wav")
    (tmp_path / "short.wav").write_bytes(b"RIFF\x04\x00\x00\x00WAVE")
    for name in ("e.wav", "c5.wav", "c25.wav", "i32.wav", "t.wav", "short.wav"):
        with pytest.raises(bz.WavFormatError):
            bz.read_ambisonic_wav(str(tmp_path / name))


def test_writer_header_matches_tool(g, tmp_path):
    n_checked = 0
    for key in g:
        if not key.endswith("/header"):
            continue
        header = g[key].tobytes()
        out = g[key[: -len("header")] + "out"]
        sr = struct.unpack_from("<I", header, 24)[0]
        assert bz.wav_header(out.shape[0], sr) == header
        path = tmp_path / "o.wav"
        bz.write_binaural_wav(str(path), sr, out)
        assert path.read_bytes() == header + out.astype("<f4").tobytes()
        n_checked += 1
    assert n_checked == 4 * 5                # 5 converted files x 4 angles


def test_skip_rule(tmp_path):
    irs = tmp_path / "amb" / "s" / "irs"
    irs.mkdir(parents=True)
    for name in ("a.wav", "b.wav", "notes.txt"):
        (irs / name).write_bytes(b"")
    d = tmp_path / "bin" / "s" / "90"
    assert not bz.angle_dir_done(str(irs), str(d))              # missing
    d.mkdir(parents=True)
    (d / "a.wav").write_bytes(b"")
    (d / "b.wav").write_bytes(b"")
    assert not bz.angle_dir_done(str(irs), str(d))              # 2 entries against 3: the script converts again
    (d / "x").write_bytes(b"")
    assert bz.angle_dir_done(str(irs), str(d))                  # equal counts: skipped, whatever the names
    assert bz.angle_dir_name(90) == "90" and bz.angle_dir_name(0.0) == "0" and bz.angle_dir_name(37.5) == "37.5"


def _direct_decode(amb, az, bank):
    """Time-domain restatement of the oracle: output n sums inputs m <= n only."""
    rot = amb.astype(np.float64) @ so.rotation_matrix(az, amb.shape[1]).T
    n = amb.shape[0]
    out = np.zeros((n + so.SH_DELAY, 2))
    for k in range(amb.shape[1]):
        for e in range(2):
            y = np.convolve(rot[:, k], bank[k, e].astype(np.float64))
            out[so.SH_DELAY:, e] += y[:n]
    return out[:n]


@pytest.mark.parametrize("n", (100, 1000, 1025, 5003, 7424, 20000))
def test_length_bucket_padding_is_exact(g, n):
    Lb = bz.length_bucket(n)
    assert n <= Lb <= max(1024, n * 9 // 8 + 1024) and Lb % 1024 == 0
    assert bz.length_bucket(Lb) == Lb
    x = mog.make_amb(n, 16, n)
    padded = np.zeros((Lb, 16), np.float32)
    padded[:n] = x
    # exact in the time domain: zeros after the input never reach an output before it
    assert np.array_equal(_direct_decode(padded, 37.5, g["bank"])[:n], _direct_decode(x, 37.5, g["bank"]))
    ref = so.sh_decode(x, 37.5, g["bank"])
    assert np.abs(so.sh_decode(padded, 37.5, g["bank"])[:n] - ref).max() <= 1e-6 * np.abs(ref).max()
