"""Ambisonic -> binaural decode at orders 0 to 3 and several azimuths per input on the H100
(ssb_sh_decode_multi_batch, BatchedAudioRenderer.sh_decode_angles, soundspaces_b200.binauralize): against the
generalised oracle, against the outputs recorded from the reference's AmbisonicBinauralizer
(tests/golden/sh_orders_golden.npz), and against the second-order entry."""
import importlib.util
import os

import numpy as np
import pytest

from oracle import sh_orders as so

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_spec = importlib.util.spec_from_file_location(
    "make_sh_orders_golden", os.path.join(ROOT, "tests", "golden", "make_sh_orders_golden.py"))
mog = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(mog)

pytestmark = pytest.mark.gpu
ANGLES = [0.0, 90.0, 180.0, 270.0]
DIRECT = 32                     # ssb_set_debug flag: force the direct form
SSB_E_INVALID_ARG = -1          # include/ssb200.h


@pytest.fixture(scope="module")
def g():
    with np.load(os.path.join(ROOT, "tests", "golden", "sh_orders_golden.npz")) as z:
        return {k: z[k] for k in z.files}


@pytest.fixture(scope="module")
def r():
    from soundspaces_b200 import BatchedAudioRenderer
    return BatchedAudioRenderer(16000, 4096, device="cuda:0")


def decode(r, amb, angles, direct):
    import torch
    r.lib.ssb_set_debug(r.ctx.handle, DIRECT if direct else 0)
    try:
        out = r.sh_decode_angles(torch.from_numpy(amb), angles)
        torch.cuda.synchronize()
        return out.cpu().numpy()
    finally:
        r.lib.ssb_set_debug(r.ctx.handle, 0)


def rirs(seed, n, L, K):
    rng = np.random.default_rng(seed)
    env = np.exp(-np.arange(L) / max(L / 5.0, 20.0))[None, :, None]
    return (rng.standard_normal((n, L, K)) * env * 0.3).astype(np.float32)


@pytest.mark.parametrize("K", (1, 4, 9, 16))
@pytest.mark.parametrize("direct", (False, True), ids=("default", "direct"))
@pytest.mark.parametrize("L", (100, 5003, 7424, 20000))
def test_decode_vs_oracle_and_single_azimuth(r, g, K, direct, L):
    """L >= 7424 takes the FFT form by default; `direct` forces the direct form at every length."""
    amb = rirs(K * 1000 + L, 2, L, K)
    bank = g["bank"]
    multi = decode(r, amb, ANGLES + [37.5], direct)
    assert multi.shape == (2, 5, L, 2)
    for a, az in enumerate(ANGLES + [37.5]):
        single = decode(r, amb, [az], direct)
        assert np.array_equal(multi[:, a], single[:, 0])               # A = 5 rows == A = 1 decodes, bit for bit
        for i in range(2):
            lti = so.sh_decode(amb[i], az, bank)
            assert np.abs(multi[i, a] - lti).max() <= 1e-4 * np.abs(lti).max()


@pytest.mark.parametrize("K", mog.ORDERS_K)
@pytest.mark.parametrize("direct", (False, True), ids=("default", "direct"))
def test_decode_vs_tool(r, g, K, direct):
    az = list(mog.AZIMUTHS)
    amb = np.stack([mog.make_amb(mog.seed_of(K, a), K) for a in az])
    out = decode(r, amb, az, direct)
    for i, a in enumerate(az):
        ref = g[f"K{K}/az{a:g}"]
        assert np.abs(out[i, i] - ref).max() <= 5e-3 * np.abs(ref).max()
    imp = np.stack([mog.impulse(16, k) for k in range(9, 16)])
    out = decode(r, imp, list(mog.IMPULSE_AZ), direct)
    for i, k in enumerate(range(9, 16)):
        for a, azi in enumerate(mog.IMPULSE_AZ):
            assert np.abs(out[i, a] - g[f"imp/k{k}/az{azi:g}"]).max() <= 1e-5


@pytest.mark.parametrize("direct", (False, True), ids=("fft", "direct"))
def test_second_order_matches_existing_entry(r, direct):
    import torch
    L = 9001 if not direct else 3000
    amb = rirs(5, 3, L, 9)
    az = [10.0, 200.0, 300.0]
    r.lib.ssb_set_debug(r.ctx.handle, DIRECT if direct else 0)
    try:
        old = r.sh_decode(torch.from_numpy(amb), az).cpu().numpy()
    finally:
        r.lib.ssb_set_debug(r.ctx.handle, 0)
    for i, a in enumerate(az):
        new = decode(r, amb[i:i + 1], [a], direct)[0, 0]
        assert np.array_equal(new, old[i])


@pytest.mark.parametrize("K", (1, 4, 16))
def test_sh_decode_other_orders(r, g, K):
    """sh_decode keeps its one-azimuth-per-RIR form at every order."""
    import torch
    amb = rirs(K, 3, 2000, K)
    az = [0.0, 45.0, 300.0]
    out = r.sh_decode(torch.from_numpy(amb), az).cpu().numpy()
    for i in range(3):
        assert np.array_equal(out[i], decode(r, amb[i:i + 1], [az[i]], False)[0, 0])
    with pytest.raises(ValueError):
        r.sh_decode(torch.zeros(1, 100, 5), [0.0])
    with pytest.raises(ValueError):
        r.sh_decode(torch.zeros(1, 100, K), [0.0], hbank=np.zeros((9, 2, 256), np.float32))


def test_refusals_launch_nothing(r):
    import torch
    dev = r.device
    K, L, n_az = 16, 8000, 4
    amb = torch.zeros((2, L, K), device=dev)
    az = torch.zeros(n_az, device=dev)
    hb = torch.zeros((K, 2, 256), device=dev)
    filt = torch.zeros((n_az, K, 256, 2), device=dev)
    out = torch.zeros((2, n_az, L, 2), device=dev)
    st = r._stream()
    f = r.lib.ssb_sh_decode_multi_batch

    def call(n=2, k=K, length=L, a=amb.data_ptr(), na=n_az, pz=az.data_ptr(), ph=hb.data_ptr(), pf=filt.data_ptr(),
             po=out.data_ptr()):
        return f(r.ctx.handle, n, k, length, a, na, pz, ph, pf, po, st)

    bad = [dict(k=0), dict(k=2), dict(k=3), dict(k=5), dict(k=10), dict(k=15), dict(k=25), dict(na=0), dict(na=-1),
           dict(n=-1), dict(length=0), dict(length=2 ** 31 - 1), dict(n=16384, na=4), dict(n=65535, na=2), dict(a=None), dict(pz=None),
           dict(ph=None), dict(pf=None), dict(po=None), dict(a=amb.data_ptr() + 2), dict(pz=az.data_ptr() + 1),
           dict(ph=hb.data_ptr() + 2), dict(pf=filt.data_ptr() + 4), dict(po=out.data_ptr() + 4)]
    before = r.ctx.launch_count
    for kw in bad:
        assert call(**kw) == SSB_E_INVALID_ARG, kw
        assert b"ssb_sh_decode_multi_batch" in r.lib.ssb_last_error(r.ctx.handle), kw
    assert r.ctx.launch_count == before
    assert call(n=0) == 0 and r.ctx.launch_count == before
    # the largest shared-memory footprint (K = 16, direct form: input tile + one filter set) launches
    r.lib.ssb_set_debug(r.ctx.handle, DIRECT)
    try:
        assert call() == 0 and r.ctx.launch_count == before + 2
    finally:
        r.lib.ssb_set_debug(r.ctx.handle, 0)
    assert call() == 0 and r.ctx.launch_count == before + 5                       # FFT form: 3 launches
    assert call(n=65535 // 4, na=4, length=100, a=torch.zeros((65535 // 4, 100, K), device=dev).data_ptr(),
                po=torch.zeros((65535 // 4, 4, 100, 2), device=dev).data_ptr()) == 0
    torch.cuda.synchronize()


def test_binauralize_tree_matches_tool(g, tmp_path):
    from soundspaces_b200 import binauralize as bz
    amb_dir, bin_dir = tmp_path / "ambisonic", tmp_path / "binaural"
    mog.write_tree(str(amb_dir))
    with pytest.warns(UserWarning, match="not converted"):
        counts = bz.binauralize_tree(str(amb_dir), str(bin_dir), device="cuda:0", max_batch_bytes=1 << 20)
    assert counts == {"converted": 5, "written": 20, "refused": 1, "skipped_dirs": 0}
    for scene in mog.TREE:
        assert sorted(os.listdir(bin_dir / scene)) == sorted(str(a) for a in mog.ANGLES)
        for angle in mog.ANGLES:
            d = bin_dir / scene / str(angle)
            names = sorted(os.listdir(d))
            assert names == list(g[f"tree/{scene}/{angle}/files"])
            for name in names:
                raw = (d / name).read_bytes()
                assert raw[:44] == g[f"tree/{scene}/{angle}/{name}/header"].tobytes()
                got = np.frombuffer(raw[44:], "<f4").reshape(-1, 2)
                ref = g[f"tree/{scene}/{angle}/{name}/out"]
                _, x = bz.read_ambisonic_wav(str(amb_dir / scene / "irs" / name))
                lti = so.sh_decode(x, angle, g["bank"])
                assert got.shape == ref.shape
                assert np.abs(got - lti).max() <= 1e-4 * np.abs(lti).max()
                assert np.abs(got - ref).max() <= 5e-3 * np.abs(ref).max()
    # the script's skip rule: sceneB's angle directories hold as many entries as its irs/ and are skipped; sceneA's
    # irs/ also holds the refused file and the text file, so (as with the script) it is converted again
    snapshot = {p: p.read_bytes() for p in bin_dir.rglob("*.wav")}
    with pytest.warns(UserWarning, match="not converted"):
        counts = bz.binauralize_tree(str(amb_dir), str(bin_dir), device="cuda:0")
    assert counts == {"converted": 3, "written": 12, "refused": 1, "skipped_dirs": 4}
    assert {p: p.read_bytes() for p in bin_dir.rglob("*.wav")} == snapshot
    # once every input produces an output, a second run skips every angle directory
    for name in ("3_9.wav", "notes.txt"):
        os.remove(amb_dir / "sceneA" / "irs" / name)
    counts = bz.binauralize_tree(str(amb_dir), str(bin_dir), device="cuda:0")
    assert counts == {"converted": 0, "written": 0, "refused": 0, "skipped_dirs": 8}


def test_cli(tmp_path):
    from soundspaces_b200 import binauralize as bz
    from soundspaces_b200.renderer import sh_hrtf_bank
    amb_dir = tmp_path / "a"
    irs = amb_dir / "s" / "irs"
    irs.mkdir(parents=True)
    x = mog.make_amb(3, 4, 700)
    mog.write_wav(str(irs / "0_1.wav"), x, 16000, "f32")
    bz.main(["--ambisonic-dir", str(amb_dir), "--binaural-dir", str(tmp_path / "b" / "c"), "--angles", "45", "0"])
    for a in (45.0, 0.0):
        sr, y = read_f32(tmp_path / "b" / "c" / "s" / f"{a:g}" / "0_1.wav")
        lti = so.sh_decode(x, a, sh_hrtf_bank(16))
        assert sr == 16000 and np.abs(y - lti).max() <= 1e-4 * np.abs(lti).max()


def read_f32(path):
    raw = path.read_bytes()
    return int.from_bytes(raw[24:28], "little"), np.frombuffer(raw[44:], "<f4").reshape(-1, 2)


@pytest.mark.parametrize("K", (4, 16))
def test_config4_chain(r, g, K):
    """BASELINE config 4 shape of work at first and third order: decode -> set_dense_rir_bank -> render."""
    import torch
    from oracle import audio_oracle as ao
    from synth import make_source
    from soundspaces_b200 import AudioRequest, BatchedAudioRenderer
    sr, L, n = 16000, 6000, 2
    rr = BatchedAudioRenderer(sr, L, device="cuda:0")
    amb = rirs(90 + K, n, L, K)
    out = rr.sh_decode_angles(torch.from_numpy(amb), ANGLES)                    # (n, 4, L, 2)
    ids = rr.set_dense_rir_bank(out.reshape(n * 4, L, 2))
    src = make_source(5, sr)
    sid = rr.add_source(src)
    spec, wave = rr.render([AudioRequest(rir=i, source=sid) for i in ids], want_wave=True)
    torch.cuda.synchronize()
    out_h = out.cpu().numpy()
    for i in range(n):
        for a, az in enumerate(ANGLES):
            rir_ref = so.sh_decode(amb[i], az, g["bank"])
            assert np.abs(out_h[i, a] - rir_ref).max() <= 1e-4 * np.abs(rir_ref).max()
            w_ref, _ = ao.render_frame(src, rir_ref, sr)
            assert np.abs(wave[i * 4 + a].cpu().numpy() - w_ref).max() <= 1e-4 * np.abs(w_ref).max()
            _, s_ref = ao.render_frame(src, out_h[i, a], sr)
            assert np.allclose(spec[i * 4 + a].cpu().numpy(), s_ref, rtol=1e-4, atol=1e-5)
