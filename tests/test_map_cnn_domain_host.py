"""The cases of tests/test_gpu_map_cnn_domain.py (tests/map_cnn_domain_cases.py) against a restatement of how
``ssb_map_encoder_batch`` tiles its work: each tile edge, kernel instance and limit the kernels have is reached by at
least one case.  Also the float32 calibration of the GPU file's accuracy bar, and the fused forwards' fallback for more
than 2^31 - 1 conv3 features.  No GPU."""
import copy
import os
import re

import pytest

torch = pytest.importorskip("torch")
nn = torch.nn

import map_cnn_domain_cases as cases  # noqa: E402
from map_cnn_models import map_obs  # noqa: E402
from soundspaces_b200 import encoder  # noqa: E402

# the tiling of soundspaces_b200/csrc/ssb200.cu
ENC_CL = 8            # CTAs per env; conv1: rank r computes rows r, r + ENC_CL, ...; conv2 / conv3: each rank computes
                      # ceil(C / ENC_CL) output channels
ENC_OCT = 2           # conv3: output channels per thread
MAP_PIX = 4           # conv1: output pixels of one row per thread
LIN_ROWS = 4          # Linear: output rows per CTA
LIN_ENVS = 16         # Linear: envs per tile
FEATURE_STRIDE = 256  # Linear: lane l of warp w sums the features l + 32 w + 256 k


def instance(c):
    """The map_encoder_conv_kernel<KW1, K2> instance ssb_map_encoder_batch launches for a case."""
    (_, kw1), (kh2, kw2), _ = c["K"]
    if kw1 == 8 and (kh2, kw2) == (4, 4):
        return "8,4"
    if kw1 == 5 and (kh2, kw2) == (3, 3):
        return "5,3"
    return "0,0"


def dispatch(kh, kw):
    """enc_conv_layer's instance of enc_conv_chw for conv3."""
    return "3x3" if (kh, kw) == (3, 3) else "4x4" if (kh, kw) == (4, 4) else "generic"


def chunk(oc):
    return -(-oc // ENC_CL)


def smem_terms(c):
    """The entry's shared-memory terms in floats: conv1 rows, the conv1 / conv2 / conv3 phases and the conv2 slice."""
    (c1, h1, w1, kh1, kw1, _, _), (c2, h2, w2, kh2, kw2, _, _), (c3, _, _, kh3, kw3, _, _) = cases.layer_shapes(c)
    C = c["C"]
    rows1 = c1 * chunk(h1) * w1
    ph1 = c1 * C * kh1 * kw1 + C * kh1 * c["W"]
    ph2 = c1 * kh2 * w1 + chunk(c2) * c1 * kh2 * kw2
    ph3 = c2 * h2 * w2 + chunk(c3) * c2 * kh3 * kw3
    return rows1, ph1, ph2, ph3, chunk(c2) * h2 * w2


def smem_bytes(c):
    rows1, ph1, ph2, ph3, s2 = smem_terms(c)
    return 4 * (max(rows1 + max(ph1, ph2), ph3) + s2)


def branch(c):
    """Which term of max(rows1 + max(conv1 phase, conv2 phase), conv3 phase) sets the footprint."""
    rows1, ph1, ph2, ph3, _ = smem_terms(c)
    if ph3 > rows1 + max(ph1, ph2):
        return "conv3"
    return "conv1" if ph1 >= ph2 else "conv2"


def fused():
    return cases.LAYOUTS + cases.LIMIT


def convs(layer):
    return [s[layer] for s in (cases.layer_shapes(c) for c in fused())]


def test_restated_tiling():
    """The constants restated above are the kernels' (by their definitions in the source), and so are the instance
    choices."""
    src = open(os.path.join(os.path.dirname(encoder.__file__), "csrc", "ssb200.cu")).read()
    for name, value in (("ENC_CL", ENC_CL), ("ENC_OCT", ENC_OCT), ("MAP_PIX", MAP_PIX), ("LIN_ROWS", LIN_ROWS),
                        ("LIN_ENVS", LIN_ENVS)):
        assert re.search(rf"constexpr int {name} = {value};", src), name
    warps = int(re.search(r"constexpr int LIN_WARPS = (\d+);", src).group(1))
    assert 32 * warps == FEATURE_STRIDE
    sel = re.search(r"auto conv = (.*?);", src, re.S).group(1)
    assert re.sub(r"\s+", " ", sel) == ("L1.kw == 8 && L2.kh == 4 && L2.kw == 4 ? map_encoder_conv_kernel<8, 4> "
                                        ": L1.kw == 5 && L2.kh == 3 && L2.kw == 3 ? map_encoder_conv_kernel<5, 3> "
                                        ": map_encoder_conv_kernel<0, 0>")
    assert "if (L.kh == 3 && L.kw == 3)" in src and "else if (L.kh == 4 && L.kw == 4)" in src
    assert encoder.MAP_SMEM_LIMIT == cases.SMEM_LIMIT and encoder.MAP_MAX_ENVS == cases.MAX_ENVS


def test_every_case_is_well_formed():
    every = cases.LAYOUTS + cases.LIMIT + cases.OVER_LIMIT + [cases.INPUT_LAYOUT, cases.BIG_B_LAYOUT, cases.HUGE_F]
    for c in every:
        assert cases.layer_shapes(c) is not None, c["name"]
        assert len(c["Cs"]) == len(c["K"]) == len(c["S"]) == 3 and len(c["bias"]) == 4, c["name"]
    names = [c["name"] for c in every]
    assert len(names) == len(set(names))
    assert cases.IDENTITY_LAYOUT in cases.LAYOUTS and cases.RELU_LAYOUT in cases.LAYOUTS


def test_map_channels():
    assert {c["C"] for c in fused()} >= {1, 2, 3, 5, 8}


def test_conv1_rows_and_columns():
    h1 = {h for _, h, *_ in convs(0)}
    assert {1, 8, 9, 17} <= h1 and any(1 < h < ENC_CL for h in h1), "H1 in {1, < 8, 8, 9, 17}"
    w1 = {w for _, _, w, *_ in convs(0)}
    assert {w % MAP_PIX for w in w1} == {0, 1, 2, 3}, "every MAP_PIX tail"
    assert any(w < MAP_PIX for w in w1), "W1 < 4"


def test_conv1_windows():
    rows = [(c, s) for c, s in zip(fused(), convs(0))]
    assert any(kh > sh for _, (_, _, _, kh, _, sh, _) in rows), "overlapping windows"
    assert any(sh > kh and sw > kw for _, (_, _, _, kh, kw, sh, sw) in rows), "strides that skip input"
    assert any((c["H"] - kh) % sh for c, (_, _, _, kh, _, sh, _) in rows), "trailing rows conv1 never reads"
    assert any((c["W"] - kw) % sw for c, (_, _, _, _, kw, _, sw) in rows), "trailing columns conv1 never reads"


def test_conv2_shapes():
    pairs = list(zip(convs(0), convs(1)))
    assert any(s2[1] == 1 and s2[3] == s1[1] > 1 for s1, s2 in pairs), "a conv2 as tall as conv1's output"
    assert any(sh > kh and sw > kw for _, _, _, kh, kw, sh, sw in convs(1)), "a conv2 stride larger than its kernel"


def test_channel_counts():
    for layer in range(3):
        oc = {s[0] for s in convs(layer)}
        assert any(c < ENC_CL for c in oc), f"C{layer + 1} < 8"
        assert any(c > ENC_CL and c % ENC_CL for c in oc), f"C{layer + 1} off a multiple of 8"
        assert any(c > ENC_CL for c in oc), f"C{layer + 1} > 8"
    assert any(chunk(c) % ENC_OCT for c, *_ in convs(2)), "an odd ceil(C3 / 8): ENC_OCT's tail"
    assert any(chunk(c) * (ENC_CL - 1) >= c > 1 for c, *_ in convs(1)), "conv2 ranks without a channel"
    assert any(c % chunk(c) and c > ENC_CL for c, *_ in convs(1)), "a short conv2 slice: a short conv3-gather owner"


def test_kernel_instances():
    got = {}
    for c in fused():
        (kh1, _), (sh1, sw1), (sh2, sw2) = c["K"][0], c["S"][0], c["S"][1]
        got.setdefault(instance(c), []).append((c, kh1, sh1 != sw1 and sh2 != sw2))
    assert any(kh1 != 8 and both for _, kh1, both in got["8,4"]), "<8, 4> at KH1 != 8, sh != sw in conv1 and conv2"
    assert any(kh1 != 5 for _, kh1, _ in got["5,3"]), "<5, 3> at KH1 != 5"
    generic = [c for c, _, _ in got["0,0"]]
    for k2 in ((3, 4), (4, 3)):
        assert any(c["K"][0][1] == 8 and c["K"][1] == k2 for c in generic), f"<0, 0>: a {k2} conv2 after a kw = 8 conv1"
    assert any(c["K"][0][1] != 8 and c["K"][1] == (4, 4) for c in generic), "<0, 0> with a 4 x 4 conv2"


def test_conv3_dispatch():
    c3 = convs(2)
    for inst in ("3x3", "4x4", "generic"):
        assert any(dispatch(kh, kw) == inst and sh != sw for _, _, _, kh, kw, sh, sw in c3), inst + " at sh != sw"
    assert any(kh == 3 and kw != 3 for _, _, _, kh, kw, _, _ in c3), "3 x k conv3"
    assert any(kh == 4 and kw != 4 for _, _, _, kh, kw, _, _ in c3), "4 x k conv3"


def test_non_square_kernels_and_strides_in_every_layer():
    for layer in range(3):
        assert any(s[3] != s[4] for s in convs(layer)), f"layer {layer + 1}: kh != kw"
        assert any(s[5] != s[6] for s in convs(layer)), f"layer {layer + 1}: sh != sw"


def test_biases():
    flags = [c["bias"] for c in cases.LAYOUTS]
    assert (False,) * 4 in flags, "bias=False on every layer"
    assert any(True in f and False in f for f in flags), "bias on some layers only"
    for i in range(4):
        assert any(f[i] for f in flags) and any(not f[i] for f in flags), f"layer {i + 1} with and without a bias"


def test_linear_edges():
    F = {cases.features(c) for c in fused()}
    assert {1, 255, 256, 257} <= F
    hidden = {c["hidden"] for c in fused()}
    assert {1, 3, 130} <= hidden
    assert {h % LIN_ROWS for h in hidden} >= {1, 2, 3}, "every LIN_ROWS tail"


def test_smem_edges_and_mirror():
    """The restated footprint equals encoder.map_encoder_smem_bytes for every case; each limit case sits at exactly
    232448 bytes through its own branch, its over-limit partner past it with no narrower over-limit shape between."""
    for c in cases.LAYOUTS + cases.LIMIT + cases.OVER_LIMIT + [cases.INPUT_LAYOUT, cases.BIG_B_LAYOUT]:
        got = encoder.map_encoder_smem_bytes(cases.make_cnn(c), c["C"], c["H"], c["W"])
        assert got == (smem_bytes(c), cases.features(c)), c["name"]
    for c in cases.LAYOUTS + [cases.INPUT_LAYOUT, cases.BIG_B_LAYOUT]:
        assert smem_bytes(c) <= cases.SMEM_LIMIT, c["name"]
    assert [smem_bytes(c) for c in cases.LIMIT] == [cases.SMEM_LIMIT] * 3
    assert [branch(c) for c in cases.LIMIT] == ["conv1", "conv2", "conv3"]
    assert [branch(c) for c in cases.OVER_LIMIT] == ["conv1", "conv2", "conv3"]
    for lim, over in zip(cases.LIMIT, cases.OVER_LIMIT):
        assert dict(lim, W=over["W"], name=over["name"]) == over and over["W"] > lim["W"]
        assert smem_bytes(over) > cases.SMEM_LIMIT
        for W in range(lim["W"] + 1, over["W"]):
            assert smem_bytes(dict(lim, W=W)) <= cases.SMEM_LIMIT, "a narrower over-limit shape exists"
    # the reference's channels reach the limit exactly in the conv1 and conv2 phases
    assert [c["Cs"] for c in cases.LIMIT[:2]] == [cases.REF_C] * 2


def _worst_ratio(c, x):
    """max over envs of max|f32 - f64| / max|f64| of torch's CPU forward, on the features and the pre-activation."""
    cnn = cases.make_cnn(c, seed=len(c["name"]))
    ref = copy.deepcopy(cnn).double()
    worst = 0.0
    with torch.no_grad():
        xx = x.permute(0, 3, 1, 2)
        for a, b in ((cnn[:6](xx), ref[:6](xx.double())), (cnn[:7](xx), ref[:7](xx.double()))):
            for e in range(a.shape[0]):
                scale = b[e].abs().max().item()
                if scale > 0:
                    worst = max(worst, (a[e].double() - b[e]).abs().max().item() / scale)
    return worst


def test_float32_calibration():
    """torch's float32 forward on the CPU against float64 on every case, with the GPU file's inputs: the worst error is
    a small fraction of the bar (1e-4 of the env's largest value)."""
    worst = 0.0
    for c in cases.LAYOUTS + cases.LIMIT:
        B = 3 if c in cases.LIMIT else 17
        worst = max(worst, _worst_ratio(c, map_obs(B, c["H"], c["W"], c["C"], seed=len(c["name"]) + 1, kind="dense")))
    c = cases.INPUT_LAYOUT
    for kind in ("gm", "am", "dense"):
        for scale in (1.0,) + cases.SCALES:
            worst = max(worst, _worst_ratio(c, map_obs(5, c["H"], c["W"], c["C"], seed=9, kind=kind) * scale))
    assert worst <= 1e-5, worst


# ------------------------------------------------------------------------------------------------ F past INT32_MAX
class FakeCuda(torch.Tensor):
    """A CPU tensor that reports ``is_cuda``, for the fused forwards' device check."""

    @property
    def is_cuda(self):
        return True


class Module(nn.Module):
    """The attributes fused_map_forward and fused_visual_forward read (depth only for the visual encoder)."""

    def __init__(self, cnn):
        super().__init__()
        self._map_type, self._n_input_gm, self._n_input_rgb, self._n_input_depth = "gm", 1, 0, 1
        self.cnn = cnn


def _huge_f_cnn(C3):
    """HUGE_F's layout with C3 channels, on the meta device (no memory)."""
    c = cases.HUGE_F
    H, W = c["H"], c["W"]
    return nn.Sequential(nn.Conv2d(1, 1, 1, device="meta"), nn.ReLU(True), nn.Conv2d(1, 1, 1, device="meta"),
                         nn.ReLU(True), nn.Conv2d(1, C3, 1, device="meta"), nn.Flatten(),
                         nn.Linear(C3 * H * W, 1, device="meta"), nn.ReLU(True))


def test_more_than_int32_max_features_run_the_original(monkeypatch):
    """Both entries refuse F > 2^31 - 1 (their Linear takes F as an int, and conv3's store index would overflow), so
    the fused forwards return None for it and the patched modules run the original; one channel fewer (F <= 2^31 - 1,
    the same shared memory) still reaches the library."""
    from soundspaces_b200 import renderer
    calls = []

    class Ops:
        def map_encoder(self, x, cnn):
            calls.append("map")
            return "fused"

        def visual_encoder(self, rgb, depth, cnn):
            calls.append("visual")
            return "fused"

    monkeypatch.setattr(renderer.WaveformOps, "get", staticmethod(lambda device: Ops()))
    c = cases.HUGE_F
    x = torch.zeros(1, c["H"], c["W"], 1).as_subclass(FakeCuda)
    C3 = c["Cs"][2]
    for n, want in ((C3, None), (C3 - 1, "fused")):
        cnn = _huge_f_cnn(n)
        nbytes, F = encoder.map_encoder_smem_bytes(cnn, 1, c["H"], c["W"])
        assert encoder.visual_encoder_smem_bytes(cnn, 1, c["H"], c["W"])[0] == nbytes
        assert nbytes <= cases.SMEM_LIMIT and (F > 2 ** 31 - 1) == (want is None)
        if n == C3:
            assert (nbytes, F) == (cases.HUGE_F_SMEM, cases.HUGE_F_FEATURES)
        m = Module(cnn)
        with torch.no_grad():
            assert encoder.fused_map_forward(m, {"gm": x}) == want
            assert encoder.fused_visual_forward(m, {"depth": x}) == want
    assert calls == ["map", "visual"]
