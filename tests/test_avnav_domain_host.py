"""The cases of tests/test_gpu_avnav_policy_domain.py (tests/avnav_domain_cases.py) against a restatement of how
``ssb_visual_encoder_batch`` and ``ssb_gru_step_batch`` tile their work: each tile edge, dispatch instance and limit
the kernels have is reached by at least one case.  Also the zero-env calls of ``WaveformOps``, which return empty
outputs without calling the library.  No GPU."""
import pytest

torch = pytest.importorskip("torch")
nn = torch.nn

import avnav_domain_cases as cases  # noqa: E402
from soundspaces_b200 import encoder  # noqa: E402

# the tiling of soundspaces_b200/csrc/ssb200.cu
ENC_CL = 8            # CTAs per env; conv2 / conv3: each computes ceil(C / ENC_CL) output channels
ENC_OCT = 2           # conv2 / conv3: output channels per thread
VIS_PIX = 4           # conv1: output pixels of one row per thread; rank r computes rows r, r + ENC_CL, ...
WARP = 32             # conv1: the lanes of a warp are 32 consecutive output channels
LIN_ROWS = 4          # Linear: output rows per CTA
LIN_ENVS = 16         # Linear and GRU: envs per tile
FEATURE_STRIDE = 256  # Linear and GRU: lane l of warp w sums the features l + 32 w + 256 k


def dispatch(kh, kw):
    """enc_conv_layer's instance of enc_conv_chw for a conv2 / conv3 kernel."""
    return "3x3" if (kh, kw) == (3, 3) else "4x4" if (kh, kw) == (4, 4) else "generic"


def smem_terms(c):
    """The entry's shared-memory terms in floats: conv1 activations, the two sides of each max."""
    (c1, h1, w1, kh1, kw1, _, _), (c2, h2, w2, kh2, kw2, _, _), (c3, _, _, kh3, kw3, _, _) = cases.layer_shapes(c)
    ic = c["IC"]
    a2, conv1 = c2 * h2 * w2, c1 * ic * kh1 * kw1 + ic * kh1 * c["W"]
    ws2, ws3 = -(-c2 // ENC_CL) * c1 * kh2 * kw2, -(-c3 // ENC_CL) * c2 * kh3 * kw3
    return c1 * h1 * w1, (a2, conv1), (ws2, ws3)


def smem_bytes(c):
    a1, region2, wslice = smem_terms(c)
    return 4 * (a1 + max(region2) + max(wslice))


def convs():
    """(case, layer index, shape) for every conv of every fused visual case."""
    return [(c, i, s) for c in cases.VISUAL + cases.LIMIT for i, s in enumerate(cases.layer_shapes(c))]


def test_restated_tiling():
    """The constants restated above are the kernels' (by their definitions in the source)."""
    import os
    import re
    src = open(os.path.join(os.path.dirname(encoder.__file__), "csrc", "ssb200.cu")).read()
    for name, value in (("ENC_CL", ENC_CL), ("ENC_OCT", ENC_OCT), ("VIS_PIX", VIS_PIX), ("LIN_ROWS", LIN_ROWS),
                        ("LIN_ENVS", LIN_ENVS)):
        assert re.search(rf"constexpr int {name} = {value};", src), name
    warps = int(re.search(r"constexpr int LIN_WARPS = (\d+);", src).group(1))
    assert WARP * warps == FEATURE_STRIDE
    assert "if (L.kh == 3 && L.kw == 3)" in src and "else if (L.kh == 4 && L.kw == 4)" in src
    assert encoder.VISUAL_SMEM_LIMIT == cases.SMEM_LIMIT and encoder.VISUAL_MAX_ENVS == cases.MAX_ENVS


def test_every_case_is_well_formed():
    for c in cases.VISUAL + cases.LIMIT + cases.OVER_LIMIT + [cases.INPUT_LAYOUT, cases.BIG_B_LAYOUT]:
        assert cases.layer_shapes(c) is not None, c["name"]
        assert c["n_rgb"] + c["n_depth"] == c["IC"] and c["n_rgb"] >= 0 and c["n_depth"] >= 0, c["name"]
    names = [c["name"] for c in cases.VISUAL + cases.LIMIT + cases.OVER_LIMIT]
    assert len(names) == len(set(names))


def test_conv1_edges():
    c1 = [s for c, i, s in convs() if i == 0]
    assert any(h < ENC_CL for _, h, *_ in c1), "H1 < 8: idle cluster ranks in conv1"
    assert any(h % ENC_CL for _, h, *_ in c1), "H1 not a multiple of 8"
    assert {w % VIS_PIX for _, _, w, *_ in c1} == {0, 1, 2, 3}, "every VIS_PIX tail"
    assert any(w < VIS_PIX for _, _, w, *_ in c1), "W1 < 4"
    assert any(oc < WARP for oc, *_ in c1), "C1 < 32"
    assert any(oc % WARP and oc > WARP for oc, *_ in c1), "C1 past a multiple of 32"


def test_conv2_conv3_edges():
    later = [s for c, i, s in convs() if i > 0]
    assert any(oc < ENC_CL for oc, *_ in later), "C < 8: idle ranks"
    assert any(oc % ENC_CL and oc > ENC_CL for oc, *_ in later), "C not a multiple of 8"
    assert any(-(-oc // ENC_CL) % ENC_OCT for oc, *_ in later), "an odd per-rank chunk"
    for inst in ("3x3", "4x4", "generic"):
        assert any(dispatch(kh, kw) == inst and sh != sw for _, _, _, kh, kw, sh, sw in later), inst + " at sh != sw"
    # a 3 x k and a 4 x k kernel must take the generic instance
    assert any(kh == 3 and kw != 3 for _, _, _, kh, kw, _, _ in later), "3 x k kernel"
    assert any(kh == 4 and kw != 4 for _, _, _, kh, kw, _, _ in later), "4 x k kernel"


def test_non_square_kernels_in_every_layer():
    for layer in range(3):
        assert any(s[3] != s[4] for c, i, s in convs() if i == layer), f"layer {layer + 1}: kh != kw"


def test_smem_edges_and_mirror():
    """The restated footprint equals encoder.visual_encoder_smem_bytes for every case; both branches of both maxes
    are taken; every fused case fits, the limit cases equal the limit and the over-limit cases exceed it."""
    region, wslice = set(), set()
    for c in cases.VISUAL + cases.LIMIT + cases.OVER_LIMIT + [cases.INPUT_LAYOUT, cases.BIG_B_LAYOUT]:
        got = encoder.visual_encoder_smem_bytes(cases.make_cnn(c), c["IC"], c["H"], c["W"])
        assert got == (smem_bytes(c), cases.features(c)), c["name"]
        _, (a2, conv1), (ws2, ws3) = smem_terms(c)
        region.add("a2" if a2 >= conv1 else "conv1")
        wslice.add("conv2" if ws2 >= ws3 else "conv3")
    assert region == {"a2", "conv1"} and wslice == {"conv2", "conv3"}
    for c in cases.VISUAL + [cases.INPUT_LAYOUT, cases.BIG_B_LAYOUT]:
        assert smem_bytes(c) <= cases.SMEM_LIMIT, c["name"]
    assert [smem_bytes(c) for c in cases.LIMIT] == [cases.SMEM_LIMIT] * 2
    assert {smem_terms(c)[1][0] >= smem_terms(c)[1][1] for c in cases.LIMIT} == {True, False}, \
        "the limit through both branches of max(C2 H2 W2, C1 IC KH KW + IC KH W)"
    assert all(smem_bytes(c) > cases.SMEM_LIMIT for c in cases.OVER_LIMIT)
    for lim, over in zip(cases.LIMIT, cases.OVER_LIMIT):
        assert (lim["IC"], lim["H"]) == (over["IC"], over["H"]) and over["W"] > lim["W"]
        for W in range(lim["W"] + 1, over["W"]):
            assert smem_bytes(dict(lim, W=W)) <= cases.SMEM_LIMIT, "a narrower over-limit shape exists"


def test_linear_edges():
    hidden = {c["hidden"] for c in cases.VISUAL + cases.LIMIT}
    F = [cases.features(c) for c in cases.VISUAL + cases.LIMIT]
    assert {h % LIN_ROWS for h in hidden} >= {1, 2, 3}, "every LIN_ROWS tail"
    assert {1, 3, 5} <= hidden
    assert 1 in F and any(f < FEATURE_STRIDE for f in F), "F < 256"
    assert any(f % FEATURE_STRIDE for f in F), "F not a multiple of 256"
    assert any(f % FEATURE_STRIDE == 1 and f > FEATURE_STRIDE for f in F), "F just past a multiple of 256"
    assert any(not c["bias"] for c in cases.VISUAL), "bias=False"
    assert {c["IC"] for c in cases.VISUAL} >= {1, 3, 4, 5} and max(c["IC"] for c in cases.VISUAL) >= 12


def test_gru_edges():
    I = {g[0] for g in cases.GRU}
    Hd = {g[1] for g in cases.GRU}
    B = {g[2] for g in cases.GRU}
    assert I | Hd <= set(cases.GRU_WIDTHS) and set(cases.GRU_WIDTHS) <= I | Hd
    for name, widths in (("I", I), ("Hd", Hd)):
        assert any(w % FEATURE_STRIDE for w in widths), f"{name} not a multiple of 256"
        assert any(w < WARP for w in widths), f"{name} < 32"
        assert any(w > FEATURE_STRIDE and w % FEATURE_STRIDE for w in widths), f"{name} past a multiple of 256"
    assert {b % LIN_ENVS for b in B} >= {0, 1, LIN_ENVS - 1}, "B mod 16 in {0, 1, 15}"
    assert B >= set(cases.GRU_BATCHES)
    masks = {v for g in cases.GRU if g[3] != "mixed" for v in g[3]}
    assert {0.5, 2.0, -1.0, float("inf"), float("-inf")} <= masks and any(v != v for v in masks)
    scales = {g[4] for g in cases.GRU}
    assert (30, 1, 1) in scales and (1, 1e3, 1) in scales and (1, 1e-6, 1) in scales and (1, 1, 0) in scales


# ------------------------------------------------------------------------------------------------ zero envs
class FakeCuda(torch.Tensor):
    """A CPU tensor that reports ``is_cuda``, for the audio encoder's device check."""

    @property
    def is_cuda(self):
        return True


class RecordingLib:
    """Stands in for libssb200 behind a WaveformOps on the CPU: records every call of the three entries."""

    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        if not name.startswith("ssb_"):
            raise AttributeError(name)

        def call(*args):
            self.calls.append(name)
            return 0
        return call


class RecordingCtx:
    handle = None
    launch_count = 0

    def __init__(self, lib):
        self.lib = lib

    def check(self, rc, what):
        assert rc == 0, what


def _cpu_ops():
    from soundspaces_b200.renderer import WaveformOps
    ops = WaveformOps.__new__(WaveformOps)
    ops.device = torch.device("cpu")
    ops.lib = RecordingLib()
    ops.ctx = RecordingCtx(ops.lib)
    ops._smt_scratch = {}
    ops._stream = lambda: None
    return ops


def test_zero_envs_return_empty_outputs_without_a_library_call():
    """An empty tensor's data pointer is NULL, which the entries refuse even at B = 0; the reference modules return
    empty outputs.  So at n = 0 the three methods return correctly shaped empty tensors and never call the library."""
    from test_encoder_host import make_cnn
    ops = _cpu_ops()
    audio = make_cnn((65, 26, 2))
    out = ops.audio_encoder(torch.zeros(0, 65, 26, 2).as_subclass(FakeCuda), audio)
    assert out.shape == (0, audio[6].out_features) and out.dtype == torch.float32
    c = cases.VISUAL[0]
    cnn = cases.make_cnn(c)
    feats = torch.zeros(0, cases.features(c)).as_subclass(FakeCuda)
    out = ops.visual_encoder(torch.zeros(0, c["H"], c["W"], 3), torch.zeros(0, c["H"], c["W"], 1), cnn, features=feats)
    assert out.shape == (0, c["hidden"]) and out.dtype == torch.float32
    out = ops.visual_encoder(None, torch.zeros(0, 36, 36, 1), cases.make_cnn(cases.BIG_B_LAYOUT))
    assert out.shape == (0, cases.BIG_B_LAYOUT["hidden"])
    gru = nn.GRU(31, 17)
    out, h = ops.gru_step(torch.zeros(0, 31), torch.zeros(0, 17), torch.zeros(0, 1), gru)
    assert out.shape == h.shape == (0, 17) and out.dtype == h.dtype == torch.float32
    out, h = ops.gru_step(torch.zeros(0, 31), torch.zeros(0, 17), torch.zeros(0), gru)
    assert out.shape == (0, 17)
    assert ops.lib.calls == []
    # malformed inputs are still refused at n = 0
    with pytest.raises(ValueError):
        ops.visual_encoder(torch.zeros(0, c["H"], c["W"], 2), torch.zeros(0, c["H"], c["W"], 1), cnn)
    with pytest.raises(ValueError):
        ops.gru_step(torch.zeros(0, 30), torch.zeros(0, 17), torch.zeros(0, 1), gru)
    # one env still reaches the library
    ops.gru_step(torch.zeros(1, 31), torch.zeros(1, 17), torch.zeros(1, 1), gru)
    assert ops.lib.calls == ["ssb_gru_step_batch"]
