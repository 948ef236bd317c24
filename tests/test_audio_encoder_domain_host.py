"""The cases of tests/test_gpu_audio_encoder_domain.py (tests/audio_encoder_domain_cases.py) against a restatement of
how ``ssb_audio_encoder_batch`` and ``ssb_audio_encoder_category_batch`` tile their work: each tile edge, dispatch
instance and limit the kernels have is reached by at least one case.  Also the host mirror of the entries' shared-memory
limit, and the dispatch of ``patch_audio_cnn``, which runs the original ``forward`` for every call the entries refuse.
No GPU: the fused path is replaced by a recorder."""
import pytest

torch = pytest.importorskip("torch")
nn = torch.nn

import audio_encoder_domain_cases as cases  # noqa: E402
from soundspaces_b200 import encoder  # noqa: E402
from test_encoder_category_host import fused_calls  # noqa: E402,F401  (the recorder fixture)
from test_encoder_host import FakeCuda, reference_classes  # noqa: E402

# the tiling of soundspaces_b200/csrc/ssb200.cu
ENC_CL = 8            # CTAs per env; each computes ceil(C / ENC_CL) output channels of every layer, conv1 included
ENC_OCT = 2           # conv2 / conv3: output channels per thread
LIN_ROWS = 4          # Linear: output rows per CTA
LIN_ENVS = 16         # Linear: envs per tile
FEATURE_STRIDE = 256  # Linear: lane l of warp w sums the features l + 32 w + 256 k


def dispatch(kh, kw):
    """enc_conv_layer's instance of enc_conv_chw for a conv2 / conv3 kernel."""
    return "3x3" if (kh, kw) == (3, 3) else "4x4" if (kh, kw) == (4, 4) else "generic"


def chunk(oc):
    return -(-oc // ENC_CL)


def smem_terms(c):
    """The entry's shared-memory terms in floats: the staged observation, the conv1 and conv2 activations, and the
    three weight slices (conv1's with its 2 + NL input channels)."""
    (c1, h1, w1, kh1, kw1, _, _), (c2, h2, w2, kh2, kw2, _, _), (c3, _, _, kh3, kw3, _, _) = cases.layer_shapes(c)
    ws = (chunk(c1) * (2 + c["NL"]) * kh1 * kw1, chunk(c2) * c1 * kh2 * kw2, chunk(c3) * c2 * kh3 * kw3)
    return c["H"] * c["W"] * 2, c1 * h1 * w1, c2 * h2 * w2, ws


def smem_bytes(c):
    obs, a1, a2, ws = smem_terms(c)
    return 4 * (obs + a1 + a2 + max(ws))


FUSED = cases.AUDIO + cases.LABELS + cases.LIMIT + cases.REF_FITS
EVERY = (FUSED + cases.OVER_LIMIT + cases.REF_OVER
         + [cases.INPUT_LAYOUT, cases.INPUT_LABELS, cases.BIG_B_LAYOUT, cases.BIG_B_LABELS])


def convs():
    """(case, layer index, shape) for every conv of every fused case."""
    return [(c, i, s) for c in FUSED for i, s in enumerate(cases.layer_shapes(c))]


def test_restated_tiling():
    """The constants restated above are the kernels' (by their definitions in the source)."""
    import os
    import re
    src = open(os.path.join(os.path.dirname(encoder.__file__), "csrc", "ssb200.cu")).read()
    for name, value in (("ENC_CL", ENC_CL), ("ENC_OCT", ENC_OCT), ("LIN_ROWS", LIN_ROWS), ("LIN_ENVS", LIN_ENVS)):
        assert re.search(rf"constexpr int {name} = {value};", src), name
    warps = int(re.search(r"constexpr int LIN_WARPS = (\d+);", src).group(1))
    assert 32 * warps == FEATURE_STRIDE
    assert "if (L.kh == 3 && L.kw == 3)" in src and "else if (L.kh == 4 && L.kw == 4)" in src
    assert "constexpr int ENC_SMEM_MAX = 227 * 1024;" in src and 227 * 1024 == cases.SMEM_LIMIT
    assert encoder.AUDIO_SMEM_LIMIT == cases.SMEM_LIMIT and encoder.AUDIO_MAX_ENVS == cases.MAX_ENVS


def test_every_case_is_well_formed():
    for c in EVERY:
        assert cases.layer_shapes(c) is not None, c["name"]
        assert c["label_stride"] >= c["NL"] >= 0 and len(c["bias"]) == 4, c["name"]
    names = [c["name"] for c in EVERY]
    assert len(names) == len(set(names))


def test_conv1_edges():
    c1 = [(c, s) for c, i, s in convs() if i == 0]
    assert {s[0] for _, s in c1} >= {1, 3, 9, 17, 33}
    assert any(s[0] < ENC_CL for _, s in c1), "C1 < 8: idle cluster ranks"
    assert any(chunk(s[0]) % 2 and s[0] % chunk(s[0]) for _, s in c1), "an odd, partial per-rank chunk"
    assert any(s[3] != s[4] for _, s in c1) and any(s[5] != s[6] for _, s in c1), "non-square kernel and stride"
    assert any(s[5] > s[3] and s[6] > s[4] for _, s in c1), "stride larger than the kernel"
    assert any((s[3], s[4]) == (c["H"], c["W"]) and s[1] == s[2] == 1 for c, s in c1), "kernel = input"
    assert any(c["W"] == 1 and s[4] == 1 and s[3] > 1 for c, s in c1), "W = 1 with a k x 1 kernel"


def test_conv2_conv3_edges():
    later = [s for c, i, s in convs() if i > 0]
    assert any(oc < ENC_CL for oc, *_ in later), "C < 8: idle ranks"
    assert any(oc % ENC_CL and oc > ENC_CL for oc, *_ in later), "C not a multiple of 8"
    assert any(chunk(oc) % ENC_OCT for oc, *_ in later), "an odd per-rank chunk (the ENC_OCT tail)"
    for inst in ("3x3", "4x4", "generic"):
        assert any(dispatch(kh, kw) == inst and sh != sw for _, _, _, kh, kw, sh, sw in later), inst + " at sh != sw"
    assert any(kh == 3 and kw != 3 for _, _, _, kh, kw, _, _ in later), "3 x k kernel"
    assert any(kh == 4 and kw != 4 for _, _, _, kh, kw, _, _ in later), "4 x k kernel"


def test_label_edges():
    assert {c["NL"] for c in cases.LABELS} == {1, 21, 222}
    kk1 = {c["K"][0][0] * c["K"][0][1] for c in cases.LABELS}
    assert 1 in kk1 and max(kk1) >= 100, "KK1 = 1 and a large KK1"
    assert any(not c["bias"][0] for c in cases.LABELS), "conv1 without a bias: the fold starts from 0"
    assert any(c["label_stride"] > c["NL"] for c in cases.LABELS), "label_stride > n_labels"
    kinds = set(cases.LABEL_KINDS)
    assert {("one_hot", 1.0), ("zero", 1.0), ("soft", 1.0), ("negative", 1.0), ("soft", 1e-3), ("soft", 1e3)} <= kinds
    x, lab = cases.make_inputs(cases.LABELS[2], 4, kind=("negative", 1.0))
    assert lab.shape == (4, 222) and lab.stride() == (230, 1) and bool((lab < 0).all())
    assert bool(lab.as_strided((4, 230), (230, 1))[:, 222:].isnan().all()), "the unread columns are NaN"
    assert bool((x[2] == 0).all()), "an all-zero env"


def test_linear_and_batch_edges():
    hidden = {c["hidden"] for c in cases.AUDIO + cases.LABELS}
    F = {cases.features(c) for c in cases.AUDIO + cases.LABELS}
    assert {1, 3, 130} <= hidden and {h % LIN_ROWS for h in hidden} >= {1, 2, 3}
    assert {1, 255, 256, 257} <= F
    assert any(not any(c["bias"]) for c in cases.AUDIO), "bias=False on every layer"
    B = {c["B"] for c in cases.AUDIO + cases.LABELS}
    assert {1, 15, 16, 17, 129} <= B and {b % LIN_ENVS for b in B} >= {0, 1, LIN_ENVS - 1}


def test_smem_mirror_and_limits():
    """The restated footprint equals encoder.audio_encoder_smem_bytes for every case; the limit cases sit exactly at
    232448 bytes through each branch of the weight-slice max (conv1's with labels), and one through the staged
    observation; each over-limit case is the nearest wider observation past it."""
    for c in EVERY:
        got = encoder.audio_encoder_smem_bytes(cases.make_cnn(c), c["NL"], c["H"], c["W"])
        assert got == (smem_bytes(c), cases.features(c)), c["name"]
    for c in FUSED + [cases.INPUT_LAYOUT, cases.INPUT_LABELS, cases.BIG_B_LAYOUT, cases.BIG_B_LABELS]:
        assert smem_bytes(c) <= cases.SMEM_LIMIT, c["name"]
    assert [smem_bytes(c) for c in cases.LIMIT] == [cases.SMEM_LIMIT] * len(cases.LIMIT)
    largest = []
    for c in cases.LIMIT:
        ws = smem_terms(c)[3]
        largest.append(ws.index(max(ws)))
    assert sorted(largest[:3]) == [0, 1, 2] and cases.LIMIT[largest.index(0)]["NL"] > 0
    obs, *_ = smem_terms(cases.LIMIT[3])
    assert 4 * obs > 0.9 * cases.SMEM_LIMIT, "the staged observation is most of the footprint"
    for lim, over in zip(cases.LIMIT + cases.REF_FITS, cases.OVER_LIMIT + cases.REF_OVER):
        assert dict(lim, W=over["W"], name=over["name"]) == over and over["W"] == lim["W"] + 1
        assert smem_bytes(over) > cases.SMEM_LIMIT, over["name"]
    assert [smem_bytes(c) for c in cases.REF_FITS] == [230328, 232280, 229912]
    assert [smem_bytes(c) for c in cases.REF_OVER] == [232768, 236256, 233888]


# ------------------------------------------------------------------------------------------------ dispatch
def _model(cls, c, **kw):
    """A stand-in AudioCNN whose ``cnn`` is the case's network."""
    m = cls((65, 26, 2), hidden=c["hidden"], **kw)
    m.cnn = cases.make_cnn(c)
    return m


def _obs(model, x, lab=None):
    obs = {getattr(model, "_audiogoal_sensor", "spectrogram"): x.as_subclass(FakeCuda)}
    if lab is not None:
        obs["category"] = lab.as_subclass(FakeCuda)
    return obs


@pytest.mark.parametrize("name", [c["name"] for c in cases.REF_FITS + cases.REF_OVER])
def test_reference_widths(name, fused_calls):  # noqa: F811
    """The reference's AudioCNN is fused up to the widest observation that fits and runs the original past it."""
    c = {x["name"]: x for x in cases.REF_FITS + cases.REF_OVER}[name]
    AvNav, AvWan, Savi = reference_classes()
    if c["NL"]:
        encoder.patch_audio_cnn(Savi, category=True)
        model = Savi((c["H"], c["W"], 2), hidden=c["hidden"], has_distractor_sound=True)
    else:
        cls = AvWan if c["C"][2] == 32 else AvNav
        encoder.patch_audio_cnn(cls)
        model = cls((c["H"], c["W"], 2), hidden=c["hidden"])
    assert encoder.audio_encoder_smem_bytes(model.cnn, c["NL"], c["H"], c["W"])[0] == smem_bytes(c)
    x, lab = cases.make_inputs(c, 2)
    with torch.no_grad():
        out = model(_obs(model, x, lab))
    assert out.shape == (2, c["hidden"])
    assert len(fused_calls) == (c in cases.REF_FITS)
    if c in cases.REF_OVER:
        with torch.no_grad():
            want = type(model).forward._ssb_original(model, {k: v.as_subclass(torch.Tensor)
                                                             for k, v in _obs(model, x, lab).items()})
        assert torch.equal(out.as_subclass(torch.Tensor), want)


@pytest.mark.parametrize("name", [c["name"] for c in cases.LIMIT + cases.OVER_LIMIT])
def test_limit_cases_dispatch(name, fused_calls):  # noqa: F811
    c = {x["name"]: x for x in cases.LIMIT + cases.OVER_LIMIT}[name]
    _, _, Savi = reference_classes()
    encoder.patch_audio_cnn(Savi, category=True)
    model = _model(Savi, c, has_distractor_sound=c["NL"] > 0)
    x, lab = cases.make_inputs(c, 1)
    with torch.no_grad():
        model(_obs(model, x, lab))
    assert len(fused_calls) == (c in cases.LIMIT)


@pytest.mark.parametrize("labels", [False, True])
def test_env_count(labels, fused_calls):  # noqa: F811
    """65535 envs are fused, 65536 run the original."""
    c = cases.BIG_B_LABELS if labels else cases.BIG_B_LAYOUT
    _, _, Savi = reference_classes()
    encoder.patch_audio_cnn(Savi, category=True)
    model = _model(Savi, c, has_distractor_sound=labels)
    x, lab = cases.make_inputs(c, cases.MAX_ENVS + 1)
    with torch.no_grad():
        model(_obs(model, x[:cases.MAX_ENVS], None if lab is None else lab[:cases.MAX_ENVS]))
        assert len(fused_calls) == 1
        out = model(_obs(model, x, lab))
    assert len(fused_calls) == 1 and out.shape == (cases.MAX_ENVS + 1, c["hidden"])


@pytest.mark.parametrize("labels", [False, True])
def test_empty_layer_and_mismatched_linear_run_the_original(labels, fused_calls):  # noqa: F811
    """The original forward runs, and raises torch's error, where the entries refuse the network."""
    c = cases.INPUT_LABELS if labels else cases.INPUT_LAYOUT
    _, _, Savi = reference_classes()
    encoder.patch_audio_cnn(Savi, category=True)
    model = _model(Savi, c, has_distractor_sound=labels)
    for W in (4, 40):                     # conv1 5 x 5 on 4 columns: empty; 40 columns: F is not in_features
        x, lab = cases.make_inputs(dict(c, W=W), 2)
        assert (encoder.audio_encoder_smem_bytes(model.cnn, c["NL"], c["H"], W) is None) == (W == 4)
        with torch.no_grad(), pytest.raises(RuntimeError):
            model(_obs(model, x, lab))
    x, lab = cases.make_inputs(c, 2)
    with torch.no_grad():
        model(_obs(model, x, lab))
    assert len(fused_calls) == 1
