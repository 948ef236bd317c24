"""The conv-stack training path on the host: stand-ins of AudioCNN, VisualCNN and MapCNN and a numpy model of the
kernels' forward and backward equations (tests/conv_stack_models.py, label fold included) pinned to the float64
golden of the unmodified reference classes (tests/golden/make_conv_stack_golden.py), and the patches' flag,
idempotence and fallback reasons that need no GPU."""
import os

import numpy as np
import pytest
import torch

import conv_stack_models as cm
from avnav_models import VisualCNN, set_params
from map_cnn_models import MapCNN
from test_encoder_host import reference_classes

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "conv_stack_golden.npz")
NAMES = ["avnav_audio16k", "avnav_audio44k", "savi_audio_category", "visual_rgbd", "visual_depth", "visual_rgb",
         "map_gm", "map_am"]


@pytest.fixture(scope="module")
def golden():
    with np.load(GOLDEN) as z:
        return {k: z[k] for k in z.files}


def stand_in(name, g):
    """The stand-in of case ``name`` with the golden's parameters, float64, its observations (regenerated from the
    case's seeds) and the upstream gradient."""
    code, N, hidden, seed = (int(v) for v in g[f"{name}/config"])
    obs, dout = cm.case_inputs(name)
    if code == 0:
        AvNav, _, Savi = reference_classes()
        shape = tuple(obs["audiogoal"].shape[1:])
        m = (Savi(shape, hidden, audiogoal_sensor="audiogoal", has_distractor_sound=True) if "category" in obs
             else AvNav(shape, hidden, audiogoal_sensor="audiogoal"))
    elif code == 1:
        n_rgb, n_depth, H, W = cm.CASES[name][1]
        m = VisualCNN(n_rgb, n_depth, H, W, hidden, "av_nav")
    else:
        kind, (H, W, C) = cm.CASES[name]
        m = MapCNN(H, W, C, hidden, map_type=kind)
    return set_params(m, seed).double(), obs, dout


def _close(got, ref, what, rel):
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    assert got.shape == ref.shape, what
    assert np.abs(got - ref).max() <= rel * np.abs(ref).max(), what


def _cnn_grads(m):
    cnn = m.cnn
    return [p.grad.numpy() for c in (cnn[0], cnn[2], cnn[4], cnn[6]) for p in (c.weight, c.bias)]


@pytest.mark.parametrize("name", NAMES)
def test_stand_in_matches_reference_golden(golden, name):
    m, obs, dout = stand_in(name, golden)
    with torch.no_grad():
        out = m(obs).numpy()
    ref = golden[f"{name}/out"]
    assert np.isnan(out[-1]).all() and np.isnan(ref[-1]).all()           # the NaN row reaches every output
    _close(out[:-1], ref[:-1], "out", 1e-12)
    y = m({k: v[:-1] for k, v in obs.items()})
    (y * dout).sum().backward()
    for j, gr in enumerate(_cnn_grads(m)):
        cm.check_grad(name, j, gr, golden, 1e-10)


def _model_args(name, m, obs):
    params = [p.detach().numpy() for c in (m.cnn[0], m.cnn[2], m.cnn[4], m.cnn[6]) for p in (c.weight, c.bias)]
    strides = [tuple(c.stride) for c in (m.cnn[0], m.cnn[2], m.cnn[4])]
    kind = cm.CASES[name][0]
    kind = "audio" if kind.startswith("audio") else kind if kind == "visual" else "map"
    if kind == "visual":
        x = obs["rgb"].numpy() if "rgb" in obs else None
        depth = obs["depth"].numpy() if "depth" in obs else None
    else:
        x, depth = next(iter(obs.values())).numpy(), None
    labels = obs["category"].numpy() if "category" in obs else None
    return kind, x, params, strides, depth, labels


@pytest.mark.parametrize("name", NAMES)
def test_model_matches_reference_golden(golden, name):
    m, obs, dout = stand_in(name, golden)
    kind, x, params, strides, depth, labels = _model_args(name, m, obs)
    out = cm.forward(kind, x, params, strides, depth, labels)[3]
    assert np.isnan(out[-1]).all()
    _close(out[:-1], golden[f"{name}/out"][:-1], "out", 1e-12)
    cut = lambda a: None if a is None else a[:-1]                       # noqa: E731
    grads = cm.backward(kind, cut(x), params, strides, dout.numpy(), cut(depth), cut(labels))
    for j, gr in enumerate(grads):
        cm.check_grad(name, j, gr, golden, 1e-10)


def test_cases_have_dead_units_and_equal_label_taps(golden):
    """The cases exercise the masks (dead conv1 units), and in the reference computation every tap of a label
    channel gets the same gradient, which is what the label fold computes once."""
    m, obs, _ = stand_in("visual_rgbd", golden)
    a1 = m.cnn[1](m.cnn[0](torch.cat([obs["rgb"].permute(0, 3, 1, 2) / 255.0, obs["depth"].permute(0, 3, 1, 2)],
                                      1)[:-1]))
    assert 0 < (a1 == 0).double().mean() < 1
    m, obs, dout = stand_in("savi_audio_category", golden)
    (m({k: v[:-1] for k, v in obs.items()}) * dout).sum().backward()
    g0 = m.cnn[0].weight.grad[:, 2:].numpy()
    assert np.abs(g0 - g0[:, :, :1, :1]).max() <= 1e-12 * np.abs(g0).max()


def test_flag_off_keeps_the_grad_path_original():
    from soundspaces_b200.encoder import patch_audio_cnn, patch_map_cnn, patch_visual_cnn
    AvNav, _, _ = reference_classes()
    original = AvNav.forward
    patch_audio_cnn(AvNav)
    assert AvNav.forward._ssb_original is original
    patch_audio_cnn(AvNav, training=True)
    patch_audio_cnn(AvNav, training=True)                                # idempotent
    assert AvNav.forward._ssb_original is original
    m = AvNav((65, 26, 2), 8)
    x = {"spectrogram": torch.rand(2, 65, 26, 2)}
    out = m(x)                                                          # CPU: the original, with autograd
    assert out.grad_fn is not None and torch.equal(out, original(m, x))
    for cls, patch in ((type("V", (VisualCNN,), {}), patch_visual_cnn), (type("M", (MapCNN,), {}), patch_map_cnn)):
        orig = cls.forward
        patch(cls, training=True)
        patch(cls)
        assert cls.forward._ssb_original is orig


def test_fallback_reasons_without_gpu():
    from soundspaces_b200.encoder import conv_stack_train_error
    v = VisualCNN(3, 1, 36, 36, 8)
    obs = {"rgb": torch.zeros(2, 36, 36, 3), "depth": torch.zeros(2, 36, 36, 1)}
    assert "CUDA" in conv_stack_train_error(v, obs)
    assert "semantic" in conv_stack_train_error(VisualCNN(3, 1, 36, 36, 8, "savi", n_semantic=6), obs)
    assert "blind" in conv_stack_train_error(VisualCNN(0, 0, 36, 36, 8), obs)
    _, _, Savi = reference_classes()
    s = Savi((65, 26, 2), 8, has_distractor_sound=True)
    assert "category" in conv_stack_train_error(s, {"audiogoal": torch.zeros(2, 65, 26, 2)})
    assert "CUDA" in conv_stack_train_error(MapCNN(20, 20, 1, 8, "am"), {"am": torch.zeros(2, 20, 20, 1)})
