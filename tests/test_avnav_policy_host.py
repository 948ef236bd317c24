"""Host side of the fused AV-Nav visual encoder and GRU state encoder (``patch_visual_cnn``, ``patch_rnn_state_encoder``):
the stand-ins against the reference classes (golden file), the structural checks, the dispatch and each fallback, and
the C prototypes.  No GPU: the fused path is replaced by a recorder."""
import ctypes
import os
import re
import subprocess

import numpy as np
import pytest

torch = pytest.importorskip("torch")
nn = torch.nn

from avnav_models import RNNStateEncoder, VisualCNN, set_params  # noqa: E402
from soundspaces_b200 import encoder, rnn as rnn_mod  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "avnav_policy_golden.npz")
VARIANTS = ("av_nav", "av_wan", "savi")


# ------------------------------------------------------------------------------------------------ golden
def _golden():
    g = np.load(GOLDEN)
    names = sorted({k.split("/")[0] for k in g.files})
    return g, names


def test_golden_covers_every_class():
    g, names = _golden()
    visual = {VARIANTS[int(g[f"{n}/config"][0])] for n in names if not n.startswith("gru")}
    assert visual == set(VARIANTS) and sum(n.startswith("gru") for n in names) >= 3


def test_visual_stand_ins_match_reference_golden():
    g, names = _golden()
    for i, n in enumerate(x for x in names if not x.startswith("gru")):
        variant, n_rgb, n_depth, H, W, hidden = (int(v) for v in g[f"{n}/config"])
        variant = VARIANTS[variant]
        seed = 10 + ["av_nav_rgbd", "av_wan_depth", "savi_rgb"].index(n)
        m = set_params(VisualCNN(n_rgb, n_depth, H, W, hidden, variant), seed).double()
        obs = {k: torch.from_numpy(g[f"{n}/{k}"]) for k in ("rgb", "depth") if f"{n}/{k}" in g.files}
        with torch.no_grad():
            y = m(obs).numpy()
        ref = g[f"{n}/out"]
        assert y.shape == ref.shape and np.abs(ref).max() > 0
        np.testing.assert_allclose(y, ref, rtol=0, atol=1e-12 * np.abs(ref).max())


def test_rnn_stand_in_matches_reference_golden():
    g, names = _golden()
    for n in (x for x in names if x.startswith("gru")):
        I, Hd, N = (int(v) for v in g[f"{n}/config"])
        seed = 30 + ["gru_mixed", "gru_zero", "gru_one"].index(n)
        m = set_params(RNNStateEncoder(I, Hd), seed).double()
        with torch.no_grad():
            y, h = m(*(torch.from_numpy(g[f"{n}/{k}"]) for k in ("x", "h", "masks")))
        np.testing.assert_allclose(y.numpy(), g[f"{n}/out"], rtol=0, atol=1e-12)
        np.testing.assert_allclose(h.numpy(), g[f"{n}/h_out"], rtol=0, atol=1e-12)


# ------------------------------------------------------------------------------------------------ layouts
def _visual(variant="av_nav", n_rgb=3, n_depth=1, H=128, W=128, hidden=512, **kw):
    return VisualCNN(n_rgb, n_depth, H, W, hidden, variant, **kw)


@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("n_rgb,n_depth", [(3, 0), (0, 1), (3, 1)])
def test_visual_layouts_accepted(variant, n_rgb, n_depth):
    m = _visual(variant, n_rgb, n_depth)
    assert encoder.conv_stack_layout_error(m.cnn, n_rgb + n_depth) == ""
    assert encoder.conv_stack_layout_error(m.cnn, n_rgb + n_depth + 1) != ""


def _deviations():
    def conv(i, **kw):
        def f(cnn):
            c = cnn[i]
            args = dict(kernel_size=c.kernel_size, stride=c.stride, bias=c.bias is not None)
            args.update(kw)
            cnn[i] = nn.Conv2d(c.in_channels, c.out_channels, **args)
        return f

    def no_relu(i):
        def f(cnn):
            cnn[i] = nn.Identity()
        return f

    def groups(cnn):
        cnn[2] = nn.Conv2d(32, 64, 4, 2, groups=2)

    return {"padding": conv(0, padding=1), "dilation": conv(2, dilation=2), "groups": groups,
            "padding_mode": conv(4, padding=1, padding_mode="reflect"), "relu1": no_relu(1), "relu2": no_relu(3),
            "relu_out": no_relu(7), "flatten": lambda cnn: cnn.__setitem__(5, nn.Identity())}


@pytest.mark.parametrize("name", sorted(_deviations()))
def test_visual_layout_deviation_refused(name):
    m = _visual()
    _deviations()[name](m.cnn)
    assert encoder.conv_stack_layout_error(m.cnn, 4) != ""


def test_audio_layout_error_unchanged():
    """encoder_layout_error keeps its audio meaning: 2 + n_category input channels, the same messages."""
    from test_encoder_host import make_cnn
    cnn = make_cnn((65, 26, 2))
    assert encoder.encoder_layout_error(cnn) == ""
    assert encoder.encoder_layout_error(make_cnn((65, 26, 2), in_ch=23), 21) == ""
    assert encoder.encoder_layout_error(make_cnn((65, 26, 2), in_ch=23)) == "module 0: in_channels 23, expected 2"
    assert encoder.encoder_layout_error(cnn, 21) == "module 0: in_channels 2, expected 23"
    assert encoder.encoder_layout_error(nn.Sequential()) == "expected an nn.Sequential of 8 modules"
    cnn[1] = nn.Identity()
    assert encoder.encoder_layout_error(cnn) == "module 1 is Identity, expected ReLU"
    assert encoder.encoder_layout_error(_visual(n_rgb=0, n_depth=2).cnn) == ""


def test_visual_smem_formula():
    """The mirror of the entry's shared-memory limit: av_nav RGB-D at 128 x 128 needs 191616 bytes; the 1024 x 1024
    interactive_demo sensor is far past the 232448-byte limit."""
    assert encoder.visual_encoder_smem_bytes(_visual().cnn, 4, 128, 128) == (191616, 2304)
    assert encoder.visual_encoder_smem_bytes(_visual("av_wan").cnn, 4, 128, 128)[1] == 4608
    big = _visual(H=1024, W=1024)
    assert encoder.visual_encoder_smem_bytes(big.cnn, 4, 1024, 1024)[0] > encoder.VISUAL_SMEM_LIMIT
    assert encoder.visual_encoder_smem_bytes(_visual(H=36, W=36).cnn, 4, 35, 36) is None


def _gru_deviations():
    return {"lstm": nn.LSTM(8, 4), "two_layers": nn.GRU(8, 4, num_layers=2), "no_bias": nn.GRU(8, 4, bias=False),
            "bidirectional": nn.GRU(8, 4, bidirectional=True), "batch_first": nn.GRU(8, 4, batch_first=True),
            "rnn": nn.RNN(8, 4)}


@pytest.mark.parametrize("name", sorted(_gru_deviations()))
def test_gru_layout_deviation_refused(name):
    assert rnn_mod.gru_layout_error(_gru_deviations()[name]) != ""
    assert rnn_mod.gru_layout_error(nn.GRU(8, 4)) == ""


# ------------------------------------------------------------------------------------------------ dispatch
class FakeCuda(torch.Tensor):
    """A CPU tensor that reports ``is_cuda``: lets the CPU suite reach the fused branch of the dispatch."""

    @property
    def is_cuda(self):
        return True


@pytest.fixture
def fused_calls(monkeypatch):
    from soundspaces_b200.renderer import WaveformOps
    calls = []

    class Recorder:
        def visual_encoder(self, rgb, depth, cnn):
            calls.append(("visual", rgb, depth, cnn))
            first = rgb if rgb is not None else depth
            return torch.full((first.shape[0], cnn[6].out_features), 7.0)

        def gru_step(self, x, h, masks, rnn):
            calls.append(("gru", x, h, masks, rnn))
            return torch.full((x.shape[0], rnn.hidden_size), 7.0), torch.full((x.shape[0], rnn.hidden_size), 7.0)

    monkeypatch.setattr(WaveformOps, "get", classmethod(lambda cls, device="cuda:0": Recorder()))
    return calls


def _patched_visual(variant="av_nav"):
    class Patched(VisualCNN):
        pass
    return encoder.patch_visual_cnn(Patched)


def _vobs(n_rgb, n_depth, N=2, H=36, W=36, fake=True):
    obs = {}
    if n_rgb:
        obs["rgb"] = torch.rand(N, H, W, n_rgb) * 255
    if n_depth:
        obs["depth"] = torch.rand(N, H, W, n_depth)
    return {k: v.as_subclass(FakeCuda) if fake else v for k, v in obs.items()}


@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("n_rgb,n_depth", [(3, 0), (0, 1), (3, 1)])
def test_visual_fused_path_taken(fused_calls, variant, n_rgb, n_depth):
    cls = _patched_visual()
    m = cls(n_rgb, n_depth, 36, 36, 8, variant)
    with torch.no_grad():
        y = m(_vobs(n_rgb, n_depth))
    assert len(fused_calls) == 1 and bool((y == 7).all())
    _, rgb, depth, cnn = fused_calls[0]
    assert (rgb is None) == (n_rgb == 0) and (depth is None) == (n_depth == 0) and cnn is m.cnn


def _visual_fallbacks():
    def semantic():
        m = _patched_visual()(3, 1, 36, 36, 8, "savi", n_semantic=6)
        m._n_input_semantic = 6
        return m, _vobs(3, 1)

    def base():
        return _patched_visual()(3, 1, 36, 36, 8), _vobs(3, 1)

    def with_obs(f):
        def g():
            m, obs = base()
            return m, f(obs)
        return g

    def with_module(f):
        def g():
            m, obs = base()
            f(m)
            return m, obs
        return g

    def blind():
        m = _patched_visual()(0, 0, 36, 36, 8)
        return m, {}

    def big():
        m = _patched_visual()(3, 1, 1024, 1024, 8)
        return m, _vobs(3, 1, N=1, H=1024, W=1024)

    return {
        "semantic": semantic, "blind": blind, "past_limit": big,
        "cpu": with_obs(lambda o: {k: v.as_subclass(torch.Tensor) for k, v in o.items()}),
        "float64": with_obs(lambda o: {**o, "depth": o["depth"].double()}),
        "non_contiguous": with_obs(lambda o: {**o, "rgb": o["rgb"].transpose(1, 2)}),
        "channel_count": with_obs(lambda o: {**o, "rgb": o["rgb"][..., :2].contiguous()}),
        "mismatched_hw": with_obs(lambda o: {**o, "depth": _vobs(0, 1, H=40)["depth"]}),
        "layout": with_module(lambda m: m.cnn.__setitem__(1, nn.Identity())),
        "linear_width": with_module(lambda m: m.cnn.__setitem__(6, nn.Linear(100, 8))),
    }


@pytest.mark.parametrize("name", sorted(_visual_fallbacks()))
def test_visual_fallback(fused_calls, name):
    m, obs = _visual_fallbacks()[name]()
    with torch.no_grad():
        assert encoder.fused_visual_forward(m, obs) is None
    assert not fused_calls


def test_visual_cpu_runs_original(fused_calls):
    m = _patched_visual()(3, 1, 36, 36, 8)
    obs = _vobs(3, 1, fake=False)
    with torch.no_grad():
        assert torch.equal(m(obs), type(m).forward._ssb_original(m, obs))
    assert not fused_calls


def test_visual_grad_enabled_runs_original(fused_calls):
    m = _patched_visual()(3, 1, 36, 36, 8)
    obs = _vobs(3, 1, fake=False)
    with torch.enable_grad():
        y = m(obs)
    assert not fused_calls
    with torch.no_grad():
        assert torch.equal(y.detach(), type(m).forward._ssb_original(m, obs))


def test_patch_visual_twice_keeps_original():
    cls = _patched_visual()
    original = cls.forward._ssb_original
    encoder.patch_visual_cnn(cls)
    assert cls.forward._ssb_original is original and original is VisualCNN.forward


def _patched_rnn():
    class Patched(RNNStateEncoder):
        pass
    return rnn_mod.patch_rnn_state_encoder(Patched)


@pytest.fixture
def cpu_dense(monkeypatch):
    """Let CPU float32 tensors pass the device check, so the CPU suite reaches the fused branch."""
    monkeypatch.setattr(rnn_mod, "_dense", lambda t, dev: (isinstance(t, torch.Tensor) and t.device == dev
                                                           and t.dtype == torch.float32 and t.is_contiguous()))


def _rnn_inputs(N=3, I=10, Hd=8):
    return torch.randn(N, I), torch.randn(1, N, Hd), torch.ones(N, 1)


def test_rnn_fused_path_taken(fused_calls, cpu_dense):
    m = _patched_rnn()(10, 8)
    with torch.no_grad():
        out, h = m(*_rnn_inputs())
    assert len(fused_calls) == 1 and out.shape == (3, 8) and h.shape == (1, 3, 8)
    _, x, h0, masks, r = fused_calls[0]
    assert x.shape == (3, 10) and h0.shape == (3, 8) and masks.shape == (3, 1) and r is m.rnn


def _rnn_fallbacks():
    return {
        "lstm": (lambda: _patched_rnn()(10, 8, rnn_type="LSTM"), lambda x, h, m: (x, torch.cat([h, h]), m)),
        "two_layers": (lambda: _patched_rnn()(10, 8, num_layers=2), lambda x, h, m: (x, torch.cat([h, h]), m)),
        "float64": (lambda: _patched_rnn()(10, 8), lambda x, h, m: (x.double(), h, m)),
        "non_contiguous": (lambda: _patched_rnn()(10, 8), lambda x, h, m: (x.t().contiguous().t(), h, m)),
        "masks_shape": (lambda: _patched_rnn()(10, 8), lambda x, h, m: (x, h, m[:, 0])),
        "input_width": (lambda: _patched_rnn()(10, 8), lambda x, h, m: (x[:, :9].contiguous(), h, m)),
    }


@pytest.mark.parametrize("name", sorted(_rnn_fallbacks()))
def test_rnn_fallback(fused_calls, cpu_dense, name):
    make, change = _rnn_fallbacks()[name]
    m = make()
    args = change(*_rnn_inputs())
    with torch.no_grad():
        assert rnn_mod.fused_single_forward(m, *args) is None
    assert not fused_calls


def test_rnn_cpu_and_grad_run_original(fused_calls):
    m = _patched_rnn()(10, 8)
    args = _rnn_inputs()
    with torch.no_grad():
        out, h = m(*args)                                  # CPU tensors: the real device check refuses them
        ref = type(m).single_forward._ssb_original(m, *args)
    assert not fused_calls and torch.equal(out, ref[0]) and torch.equal(h, ref[1])
    out_g, _ = m(*args)                                    # grad enabled
    assert out_g.requires_grad and not fused_calls


def test_patch_rnn_twice_keeps_original():
    cls = _patched_rnn()
    original = cls.single_forward._ssb_original
    rnn_mod.patch_rnn_state_encoder(cls)
    assert cls.single_forward._ssb_original is original and original is RNNStateEncoder.single_forward


# ------------------------------------------------------------------------------------------------ C ABI
def _header_params(name):
    text = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "ssb200.h")).read(), flags=re.S)
    m = re.search(r"\b" + name + r"\s*\(([^)]*)\)", text)
    return [p.strip() for p in m.group(1).split(",")]


def _kind(param):
    if "*" in param or "[" in param:
        return "ptr"
    return param.rsplit(None, 1)[0]


@pytest.mark.parametrize("name", ["ssb_visual_encoder_batch", "ssb_gru_step_batch"])
def test_prototypes_match_header(name):
    from soundspaces_b200 import _lib
    restype, argtypes = _lib.EXPORTS[name]
    params = _header_params(name)
    assert restype is ctypes.c_int and len(argtypes) == len(params)
    for p, a in zip(params, argtypes):
        want = {"ptr": (ctypes.c_void_p,), "int": (ctypes.c_int,)}[_kind(p)]
        assert a in want or (_kind(p) == "ptr" and hasattr(a, "_type_")), (name, p, a)


def test_conv2d_layer_struct_matches_c(tmp_path):
    from soundspaces_b200 import _lib
    src = tmp_path / "layout.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "ssb200.h"\n'
                   'int main(){printf("%zu %zu %zu %zu\\n", sizeof(ssb_conv2d_layer), offsetof(ssb_conv2d_layer, '
                   'out_channels), offsetof(ssb_conv2d_layer, sw), offsetof(ssb_conv2d_layer, relu));return 0;}\n')
    exe = tmp_path / "layout"
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    vals = [int(v) for v in subprocess.check_output([str(exe)]).split()]
    L = _lib.Conv2dLayer
    assert vals == [ctypes.sizeof(L), L.out_channels.offset, L.sw.offset, L.relu.offset]
