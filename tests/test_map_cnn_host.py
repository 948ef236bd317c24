"""Host side of the fused AV-WaN map encoder (``patch_map_cnn``, ``map_encoder_smem_bytes``): the stand-in against the
reference class (golden file), the shared-memory formula, the structural checks, the dispatch and each fallback, and
the C prototype.  No GPU: the fused path is replaced by a recorder."""
import ctypes
import os

import numpy as np
import pytest

torch = pytest.importorskip("torch")
nn = torch.nn

from avnav_models import set_params  # noqa: E402
from map_cnn_models import REFERENCE_SHAPES, MapCNN, map_obs  # noqa: E402
from soundspaces_b200 import encoder  # noqa: E402
from test_avnav_policy_host import _header_params, _kind  # noqa: E402
from test_encoder_host import Flatten  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "map_cnn_golden.npz")


# ------------------------------------------------------------------------------------------------ golden
@pytest.mark.parametrize("name", sorted(REFERENCE_SHAPES))
def test_stand_in_matches_reference_golden(name):
    g = np.load(GOLDEN)
    H, W, C, hidden, N, pseed, xseed = (int(v) for v in g[f"{name}/config"])
    map_type = REFERENCE_SHAPES[name][0]
    assert (H, W, C) == REFERENCE_SHAPES[name][1:]
    m = set_params(MapCNN(H, W, C, hidden, map_type), pseed).double()
    x = map_obs(N, H, W, C, seed=xseed, kind=map_type).double()
    with torch.no_grad():
        y = m({map_type: x}).numpy()
    ref = g[f"{name}/out"]
    assert y.shape == ref.shape == (N, hidden) and np.abs(ref).max() > 0
    np.testing.assert_allclose(y, ref, rtol=0, atol=1e-12 * np.abs(ref).max())


# ------------------------------------------------------------------------------------------------ shared memory
def test_smem_formula_reference_shapes():
    """The header's values: the geometric maps fit once conv1 is spread over the cluster (the copy-per-CTA visual
    kernel needs 459136 and 907648 bytes for them); the acoustic map is small."""
    want = {"gm200": (161568, 14112), "gm400": (169504, 2592), "am20": (19584, 512)}
    for name, (map_type, H, W, C) in REFERENCE_SHAPES.items():
        cnn = MapCNN(H, W, C, 512, map_type).cnn
        assert encoder.map_encoder_smem_bytes(cnn, C, H, W) == want[name], name
        assert want[name][0] <= encoder.MAP_SMEM_LIMIT
    assert encoder.visual_encoder_smem_bytes(MapCNN(200, 200, 2, 8).cnn, 2, 200, 200)[0] == 459136
    assert encoder.visual_encoder_smem_bytes(MapCNN(400, 400, 2, 8).cnn, 2, 400, 400)[0] == 907648


def test_smem_formula_terms():
    """Each phase of the formula, on a shape where it is the largest."""
    geo = ((8, 4, 3), (5, 4, 2))
    cnn = MapCNN(400, 400, 2, 8, layers=geo).cnn
    # conv2 phase dominates at 400: 25280 + 10112 + 4096 + 2888 floats
    assert encoder.map_encoder_smem_bytes(cnn, 2, 400, 400)[0] == 4 * (25280 + 10112 + 4096 + 2888)
    # conv1 phase dominates for a wide 3-channel map: the staged input rows C KH1 W grow with W.  H1 x W1 = 15 x 375,
    # H2 x W2 = 3 x 93
    wide = MapCNN(120, 3000, 3, 8, layers=((8, 4, 3), (8, 4, 2))).cnn
    rows1, ph1, ph2, ph3 = 32 * 2 * 375, 32 * 3 * 64 + 3 * 8 * 3000, 32 * 4 * 375 + 8 * 32 * 16, 64 * 3 * 93 + 4 * 64 * 9
    assert ph1 > ph2 and rows1 + ph1 > ph3
    assert encoder.map_encoder_smem_bytes(wide, 3, 120, 3000)[0] == 4 * (rows1 + ph1 + 8 * 3 * 93)
    # conv3 phase dominates at 200 (the gathered conv2 output): 33856 + 2304 + 4232 floats
    assert encoder.map_encoder_smem_bytes(MapCNN(200, 200, 2, 8).cnn, 2, 200, 200)[0] == 4 * (33856 + 2304 + 4232)
    assert encoder.map_encoder_smem_bytes(cnn, 2, 400, 20) is None                     # conv2 output empty
    big = MapCNN(1000, 1000, 2, 8, layers=geo).cnn
    assert encoder.map_encoder_smem_bytes(big, 2, 1000, 1000)[0] > encoder.MAP_SMEM_LIMIT


# ------------------------------------------------------------------------------------------------ layouts
@pytest.mark.parametrize("name", sorted(REFERENCE_SHAPES))
def test_reference_layouts_accepted(name):
    map_type, H, W, C = REFERENCE_SHAPES[name]
    cnn = MapCNN(H, W, C, 512, map_type).cnn
    assert encoder.conv_stack_layout_error(cnn, C) == ""
    assert encoder.conv_stack_layout_error(cnn, C + 1) != ""


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

    def channels(cnn):
        cnn[2] = nn.Conv2d(16, 64, 4, 2)

    return {"padding": conv(0, padding=1), "dilation": conv(2, dilation=2), "groups": groups,
            "padding_mode": conv(4, padding=1, padding_mode="reflect"), "conv2_channels": channels,
            "relu1": no_relu(1), "relu2": no_relu(3), "relu_out": no_relu(7),
            "no_flatten": lambda cnn: cnn.__setitem__(5, nn.Identity()),
            "flatten_start": lambda cnn: cnn.__setitem__(5, nn.Flatten(start_dim=2)),
            "flatten_end": lambda cnn: cnn.__setitem__(5, nn.Flatten(end_dim=2)),
            "extra_relu": lambda cnn: cnn.insert(5, nn.ReLU())}


@pytest.mark.parametrize("name", sorted(_deviations()))
def test_layout_deviation_refused(name):
    m = MapCNN(200, 200, 2, 8)
    _deviations()[name](m.cnn)
    assert encoder.conv_stack_layout_error(m.cnn, 2) != ""


def test_reference_flatten_accepted():
    """The reference's ss_baselines.common.utils.Flatten is accepted like nn.Flatten()."""
    m = MapCNN(20, 20, 1, 8, "am")
    m.cnn[5] = Flatten()
    assert encoder.conv_stack_layout_error(m.cnn, 1) == ""


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
        def map_encoder(self, x, cnn):
            calls.append((x, cnn))
            return torch.full((x.shape[0], cnn[6].out_features), 7.0)

    monkeypatch.setattr(WaveformOps, "get", classmethod(lambda cls, device="cuda:0": Recorder()))
    return calls


def _patched():
    class Patched(MapCNN):
        pass
    return encoder.patch_map_cnn(Patched)


def _obs(map_type, N, H, W, C, fake=True):
    x = map_obs(N, H, W, C, seed=1, kind=map_type)
    return {map_type: x.as_subclass(FakeCuda) if fake else x}


@pytest.mark.parametrize("name", sorted(REFERENCE_SHAPES))
def test_fused_path_taken(fused_calls, name):
    map_type, H, W, C = REFERENCE_SHAPES[name]
    m = _patched()(H, W, C, 8, map_type)
    obs = _obs(map_type, 2, H, W, C)
    other = "am" if map_type == "gm" else "gm"
    obs[other] = torch.zeros(2, 3, 3, 5).as_subclass(FakeCuda)          # the other map is not read
    with torch.no_grad():
        y = m(obs)
    assert len(fused_calls) == 1 and y.shape == (2, 8) and bool((y == 7).all())
    x, cnn = fused_calls[0]
    assert x is obs[map_type] and cnn is m.cnn


def test_zero_envs_take_fused_path(fused_calls):
    """N = 0 qualifies; WaveformOps.map_encoder returns (0, hidden) without calling the library."""
    m = _patched()(20, 20, 1, 8, "am")
    with torch.no_grad():
        y = m(_obs("am", 0, 20, 20, 1))
    assert len(fused_calls) == 1 and y.shape == (0, 8)


def _fallbacks():
    def base():
        return _patched()(200, 200, 2, 8), _obs("gm", 2, 200, 200, 2)

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

    def big():
        geo = ((8, 4, 3), (5, 4, 2))
        return _patched()(1000, 1000, 2, 8, layers=geo), _obs("gm", 1, 1000, 1000, 2)

    def too_many_envs():
        m = _patched()(20, 20, 1, 8, "am")
        return m, {"am": torch.empty(encoder.MAP_MAX_ENVS + 1, 20, 20, 1).as_subclass(FakeCuda)}

    return {
        "past_limit": big, "too_many_envs": too_many_envs,
        "cpu": with_obs(lambda o: {"gm": o["gm"].as_subclass(torch.Tensor)}),
        "float64": with_obs(lambda o: {"gm": o["gm"].double()}),
        "non_contiguous": with_obs(lambda o: {"gm": o["gm"].transpose(1, 2)}),
        "channels_first": with_obs(lambda o: {"gm": o["gm"].permute(0, 3, 1, 2).contiguous()}),
        "three_dims": with_obs(lambda o: {"gm": o["gm"][..., 0].contiguous()}),
        "channel_count": with_obs(lambda o: {"gm": o["gm"][..., :1].contiguous()}),
        "missing_map": with_obs(lambda o: {"am": o["gm"]}),
        "layer_output_empty": with_obs(lambda o: {"gm": o["gm"][:, :30, :30].contiguous()}),
        "linear_vs_input": with_obs(lambda o: {"gm": o["gm"][:, :150, :150].contiguous()}),
        "layout": with_module(lambda m: m.cnn.__setitem__(1, nn.Identity())),
        "padding": with_module(lambda m: m.cnn.__setitem__(0, nn.Conv2d(2, 32, 8, 4, padding=1))),
        "linear_width": with_module(lambda m: m.cnn.__setitem__(6, nn.Linear(100, 8))),
        "n_input_gm": with_module(lambda m: setattr(m, "_n_input_gm", 3)),
    }


@pytest.mark.parametrize("name", sorted(_fallbacks()))
def test_fallback(fused_calls, name):
    m, obs = _fallbacks()[name]()
    with torch.no_grad():
        assert encoder.fused_map_forward(m, obs) is None
    assert not fused_calls


def test_cpu_runs_original(fused_calls):
    m = _patched()(20, 20, 1, 8, "am")
    obs = _obs("am", 3, 20, 20, 1, fake=False)
    with torch.no_grad():
        assert torch.equal(m(obs), type(m).forward._ssb_original(m, obs))
    assert not fused_calls


def test_grad_enabled_runs_original(fused_calls):
    m = _patched()(20, 20, 1, 8, "am")
    obs = _obs("am", 3, 20, 20, 1)
    with torch.enable_grad():
        y = m(obs)
    assert not fused_calls and y.requires_grad
    with torch.no_grad():
        assert torch.equal(y.detach(), type(m).forward._ssb_original(m, obs))


def test_patch_twice_keeps_original():
    cls = _patched()
    original = cls.forward._ssb_original
    encoder.patch_map_cnn(cls)
    assert cls.forward._ssb_original is original and original is MapCNN.forward


# ------------------------------------------------------------------------------------------------ C ABI
def test_prototype_matches_header():
    from soundspaces_b200 import _lib
    restype, argtypes = _lib.EXPORTS["ssb_map_encoder_batch"]
    params = _header_params("ssb_map_encoder_batch")
    assert restype is ctypes.c_int and len(argtypes) == len(params) == 14
    for p, a in zip(params, argtypes):
        want = {"ptr": (ctypes.c_void_p,), "int": (ctypes.c_int,)}[_kind(p)]
        assert a in want or (_kind(p) == "ptr" and hasattr(a, "_type_")), (p, a)
    assert argtypes[6]._type_ is _lib.Conv2dLayer
