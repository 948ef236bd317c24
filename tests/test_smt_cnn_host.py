"""Host side of the fused SMTCNN (SAVi's visual encoder): the stand-in against the reference's recorded float64
outputs, the resize / crop geometry the host sends to ``ssb_smt_cnn_batch``, the structural check behind
``patch_smt_cnn`` and its dispatch.  No GPU: the fused path is replaced by a recorder."""
import os

import numpy as np
import pytest

torch = pytest.importorskip("torch")
nn = torch.nn

from smt_cnn_models import SMTCNN, ResizeCenterCropper, geometry, observations, set_params  # noqa: E402
from soundspaces_b200 import encoder  # noqa: E402

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "smt_cnn_golden.npz")


class FakeCuda(torch.Tensor):
    """A CPU tensor that reports ``is_cuda``: lets the CPU suite reach the fused branch of the dispatch."""

    @property
    def is_cuda(self):
        return True


def _golden():
    g = np.load(GOLDEN)
    names = sorted({k.split("/")[0] for k in g.files if "/" in k})
    return g, names


def test_golden_shapes_cover_the_issue_cases():
    g, names = _golden()
    shapes = {tuple(int(v) for v in g[f"{n}/config"][1:3]) for n in names}
    assert shapes == {(128, 128), (96, 128), (100, 100), (48, 48), (256, 256)}
    assert geometry(96, 128)[:2] == (64, 85)


@pytest.mark.parametrize("name", ["s128", "s96x128", "s100", "s48", "s256"])
def test_stand_in_matches_reference(name):
    g, _ = _golden()
    B, H, W, seed = (int(v) for v in g[f"{name}/config"])
    obs = observations(B, H, W, seed)
    assert obs["rgb"].double().sum().item() == float(g[f"{name}/rgb_sum"])
    assert obs["depth"].double().sum().item() == float(g[f"{name}/depth_sum"])
    model = set_params(SMTCNN({"rgb": 3, "depth": 1}), int(g["param_seed"])).double().eval()
    obs64 = {k: v.double() for k, v in obs.items()}
    with torch.no_grad():
        rgb_img = model.obs_transform(obs64["rgb"].permute(0, 3, 1, 2) / 255.0)
        depth_img = model.obs_transform(obs64["depth"].permute(0, 3, 1, 2))
        out = model(obs64)
    # the reference resizes in float32: its images carry float32 rounding
    for got, key in ((rgb_img, "rgb_img"), (depth_img, "depth_img")):
        ref = torch.from_numpy(g[f"{name}/{key}"]).double()
        assert got.shape == ref.shape == (B, 3 if key == "rgb_img" else 1, 64, 64)
        assert (got - ref).abs().max().item() <= 1e-6 * ref.abs().max().item()
    ref = torch.from_numpy(g[f"{name}/out"])
    assert out.shape == ref.shape == (B, 128)
    assert (out - ref).abs().max().item() <= 1e-4 * ref.abs().max().item()


def _reference_expression(h, w, size=64):
    scale = size / min(h, w)
    h2, w2 = int(h * scale), int(w * scale)
    return h2, w2, h2 // 2 - size // 2, w2 // 2 - size // 2


def test_geometry_matches_reference_expression_and_flags_63():
    bad = []
    for m in range(1, 1025):
        for h, w in ((m, m), (m, m + 1), (m + 37, m), (m, 2 * m + 3)):
            got = encoder.resize_center_crop_geometry(h, w)
            assert got == _reference_expression(h, w), (h, w)
            h2, w2, cy, cx = got
            inside = cy >= 0 and cx >= 0 and cy + 64 <= h2 and cx + 64 <= w2
            assert encoder.crop_inside(*got) == inside
        if not encoder.crop_inside(*encoder.resize_center_crop_geometry(m, m)):
            bad.append(m)
    # exactly the short edges where int(m * (64 / m)) rounds down to 63
    assert bad == [m for m in range(1, 1025) if int(m * (64 / m)) != 64]
    assert bad[:7] == [49, 98, 103, 107, 161, 187, 196]
    assert sum(1 for m in range(1, 4097) if int(m * (64 / m)) != 64) == 505


def _model(channels=None, **kw):
    return set_params(SMTCNN(channels or {"rgb": 3, "depth": 1}, **kw), 3).eval()


def test_layout_accepts_reference_shapes():
    assert encoder.smt_cnn_layout_error(_model()) == ""
    assert encoder.smt_cnn_layout_error(_model({"rgb": 3})) == ""
    assert encoder.smt_cnn_layout_error(_model({"depth": 1})) == ""
    assert encoder.smt_cnn_layout_error(_model(obs_transform=None)) == ""


def test_layout_refusals_give_reasons():
    m = _model()
    m.input_modalities = ["rgb", "depth", "semantic", "semantic_object"]
    assert "only 'rgb'" in encoder.smt_cnn_layout_error(m)
    m = _model()
    m.obs_transform = ResizeCenterCropper(size=(128, 128))
    assert "obs_transform" in encoder.smt_cnn_layout_error(m)
    m.obs_transform = ResizeCenterCropper(channels_last=True)
    assert "obs_transform" in encoder.smt_cnn_layout_error(m)
    m.obs_transform = nn.Identity()
    assert "obs_transform is Identity" in encoder.smt_cnn_layout_error(m)
    m = _model()
    m.depth_encoder.fc = nn.Linear(4608, 64)
    assert encoder.smt_cnn_layout_error(m).startswith("depth_encoder: fc takes 4608")
    m = _model()
    m.rgb_encoder.bn1 = nn.BatchNorm2d(16)
    assert encoder.smt_cnn_layout_error(m).startswith("rgb_encoder: bn1 is BatchNorm2d")


@pytest.fixture
def fused_calls(monkeypatch):
    """Replace the fused path with a recorder that returns zeros of the right shape."""
    from soundspaces_b200.renderer import WaveformOps
    calls = []

    class Recorder:
        def smt_cnn(self, rgb, depth, rgb_encoder, depth_encoder, resize=True):
            calls.append(dict(rgb=rgb, depth=depth, rgb_encoder=rgb_encoder, depth_encoder=depth_encoder, resize=resize))
            B = (rgb if rgb is not None else depth).shape[0]
            return torch.zeros(B, 64 * ((rgb is not None) + (depth is not None)))

    monkeypatch.setattr(WaveformOps, "get", classmethod(lambda cls, device="cuda:0": Recorder()))
    return calls


def _patched_class():
    cls = type("SMTCNN", (SMTCNN,), {})
    encoder.patch_smt_cnn(cls)
    return cls


def _fake(obs):
    return {k: v.as_subclass(FakeCuda) for k, v in obs.items()}


def test_dispatch_takes_fused_path(fused_calls):
    cls = _patched_class()
    model = set_params(cls({"rgb": 3, "depth": 1}), 3).eval()
    obs = observations(3, 128, 128, 0)
    with torch.no_grad():
        out = model(_fake(obs))
    assert out.shape == (3, 128) and len(fused_calls) == 1
    c = fused_calls[0]
    assert c["rgb_encoder"] is model.rgb_encoder and c["depth_encoder"] is model.depth_encoder and c["resize"]
    depth_only = set_params(cls({"depth": 1}, obs_transform=None), 3).eval()
    with torch.no_grad():
        depth_only(_fake(observations(2, 64, 64, 1, rgb=0)))
    assert fused_calls[1]["rgb"] is None and fused_calls[1]["resize"] is False
    assert cls.forward._ssb_original is SMTCNN.forward
    encoder.patch_smt_cnn(cls)
    assert cls.forward._ssb_original is SMTCNN.forward          # patching twice changes nothing


def _run_falls_back(model, obs, calls, grad=False):
    with torch.set_grad_enabled(grad):
        try:
            model(obs)
        except Exception:
            pass                      # the original may raise (the 63-pixel case): it ran, the fused path did not
    return not calls


def test_fallbacks(fused_calls):
    cls = _patched_class()
    model = set_params(cls({"rgb": 3, "depth": 1}), 3).eval()
    obs = observations(2, 128, 128, 0)
    assert _run_falls_back(model, _fake(obs), fused_calls, grad=True)                         # PPO update
    assert _run_falls_back(model, obs, fused_calls)                                            # CPU
    assert _run_falls_back(model, _fake({k: v.double() for k, v in obs.items()}), fused_calls)  # float64
    nc = {k: v.transpose(1, 2).contiguous().transpose(1, 2) for k, v in obs.items()}
    assert _run_falls_back(model, _fake(nc), fused_calls)                                      # non-contiguous
    assert _run_falls_back(model, _fake({"rgb": obs["rgb"]}), fused_calls)                     # missing modality
    assert _run_falls_back(model, _fake({"rgb": obs["rgb"], "depth": obs["depth"][:1]}), fused_calls)   # unequal B
    assert _run_falls_back(model, _fake(observations(2, 98, 130, 0)), fused_calls)             # 98: resizes to 63
    assert _run_falls_back(model, _fake(observations(0, 128, 128, 0)), fused_calls)            # B = 0
    assert _run_falls_back(model, _fake(observations(1, 1025, 64, 0, rgb=0) | {"rgb": obs["rgb"][:1]}), fused_calls)
    sem = set_params(cls({"rgb": 3, "depth": 1}), 3).eval()
    sem.input_modalities = sem.input_modalities + ["semantic", "semantic_object"]
    assert _run_falls_back(sem, _fake(obs), fused_calls)                                       # semantic
    for t in (ResizeCenterCropper(size=(96, 96)), ResizeCenterCropper(channels_last=True), nn.Identity()):
        other = set_params(cls({"rgb": 3, "depth": 1}), 3).eval()
        other.obs_transform = t
        assert _run_falls_back(other, _fake(obs), fused_calls)                                 # obs_transform
    no_t = set_params(cls({"rgb": 3, "depth": 1}, obs_transform=None), 3).eval()
    assert _run_falls_back(no_t, _fake(obs), fused_calls)                                      # 128 x 128, no resize
    wide = set_params(cls({"depth": 1}, obs_transform=None), 3).eval()
    assert _run_falls_back(wide, _fake(observations(1025, 64, 64, 0, rgb=0)), fused_calls)    # B > 1024
    model.depth_encoder.double()
    assert _run_falls_back(model, _fake(obs), fused_calls)                                     # float64 parameters


def test_patched_falls_back_to_identical_result():
    """On CPU the patched class computes exactly what the unpatched one does."""
    cls = _patched_class()
    model = set_params(cls({"rgb": 3, "depth": 1}), 3).eval()
    plain = set_params(SMTCNN({"rgb": 3, "depth": 1}), 3).eval()
    obs = observations(2, 100, 100, 0)
    with torch.no_grad():
        assert torch.equal(model(obs), plain(obs))
