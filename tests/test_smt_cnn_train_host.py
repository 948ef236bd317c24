"""Host-side tests of SAVi's visual encoder trained in the PPO update: the float64 stand-in the GPU tests measure
against is pinned to the unmodified reference's forward and gradients (tests/golden/smt_cnn_train_golden.npz),
smt_cnn_train_error's reasons, and patch_smt_cnn(training=True)'s routing with a fake library."""
import os

import numpy as np
import pytest
import torch

from smt_cnn_models import SMTCNN, set_params
from smt_cnn_train_models import CASES, PARAM_SEED, case_grad, case_observations, forward_backward, standin
from smt_resnet_train_models import check_grad
from soundspaces_b200 import encoder
from soundspaces_b200.encoder import SmtCnnFunction, patch_smt_cnn, smt_cnn_params, smt_cnn_train_error

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "smt_cnn_train_golden.npz")


@pytest.fixture(scope="module")
def golden():
    return dict(np.load(GOLDEN))


@pytest.mark.parametrize("name", sorted(CASES))
def test_standin_matches_reference(golden, name):
    mods = CASES[name][3]
    out, grads = forward_backward(standin(name), case_observations(name), case_grad(name, 64 * len(mods)))
    ref = golden[f"{name}/out"]
    # the reference resizes in float32 (interpolate keeps the float32 the crop arrives in), the stand-in in float64
    assert np.abs(out.numpy() - ref).max() <= 1e-5 * np.abs(ref).max()
    assert len(grads) == 62 * len(mods)
    for j, g in enumerate(grads):
        check_grad(name, j, g.numpy(), golden, 1e-5)


def _module(mods=("rgb", "depth")):
    return set_params(SMTCNN({m: 3 if m == "rgb" else 1 for m in mods}), PARAM_SEED)


def test_params_order():
    m = _module()
    ps = smt_cnn_params(m)
    assert len(ps) == 124
    assert ps[0] is m.rgb_encoder.conv1.weight and ps[62] is m.depth_encoder.conv1.weight
    assert ps[61] is m.rgb_encoder.fc.bias and ps[123] is m.depth_encoder.fc.bias


def test_train_error_reasons():
    m = _module()
    obs = case_observations("rgbd128")
    assert "not a CUDA tensor" in smt_cnn_train_error(m, obs)
    sem = _module()
    sem.input_modalities = ["rgb", "depth", "semantic"]
    assert "only 'rgb' and / or 'depth'" in smt_cnn_train_error(sem, obs)
    assert "not a CUDA tensor" in smt_cnn_train_error(m, {})


class _FakeOps:
    def __init__(self):
        self.calls = []

    def smt_cnn_train_forward(self, rgb, depth, params, eps, resize):
        self.calls.append(("fwd", rgb.shape[0], len(params), len(eps), resize))
        return torch.zeros(rgb.shape[0], 128), torch.zeros(16, dtype=torch.uint8)

    def smt_cnn_train_backward(self, rgb, depth, params, eps, resize, ws, grad_out, need=None):
        self.calls.append(("bwd", tuple(need)))
        return tuple(torch.ones_like(p) if n else None for p, n in zip(params, need))


def test_routing(monkeypatch):
    class Net(SMTCNN):
        pass

    orig = Net.forward
    patch_smt_cnn(Net, training=True)
    assert Net.forward._ssb_original is orig
    m = set_params(Net({"rgb": 3, "depth": 1}), PARAM_SEED)
    obs = case_observations("rgbd128")
    # refused: the original runs, and differentiates as usual
    out = m(obs)
    assert out.requires_grad and out.shape == (4, 128)
    fake = _FakeOps()
    from soundspaces_b200.renderer import WaveformOps
    monkeypatch.setattr(encoder, "smt_cnn_train_error", lambda module, o: "")
    monkeypatch.setattr(WaveformOps, "get", staticmethod(lambda device: fake))
    # trainable: SmtCnnFunction with all 124 parameters and 40 eps
    m.depth_encoder.requires_grad_(False)
    out = m(obs)
    assert out.requires_grad and fake.calls == [("fwd", 4, 124, 40, True)]
    out.sum().backward()
    need = fake.calls[1][1]
    assert need == (True,) * 62 + (False,) * 62
    assert torch.equal(m.rgb_encoder.conv1.weight.grad, torch.ones_like(m.rgb_encoder.conv1.weight))
    # frozen: the rollout entry in chunks of at most 1024 rows under no_grad
    m.requires_grad_(False)
    chunks = []

    def fused(module, o):
        assert not torch.is_grad_enabled() and set(o) == {"rgb", "depth"}
        chunks.append(o["rgb"].shape[0])
        return torch.zeros(o["rgb"].shape[0], 128)

    monkeypatch.setattr(encoder, "fused_smt_cnn_forward", fused)
    big = {k: v[:1].expand(2500, *v.shape[1:]).contiguous() for k, v in obs.items()}
    out = m(big)
    assert chunks == [1024, 1024, 452] and out.shape == (2500, 128) and not out.requires_grad
    # no grad: the rollout path, not the train route
    chunks.clear()
    with torch.no_grad():
        m(obs)
    assert chunks == [4]
    assert len(fake.calls) == 2


def test_function_saves_nothing_when_frozen(monkeypatch):
    fake = _FakeOps()
    from soundspaces_b200.renderer import WaveformOps
    monkeypatch.setattr(WaveformOps, "get", staticmethod(lambda device: fake))
    m = _module(("rgb",)).requires_grad_(False)
    x = case_observations("rgb128")["rgb"]
    out = SmtCnnFunction.apply(True, (1e-5,) * 20, True, x, None, *smt_cnn_params(m))
    assert not out.requires_grad and out.grad_fn is None
