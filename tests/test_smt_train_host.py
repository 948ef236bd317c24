"""Host-side tests of SAVi's scene memory transformer trained in the PPO update: the float64 stand-in the GPU tests
measure against is pinned to the unmodified reference's forward and gradients (tests/golden/smt_train_golden.npz),
the parameter order, smt_train_error's reasons, and patch_smt_state_encoder(training=True)'s routing with a fake
library."""
import os

import numpy as np
import pytest
import torch

from smt_models import make_smt
from smt_train_models import CASES, SMTStandIn, case_inputs, case_module, forward_backward
from soundspaces_b200 import smt
from soundspaces_b200.smt import SmtFunction, patch_smt_state_encoder, smt_train_error, smt_train_parameters

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "smt_train_golden.npz")


@pytest.fixture(scope="module")
def golden():
    return dict(np.load(GOLDEN))


def _close(got, ref):
    # the golden stores the float64 reference rounded to float32
    assert got.shape == ref.shape
    assert np.abs(got - ref).max() <= 1e-6 * max(np.abs(ref).max(), 1e-30)


@pytest.mark.parametrize("name", sorted(CASES))
def test_standin_matches_reference(golden, name):
    out, grads, dx, dgoal = forward_backward(case_module(SMTStandIn, name), *case_inputs(name))
    _close(out.numpy(), golden[f"{name}/out"])
    _close(dx.numpy(), golden[f"{name}/dx"])
    if dgoal is not None:
        _close(dgoal.numpy(), golden[f"{name}/dgoal"])
    pose = CASES[name][1] is not None
    assert len(grads) == (40 if pose else 38)
    for j, g in enumerate(grads):
        _close(g.numpy(), golden[f"{name}/g{j}"])


def test_golden_pose_columns():
    """The agent pose's columns of dx: finite, and exactly 0 on x, y and heading without valid memory."""
    z = np.load(GOLDEN)
    for name, (D, pi, *_rest) in CASES.items():
        assert np.isfinite(z[f"{name}/dx"]).all()
    dx = z["current_only/dx"]
    assert (dx[:, 16:19] == 0).all() and (dx[:, 19] != 0).all()


def test_params_order():
    m = make_smt(20, 16, 32, 4)
    tr = m.transformer
    enc, dec = tr.encoder.layers[0], tr.decoder.layers[0]
    ps = smt_train_parameters(m)
    assert len(ps) == 40
    expect = [m.pose_encoder.weight, m.pose_encoder.bias, m.fusion_encoder[0].weight, m.fusion_encoder[0].bias,
              m.fusion_encoder[2].weight, m.fusion_encoder[2].bias, enc.self_attn.in_proj_weight,
              enc.self_attn.in_proj_bias, enc.self_attn.out_proj.weight, enc.self_attn.out_proj.bias,
              enc.linear1.weight, enc.linear1.bias, enc.linear2.weight, enc.linear2.bias, enc.norm1.weight,
              enc.norm1.bias, enc.norm2.weight, enc.norm2.bias, tr.encoder.norm.weight, tr.encoder.norm.bias,
              dec.self_attn.in_proj_weight, dec.self_attn.in_proj_bias, dec.self_attn.out_proj.weight,
              dec.self_attn.out_proj.bias, dec.multihead_attn.in_proj_weight, dec.multihead_attn.in_proj_bias,
              dec.multihead_attn.out_proj.weight, dec.multihead_attn.out_proj.bias, dec.linear1.weight,
              dec.linear1.bias, dec.linear2.weight, dec.linear2.bias, dec.norm1.weight, dec.norm1.bias,
              dec.norm2.weight, dec.norm2.bias, dec.norm3.weight, dec.norm3.bias, tr.decoder.norm.weight,
              tr.decoder.norm.bias]
    assert all(a is b for a, b in zip(ps, expect))
    assert {id(p) for p in ps} == {id(p) for p in m.parameters()}
    m2 = make_smt(12, None, 16, 2)
    assert len(smt_train_parameters(m2)) == 38 and smt_train_parameters(m2)[0] is m2.fusion_encoder[0].weight


def test_train_error_reasons(monkeypatch):
    m = make_smt(20, 16, 32, 4)
    x, memory, masks, goal, _ = case_inputs("pose_goal")
    assert smt_train_error(m, x, memory, masks, goal) == "x is not a CUDA tensor"
    two = make_smt(20, 16, 32, 4)
    two.transformer.encoder.layers.append(two.transformer.encoder.layers[0])
    assert "expected 1 encoder and 1 decoder layer" in smt_train_error(two, x, memory, masks, goal)
    m.train()
    m.transformer.encoder.layers[0].dropout.p = 0.1
    assert smt_train_error(m, x, memory, masks, goal) == "dropout > 0 in training mode"
    monkeypatch.setattr(torch, "is_autocast_enabled", lambda *a: True)
    assert smt_train_error(m, x, memory, masks, goal) == "autocast is on"


class _FakeOps:
    def __init__(self):
        self.calls = []

    def smt_train_forward(self, module, x, memory, masks, goal):
        self.calls.append(("fwd", x.shape[0], goal is not None))
        return torch.zeros(x.shape[0], module.transformer.d_model), torch.zeros(16, dtype=torch.uint8)

    def smt_train_backward(self, module, x, memory, masks, goal, ws, grad_out, need=None):
        self.calls.append(("bwd", tuple(need)))
        ps = smt_train_parameters(module)
        grads = tuple(torch.ones_like(p) if n else None for p, n in zip(ps, need))
        return grads + (torch.ones_like(x) if need[len(ps)] else None,
                        torch.ones_like(goal) if goal is not None and need[len(ps) + 1] else None)

    def smt_state_encoder(self, module, x, memory, masks, goal=None):
        self.calls.append(("rollout", x.shape[0]))
        return torch.zeros(x.shape[0], module.transformer.d_model)


def test_routing(monkeypatch):
    class Net(SMTStandIn):
        pass

    orig = Net.single_forward
    patch_smt_state_encoder(Net, training=True)
    assert Net.single_forward._ssb_original is orig
    patch_smt_state_encoder(Net, training=True)
    assert Net.single_forward._ssb_original is orig
    m = Net(20, 4, 32, 0.0, 16, False)
    x, memory, masks, goal, _ = case_inputs("pose_goal")
    # refused (CPU tensors): the original runs and differentiates as usual
    out = m.single_forward(x, memory, masks, goal)
    assert out.requires_grad and out.shape == (3, 32)
    fake = _FakeOps()
    from soundspaces_b200.renderer import WaveformOps
    monkeypatch.setattr(WaveformOps, "get", staticmethod(lambda device: fake))
    monkeypatch.setattr(smt, "smt_train_error", lambda *a: "")
    # grad mode: SmtFunction with all 40 parameters; x and goal get gradients when they require them
    goal = goal.clone().requires_grad_(True)
    out = m.single_forward(x, memory, masks, goal)
    assert out.requires_grad and fake.calls == [("fwd", 3, True)]
    out.sum().backward()
    assert fake.calls[1] == ("bwd", (True,) * 40 + (False, True))
    assert torch.equal(goal.grad, torch.ones_like(goal))
    assert torch.equal(m.pose_encoder.weight.grad, torch.ones_like(m.pose_encoder.weight))
    # no grad: the rollout path
    monkeypatch.setattr(smt, "fused_single_forward", lambda module, *a: fake.smt_state_encoder(module, *a))
    with torch.no_grad():
        m.single_forward(x, memory, masks, None)
    assert fake.calls[-1] == ("rollout", 3) and len(fake.calls) == 3


def test_untrained_patch_keeps_grad_calls_on_the_original(monkeypatch):
    class Net(SMTStandIn):
        pass

    patch_smt_state_encoder(Net)
    fake = _FakeOps()
    from soundspaces_b200.renderer import WaveformOps
    monkeypatch.setattr(WaveformOps, "get", staticmethod(lambda device: fake))
    monkeypatch.setattr(smt, "smt_train_error", lambda *a: "")
    m = Net(20, 4, 32, 0.0, 16, False)
    out = m.single_forward(*case_inputs("pose_goal")[:4])
    assert out.requires_grad and fake.calls == []


def test_function_saves_nothing_without_grad(monkeypatch):
    fake = _FakeOps()
    from soundspaces_b200.renderer import WaveformOps
    monkeypatch.setattr(WaveformOps, "get", staticmethod(lambda device: fake))
    m = make_smt(20, 16, 32, 4).requires_grad_(False)
    x, memory, masks, goal, _ = case_inputs("pose_goal")
    out = SmtFunction.apply(True, m, x, memory, masks, goal, *smt_train_parameters(m))
    assert not out.requires_grad and out.grad_fn is None
    m.requires_grad_(True)
    out = SmtFunction.apply(False, m, x, memory, masks, goal, *smt_train_parameters(m))
    assert out.grad_fn is not None and len(out.grad_fn.saved_tensors) == 0
