"""CPU tests of the heads of ``evaluate_actions`` in PPO's update (soundspaces_b200/policy.py, ``training=True``): the
stand-ins against the reference golden, the routing through ``PolicyHeadFunction``, every fall-back reason, the flag
leaving ``evaluate_actions`` alone when off, patch idempotence and the ABI prototypes."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch
import torch.nn as nn

import policy_head_train_models as ptm
from soundspaces_b200 import policy as ph

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "policy_head_train_golden.npz")


@pytest.fixture(scope="module")
def golden():
    with np.load(GOLDEN) as z:
        return {k: z[k] for k in z.files}


@pytest.mark.parametrize("name", sorted(ptm.CASES))
def test_stand_ins_match_reference_golden(golden, name):
    trainer, H, A, N, seed, gain, masking, special = ptm.CASES[name]
    policy = ptm.make_policy(trainer, H, A, seed, gain, masking, special).double()
    inputs = ptm.case_inputs(name)
    np.testing.assert_array_equal(inputs[0].numpy(), golden[f"{name}/features"])
    np.testing.assert_array_equal(inputs[2].numpy(), golden[f"{name}/actions"])
    for key, got in zip(ptm.OUTPUTS, ptm.forward_backward(policy, trainer, *inputs)):
        np.testing.assert_allclose(got.numpy(), golden[f"{name}/{key}"], rtol=1e-12, atol=1e-12, err_msg=key)
        assert np.isfinite(golden[f"{name}/{key}"]).all() or key == "log_prob", key


def test_golden_covers_neg_inf_logits_and_masked_out_actions(golden):
    b = golden["av_nav_neg_inf/dactor_bias"]
    assert b[ptm.NEG_INF_ACTION] == 0.0 and np.isfinite(b).all()
    amap, actions = golden["av_wan_masked_taken/action_map"], golden["av_wan_masked_taken/actions"][:, 0]
    taken = amap[np.arange(len(actions)), actions]
    assert (taken == 0).sum() >= 3 and (taken == 1).sum() >= 3


def _cpu_dense(monkeypatch):
    """Let CPU tensors qualify, so that the routing runs without a GPU."""
    monkeypatch.setattr(ph, "_dense", lambda t, device: isinstance(t, torch.Tensor) and t.device == device
                        and t.dtype == torch.float32 and t.is_contiguous())


def _case(trainer, N=5, masking=True):
    H, A = 16, 9 if trainer == "av_wan" else 4
    policy = ptm.make_policy(trainer, H, A, 3, 3.0, masking)
    features = torch.tanh(torch.randn((N, H), generator=torch.Generator().manual_seed(1)))
    obs = {"features": features}
    if trainer == "av_wan":
        obs["action_map"] = ptm.phm.action_map(N, A, 2)
    action = torch.randint(0, A, (N, 1), generator=torch.Generator().manual_seed(2))
    return policy, obs, action


def test_evaluate_inputs_reasons(monkeypatch):
    policy, obs, action = _case("av_wan")
    f = obs["features"]
    assert ph._evaluate_inputs(policy, f, obs, action) is None               # CPU features
    _cpu_dense(monkeypatch)
    masked, mask, act = ph._evaluate_inputs(policy, f, obs, action)
    assert masked and torch.equal(mask, obs["action_map"]) and act.dtype == torch.int64
    assert ph._evaluate_inputs(policy, f, obs, action.int())[2].dtype == torch.int64
    refusals = {
        "features not float32": (f.double(), obs, action),
        "features not contiguous": (f.t().contiguous().t(), obs, action),
        "actions float": (f, obs, action.float()),
        "actions bool": (f, obs, action.bool()),
        "actions (N,)": (f, obs, action.view(-1)),
        "actions (N, 2)": (f, obs, action.repeat(1, 2)),
        "actions not a tensor": (f, obs, action.tolist()),
        "action_map requires grad": (f, dict(obs, action_map=obs["action_map"].clone().requires_grad_(True)), action),
        "action_map short": (f, dict(obs, action_map=obs["action_map"][:, :5]), action),
    }
    for why, (x, o, a) in refusals.items():
        assert ph._evaluate_inputs(policy, x, o, a) is None, why
    monkeypatch.setattr(ph, "MAX_TRAIN_ROWS", 4)
    assert ph._evaluate_inputs(policy, f, obs, action) is None
    monkeypatch.setattr(ph, "MAX_TRAIN_ROWS", 5)
    assert ph._evaluate_inputs(policy, f, obs, action) is not None
    monkeypatch.setattr(torch, "is_autocast_enabled", lambda *a: True)
    assert ph._evaluate_inputs(policy, f, obs, action) is None


def test_evaluate_inputs_refuse_parameters(monkeypatch):
    _cpu_dense(monkeypatch)
    policy, obs, action = _case("av_nav")
    policy.critic.fc.double()
    assert ph._evaluate_inputs(policy, obs["features"], obs, action) is None


def test_row_limit_is_the_largest_minibatch():
    assert ph.MAX_TRAIN_ROWS == 4096 * 256


def _patched(trainer, training=True):
    cls = type("Patched", (ptm.POLICIES[trainer],), {})
    return ph.patch_policy(cls, training=training)


class _FakeOps:
    """Records the library calls and runs the heads in eager float32 on the CPU."""

    def __init__(self):
        self.calls = []

    def policy_head_train_forward(self, features, actor, critic, masked, mask, action):
        self.calls.append(("fwd", features.shape[0], masked, mask is not None))
        z = features @ actor.weight.t() + actor.bias
        if masked:
            p = torch.softmax(z, 1) * (mask if mask is not None else 1)
            d = torch.distributions.Categorical(probs=p)
        else:
            d = torch.distributions.Categorical(logits=z)
        value = features @ critic.weight.t() + critic.bias
        lp = d.log_prob(action[:, 0]).unsqueeze(1)
        return value, lp, d.entropy(), torch.zeros_like(z), torch.zeros(1, dtype=torch.int32)

    def policy_head_train_backward(self, features, aw, cw, masked, mask, action, saved, gv, glp, ge, need):
        self.calls.append(("bwd", tuple(need)))
        ts = (features, aw, aw[:, 0], cw, cw[:, 0])
        return tuple(torch.ones_like(t) if n else None for t, n in zip(ts, need))


@pytest.mark.parametrize("trainer", ptm.TRAINERS)
def test_routing(monkeypatch, trainer):
    """The patched evaluate_actions hands the net the original's arguments, runs the heads through
    PolicyHeadFunction with the mask and int64 actions, returns the original's tuple with the entropy's mean, and
    asks the backward for the gradients autograd needs."""
    _cpu_dense(monkeypatch)
    fake = _FakeOps()
    from soundspaces_b200.renderer import WaveformOps
    monkeypatch.setattr(WaveformOps, "get", staticmethod(lambda device: fake))
    policy, obs, action = _case(trainer)
    patched = _patched(trainer)(policy.net, policy.action_distribution.linear.out_features)
    patched.load_state_dict(policy.state_dict())
    args, kw = ptm.evaluate_args(trainer, obs, action)
    want = policy.evaluate_actions(*args, **kw)
    got = patched.evaluate_actions(*args, **kw)
    assert fake.calls == [("fwd", 5, trainer == "av_wan", trainer == "av_wan")]
    assert len(got) == len(want) == (5 if trainer == "savi" else 4)
    for a, b in zip(got[:3], want[:3]):
        torch.testing.assert_close(a, b, rtol=1e-6, atol=1e-6)
        assert a.requires_grad
    for a, b in zip(got[3:], want[3:]):
        assert torch.equal(a, b)
    (got[0].sum() + got[1].sum() + got[2]).backward()
    assert fake.calls[1] == ("bwd", (False, True, True, True, True))
    assert torch.equal(patched.critic.fc.bias.grad, torch.ones(1))
    # keyword arguments bind to the same places
    names = ["observations", "rnn_hidden_states", "prev_actions", "masks", "action", "ext_memory", "ext_memory_masks"]
    got = patched.evaluate_actions(**dict(zip(names, args)))
    assert fake.calls[-1][0] == "fwd" and len(got) == len(want)


def test_features_that_require_grad_get_gradients(monkeypatch):
    _cpu_dense(monkeypatch)
    fake = _FakeOps()
    from soundspaces_b200.renderer import WaveformOps
    monkeypatch.setattr(WaveformOps, "get", staticmethod(lambda device: fake))
    policy, obs, action = _case("av_nav")
    patched = _patched("av_nav")(policy.net, 4)
    patched.requires_grad_(False)
    obs["features"].requires_grad_(True)
    out = patched.evaluate_actions(*ptm.evaluate_args("av_nav", obs, action)[0])
    out[1].sum().backward()
    assert fake.calls[1] == ("bwd", (True, False, False, False, False))
    assert torch.equal(obs["features"].grad, torch.ones_like(obs["features"]))


@pytest.mark.parametrize("reason", ["layout", "host", "actions"])
def test_original_head_lines_run_when_the_call_does_not_qualify(monkeypatch, reason):
    cls = _patched("av_wan")
    policy, obs, action = _case("av_wan")
    patched = cls(policy.net, 9)
    patched.load_state_dict(policy.state_dict())
    if reason == "layout":
        patched.critic.fc = nn.Linear(16, 1, bias=False)
        policy.critic.fc = patched.critic.fc
    if reason != "host":
        _cpu_dense(monkeypatch)
    if reason == "actions":
        action = action.view(-1, 1).float()
    calls = []
    monkeypatch.setattr(ph.PolicyHeadFunction, "apply", lambda *a: calls.append(a))
    args, kw = ptm.evaluate_args("av_wan", obs, action)
    got = patched.evaluate_actions(*args, **kw)
    want = policy.evaluate_actions(*args, **kw)
    assert calls == []
    for a, b in zip(got, want):
        assert torch.equal(a, b)


def test_flag_off_leaves_evaluate_actions_alone():
    cls = type("Patched", (ptm.AvWanPolicy,), {})
    original = cls.evaluate_actions
    ph.patch_policy(cls)
    assert cls.evaluate_actions is original and not hasattr(cls.evaluate_actions, "_ssb_original")
    assert hasattr(cls.act, "_ssb_original")
    ph.patch_policy(cls, training=True)
    assert cls.evaluate_actions._ssb_original is original


def test_patch_is_idempotent():
    cls = type("Patched", (ptm.SaviPolicy,), {})
    original, original_act = cls.evaluate_actions, cls.act
    ph.patch_policy(cls, training=True)
    first = cls.evaluate_actions
    ph.patch_policy(cls, training=True)
    assert cls.evaluate_actions._ssb_original is original and cls.act._ssb_original is original_act
    assert cls.evaluate_actions is not first and cls.evaluate_actions.__doc__ == original.__doc__
    assert ptm.SaviPolicy.evaluate_actions is original


def _header_params(name):
    text = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "ssb200.h")).read(), flags=re.S)
    m = re.search(r"\b" + name + r"\s*\(([^)]*)\)", text)
    return [p.strip() for p in m.group(1).split(",")]


@pytest.mark.parametrize("name,n", [("ssb_policy_head_train_forward_batch", 18),
                                    ("ssb_policy_head_train_backward_batch", 21),
                                    ("ssb_policy_head_train_workspace_bytes", 3)])
def test_prototypes_match_header(name, n):
    from soundspaces_b200 import _lib
    restype, argtypes = _lib.EXPORTS[name]
    params = _header_params(name)
    assert len(argtypes) == len(params) == n
    assert restype is (ctypes.c_int64 if name.endswith("bytes") else ctypes.c_int)
    for p, a in zip(params, argtypes):
        want = ctypes.c_void_p if "*" in p else ctypes.c_int
        assert a is want, (p, a)
