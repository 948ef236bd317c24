"""CPU tests of the fused policy heads (soundspaces_b200/policy.py): the stand-ins against the reference golden, the
sampling identity the fused path relies on, layout recognition, fallbacks, signature binding, patch idempotence and
the ABI prototype."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch
import torch.nn as nn

import policy_head_models as phm
from soundspaces_b200 import policy as ph

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "policy_head_golden.npz")
TRAINERS = ("av_nav", "savi", "av_wan")


@pytest.fixture(scope="module")
def golden():
    with np.load(GOLDEN) as z:
        return {k: z[k] for k in z.files}


def _cases(g):
    return sorted({k.split("/")[0] for k in g if "/" in k})


def test_stand_ins_match_reference_golden(golden):
    names = _cases(golden)
    assert len(names) == 5
    for name in names:
        c = golden[f"{name}/config"]
        trainer, (H, A, N, n_in, seed), gain, masking = TRAINERS[int(c[0])], map(int, c[1:6]), c[6], bool(c[7])
        policy = phm.make_policy(trainer, H, A, n_in, seed, gain, masking).double().eval()
        obs = {"x": torch.from_numpy(golden[f"{name}/x"])}
        if trainer == "av_wan":
            obs["action_map"] = torch.from_numpy(golden[f"{name}/action_map"])
        args, kw = phm.act_args(trainer, obs, N, True)
        with torch.no_grad():
            res = policy.act(*args, **kw)
            np.testing.assert_allclose(res[0].numpy(), golden[f"{name}/value"], rtol=1e-12, atol=1e-12)
            np.testing.assert_array_equal(res[1].numpy(), golden[f"{name}/mode"])
            np.testing.assert_allclose(res[2].numpy(), golden[f"{name}/mode_log_prob"], rtol=1e-12, atol=1e-12)
            features = policy.net(*args[:4])[0]
            dist = (policy.action_distribution(features, obs["action_map"]) if trainer == "av_wan"
                    else policy.action_distribution(features))
            lp = dist.log_probs(torch.from_numpy(golden[f"{name}/actions"]))
            np.testing.assert_allclose(lp.numpy(), golden[f"{name}/log_probs"], rtol=1e-12, atol=1e-12)
            for i, s in enumerate(golden["sample_seeds"]):
                torch.manual_seed(int(s))
                args, kw = phm.act_args(trainer, obs, N, False)
                np.testing.assert_array_equal(policy.act(*args, **kw)[1][:, 0].numpy(), golden[f"{name}/samples"][i])


@pytest.mark.parametrize("seed", range(15))
def test_multinomial_is_argmax_of_p_over_exponential(seed):
    # torch.multinomial(p, 1, True) draws q = empty_like(p).exponential_(1) and takes argmax(p / q)
    g = torch.Generator().manual_seed(seed)
    p = torch.softmax(torch.randn((64, 81), generator=g) * 3, dim=1) * phm.action_map(64, 81, seed)
    p = p / p.sum(-1, keepdim=True)
    gen = torch.Generator().manual_seed(1000 + seed)
    want = torch.multinomial(p, 1, True, generator=gen)
    gen.manual_seed(1000 + seed)
    q = torch.empty_like(p).exponential_(1, generator=gen)
    assert torch.equal(torch.argmax(p / q, dim=-1, keepdim=True), want)


def _policy(trainer="av_nav", H=16, A=4, **kw):
    return phm.make_policy(trainer, H, A, **kw).eval()


def test_layout_recognition():
    for t in TRAINERS:
        assert ph.policy_head_layout_error(_policy(t, A=9 if t == "av_wan" else 4)) == ""
    p = _policy()
    p.action_distribution.linear = nn.Sequential(nn.Linear(16, 4))
    assert "not nn.Linear" in ph.policy_head_layout_error(p)
    p = _policy()
    p.critic.fc = nn.Linear(16, 1, bias=False)
    assert "no bias" in ph.policy_head_layout_error(p)
    p = _policy()
    p.critic.fc = nn.Linear(16, 2)
    assert "expected 1" in ph.policy_head_layout_error(p)
    p = _policy()
    p.critic.fc = nn.Linear(15, 1)
    assert "takes 15 features" in ph.policy_head_layout_error(p)
    assert "at most 256" in ph.policy_head_layout_error(_policy(A=257))
    assert "at most 256 and 2048" in ph.policy_head_layout_error(_policy(H=2049))
    assert ph.policy_head_layout_error(_policy(A=256, H=2048)) == ""
    assert "not nn.Linear" in ph.policy_head_layout_error(nn.Module())


def test_head_inputs_refuse_host_features():
    p = _policy()
    assert ph._head_inputs(p, torch.zeros((3, 16)), {}) is None


def _patched(trainer):
    cls = type("Patched", (phm.POLICIES[trainer],), {})
    return ph.patch_policy(cls)


@pytest.mark.parametrize("trainer", TRAINERS)
@pytest.mark.parametrize("deterministic", [False, True])
@pytest.mark.parametrize("positional", [False, True])
def test_signature_binding(monkeypatch, trainer, deterministic, positional):
    """The patched act hands the net the original's arguments and the head the right ``deterministic``, whichever
    way it arrives; on host features it falls back to the reference head with the original's outputs."""
    A = 9 if trainer == "av_wan" else 4
    policy = _policy(trainer, A=A)
    patched = _patched(trainer)(policy.net, A)
    patched.load_state_dict(policy.state_dict())
    seen = []
    real = ph.fused_head

    def spy(pol, features, observations, det):
        seen.append(det)
        return real(pol, features, observations, det)
    monkeypatch.setattr(ph, "fused_head", spy)
    obs = {"x": torch.randn((5, 8)), "action_map": phm.action_map(5, A, 0)}
    args, kw = phm.act_args(trainer, obs, 5, deterministic, positional)
    with torch.no_grad():
        torch.manual_seed(7)
        want = policy.act(*args, **kw)
        torch.manual_seed(7)
        got = patched.act(*args, **kw)
    assert seen == [deterministic]
    assert len(got) == len(want) == (5 if trainer != "av_nav" else 4)
    for a, b in zip(got[:4], want[:4]):
        assert torch.equal(a, b)
    if trainer == "savi":
        assert torch.equal(got[4], want[4])
    if trainer == "av_wan":
        assert torch.equal(got[4].probs, want[4].probs)


@pytest.mark.parametrize("reason", ["grad", "layout"])
def test_original_runs_without_the_fused_head(monkeypatch, reason):
    cls = _patched("av_nav")
    policy = cls(phm.StubNet(8, 16), 4)
    if reason == "layout":
        policy.critic.fc = nn.Linear(16, 1, bias=False)
    calls = []
    monkeypatch.setattr(ph, "fused_head", lambda *a: calls.append(a))
    original = cls.act._ssb_original
    args, kw = phm.act_args("av_nav", {"x": torch.randn((3, 8))}, 3, True)
    ctx = torch.enable_grad() if reason == "grad" else torch.no_grad()
    with ctx:
        out = cls.act(policy, *args, **kw)
        with torch.no_grad():
            ref = original(policy, *args, **kw)
    assert calls == []
    for a, b in zip(out, ref):
        assert torch.equal(a, b)


def test_patch_is_idempotent():
    cls = type("Patched", (phm.AvWanPolicy,), {})
    original = cls.act
    ph.patch_policy(cls)
    first = cls.act
    ph.patch_policy(cls)
    assert cls.act._ssb_original is original
    assert cls.act is not first and cls.act._ssb_original is first._ssb_original
    assert phm.AvWanPolicy.act is original


def _header_params(name):
    text = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "ssb200.h")).read(), flags=re.S)
    m = re.search(r"\b" + name + r"\s*\(([^)]*)\)", text)
    return [p.strip() for p in m.group(1).split(",")]


def test_prototype_matches_header():
    from soundspaces_b200 import _lib
    restype, argtypes = _lib.EXPORTS["ssb_policy_head_batch"]
    params = _header_params("ssb_policy_head_batch")
    assert restype is ctypes.c_int and len(argtypes) == len(params) == 18
    for p, a in zip(params, argtypes):
        want = ctypes.c_void_p if "*" in p else ctypes.c_int
        assert p.rsplit(None, 1)[0].startswith(("int", "const", "float", "ssb_ctx", "void")) and a is want, (p, a)
