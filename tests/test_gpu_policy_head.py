"""GPU tests of the fused policy heads (``ssb_policy_head_batch`` through soundspaces_b200/policy.py) at the shapes the
trainers run: AV-Nav H = 512, A = 4; AV-WaN H = 512, A = 81 with masking on and off; SAVi's SMT width H = 128, A = 4.
Eager reference: the stand-ins of tests/policy_head_models.py (pinned to the reference by the golden file)."""
import ctypes
import warnings

import pytest
import torch

import policy_head_models as phm
from soundspaces_b200 import policy as ph

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)
# name: (trainer, masking)
CASES = {"av_nav": ("av_nav", None), "savi": ("savi", None), "av_wan_masked": ("av_wan", True),
         "av_wan_unmasked": ("av_wan", False)}
NEAR_TIE = 1e-5


def _setup(name, N, seed=0, gain=3.0):
    trainer, masking = CASES[name]
    H, A = phm.SHAPES[trainer]
    policy = phm.make_policy(trainer, H, A, seed=seed, gain=gain, masking=bool(masking)).to(DEV).eval()
    g = torch.Generator().manual_seed(50 + seed)
    features = torch.tanh(torch.randn((N, H), generator=g) * 2).to(DEV)
    obs = {"x": torch.zeros((N, 8), device=DEV)}
    if trainer == "av_wan":
        obs["action_map"] = phm.action_map(N, A, seed).reshape(N, 9, 9).to(DEV)
    return policy, features, obs


def _eager(policy, features, obs, deterministic):
    return policy._head(features, obs, deterministic)


def _ops():
    from soundspaces_b200.renderer import WaveformOps
    return WaveformOps.get(DEV)


def _ratio_margin(probs, q):
    """Relative gap between the two largest p / q of each row."""
    top = torch.topk((probs / q).double(), 2, dim=-1).values
    return (top[:, 0] - top[:, 1]) / top[:, 0]


@pytest.mark.parametrize("name", list(CASES))
@pytest.mark.parametrize("N", [16, 128, 512])
def test_random_stream_and_generator_state(name, N):
    policy, features, obs = _setup(name, N, seed=N)
    with torch.no_grad():
        torch.cuda.manual_seed(1234 + N)
        start = torch.cuda.get_rng_state()
        value, action, lp, dist = _eager(policy, features, obs, False)
        after_eager = torch.cuda.get_rng_state()
        torch.cuda.set_rng_state(start)
        q = torch.empty_like(dist.probs).exponential_(1)
        margin = _ratio_margin(dist.probs, q)
        torch.cuda.set_rng_state(start)
        f_value, f_action, f_lp, _ = ph.fused_head(policy, features, obs, False)
        after_fused = torch.cuda.get_rng_state()
    assert torch.equal(after_eager, after_fused), "the fused head consumed different random numbers"
    clear = margin > NEAR_TIE
    near = int((~clear).sum())
    print(f"{name} N={N}: {near} near-ties")
    assert torch.equal(f_action[clear], action[clear])
    assert near <= max(1, N // 100)


@pytest.mark.parametrize("name", list(CASES))
def test_accuracy_against_float64(name):
    N = 128
    policy, features, obs = _setup(name, N, seed=3)
    p64 = phm.make_policy(CASES[name][0], *phm.SHAPES[CASES[name][0]], seed=3, gain=3.0,
                          masking=bool(CASES[name][1])).to(DEV).double().eval()
    obs64 = {k: v.double() for k, v in obs.items()}
    with torch.no_grad():
        v_ref, a_ref, _, d_ref = _eager(p64, features.double(), obs64, True)
        value, action, lp, _ = ph.fused_head(policy, features, obs, True)
        lp_all = torch.log(d_ref.probs.clamp(torch.finfo(torch.float32).eps, 1 - torch.finfo(torch.float32).eps)) \
            if CASES[name][1] is not None else d_ref.logits
        top = torch.topk(d_ref.probs, 2, dim=-1).values
        clear = (top[:, 0] - top[:, 1]) / top[:, 0] > NEAR_TIE
    assert torch.equal(action[clear], a_ref[clear]) and int((~clear).sum()) <= 1
    lp_ref = lp_all.gather(1, action)
    bar_lp = 1e-4 * lp_all.abs().amax(dim=1, keepdim=True)
    assert bool(((lp.double() - lp_ref).abs() <= bar_lp).all())
    assert bool(((value.double() - v_ref).abs() <= 1e-4 * v_ref.abs().clamp_min(1.0)).all())


@pytest.mark.parametrize("name", list(CASES))
def test_bit_identical_across_batch_sizes_and_positions(name):
    trainer, masking = CASES[name]
    policy, features, obs = _setup(name, 513, seed=5)
    A = policy.action_distribution.linear.out_features
    mask = obs["action_map"].reshape(513, A).contiguous() if masking else None
    q = torch.empty((513, A), device=DEV).exponential_(1)
    args = (policy.action_distribution.linear, policy.critic.fc, masking is not None)
    ops = _ops()
    for qq in (None, q):
        full = ops.policy_head(features, *args, mask, qq, want_probs=True)
        for B in (1, 7, 128):
            part = ops.policy_head(features[:B].contiguous(), *args, None if mask is None else mask[:B].contiguous(),
                                   None if qq is None else qq[:B].contiguous(), want_probs=True)
            for a, b in zip(part[:4], full[:4]):
                assert torch.equal(a, b[:B])
        perm = torch.randperm(513, generator=torch.Generator().manual_seed(1)).to(DEV)
        shuf = ops.policy_head(features[perm].contiguous(), *args, None if mask is None else mask[perm].contiguous(),
                               None if qq is None else qq[perm].contiguous(), want_probs=True)
        for a, b in zip(shuf[:4], full[:4]):
            assert torch.equal(a, b[perm])
        assert int(full[4].item()) == 0


def test_refused_rows_raise_like_the_reference():
    policy, features, obs = _setup("av_nav", 8)
    bad = features.clone()
    bad[3, 7] = float("nan")
    with torch.no_grad():
        with pytest.raises(ValueError):
            _eager(policy, bad, obs, False)
        with pytest.raises(ValueError, match=r"env rows \[3\]"):
            ph.fused_head(policy, bad, obs, False)
        with pytest.raises(ValueError, match=r"env rows \[3\]"):
            ph.fused_head(policy, bad, obs, True)
    policy, features, obs = _setup("av_wan_masked", 8)
    obs["action_map"][2] = 0
    obs["action_map"][6] = 0
    with torch.no_grad():
        with pytest.raises(ValueError):
            _eager(policy, features, obs, False)
        with pytest.raises(ValueError, match=r"env rows \[2, 6\]"):
            ph.fused_head(policy, features, obs, False)
        value, action, lp, probs, status = _ops().policy_head(
            features, policy.action_distribution.linear, policy.critic.fc, True,
            obs["action_map"].reshape(8, -1).contiguous(), None, want_probs=True)
    assert int(status.item()) == 2
    assert action[[2, 6], 0].tolist() == [-1, -1] and bool((action[[0, 1, 3, 4, 5, 7]] >= 0).all())
    assert bool(lp[[2, 6]].isnan().all()) and bool(probs[[2, 6]].isnan().all())
    assert not bool(lp[[0, 1, 3, 4, 5, 7]].isnan().any())


def test_entry_refusals_launch_nothing():
    ops = _ops()
    lib, ctx = ops.lib, ops.ctx
    f = torch.zeros((4, 64), device=DEV)
    w, b, cw, cb = (torch.zeros(s, device=DEV) for s in ((8, 64), (8,), (1, 64), (1,)))
    v, lp = torch.empty(4, device=DEV), torch.empty(4, device=DEV)
    a = torch.empty(5, dtype=torch.int64, device=DEV)
    st = torch.empty(2, dtype=torch.int32, device=DEV)

    def call(B=4, H=64, A=8, feat=f.data_ptr(), masked=0, mask=None, action=a.data_ptr(), status=st.data_ptr()):
        return lib.ssb_policy_head_batch(ctx.handle, B, H, A, feat, w.data_ptr(), b.data_ptr(), cw.data_ptr(),
                                         cb.data_ptr(), masked, mask, None, v.data_ptr(), action, lp.data_ptr(),
                                         None, status, ctypes.c_void_p(0))
    torch.cuda.synchronize()
    n0 = ctx.launch_count
    for kw in ({"B": -1}, {"B": 65536}, {"H": 0}, {"A": 0}, {"masked": 2}, {"mask": f.data_ptr()}, {"feat": None},
               {"feat": f.data_ptr() + 2}, {"action": a.data_ptr() + 4}, {"status": None},
               {"status": st.data_ptr() + 2}):
        assert call(**kw) == -1, kw
    assert call(A=257) == -4 and "A <= 256" in lib.ssb_last_error(ctx.handle).decode()
    assert call(H=2049) == -4 and "H <= 2048" in lib.ssb_last_error(ctx.handle).decode()
    assert call(B=0) == 0
    assert ctx.launch_count == n0


def _count_syncs(fn):
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        torch.cuda.set_sync_debug_mode("warn")
        try:
            fn()
        finally:
            torch.cuda.set_sync_debug_mode(0)
    found = [f"{w.filename}:{w.lineno}" for w in caught if "synchroniz" in str(w.message)]
    print("syncs at", found)
    return len(found)


@pytest.mark.parametrize("name", list(CASES))
@pytest.mark.parametrize("deterministic", [False, True])
def test_one_sync_and_one_library_launch(name, deterministic):
    policy, features, obs = _setup(name, 128)
    ops = _ops()
    with torch.no_grad():
        _count_syncs(lambda: ph.fused_head(policy, features, obs, deterministic))   # warm up: one-time syncs
        _count_syncs(lambda: _eager(policy, features, obs, deterministic))
        torch.cuda.synchronize()
        n0 = ops.ctx.launch_count
        fused = _count_syncs(lambda: ph.fused_head(policy, features, obs, deterministic))
        assert ops.ctx.launch_count - n0 == 1
        eager = _count_syncs(lambda: _eager(policy, features, obs, deterministic))
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            ph.fused_head(policy, features, obs, deterministic)
            torch.cuda.synchronize()
    kernels = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA
               and "emcpy" not in e.name and "emset" not in e.name]
    print(f"{name} deterministic={deterministic}: fused {fused} sync(s), eager {eager}; fused kernels {kernels}")
    assert fused == 1
    assert sum("policy_head_kernel" in k for k in kernels) == 1
    # plus torch's exponential_ when sampling, and the sum and divide of Categorical(probs=...) for AV-WaN's head
    assert len(kernels) == 1 + (not deterministic) + 2 * (CASES[name][0] == "av_wan")


@pytest.mark.parametrize("name", list(CASES))
@pytest.mark.parametrize("deterministic", [False, True])
def test_patched_act_matches_original(name, deterministic):
    trainer, masking = CASES[name]
    H, A = phm.SHAPES[trainer]
    N = 64
    policy = phm.make_policy(trainer, H, A, seed=9, gain=3.0, masking=bool(masking)).to(DEV).eval()
    patched = ph.patch_policy(type("Patched", (phm.POLICIES[trainer],), {}))(policy.net, A, *(
        [bool(masking)] if trainer == "av_wan" else []))
    patched.load_state_dict(policy.state_dict())
    patched.to(DEV).eval()
    obs = {"x": torch.randn((N, 8), generator=torch.Generator().manual_seed(2)).to(DEV)}
    if trainer == "av_wan":
        obs["action_map"] = phm.action_map(N, A, 2).to(DEV)
    args, kw = phm.act_args(trainer, obs, N, deterministic, positional=deterministic)
    with torch.no_grad():
        torch.cuda.manual_seed(77)
        want = policy.act(*args, **kw)
        torch.cuda.manual_seed(77)
        got = patched.act(*args, **kw)
        features = policy.net(*args[:4])[0]
        probs = _eager(policy, features, obs, True)[3].probs
        torch.cuda.manual_seed(77)
        q = torch.empty_like(probs).exponential_(1)
    clear = (_ratio_margin(probs, torch.ones_like(q) if deterministic else q) > NEAR_TIE)
    assert len(got) == len(want)
    assert torch.equal(got[1][clear], want[1][clear]) and int((~clear).sum()) <= 1
    torch.testing.assert_close(got[0], want[0], rtol=1e-5, atol=1e-5)
    torch.testing.assert_close(got[2][clear], want[2][clear], rtol=1e-4, atol=1e-5)
    assert torch.equal(got[3], want[3])
    if trainer == "savi":
        assert torch.equal(got[4], want[4])
    if trainer == "av_wan":
        assert type(got[4]) is phm.CustomFixedCategorical
        torch.testing.assert_close(got[4].probs, want[4].probs, rtol=1e-5, atol=1e-6)
