"""The policies' action and value heads in the PPO update through the library (ssb_policy_head_train_*,
PolicyHeadFunction and ``patch_policy(..., training=True)``): forward bits against the rollout entry, PPO's first
ratio after a rollout through the patched storage, accuracy against float64, determinism, launch counts, host syncs,
refusals and a three-step Adam round."""
import copy
import ctypes
import os
import warnings

import numpy as np
import pytest

import policy_head_models as phm
import policy_head_train_models as ptm

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "policy_head_train_golden.npz")
# (trainer, H, A, masking): the trainers' heads, AV-WaN's masked and unmasked
HEADS = [("av_nav", 512, 4, True), ("savi", 128, 4, True), ("av_wan", 512, 81, True), ("av_wan", 512, 81, False)]


@pytest.fixture(scope="module")
def ops():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    from soundspaces_b200.renderer import WaveformOps
    return WaveformOps.get("cuda:0")


def _patched(trainer, H, A, seed=0, gain=3.0, masking=True, special=""):
    from soundspaces_b200.policy import patch_policy
    cls = patch_policy(type("Patched", (ptm.POLICIES[trainer],), {}), training=True)
    return ptm.make_policy(trainer, H, A, seed, gain, masking, special, classes={trainer: cls}).cuda()


def _unpatched(policy, trainer, dtype=torch.float32):
    ref = copy.deepcopy(policy).to(dtype)
    ref.__class__ = ptm.POLICIES[trainer]
    return ref


def _inputs(trainer, H, A, B, seed):
    g = torch.Generator().manual_seed(seed)
    features = torch.tanh(torch.randn((B, H), generator=g) * 2).cuda()
    amap = phm.action_map(B, A, seed).cuda() if trainer == "av_wan" else None
    return features, amap, g


def _rel(a, b):
    return (a.double() - b.double()).abs().max().item() / max(b.double().abs().max().item(), 1e-30)


# ------------------------------------------------------------------------------------------------------------ bits
@pytest.mark.parametrize("head", HEADS, ids=lambda h: f"{h[0]}-{h[2]}-{'m' if h[3] else 'u'}")
@pytest.mark.parametrize("B", [1, 17, 1500, 70000])
def test_forward_bits_match_rollout_mode(ops, head, B):
    trainer, H, A, masking = head
    policy = _patched(trainer, H, A, masking=masking)
    features, amap, _ = _inputs(trainer, H, A, B, 5)
    actor, critic = policy.action_distribution.linear, policy.critic.fc
    masked = trainer == "av_wan"
    mask = amap if masked and masking else None
    with torch.no_grad():
        rows = []
        for i in range(0, B, 65535):            # the rollout entry takes up to 65535 rows a call
            sl = slice(i, min(B, i + 65535))
            rows.append(ops.policy_head(features[sl], actor, critic, masked,
                                        None if mask is None else mask[sl].contiguous()))
        value, action, log_prob = (torch.cat([r[k] for r in rows]) for k in range(3))
        assert all(r[4].item() == 0 for r in rows)
        v2, lp2, ent, saved, status = ops.policy_head_train_forward(features, actor, critic, masked, mask, action)
    assert status.item() == 0
    assert torch.equal(v2, value) and torch.equal(lp2, log_prob)
    assert (torch.exp(lp2 - log_prob) == 1.0).all()
    assert torch.isfinite(ent).all()


def test_first_ppo_ratio_is_one_after_a_patched_rollout(ops):
    """A rollout through the patched act and patch_rollout_storage, then the first minibatch of PPO's update
    through the patched evaluate_actions: ratio exactly 1 and values equal to value_preds for every row."""
    import rollout_models as rm
    from soundspaces_b200 import rollout as ro
    T, N, H, A = 150, 10, 512, 4
    policy = _patched("av_nav", H, A, seed=3, gain=1.0)
    st = ro.patch_rollout_storage(type("Storage", (rm.CommonRolloutStorage,), {}))(
        T, N, rm.spaces({"features": (H,)}), rm.ActionSpace(), 4, 1)
    st.to("cuda")
    g = torch.Generator().manual_seed(9)
    torch.manual_seed(9)
    dev = torch.device("cuda")
    frames = torch.tanh(torch.randn((T + 1, N, H), generator=g) * 2).to(dev)
    st.observations["features"][0].copy_(frames[0])     # insert stores the observation after the step
    h, prev, masks = torch.zeros((1, N, 4), device=dev), torch.zeros((N, 1), dtype=torch.long, device=dev), \
        torch.ones((N, 1), device=dev)
    for t in range(T):
        with torch.no_grad():
            value, action, log_prob, _ = policy.act({"features": frames[t]}, h, prev, masks)
        st.insert({"features": frames[t + 1]}, h, action, log_prob, value, torch.randn((N, 1), generator=g).to(dev),
                  masks)
    st.compute_returns(torch.zeros((N, 1), device=dev), True, 0.99, 0.95)
    adv = st.returns[:-1] - st.value_preds[:-1]
    obs_b, h_b, actions_b, prev_b, value_preds_b, _, masks_b, old_lp_b, adv_b = \
        next(iter(st.recurrent_generator(adv, 1)))
    assert actions_b.shape == (T * N, 1)
    values, lp, ent, _ = policy.evaluate_actions(obs_b, h_b, prev_b, masks_b, actions_b)
    ratio = torch.exp(lp - old_lp_b)
    assert (ratio == 1.0).all() and torch.equal(values, value_preds_b)
    # the reference's surrogate differentiates through the patched heads
    loss = -torch.min(ratio * adv_b, torch.clamp(ratio, 0.8, 1.2) * adv_b).mean() + \
        0.5 * (adv_b + value_preds_b - values).pow(2).mean() - 0.01 * ent
    loss.backward()
    assert all(torch.isfinite(p.grad).all() for p in policy.parameters())
    eager = _unpatched(policy, "av_nav")
    with torch.no_grad():
        lp_e = eager.evaluate_actions(obs_b, h_b, prev_b, masks_b, actions_b)[1]
    dev_eager = (torch.exp(lp_e - old_lp_b) - 1).abs().max().item()
    print(f"eager heads: max |ratio - 1| = {dev_eager:.3g} over {T * N} rows")


# -------------------------------------------------------------------------------------------------------- accuracy
def _fused_and_eager(policy, trainer, features, amap, actions, gv, glp, ge):
    fused = ptm.forward_backward(policy, trainer, features, amap, actions, gv, glp, ge)
    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        eager = ptm.forward_backward(_unpatched(policy, trainer), trainer, features, amap, actions, gv, glp, ge)
    finally:
        torch.backends.cuda.matmul.allow_tf32 = prev
    return fused, eager


def _check(fused, eager, want, what):
    for key, f, e, w in zip(ptm.OUTPUTS, fused, eager, want):
        bound = max(1e-4, 2 * _rel(e, w))
        assert _rel(f, w) <= bound, f"{what} {key}: {_rel(f, w):.3g} > {bound:.3g}"


@pytest.mark.parametrize("name", sorted(ptm.CASES))
def test_matches_float64_golden(ops, name):
    trainer, H, A, N, seed, gain, masking, special = ptm.CASES[name]
    with np.load(GOLDEN) as z:
        want = [torch.from_numpy(z[f"{name}/{k}"]) for k in ptm.OUTPUTS]
        features = torch.from_numpy(z[f"{name}/features"]).float().cuda()
        amap = torch.from_numpy(z[f"{name}/action_map"]).float().cuda() if trainer == "av_wan" else None
        actions = torch.from_numpy(z[f"{name}/actions"]).cuda()
        gv, glp = (torch.from_numpy(z[f"{name}/{k}"]).float().cuda() for k in ("gv", "glp"))
        ge = float(z[f"{name}/ge"])
    policy = _patched(trainer, H, A, seed, gain, masking, special)
    fused, eager = _fused_and_eager(policy, trainer, features, amap, actions, gv, glp, ge)
    assert all(torch.isfinite(t).all() for t in fused[3:])
    _check([t.cpu() for t in fused], [t.cpu() for t in eager], want, name)


@pytest.mark.parametrize("head", HEADS[:3], ids=lambda h: h[0])
def test_matches_float64_at_1500_rows(ops, head):
    trainer, H, A, masking = head
    B = 1500
    policy = _patched(trainer, H, A, seed=11)
    features, amap, g = _inputs(trainer, H, A, B, 11)
    actions = torch.randint(0, A, (B, 1), generator=g).cuda()
    gv, glp = (torch.randn((B, 1), generator=g).cuda() for _ in range(2))
    fused, eager = _fused_and_eager(policy, trainer, features, amap, actions, gv, glp, 0.7)
    want = ptm.forward_backward(_unpatched(policy, trainer, torch.float64), trainer, features.double(),
                                None if amap is None else amap.double(), actions, gv.double(), glp.double(), 0.7)
    _check(fused, eager, want, trainer)


# ----------------------------------------------------------------------------------------------------- determinism
def test_backward_is_deterministic_and_rows_independent_of_batch(ops):
    trainer, H, A = "av_wan", 512, 81
    policy = _patched(trainer, H, A, seed=13)
    B = 1500
    features, amap, g = _inputs(trainer, H, A, B, 13)
    actions = torch.randint(0, A, (B, 1), generator=g).cuda()
    gv, glp, gh = (torch.randn(B, generator=g).cuda() for _ in range(3))
    actor, critic = policy.action_distribution.linear, policy.critic.fc

    def run(rows):
        f, m, a = features[rows].contiguous(), amap[rows].contiguous(), actions[rows].contiguous()
        saved = ops.policy_head_train_forward(f, actor, critic, True, m, a)[3]
        return ops.policy_head_train_backward(f, actor.weight, critic.weight, True, m, a, saved, gv[rows],
                                              glp[rows], gh[rows])

    full = run(torch.arange(B, device="cuda"))
    again = run(torch.arange(B, device="cuda"))
    assert all(torch.equal(x, y) for x, y in zip(full, again))
    for rows in ([700], [3, 1499, 700], list(range(17, 34))):
        part = run(torch.tensor(rows, device="cuda"))
        assert torch.equal(part[0], full[0][rows])


# ------------------------------------------------------------------------------------------- launches and syncs
@pytest.mark.parametrize("want,launches", [("all", 2), ("features", 1), ("params", 2)])
def test_launch_counts_and_one_sync(ops, want, launches):
    trainer, H, A = "av_wan", 512, 81
    policy = _patched(trainer, H, A, seed=17)
    B = 600
    features, amap, g = _inputs(trainer, H, A, B, 17)
    features.requires_grad_(want != "params")
    policy.requires_grad_(want != "features")
    obs = {"features": features, "action_map": amap}
    actions = torch.randint(0, A, (B, 1), generator=g).cuda()
    torch.cuda.synchronize()
    n0 = ops.ctx.launch_count
    torch.cuda.set_sync_debug_mode("warn")
    try:
        with warnings.catch_warnings(record=True) as caught:
            warnings.simplefilter("always")
            out = policy.evaluate_actions(*ptm.evaluate_args(trainer, obs, actions)[0])
    finally:
        torch.cuda.set_sync_debug_mode(0)
    syncs = [w for w in caught if "synchroniz" in str(w.message)]
    assert len(syncs) == 1, [str(w.message) for w in caught]
    assert ops.ctx.launch_count - n0 == 1
    (out[0].sum() + out[1].sum() + out[2]).backward()
    assert ops.ctx.launch_count - n0 == 1 + launches


# ------------------------------------------------------------------------------------------------------- refusals
def _refused(policy, trainer, features, amap, actions, rows):
    obs = {"features": features}
    if amap is not None:
        obs["action_map"] = amap
    with pytest.raises(ValueError, match=rf"rows \[{', '.join(map(str, rows))}\]"):
        policy.evaluate_actions(*ptm.evaluate_args(trainer, obs, actions)[0])


def test_refused_rows_raise_value_error(ops):
    B, H, A = 9, 32, 4
    policy = _patched("av_nav", H, A, seed=19)
    with torch.no_grad():                       # one sign per action row, so a large feature row overflows them all
        policy.action_distribution.linear.weight.abs_()
    features, _, g = _inputs("av_nav", H, A, B, 19)
    actions = torch.randint(0, A, (B, 1), generator=g).cuda()
    f = features.clone()
    f[2, 5] = float("nan")
    _refused(policy, "av_nav", f, None, actions, [2])
    f = features.clone()
    f[4] = 3e38                                 # every logit +Inf
    _refused(policy, "av_nav", f, None, actions, [4])
    f = features.clone()
    f[6] = -3e38                                # every logit -Inf
    _refused(policy, "av_nav", f, None, actions, [6])
    a = actions.clone()
    a[1, 0], a[8, 0] = A, -1
    _refused(policy, "av_nav", features, None, a, [1, 8])
    wan = _patched("av_wan", H, 9, seed=19)
    features, amap, g = _inputs("av_wan", H, 9, B, 20)
    amap[3] = 0
    _refused(wan, "av_wan", features, amap, torch.zeros((B, 1), dtype=torch.long, device="cuda"), [3])


def test_abi_refusals_launch_nothing(ops):
    lib, h = ops.lib, ops.ctx.handle
    f = torch.zeros((8, 16), device="cuda")
    aw, ab, cw, cb = torch.zeros((4, 16), device="cuda"), torch.zeros(4, device="cuda"), \
        torch.zeros(16, device="cuda"), torch.zeros(1, device="cuda")
    act = torch.zeros((8, 1), dtype=torch.long, device="cuda")
    out = torch.zeros((4, 8 * 4), device="cuda")
    status = torch.zeros(1, dtype=torch.int32, device="cuda")
    ws = torch.zeros(1 << 20, dtype=torch.uint8, device="cuda")
    p = lambda t, off=0: t.data_ptr() + off                                 # noqa: E731

    def fwd(B=8, H=16, A=4, masked=0, feat=None, action=None):
        return lib.ssb_policy_head_train_forward_batch(h, B, H, A, feat if feat is not None else p(f), p(aw), p(ab),
                                                       p(cw), p(cb), masked, None,
                                                       action if action is not None else p(act), p(out[0]),
                                                       p(out[1]), p(out[2]), p(out[3]), p(status), None)

    def bwd(B=8, H=16, A=4, workspace=None):
        return lib.ssb_policy_head_train_backward_batch(h, B, H, A, p(f), p(aw), p(cw), 0, None, p(act), p(out[3]),
                                                        p(out[0]), p(out[1]), p(out[2]),
                                                        workspace if workspace is not None else p(ws), None,
                                                        p(out[0]), None, None, None, None)
    calls = [lambda: fwd(B=-1), lambda: fwd(B=4096 * 256 + 1), lambda: fwd(A=257), lambda: fwd(H=2049),
             lambda: fwd(masked=2), lambda: fwd(feat=p(f, 2)), lambda: fwd(action=p(act, 4)),
             lambda: bwd(B=-1), lambda: bwd(A=0), lambda: bwd(workspace=p(ws, 8)), lambda: bwd(A=257)]
    torch.cuda.synchronize()
    for i, c in enumerate(calls):
        n0 = ops.ctx.launch_count
        assert c() != 0 and ops.ctx.launch_count == n0, i
    n0 = ops.ctx.launch_count
    assert fwd(B=0) == 0 and bwd(B=0) == 0 and ops.ctx.launch_count == n0
    assert lib.ssb_policy_head_train_workspace_bytes(4096 * 256 + 1, 16, 4) == -1
    assert lib.ssb_policy_head_train_workspace_bytes(8, 16, 4) <= ws.numel()


# ------------------------------------------------------------------------------------------------------- training
def test_adam_round_matches_unpatched(ops):
    trainer, H, A = "av_wan", 512, 81
    B = 1500
    fused = _patched(trainer, H, A, seed=23, gain=1.0)
    eager, ref = _unpatched(fused, trainer), _unpatched(fused, trainer, torch.float64)
    features, amap, g = _inputs(trainer, H, A, B, 23)
    actions = torch.randint(0, A, (B, 1), generator=g).cuda()
    adv = torch.randn((B, 1), generator=g).cuda()
    opts = [torch.optim.Adam(m.parameters(), lr=1e-3) for m in (fused, eager, ref)]

    def loss(policy, dtype):
        obs = {"features": features.to(dtype), "action_map": amap.to(dtype)}
        v, lp, ent = policy.evaluate_actions(*ptm.evaluate_args(trainer, obs, actions)[0])[:3]
        return -(lp * adv.to(dtype)).mean() + 0.5 * (v - adv.to(dtype)).pow(2).mean() - 0.01 * ent

    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        for _ in range(3):
            for o in opts:
                o.zero_grad()
            for m, dt in ((fused, torch.float32), (eager, torch.float32), (ref, torch.float64)):
                loss(m, dt).backward()
            for o in opts:
                o.step()
    finally:
        torch.backends.cuda.matmul.allow_tf32 = prev
    pf, pe, pr = (list(m.parameters()) for m in (fused, eager, ref))
    bound = max(1e-4, 2 * max(_rel(e, r) for e, r in zip(pe, pr)))
    for i, (a, r) in enumerate(zip(pf, pr)):
        assert _rel(a, r) <= bound, f"parameter {i}: {_rel(a, r):.3g}, bound {bound:.3g}"
