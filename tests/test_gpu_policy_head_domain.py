"""GPU tests of ``ssb_policy_head_batch`` across what its entry accepts (tests/policy_head_domain_cases.py): every
action slot count, critic pass, feature tail and tail CTA, both limits, all three heads, logit spreads from exact ties
to one-hot rows, action maps with fractional, subnormal, huge and -0.0 values, constructed draws, every refusal class,
the refused-row ticket at B = 65535, and the patched ``act``'s host path.  References: the heads in float64 on the
device, and the eager float32 stand-ins of tests/policy_head_models.py on the CPU for what the reference refuses."""
import ctypes

import pytest
import torch

import policy_head_domain_cases as cases
import policy_head_models as phm
from soundspaces_b200 import policy as ph

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)
B = 129
EPS32 = torch.finfo(torch.float32).eps


def _ops():
    from soundspaces_b200.renderer import WaveformOps
    return WaveformOps.get(DEV)


def _linears(prm):
    aw, ab, cw, cb = prm
    actor, critic = torch.nn.Linear(aw.shape[1], aw.shape[0]), torch.nn.Linear(aw.shape[1], 1)
    with torch.no_grad():
        for lin, w, b in ((actor, aw, ab), (critic, cw, cb)):
            lin.weight.copy_(w)
            lin.bias.copy_(b)
    return actor.to(DEV), critic.to(DEV)


def _call(lins, x, head, mask=None, q=None, want_probs=True):
    """(value (n,), action (n,), log_prob (n,), probs, status) of one launch."""
    v, a, lp, p, st = _ops().policy_head(x.to(DEV).contiguous(), *lins, head != "logits",
                                         None if mask is None else mask.to(DEV).contiguous(),
                                         None if q is None else q.to(DEV).contiguous(), want_probs=want_probs)
    return v.view(-1), a.view(-1), lp.view(-1), p, st


def _check_accuracy(out, ref, what):
    v, a, lp, p, st = out
    assert int(st.item()) == 0, what
    e = cases.errors(v, a, lp, p, ref)
    assert max(e) <= 1.0, (what, e)


def _check_sample_identity(out, q, what):
    """The sampled action is argmax(P / q) of the kernel's own probabilities in float32, bit for bit."""
    _, a, _, p, _ = out
    assert torch.equal(a, torch.argmax(p / q.to(DEV), dim=1)), what


def _cases():
    return [(H, A, head) for (H, A) in cases.ALL_SHAPES for head in cases.HEADS]


def _id(v):
    return f"{v[0]}x{v[1]}-{v[2]}"


# ------------------------------------------------------------------------------------------------------ accuracy
@pytest.mark.parametrize("H,A,head", _cases(), ids=[_id(c) for c in _cases()])
def test_accuracy_and_exact_identities(H, A, head):
    """Per env against float64 at every gain, mask kind and draw; the mode is argmax(P) and a draw argmax(P / q) of
    the kernel's own P; gain-0 rows (exact ties everywhere) take the float64 argmax, the lowest tied index."""
    seed = 31 * H + A
    x = cases.features(B, H, seed)
    for gain in cases.GAINS:
        prm = cases.params(H, A, gain, seed)
        lins = _linears(prm)
        z64 = x.double() @ prm[0].double().t() + prm[1].double()
        kinds = cases.mask_kinds(A, gain) if head == "masked" else [None]
        for kind in kinds:
            mask = None if kind is None else cases.make_mask(kind, B, A, seed, z64)
            what = (H, A, head, gain, kind)
            ref = cases.reference64(prm, x.to(DEV), head, mask)
            mode = _call(lins, x, head, mask)
            _check_accuracy(mode, ref, what)
            p64 = ref[2]
            a_ref = p64.argmax(dim=1)
            keep = torch.ones_like(a_ref, dtype=torch.bool) if gain == 0 else cases.clear_mode(p64)
            assert torch.equal(mode[1][keep], a_ref[keep]), what
            assert int((~keep).sum()) <= 2, what
            assert torch.equal(mode[1], torch.argmax(mode[3], dim=1)), what
            if A == 1:
                want = torch.log(torch.tensor([1 - EPS32], device=DEV)) if head != "logits" else \
                    torch.zeros(1, device=DEV)
                assert torch.equal(mode[2], want.expand(B)), what
            # the constructed draws need the kernel's own probabilities
            for draw in cases.DRAWS:
                q = cases.make_draw(draw, B, A, seed + len(draw), mode[3].cpu())
                out = _call(lins, x, head, mask, q)
                _check_accuracy(out, ref, what + (draw,))
                _check_sample_identity(out, q, what + (draw,))
                assert torch.equal(out[3], mode[3]) and torch.equal(out[0], mode[0]), what
                if draw == "ones":
                    assert torch.equal(out[1], mode[1]), what
                if draw == "ratio_tie":
                    first = torch.argmax((mode[3] > 0).to(torch.int8), dim=1)
                    assert torch.equal(out[1], first), what


@pytest.mark.parametrize("H,A,head", _cases(), ids=[_id(c) for c in _cases()])
def test_constructed_ties_take_the_lowest_index(H, A, head):
    """Exact ties at action pairs across lanes and slots: mode, all-ones draws and p / q ties pick the lower action."""
    pairs = cases.tie_pairs(A)
    if not pairs:
        pytest.skip(f"A = {A} has no tie pair")
    for k, pair in enumerate(pairs):
        prm, x = cases.tie_inputs(B, H, A, pair, seed=H + k)
        lins = _linears(prm)
        mask = None
        if head == "masked":
            mask = cases.make_mask("binary", B, A, k, torch.zeros((B, A)))
            mask[:, list(pair)] = 1.0
        mode = _call(lins, x, head, mask)
        assert int(mode[4].item()) == 0
        assert bool((mode[3][:, pair[0]] == mode[3][:, pair[1]]).all()), pair
        assert bool((mode[1] == pair[0]).all()), pair
        ref = cases.reference64(prm, x.to(DEV), head, mask)
        _check_accuracy(mode, ref, pair)
        for draw in ("ones", "ratio_tie"):
            q = cases.make_draw(draw, B, A, k, mode[3].cpu())
            out = _call(lins, x, head, mask, q)
            _check_sample_identity(out, q, (pair, draw))
            if draw == "ones":
                assert bool((out[1] == pair[0]).all()), pair


# ------------------------------------------------------------------------------------------------ bit-identity
@pytest.mark.parametrize("H,A,head", _cases(), ids=[_id(c) for c in _cases()])
def test_bit_identical_across_batch_sizes_positions_and_probs(H, A, head):
    seed = 7 * H + A
    x = cases.features(B, H, seed)
    prm = cases.params(H, A, 3.0, seed)
    lins = _linears(prm)
    z64 = x.double() @ prm[0].double().t()
    mask = cases.make_mask("fraction", B, A, seed, z64) if head == "masked" else None
    q = torch.empty((B, A)).exponential_(1, generator=torch.Generator().manual_seed(seed))
    perm = torch.randperm(B, generator=torch.Generator().manual_seed(seed))
    for qq in (None, q):
        full = _call(lins, x, head, mask, qq)
        no_probs = _call(lins, x, head, mask, qq, want_probs=False)
        for s, t in zip(full[:3], no_probs[:3]):
            assert torch.equal(s, t)
        for b in cases.BATCHES:
            part = _call(lins, x[:b], head, None if mask is None else mask[:b], None if qq is None else qq[:b])
            for s, t in zip(part[:4], full[:4]):
                assert torch.equal(s, t[:b]), b
            assert int(part[4].item()) == 0
        shuf = _call(lins, x[perm], head, None if mask is None else mask[perm], None if qq is None else qq[perm])
        pd = perm.to(DEV)
        for s, t in zip(shuf[:4], full[:4]):
            assert torch.equal(s, t[pd])


@pytest.mark.parametrize("H,A", cases.BIG_B_SHAPES)
@pytest.mark.parametrize("head", cases.HEADS)
def test_largest_batch(H, A, head):
    """B = 65535 (16,384 CTAs, the last with 3 envs): within the float64 bars and bit-identical to small calls."""
    n = cases.MAX_B
    x = cases.features(n, H, 5)
    prm = cases.params(H, A, 3.0, 5)
    lins = _linears(prm)
    z64 = (x.to(DEV).double() @ prm[0].to(DEV).double().t()).cpu()
    mask = cases.make_mask("binary", n, A, 5, z64) if head == "masked" else None
    q = torch.empty((n, A)).exponential_(1, generator=torch.Generator().manual_seed(5))
    for qq in (None, q):
        out = _call(lins, x, head, mask, qq)
        _check_accuracy(out, cases.reference64(prm, x.to(DEV), head, mask), (H, A, head))
        if qq is not None:
            _check_sample_identity(out, qq, (H, A, head))
        for lo in (0, n - 7):
            part = _call(lins, x[lo:], head, None if mask is None else mask[lo:], None if qq is None else qq[lo:])
            for s, t in zip(part[:4], out[:4]):
                assert torch.equal(s, t[lo:]), lo


# ------------------------------------------------------------------------------------------------------ refusals
def _refusal_params():
    out = []
    for name, head, applies, refused in cases.REFUSALS:
        for H, A in cases.REFUSE_SHAPES:
            if name == "mask_underflow" and A < 2:
                continue
            out.append(pytest.param(name, head, applies, refused, H, A, id=f"{name}-{head}-{H}x{A}"))
    return out


def _raises_on_cpu(policy, x, mask, deterministic):
    """Whether the eager float32 stand-in raises ValueError on one row (with masking off its action map is unread)."""
    obs = {"x": torch.zeros((1, 8)), "action_map": mask if mask is not None else torch.ones((1, x.shape[1]))}
    try:
        with torch.no_grad():
            policy._head(x, obs, deterministic)
    except ValueError:
        return True
    return False


@pytest.mark.parametrize("name,head,applies,refused,H,A", _refusal_params())
def test_refusals(name, head, applies, refused, H, A):
    prm, x, mask = cases.refusal_input(name, head, H, A)
    lins = _linears(prm)
    n = cases.REFUSE_B
    rows = cases.refusal_expected_rows(name, head, applies) if refused else []
    q = torch.empty((n, A)).exponential_(1, generator=torch.Generator().manual_seed(H))
    # a clean call: the refused rows' features replaced, their action maps all open
    cx, cmask = x.clone(), None if mask is None else mask.clone()
    cx[rows] = cases.features(n, H, 99)[rows]
    if cmask is not None:
        cmask[rows] = 1.0
    keep = torch.ones(n, dtype=torch.bool)
    keep[rows] = False
    keep_d = keep.to(DEV)
    policy = cases.stand_in(H, A, head, prm)
    for qq in (None, q):
        out = _call(lins, x, head, mask, qq)
        v, a, lp, p, st = out
        assert int(st.item()) == len(rows), (name, H, A)
        assert bool((a[~keep_d] == -1).all()) and bool(v[~keep_d].isnan().all())
        assert bool(lp[~keep_d].isnan().all()) and bool(p[~keep_d].isnan().all())
        assert bool((a[keep_d] >= 0).all())
        if applies == "rows":
            clean = _call(lins, cx, head, cmask, qq)
            assert int(clean[4].item()) == 0
            for s, t in zip(out[:4], clean[:4]):
                assert torch.equal(s[keep_d], t[keep_d])
        elif not refused:
            assert not bool(v.isnan().any()) and not bool(lp.isnan().any()) and not bool(p.isnan().any())
            if qq is not None:
                _check_sample_identity(out, qq, name)
        # what the reference does, row by row on the CPU, in mode and when sampling
        check = sorted(set(rows[:6] + [r for r in (0, 1, 4, 63, n - 1) if keep[r]]))
        for r in check:
            got = _raises_on_cpu(policy, x[r:r + 1], None if mask is None else mask[r:r + 1], qq is None)
            assert got == (r in rows), (name, r, qq is None)
    # through the patched act's head: the ValueError names exactly the refused rows
    pol = policy.to(DEV)
    obs = {"x": torch.zeros((n, 8), device=DEV)}
    if head == "masked":
        obs["action_map"] = mask.to(DEV)
    with torch.no_grad():
        for det in (True, False):
            if refused:
                with pytest.raises(ValueError, match=rf"env rows \[{', '.join(map(str, rows))}\]:"):
                    ph.fused_head(pol, x.to(DEV), obs, det)
            else:
                assert ph.fused_head(pol, x.to(DEV), obs, det) is not None


# -------------------------------------------------------------------------------------------------------- ticket
def test_ticket_counts_at_the_largest_batch():
    """At B = 65535 the count is exact with refused rows in the first, a middle and the last CTA, with every row
    refused, and over back-to-back calls whose counts vary (refused, then clean, reports 0), each status kept."""
    n, H, A = cases.MAX_B, 32, 16
    prm = cases.params(H, A, 3.0, 11)
    lins = _linears(prm)
    x = cases.features(n, H, 11)
    sets = [[0, 1, 2, 3], [n // 2, n // 2 + 3], [n - 1], [0, 5, 8190 * 4 + 2, n - 3, n - 2, n - 1], [],
            list(range(0, n, 97)), [], list(range(n)), [], [7]]
    statuses = []
    for s in sets:
        bad = x.clone()
        if s:
            bad[s, 3] = float("nan")
        statuses.append(_call(lins, bad, "logits")[4])
    assert [int(t.item()) for t in statuses] == [len(s) for s in sets]
    # one side-stream call against the default stream's, with a refused row
    bad = x.clone()
    bad[[9, n - 1], 0] = float("inf")
    want = _call(lins, bad, "logits")
    side = torch.cuda.Stream(device=DEV)
    side.wait_stream(torch.cuda.current_stream(DEV))
    with torch.cuda.stream(side):
        got = _call(lins, bad, "logits")
    torch.cuda.current_stream(DEV).wait_stream(side)
    for s, t in zip(got, want):
        torch.testing.assert_close(s, t, rtol=0, atol=0, equal_nan=True)
    assert int(got[4].item()) == 2


# ----------------------------------------------------------------------------------------------------- host path
def _avwan(N, A=81, H=512):
    policy = phm.make_policy("av_wan", H, A, seed=4, gain=3.0, masking=True).to(DEV).eval()
    g = torch.Generator().manual_seed(4)
    features = torch.tanh(torch.randn((N, H), generator=g) * 2).to(DEV)
    return policy, features


@pytest.mark.parametrize("dtype", [torch.bool, torch.uint8, torch.int64, torch.float64, torch.float32])
@pytest.mark.parametrize("shape", [(81,), (9, 9), (1, 9, 9)])
def test_action_map_dtypes_and_shapes_take_the_fused_path(dtype, shape):
    N = 64
    policy, features = _avwan(N)
    amap = phm.action_map(N, 81, 3).reshape((N,) + shape).to(dtype).to(DEV)
    obs = {"action_map": amap}
    ops = _ops()
    with torch.no_grad():
        want = policy._head(features, obs, True)
        torch.cuda.synchronize()
        n0 = ops.ctx.launch_count
        got = ph.fused_head(policy, features, obs, True)
        assert ops.ctx.launch_count - n0 == 1
    clear = cases.clear_mode(want[3].probs.double())
    assert torch.equal(got[1][clear], want[1][clear])
    torch.testing.assert_close(got[3].probs, want[3].probs, rtol=1e-5, atol=1e-6)
    torch.testing.assert_close(got[0], want[0], rtol=1e-5, atol=1e-5)


class _ShapedNet(phm.StubNet):
    """StubNet whose features come out float64, non-contiguous or as they are."""

    def __init__(self, n_in, H, form):
        super().__init__(n_in, H)
        self.form = form

    def forward(self, observations, rnn_hidden_states, prev_actions, masks, *ext):
        f, h = super().forward(observations, rnn_hidden_states, prev_actions, masks)
        if self.form == "noncontig":
            f = f.t().contiguous().t()
        return f, h


@pytest.mark.parametrize("form,N", [("float64", 16), ("noncontig", 16), ("plain", 65536)])
@pytest.mark.parametrize("trainer", ["av_nav", "av_wan"])
def test_unqualified_features_fall_back_bit_for_bit(form, N, trainer):
    H, A = phm.SHAPES[trainer]
    net = _ShapedNet(8, H, form)
    masking = [True] if trainer == "av_wan" else []
    policy = phm.POLICIES[trainer](net, A, *masking)
    phm.set_params(policy, 6, 3.0)
    patched = ph.patch_policy(type("Patched", (phm.POLICIES[trainer],), {}))(net, A, *masking)
    patched.load_state_dict(policy.state_dict())
    dt = torch.float64 if form == "float64" else torch.float32
    policy.to(DEV, dt).eval()
    patched.to(DEV, dt).eval()
    obs = {"x": torch.randn((N, 8), generator=torch.Generator().manual_seed(6)).to(DEV, dt)}
    if trainer == "av_wan":
        obs["action_map"] = phm.action_map(N, A, 6).to(DEV)
    ops = _ops()
    for det in (True, False):
        args, kw = phm.act_args(trainer, obs, N, det)
        with torch.no_grad():
            torch.cuda.manual_seed(5)
            want = policy.act(*args, **kw)
            torch.cuda.synchronize()
            n0 = ops.ctx.launch_count
            torch.cuda.manual_seed(5)
            got = patched.act(*args, **kw)
            assert ops.ctx.launch_count == n0, form
        for s, t in zip(got[:4], want[:4]):
            assert torch.equal(s, t), form
        if trainer == "av_wan":
            assert torch.equal(got[4].probs, want[4].probs)


# -------------------------------------------------------------------------------------------------- entry limits
def test_entry_accepts_the_limits_and_refuses_past_them():
    ops = _ops()
    lib, ctx = ops.lib, ops.ctx
    H, A, n = cases.MAX_H, cases.MAX_A, 4
    t = {k: torch.zeros(s, device=DEV) for k, s in (("f", (n, H + 1)), ("w", (A + 1, H + 1)), ("b", (A + 1,)),
                                                    ("cw", (H + 1,)), ("cb", (1,)), ("v", (n,)), ("lp", (n,)))}
    a = torch.empty(n, dtype=torch.int64, device=DEV)
    st = torch.full((1,), -5, dtype=torch.int32, device=DEV)

    def call(H, A):
        return lib.ssb_policy_head_batch(ctx.handle, n, H, A, t["f"].data_ptr(), t["w"].data_ptr(),
                                         t["b"].data_ptr(), t["cw"].data_ptr(), t["cb"].data_ptr(), 0, None, None,
                                         t["v"].data_ptr(), a.data_ptr(), t["lp"].data_ptr(), None, st.data_ptr(),
                                         ctypes.c_void_p(0))
    torch.cuda.synchronize()
    n0 = ctx.launch_count
    assert call(H, A) == 0
    torch.cuda.synchronize()
    assert ctx.launch_count == n0 + 1 and int(st.item()) == 0
    assert bool((a == 0).all()) and bool((t["v"] == 0).all())
    assert call(H + 1, A) == -4 and "H <= 2048" in lib.ssb_last_error(ctx.handle).decode()
    assert call(H, A + 1) == -4 and "A <= 256" in lib.ssb_last_error(ctx.handle).decode()
    assert ctx.launch_count == n0 + 1
