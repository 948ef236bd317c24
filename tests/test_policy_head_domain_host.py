"""The cases of tests/test_gpu_policy_head_domain.py (tests/policy_head_domain_cases.py) against ``policy_head_kernel``'s
tiling: every action slot count, a critic row on a second pass, short feature tails, every tail CTA, both limits, ties
across lanes and slots, and every refusal class.  The kernel's refusal rule restated in float32 against the eager
stand-in, and the float32 calibration of the GPU file's bars.  No GPU."""
import os
import re

import numpy as np
import pytest

torch = pytest.importorskip("torch")
from torch.distributions import Categorical  # noqa: E402

import policy_head_domain_cases as cases  # noqa: E402

SRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "soundspaces_b200", "csrc",
                   "ssb200.cu")

# the kernel's tiling, restated
PH_ENVS, PH_WARPS, PH_SLOTS = 4, 16, 8


def slots(A):
    """Action slots a lane holds: actions l + 32 k for k < slots."""
    return -(-A // 32)


def critic_pass(A):
    """(warp, pass) of the critic row A in the round robin r = warp + PH_WARPS * pass."""
    return A % PH_WARPS, A // PH_WARPS


def tail_envs(B):
    """Envs of the last CTA."""
    return B - PH_ENVS * ((B - 1) // PH_ENVS)


def test_tiling_matches_the_source():
    src = open(SRC).read()
    k0 = src.index("policy_head_kernel(PolicyHeadParams p)")
    body = src[k0:src.index("// SAVi belief update", k0)]
    for name, value in (("PH_ENVS", PH_ENVS), ("PH_WARPS", PH_WARPS), ("PH_MAX_A", cases.MAX_A),
                        ("PH_MAX_H", cases.MAX_H)):
        assert re.search(rf"#define {name} {value}\n", src), name
    assert "#define PH_SLOTS (PH_MAX_A / 32)" in src and cases.MAX_A // 32 == PH_SLOTS
    assert "for (int r = warp; r <= A; r += PH_WARPS)" in body            # row A, the critic, is one more row
    assert "for (int f = lane; f < H; f += 32)" in body
    assert "const int a = lane + 32 * k;" in body
    assert "ne = min(PH_ENVS, p.B - e0)" in body
    assert re.search(r"B < 0 \|\| B > 65535", src)


# -------------------------------------------------------------------------------------------------------- coverage
def test_every_slot_count_and_critic_pass_is_reached():
    assert {slots(A) for _, A in cases.SHAPES} == set(range(1, PH_SLOTS + 1))
    passes = {critic_pass(A)[1] for _, A in cases.SHAPES}
    assert {0, 1} <= passes and max(passes) == critic_pass(cases.MAX_A)[1] == 16
    # A + 1 at 16 (the last warp's first row) and 17 (a second pass), and at 16 k + 1 beyond
    assert {15, 16} <= {A for _, A in cases.SHAPES}
    assert any(A >= 32 and (A + 1) % 16 == 1 for _, A in cases.SHAPES)
    assert {H % 32 for H, _ in cases.SHAPES} >= {0, 1, 31}
    assert (1, 1) in cases.SHAPES and (cases.MAX_H, cases.MAX_A) in cases.SHAPES
    assert set(cases.TRAINER_SHAPES) <= set(cases.ALL_SHAPES)
    assert all(1 <= H <= cases.MAX_H and 1 <= A <= cases.MAX_A for H, A in cases.ALL_SHAPES)


def test_every_tail_cta_and_both_batch_limits():
    assert {tail_envs(b) for b in cases.BATCHES} == {1, 2, 3, 4}
    assert 1 in cases.BATCHES and max(cases.BATCHES) > 4 * PH_ENVS
    assert cases.MAX_B == 65535 and tail_envs(cases.MAX_B) == 3
    assert (cases.MAX_H, cases.MAX_A) in cases.BIG_B_SHAPES and any(A <= 32 for _, A in cases.BIG_B_SHAPES)


def test_ties_cross_lanes_and_slots():
    lanes = [p for p in cases.TIE_PAIRS if p[0] // 32 == p[1] // 32 and p[0] % 32 != p[1] % 32]
    slot_pairs = [p for p in cases.TIE_PAIRS if p[0] // 32 != p[1] // 32]
    assert lanes and slot_pairs
    assert any(p[0] % 32 == p[1] % 32 for p in slot_pairs)            # one lane, two slots
    assert any(p[0] % 32 != p[1] % 32 for p in slot_pairs)            # two lanes, two slots
    assert (0, cases.MAX_A - 1) in cases.TIE_PAIRS
    for p in cases.TIE_PAIRS:
        assert any(p in cases.tie_pairs(A) for _, A in cases.SHAPES), p


@pytest.mark.parametrize("H,A", cases.SHAPES[:6] + [(2048, 256)])
def test_tie_inputs_tie_exactly_in_float32(H, A):
    for pair in cases.tie_pairs(A):
        (aw, ab, cw, cb), x = cases.tie_inputs(8, H, A, pair, seed=3)
        z32 = torch.nn.functional.linear(x, aw, ab)
        z64 = x.double() @ aw.double().t() + ab.double()
        assert torch.equal(z32.double(), z64)
        top = z64.max(dim=1).values
        assert bool((z64[:, pair[0]] == top).all() and (z64[:, pair[1]] == top).all())
        assert int((z64 == top[:, None]).sum()) == 2 * 8


def test_every_refusal_class_is_placed():
    rows = cases.refuse_rows()
    last = (cases.REFUSE_B - 1) // PH_ENVS
    assert {c for c, _ in cases.REFUSE_AT} == {0, 16, last} and 0 < 16 < last
    assert {s for _, s in cases.REFUSE_AT} == {0, 1, 2, 3}
    assert all(r < cases.REFUSE_B for r in rows) and len(set(rows)) == len(rows)
    names = {(n, h) for n, h, _, _ in cases.REFUSALS}
    for n in ("nan_feature", "pinf_feature", "ninf_feature", "overflow_feature"):
        assert (n, "logits") in names and (n, "masked") in names, n
    for n in ("pinf_bias", "ninf_biases_all", "ninf_biases_some"):
        assert (n, "logits") in names and (n, "nomask") in names, n
    for n in ("mask_zero", "mask_underflow", "mask_negative", "mask_nan", "mask_pinf"):
        assert (n, "masked") in names, n
    assert [r[3] for r in cases.REFUSALS if r[0] == "ninf_biases_some"] == [False, False]


# ------------------------------------------------------------------------------------------------- refusal rule
def kernel_refuses(z, head, mask, sampling, old=False):
    """The kernel's refusal rule on one row's float32 logits z (numpy), restated: fmaxf skips NaN, a NaN z, with the
    logits head a NaN normalised logit (``old``: the rule before, a NaN z only), with the masked head a zero sum or a
    NaN or negative normalised entry, and when sampling a non-finite probability."""
    f = np.float32
    with np.errstate(all="ignore"):
        bad = bool(np.isnan(z).any())
        m = np.fmax.reduce(z, initial=f(-np.inf))
        s = np.exp(z - m).sum(dtype=f)
        if head == "logits":
            l = z - (m + np.log(s))
            if not old:
                bad |= bool(np.isnan(l).any())
            m2 = np.fmax.reduce(l, initial=f(-np.inf))
            e = np.exp(l - m2)
            p = e / e.sum(dtype=f)
        else:
            p = np.exp(z - m) / s
            if mask is not None:
                p = p * mask
            t = p.sum(dtype=f)
            bad |= bool(t == 0)
            p = p / t
            bad |= not bool((p >= 0).all())
        if sampling:
            bad |= not bool(np.isfinite(p).all())
    return bad


def _raises(policy, x, mask, deterministic):
    obs = {"x": torch.zeros((1, 8)), "action_map": mask if mask is not None else torch.ones((1, x.shape[1]))}
    try:
        with torch.no_grad():
            policy._head(x, obs, deterministic)
    except ValueError:
        return True
    return False


def _refusal_inputs():
    for name, head, applies, refused in cases.REFUSALS:
        for H, A in cases.REFUSE_SHAPES:
            if name == "mask_underflow" and A < 2:
                continue
            yield pytest.param(name, head, applies, refused, H, A, id=f"{name}-{head}-{H}x{A}")


ROW_CHECKS = (1, 2, 64, cases.REFUSE_B - 1)


@pytest.mark.parametrize("name,head,applies,refused,H,A", list(_refusal_inputs()))
def test_refusal_rule_matches_the_reference(name, head, applies, refused, H, A):
    """The restated rule equals "the stand-in raises ValueError" on every checked row, in mode and when sampling; the
    rule before this fix (a NaN z only) disagrees on every logits-head input whose z holds +Inf or only -Inf."""
    prm, x, mask = cases.refusal_input(name, head, H, A)
    policy = cases.stand_in(H, A, head, prm)
    want = set(cases.refusal_expected_rows(name, head, applies)) if refused else set()
    old_disagrees = 0
    for r in sorted(set(cases.refuse_rows()) | set(ROW_CHECKS)):
        with torch.no_grad():
            z = policy.action_distribution.linear(x[r:r + 1])[0].numpy()
        m = None if mask is None else mask[r].numpy()
        for det in (True, False):
            raised = _raises(policy, x[r:r + 1], None if mask is None else mask[r:r + 1], det)
            assert raised == (r in want), (name, r, det)
            assert kernel_refuses(z, head, m, not det) == raised, (name, r, det)
            old_disagrees += kernel_refuses(z, head, m, not det, old=True) != raised
    inf_logits = head == "logits" and name in ("pinf_feature", "ninf_feature", "pinf_bias", "ninf_biases_all",
                                               "overflow_feature")
    if inf_logits:
        # in mode every refused row escapes the old rule; when sampling the NaN probabilities catch it
        assert old_disagrees == len([r for r in set(cases.refuse_rows()) | set(ROW_CHECKS) if r in want])
    else:
        assert old_disagrees == 0


# -------------------------------------------------------------------------------------------------- calibration
def _f32_head(prm, x, head, mask):
    """torch's float32 CPU head, the reference's computation: (value, mode action, log_prob, probs)."""
    aw, ab, cw, cb = prm
    F = torch.nn.functional
    z = F.linear(x, aw, ab)
    value = F.linear(x, cw, cb)[:, 0]
    if head == "logits":
        d = Categorical(logits=z, validate_args=False)
        a = d.probs.argmax(1)
        lp = d.logits.gather(1, a[:, None])[:, 0]
    else:
        p = torch.softmax(z, 1)
        if mask is not None:
            p = p * mask
        d = Categorical(probs=p, validate_args=False)
        a = d.probs.argmax(1)
        lp = torch.log(d.probs.clamp(cases.EPS, 1 - cases.EPS)).gather(1, a[:, None])[:, 0]
    return value, a, lp, d.probs


WORST = {}


@pytest.mark.parametrize("H,A", cases.ALL_SHAPES)
def test_float32_calibration_of_the_bars(H, A):
    """torch's float32 head against float64 on every accuracy input and tie input; every error is at most half of
    its bar.  The masked head's bar on a subnormal row adds one float32 step of its product (cases.reference64)."""
    B = 129
    seed = 31 * H + A
    x = cases.features(B, H, seed)
    worst = [0.0, 0.0, 0.0]
    for head in cases.HEADS:
        inputs = []
        for gain in cases.GAINS:
            prm = cases.params(H, A, gain, seed)
            z64 = x.double() @ prm[0].double().t() + prm[1].double()
            for kind in (cases.mask_kinds(A, gain) if head == "masked" else [None]):
                inputs.append((prm, x, None if kind is None else cases.make_mask(kind, B, A, seed, z64)))
        for k, pair in enumerate(cases.tie_pairs(A)):
            prm, xt = cases.tie_inputs(B, H, A, pair, seed=H + k)
            inputs.append((prm, xt, torch.ones((B, A)) if head == "masked" else None))
        for prm, xx, mask in inputs:
            out = _f32_head(prm, xx, head, mask)
            e = cases.errors(*out, cases.reference64(prm, xx, head, mask))
            worst = [max(u, v) for u, v in zip(worst, e)]
    WORST[(H, A)] = worst
    print(f"H={H} A={A}: worst error / bar: value {worst[0]:.3g}, log_prob {worst[1]:.3g}, probs {worst[2]:.3g}")
    assert max(worst) <= 0.5, worst
