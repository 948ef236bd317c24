"""The cases of tests/test_gpu_policy_head_domain.py as plain data and seeded inputs, shared with
tests/test_policy_head_domain_host.py, which checks that they reach every action slot count, critic pass, feature tail,
tail CTA, tie position and refusal class ``ssb_policy_head_batch`` accepts, and calibrates the GPU file's bars on the CPU.

Heads: ``logits`` (CategoricalNet: AV-Nav, SAVi), ``masked`` (CategoricalNetWithMask with an action map) and ``nomask``
(CategoricalNetWithMask with masking off: the kernel's masked head with no mask).  Every input is built on the CPU in
float32 and moved where a test needs it.
"""
import torch

import policy_head_models as phm

MAX_A, MAX_H, MAX_B = 256, 2048, 65535
HEADS = ("logits", "masked", "nomask")

# (H, A).  A mod 32 = 1, 2, 0, 15, 16, 17, 31, 0, 1, 0, 1, 4, 22, 0, 0, 31, 0 with 1 to 8 action slots per lane
# (A = 100, 150, 192 and 224 for 4 to 7); A + 1 = 16, 17, 33, 65, 193, 225, 257 rows put the critic on a first,
# second or later pass of the 16 warps; H mod 32 = 1, 2, 31, 0, 1, 4, 31, 1, 8, 12, 16, 0, 31, 0 with both limits.
SHAPES = [(1, 1), (1, 2), (2, 256), (31, 15), (32, 16), (33, 17), (64, 31), (100, 32), (511, 33), (513, 64),
          (1000, 65), (200, 100), (300, 150), (400, 192), (160, 224), (2047, 255), (2048, 256)]
TRAINER_SHAPES = [(512, 4), (128, 4), (512, 81)]
ALL_SHAPES = SHAPES + TRAINER_SHAPES
# every tail-CTA size ne = B mod 4 (1 to 4) and one CTA, two and 33
BATCHES = (1, 2, 3, 4, 5, 8, 129)
BIG_B_SHAPES = [(32, 16), (2048, 256)]
# actor weights N(0, gain^2 / H): 0 ties every logit (the bias is 0 too), 30 underflows probabilities to exactly 0,
# 300 makes most rows one-hot
GAINS = (0.0, 1.0, 3.0, 30.0, 300.0)

# action pairs sharing the row's maximum by construction: across a lane boundary in one slot, across slots in one
# lane, the first and last action, and two slots of lane 0
TIE_PAIRS = [(1, 33), (31, 63), (0, 255), (32, 224), (0, 1), (15, 16)]

# action-map kinds for the masked head; "open_j" opens the one action j of every row
MASKS = ("binary", "open_0", "open_31", "open_32", "open_last", "fraction", "subnormal", "huge", "negzero")
SUBNORMAL, HUGE = 1e-40, 1e30
# draws: torch's Exp(1), all ones (the draw is the mode), q = p (every action with p > 0 ties at 1), and Exp(1)
# with subnormal, huge and +Inf entries, +Inf on each row's most likely action
DRAWS = ("exp", "ones", "ratio_tie", "extreme")


def mask_actions(kind, A):
    """The open action of an ``open_*`` kind, or None."""
    return {"open_0": 0, "open_31": 31, "open_32": 32, "open_last": A - 1}.get(kind)


def mask_kinds(A, gain):
    """The mask kinds a masked case at A actions runs: one-action maps where that action exists, and only at gains
    whose probabilities cannot underflow (a single open action with probability 0 is a refused row)."""
    out, opened = [], set()
    for k in MASKS:
        j = mask_actions(k, A)
        if j is not None:
            if j >= A or j in opened or gain > 3.0:
                continue
            opened.add(j)
        out.append(k)
    return out


def params(H, A, gain, seed):
    """(actor weight [A][H], actor bias [A], critic weight [1][H], critic bias [1]) in float32."""
    g = torch.Generator().manual_seed(seed)
    aw = torch.randn((A, H), generator=g) * (gain / H ** 0.5)
    ab = torch.randn((A,), generator=g) * (0.1 if gain else 0.0)
    cw = torch.randn((1, H), generator=g) / H ** 0.5
    cb = torch.randn((1,), generator=g) * 0.1
    return aw, ab, cw, cb


def features(B, H, seed):
    g = torch.Generator().manual_seed(1000 + seed)
    return torch.tanh(torch.randn((B, H), generator=g) * 2)


def tie_pairs(A):
    return [p for p in TIE_PAIRS if p[1] < A]


def tie_inputs(B, H, A, pair, seed):
    """Parameters and features whose logits are exact in any summation order (integer weights in [-2, 2], features in
    multiples of 1/4, integer biases: every partial sum is a multiple of 1/4 below 2^15), with every row's maximum
    shared by the two actions of ``pair``: they get the same weights and the smallest integer bias that puts them
    above every other action of every row."""
    g = torch.Generator().manual_seed(seed)
    aw = torch.randint(-2, 3, (A, H), generator=g).float()
    cw = torch.randint(-2, 3, (1, H), generator=g).float()
    x = torch.randint(-4, 5, (B, H), generator=g).float() / 4
    i, j = pair
    aw[j] = aw[i]
    z = x.double() @ aw.double().t()
    others = torch.ones(A, dtype=torch.bool)
    others[[i, j]] = False
    ab = torch.zeros(A)
    gap = (z[:, others] - z[:, i:i + 1]).max().item() if bool(others.any()) else 0.0
    ab[i] = ab[j] = float(int(gap) + 1)
    return (aw, ab, cw, torch.zeros(1)), x


def make_mask(kind, B, A, seed, z64):
    """(B, A) float32 action map of ``kind``; every kind but ``open_*`` opens each row's float64 argmax of z, so no
    row normalises to zero."""
    g = torch.Generator().manual_seed(2000 + seed)
    j = mask_actions(kind, A)
    if j is not None:
        m = torch.zeros((B, A))
        m[:, j] = 1.0
        return m
    top = z64.argmax(dim=1)
    rows = torch.arange(B)
    if kind == "fraction":
        m = torch.randint(0, 11, (B, A), generator=g).float() * 0.1
        m[rows, top] = 0.7
        return m
    m = (torch.rand((B, A), generator=g) < 0.6).float()
    m[rows, top] = 1.0
    if kind == "subnormal":
        m = m * SUBNORMAL
    elif kind == "huge":
        m = m * HUGE
    elif kind == "negzero":
        m = torch.where(m == 0, torch.full_like(m, -0.0), m)
    return m


def make_draw(kind, B, A, seed, p):
    """(B, A) float32 draws q of ``kind`` for probabilities ``p`` (float32, the kernel's own for ``ratio_tie``)."""
    g = torch.Generator().manual_seed(3000 + seed)
    if kind == "ones":
        return torch.ones((B, A))
    if kind == "ratio_tie":
        return torch.where(p > 0, p, torch.ones_like(p))
    q = torch.empty((B, A)).exponential_(1, generator=g)
    if kind == "extreme":
        r = torch.rand((B, A), generator=g)
        q = torch.where(r < 0.1, torch.full_like(q, SUBNORMAL), q)
        q = torch.where((r >= 0.1) & (r < 0.2), torch.full_like(q, 1e30), q)
        q = torch.where((r >= 0.2) & (r < 0.25), torch.full_like(q, float("inf")), q)
        q[torch.arange(B), p.argmax(dim=1)] = float("inf")
    return q


EPS = float(torch.finfo(torch.float32).eps)
# the GPU file's bars: value relative to max(1, |ref|), log_prob relative to the row's largest |log-probability|,
# probs absolute
BAR_VALUE, BAR_LOG_PROB, BAR_PROBS = 1e-4, 1e-4, 1e-5


def reference64(prm, x, head, mask):
    """The heads in float64 on ``x``'s device -> (value (B,), z, p, lp, grid) with lp the table ``log_prob`` gathers
    from: z - logsumexp(z) for the logits head, log(clamp(p, eps, 1 - eps)) for the masked head.  The masked product
    p * mask is rounded to float32, as the reference's float32 product and the kernel round it; ``grid`` (B, 1) is one
    float32 step of that product at the row's smallest magnitude (2^-149) relative to its sum, 0 elsewhere: in a row
    whose every product is subnormal it is more than the probability bar, and it is added to it."""
    aw, ab, cw, cb = (t.to(x.device, torch.float64) for t in prm)
    x = x.double()
    z = x @ aw.t() + ab
    value = (x @ cw.t() + cb)[:, 0]
    grid = torch.zeros((x.shape[0], 1), dtype=torch.float64, device=x.device)
    if head == "logits":
        lp = z - torch.logsumexp(z, 1, keepdim=True)
        p = torch.softmax(lp, 1)
    else:
        p = torch.softmax(z, 1)
        if mask is not None:
            p = (p * mask.to(x.device, torch.float64)).float().double()
        t = p.sum(1, keepdim=True)
        grid = 2.0 ** -149 / t
        p = p / t
        lp = torch.log(p.clamp(EPS, 1 - EPS))
    return value, z, p, lp, grid


def errors(value, action, log_prob, probs, ref):
    """Worst |error| / bar of (value, log_prob, probs) over the rows, log_prob gathered at ``action``."""
    v64, _, p64, lp64, grid = ref
    a = action.view(-1, 1)
    fin = torch.where(lp64.isfinite(), lp64.abs(), torch.zeros_like(lp64))
    bar_lp = BAR_LOG_PROB * fin.amax(1, keepdim=True) + 2 * grid / p64.gather(1, a).clamp_min(EPS)
    bar_lp = bar_lp.clamp_min(1e-30)
    e_v = ((value.view(-1).double() - v64).abs() / (BAR_VALUE * v64.abs().clamp_min(1.0))).max().item()
    e_lp = ((log_prob.view(-1, 1).double() - lp64.gather(1, a)).abs() / bar_lp).max().item()
    e_p = ((probs.double() - p64).abs() / probs_bar(ref)).max().item() if probs is not None else 0.0
    return e_v, e_lp, e_p


def probs_bar(ref):
    """(B, 1) bar on the probabilities: 1e-5, plus 4 float32 roundings of the row's largest |z| (a float32 logit is
    only that exact, and exp turns an error in z into the same relative error in p: at gain 300, |z| near 1000, that
    is 4.6e-4), plus 4 float32 steps of a subnormal masked product (``grid``)."""
    z64, grid = ref[1], ref[4]
    zmax = torch.where(z64.isfinite(), z64.abs(), torch.zeros_like(z64)).amax(1, keepdim=True)
    return BAR_PROBS + 4 * EPS * zmax + 4 * grid


def clear_mode(p64, gap=1e-5):
    """Rows whose top two float64 probabilities differ by more than ``gap`` relative."""
    if p64.shape[1] == 1:
        return torch.ones(p64.shape[0], dtype=torch.bool, device=p64.device)
    top = torch.topk(p64, 2, dim=1).values
    return (top[:, 0] - top[:, 1]) > gap * top[:, 0]


# ---------------------------------------------------------------------------------------------------------- refusals
# one call of B = REFUSE_B envs (CTAs 0 to 32, the last with 2 envs) per input; a per-row input is placed at rows
# 4 * cta + slot for (cta, slot) in REFUSE_AT: the first CTA, a middle one and the last, slots 0 to 3
REFUSE_B = 130
REFUSE_AT = [(0, 0), (0, 3), (16, 1), (16, 2), (32, 1)]
# (name, head, rows it applies to: "rows" the REFUSE_AT rows, "all" every row (a parameter), whether refused)
REFUSALS = [
    ("nan_feature", "logits", "rows", True),
    ("pinf_feature", "logits", "rows", True),
    ("ninf_feature", "logits", "rows", True),
    ("pinf_bias", "logits", "all", True),
    ("ninf_biases_all", "logits", "all", True),
    ("ninf_biases_some", "logits", "all", False),
    ("overflow_feature", "logits", "rows", True),
    ("nan_feature", "masked", "rows", True),
    ("pinf_feature", "masked", "rows", True),
    ("ninf_feature", "masked", "rows", True),
    ("pinf_bias", "nomask", "all", True),
    ("ninf_biases_all", "nomask", "all", True),
    ("ninf_biases_some", "nomask", "all", False),
    ("overflow_feature", "masked", "rows", True),
    ("mask_zero", "masked", "rows", True),
    ("mask_underflow", "masked", "rows", True),
    ("mask_negative", "masked", "rows", True),
    ("mask_nan", "masked", "rows", True),
    ("mask_pinf", "masked", "rows", True),
]
REFUSE_SHAPES = [(512, 4), (128, 4), (512, 81), (33, 17), (2048, 256)]


def refuse_rows():
    return sorted(4 * c + s for c, s in REFUSE_AT)


def refusal_input(name, head, H, A, seed=7):
    """(params, features (REFUSE_B, H), mask or None) of a refusal input.  ``mask_underflow`` runs at gain 300 and
    opens only actions whose float64 probability is below e^-120 (float32 rounds it to 0 in any order)."""
    gain = 300.0 if name == "mask_underflow" else 3.0
    aw, ab, cw, cb = params(H, A, gain, seed)
    x = features(REFUSE_B, H, seed)
    rows = refuse_rows()
    col = H // 2
    if name == "nan_feature":
        x[rows, col] = float("nan")
    elif name == "pinf_feature":
        x[rows, col] = float("inf")
    elif name == "ninf_feature":
        x[rows, col] = float("-inf")
    elif name == "overflow_feature":
        # positive weights: every product positive and every sum past FLT_MAX, so every z is +Inf in any summation
        # order, never NaN
        aw = aw.abs()
        x[rows] = 3e38
    elif name == "pinf_bias":
        ab[A // 2] = float("inf")
    elif name == "ninf_biases_all":
        ab[:] = float("-inf")
    elif name == "ninf_biases_some":
        ab[::2] = float("-inf") if A > 1 else 0.0
    mask = None
    if head == "masked":
        z64 = x.double() @ aw.double().t() + ab.double()
        z64 = torch.nan_to_num(z64, nan=0.0, posinf=0.0, neginf=0.0)
        mask = make_mask("binary", REFUSE_B, A, seed, z64)
        top = z64.argmax(dim=1)
        for r in rows:
            if name == "mask_zero":
                mask[r] = 0.0
            elif name == "mask_underflow":
                lp = torch.log_softmax(z64[r], 0)
                mask[r] = (lp < -120).float()
            elif name == "mask_negative":
                # beside the open argmax: the sum stays positive, that entry negative (a -1 at a row's only open
                # action would normalise to a valid 1 beside -0.0)
                mask[r, (top[r] + 1) % A] = -1.0
            elif name == "mask_nan":
                mask[r, (top[r] + 1) % A] = float("nan")
            elif name == "mask_pinf":
                mask[r, (top[r] + 1) % A] = float("inf")
    return (aw, ab, cw, cb), x, mask


def refusal_expected_rows(name, head, applies):
    if applies == "all":
        return list(range(REFUSE_B))
    return refuse_rows()


def stand_in(H, A, head, prm):
    """The eager stand-in policy (tests/policy_head_models.py) with parameters ``prm``, on the CPU in float32."""
    trainer = "av_nav" if head == "logits" else "av_wan"
    policy = phm.make_policy(trainer, H, A, masking=head == "masked").eval()
    with torch.no_grad():
        for lin, (w, b) in ((policy.action_distribution.linear, prm[:2]), (policy.critic.fc, prm[2:])):
            lin.weight.copy_(w)
            lin.bias.copy_(b)
    return policy
