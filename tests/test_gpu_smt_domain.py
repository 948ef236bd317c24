"""SAVi's scene memory transformer on the GPU across the inputs ``ssb_smt_state_encoder_batch`` accepts: widths and
head sizes off the kernels' tile grid, fusion input widths across the 64-wide K tiles, per-env token counts at the 16-row
query and 64-key tile edges in contiguous, wrapped and scattered slot layouts, the largest shared-memory footprints,
decoder groups of 4 envs, every kind of mask value, distinct LayerNorm eps, a zero-variance LayerNorm input, badly
scaled inputs and pose edges.  Each env is compared with a float64 forward of the stand-in on its own scale:
``max|got_b - ref_b| <= 1e-4 max|ref_b|`` for every env b (``test_gpu_smt._check``).  The C entry is also called
directly: every refusal returns its code and message and launches nothing, and every limit runs.

The cases are listed in tests/smt_domain_cases.py; tests/test_smt_host.py checks through a restatement of the host's
tiling that they reach every kernel's tile edges.

Calibration (torch's float32 forward of the stand-in on a CPU against float64, max over envs of
max|d_b| / max|ref_b|): 2e-7 .. 8e-7 at head dims 1, 9, 25 and 125, d 512 with T = 1024, D = 1024 with pose index
1020, D = 2 without pose encoding, pose index 0 and inputs scaled by 1e3 and 1e-6.  The cases calibrated here give
their figures in their docstrings.  1e-4 leaves two orders of magnitude over float32 rounding and still catches a wrong
tile tail or a wrong eps.
"""
import ctypes as C
import math

import pytest

import smt_domain_cases as cases
from smt_models import make_inputs, make_smt
from test_gpu_smt import DEV, LAUNCHES, _check, _cuda, _ops, _ref64, _run

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")


def masks_for(c):
    """(B, M) masks with ``c["valid"][b]`` valid slots for env b: ``contiguous`` from slot 0, ``wrapped`` around the
    end of the ring, ``scattered`` every (M // valid)-th slot, or by default make_inputs' ring ending before slot 7 b."""
    B, M = c["B"], c["M"]
    masks = torch.zeros(B, M)
    layout = c.get("layout")
    for b, v in enumerate(c["valid"]):
        i = torch.arange(v)
        if layout == "contiguous":
            slots = i
        elif layout == "wrapped":
            slots = (M - v // 2 + i) % M
        elif layout == "scattered":
            slots = i * max(1, M // max(v, 1))
        else:
            slots = ((7 * b) % max(M, 1) - 1 - i) % max(M, 1)
        masks[b, slots] = 1.0
    return masks


def model_for(c):
    return make_smt(D=c["D"], pose_index=c["pose_index"], d_model=c["d_model"], nhead=c["nhead"],
                    pretraining=c["pretraining"], seed=c["seed"])


def inputs_for(c, goal=True):
    """x, memory, masks, goal of a case (goal None without one)."""
    return make_inputs(c["B"], c["M"], D=c["D"], d_model=c["d_model"], pose_index=c["pose_index"], seed=c["seed"],
                       goal=goal, masks=masks_for(c))


def _subset(envs, x, memory, masks, goal):
    i = torch.tensor(envs)
    return x[i], memory[:, i], masks[i], None if goal is None else goal[i]


def accuracy(m, x, memory, masks, goal, envs=None, mc=None):
    """The library's output for the batch, checked per env against float64 (only ``envs`` when given)."""
    out = _run(mc if mc is not None else _cuda(m), x, memory, masks, goal)
    if envs is None:
        _check(out, _ref64(m, x, memory, masks, goal))
    else:
        _check(out[torch.tensor(envs).to(DEV)], _ref64(m, *_subset(envs, x, memory, masks, goal)))
    return out


def _by_name(cs):
    return {c["name"]: c for c in cs}


# ---------------------------------------------------------------------------
# widths, heads and fusion input widths
# ---------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(_by_name(cases.width_cases())))
def test_widths_and_heads(name):
    c = _by_name(cases.width_cases())[name]
    m = model_for(c)
    mc = _cuda(m)
    for goal in (True, False):
        accuracy(m, *inputs_for(c, goal), mc=mc)


@pytest.mark.parametrize("name", list(_by_name(cases.fusion_cases())))
def test_fusion_widths(name):
    """Without pose encoding F = D (D = 1 and 2 included), with it F = pose index + 16.  Where D > pose index + 4,
    NaN in the columns past the pose (dropped by the module) gives the finite run's output bit for bit."""
    c = _by_name(cases.fusion_cases())[name]
    m = model_for(c)
    mc = _cuda(m)
    x, memory, masks, goal = inputs_for(c)
    out = accuracy(m, x, memory, masks, goal, mc=mc)
    accuracy(m, x, memory, masks, None, mc=mc)
    pi = c["pose_index"]
    if pi is not None and c["D"] > pi + 4:
        x, memory = x.clone(), memory.clone()
        x[:, pi + 4:] = float("nan")
        memory[..., pi + 4:] = float("nan")
        assert torch.equal(_run(mc, x, memory, masks, goal), out)


# ---------------------------------------------------------------------------
# token counts at the tile edges
# ---------------------------------------------------------------------------
@pytest.mark.parametrize("goal", [True, False], ids=["goal", "no_goal"])
@pytest.mark.parametrize("layout", cases.LAYOUTS)
def test_token_counts(layout, goal):
    """Counts 1 .. 1024 (current token included) in one batch of 1023 slots; without a goal the decoder's target is
    the fused token at row count - 1."""
    c = _by_name(cases.count_cases())[f"counts_{layout}"]
    x, memory, masks, g = inputs_for(c, goal)
    assert [int(v) for v in masks.sum(1)] == c["valid"]
    accuracy(model_for(c), x, memory, masks, g)


# ---------------------------------------------------------------------------
# the largest footprints
# ---------------------------------------------------------------------------
def _check_envs(c):
    """Every env, or at B = 1024 the first and last 4-env groups, the middle, and the envs with the fewest and most
    tokens (the float64 reference of all 1024 envs x 1024 tokens would dominate the file's time)."""
    if c["B"] <= 64:
        return None
    v = c["valid"]
    return sorted({0, 1, 2, 3, c["B"] // 2, c["B"] - 4, c["B"] - 3, c["B"] - 2, c["B"] - 1,
                   v.index(min(v)), v.index(max(v))})


@pytest.mark.parametrize("name", list(_by_name(cases.largest_cases())))
def test_largest_footprints(name):
    c = _by_name(cases.largest_cases())[name]
    m = model_for(c)
    mc = _cuda(m)
    for goal in (True, False):
        accuracy(m, *inputs_for(c, goal), envs=_check_envs(c), mc=mc)
    torch.cuda.synchronize()


# ---------------------------------------------------------------------------
# decoder groups of 4 envs
# ---------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(_by_name(cases.decoder_cases())))
def test_decoder_batch_sizes(name):
    c = _by_name(cases.decoder_cases())[name]
    m = model_for(c)
    mc = _cuda(m)
    x, memory, masks, goal = inputs_for(c)
    envs = _check_envs(c)
    out = accuracy(m, x, memory, masks, goal, envs=envs, mc=mc)
    b = c["B"] - 1                                              # the last env alone
    one = _run(mc, x[b:].contiguous(), memory[:, b:].contiguous(), masks[b:].contiguous(), goal[b:].contiguous())
    assert torch.equal(one[0], out[b])


def test_decoder_group_positions():
    """One env at positions 0 .. 3 of a 4-env decoder group and across the last, partial group of 11 gives its own
    output bit for bit."""
    probes = cases.probe_cases()
    c = probes[0]
    m = model_for(c)
    mc = _cuda(m)
    x, memory, masks, goal = inputs_for(c)
    px, pmem, pmasks, pgoal = inputs_for(dict(c, B=1, seed=c["seed"] + 1, valid=[17]))
    alone = _run(mc, px, pmem, pmasks, pgoal)[0]
    for p in (pc["probe"] for pc in probes):
        bx, bmem, bmasks, bgoal = x.clone(), memory.clone(), masks.clone(), goal.clone()
        bx[p], bmem[:, p], bmasks[p], bgoal[p] = px[0], pmem[:, 0], pmasks[0], pgoal[0]
        out = accuracy(m, bx, bmem, bmasks, bgoal, mc=mc) if p == probes[-1]["probe"] else _run(mc, bx, bmem, bmasks, bgoal)
        assert torch.equal(out[p], alone), p


# ---------------------------------------------------------------------------
# mask values
# ---------------------------------------------------------------------------
def test_mask_values():
    """1, 2, 0.5, 0, -1, +inf, -inf and NaN in every env (slot j of env b holds value (j + b) mod 8): a slot is padding
    iff 1 - m > 0, so 1, 2, +inf and NaN are valid.  float32 on a CPU: 2.2e-7 of float64."""
    c = _by_name(cases.mask_cases())["mask_values"]
    x, memory, _, goal = inputs_for(c)
    vals = torch.tensor(cases.MASK_VALUES)
    j = torch.arange(c["M"])
    masks = torch.stack([vals[(j + b) % len(vals)] for b in range(c["B"])])
    assert [int(v) for v in (~((1 - masks) > 0)).sum(1)] == c["valid"]
    accuracy(model_for(c), x, memory, masks, goal)


def test_pretraining_ignores_non_zero_masks():
    """Only the current token is valid.  float32 on a CPU: 4.9e-7 of float64."""
    c =_by_name(cases.mask_cases())["pretraining"]
    x, memory, _, goal = inputs_for(c)
    masks = 1.0 + torch.rand(c["B"], c["M"], generator=torch.Generator().manual_seed(7))
    m = model_for(c)
    assert m._pretraining
    accuracy(m, x, memory, masks, goal)


# ---------------------------------------------------------------------------
# numerics
# ---------------------------------------------------------------------------
def _norms(m):
    enc, dec = m.transformer.encoder.layers[0], m.transformer.decoder.layers[0]
    return [enc.norm1, enc.norm2, m.transformer.encoder.norm, dec.norm1, dec.norm2, dec.norm3, m.transformer.decoder.norm]


def eps_model(c):
    """Seven distinct eps; norm2 and norm3 shrunk to gamma, beta ~ 0.05, so that the final norms, which run as a
    second pass over their output, see a variance near their eps."""
    m = model_for(c)
    norms = _norms(m)
    for n, eps in zip(norms, cases.EPS):
        n.eps = eps
    with torch.no_grad():
        for n in (norms[1], norms[5]):
            n.weight.mul_(0.05)
            n.bias.mul_(0.05)
    return m


def constant_norm1_model(c):
    """encoder norm1's input is 0.5 in every column of every row (fusion_encoder[2] and the encoder's out_proj reduced
    to their biases 0.5 and 0; sums of 0.5 are exact in float32), so its variance is exactly 0 and its output is its
    beta."""
    m = model_for(c)
    with torch.no_grad():
        m.fusion_encoder[2].weight.zero_()
        m.fusion_encoder[2].bias.fill_(0.5)
        out_proj = m.transformer.encoder.layers[0].self_attn.out_proj
        out_proj.weight.zero_()
        out_proj.bias.zero_()
    return m


def test_layer_norm_eps():
    """float32 on a CPU: 4.7e-7 of float64."""
    c =_by_name(cases.numeric_cases())["eps"]
    m = eps_model(c)
    assert len({n.eps for n in _norms(m)}) == 7
    mc = _cuda(m)
    for goal in (True, False):
        accuracy(m, *inputs_for(c, goal), mc=mc)


def test_zero_variance_layer_norm_input():
    """norm1 returns its beta: rstd = 1 / sqrt(eps) multiplies an exact 0.  float32 on a CPU: 3.8e-7 of float64."""
    c =_by_name(cases.numeric_cases())["constant_norm1"]
    m = constant_norm1_model(c)
    mc = _cuda(m)
    for goal in (True, False):
        accuracy(m, *inputs_for(c, goal), mc=mc)


def scaled_inputs(c, goal=True):
    """The case's inputs with every feature column (not the pose) and the goal scaled by ``c["scale"]``."""
    x, memory, masks, g = inputs_for(c, goal)
    s, pi = c["scale"], c["pose_index"]
    x[:, :pi] *= s
    memory[..., :pi] *= s
    return x, memory, masks, None if g is None else g * s


@pytest.mark.parametrize("scale", cases.SCALES)
def test_input_scales(scale):
    """1e-6 and 1e3 (where the softmax saturates).  float32 on a CPU: 3.4e-7 and 5.3e-7 of float64."""
    c = _by_name(cases.numeric_cases())[f"scale{scale:g}"]
    m = model_for(c)
    mc = _cuda(m)
    for goal in (True, False):
        accuracy(m, *scaled_inputs(c, goal), mc=mc)


def pose_edge_inputs(c, goal=True):
    """Env 0: memory poses at the agent's exact position (atan2(0, 0)); env 1: headings on both sides of +-pi; envs 2
    and 3: headings near +1e3 and -1e3 rad; env 4: times 0 and 200 (exp(-t) underflows in float32); env 5: all of it;
    envs 6, 7: make_inputs' trajectories."""
    x, memory, masks, g = inputs_for(c, goal)
    pi, M = c["pose_index"], c["M"]
    h = slice(pi + 2, pi + 3)
    for b in (0, 5):
        memory[::2, b, pi:pi + 2] = x[b, pi:pi + 2]
    for b, centre in ((1, math.pi), (2, 1000.0), (3, -1000.0), (5, 1000.0)):
        x[b, h] = centre - 0.01
        memory[:, b, h] = (centre + torch.linspace(-0.5, 0.5, M) * (-1) ** b)[:, None]
    x[1, h] = math.pi - 0.01
    memory[1::2, 1, h] = -math.pi + 0.02                    # across the +-pi seam
    for b in (4, 5):
        x[b, pi + 3] = 0.0
        memory[::3, b, pi + 3] = 200.0
        memory[1::3, b, pi + 3] = 0.0
    return x, memory, masks, g


def test_pose_edges():
    """float32 on a CPU: 2.2e-6 of float64, the most of any case here: near 1e3 rad the relative bearing
    atan2(dy, dx) + heading rounds to float32's 6e-5 spacing before its sine and cosine are taken."""
    c =_by_name(cases.numeric_cases())["pose_edges"]
    m = model_for(c)
    mc = _cuda(m)
    for goal in (True, False):
        accuracy(m, *pose_edge_inputs(c, goal), mc=mc)


# ---------------------------------------------------------------------------
# the C entry called directly
# ---------------------------------------------------------------------------
SSB_E_INVALID_ARG, SSB_E_SHAPE = -1, -4


class Entry:
    """Device inputs of one direct ``ssb_smt_state_encoder_batch`` call and the call itself, any argument replaced."""

    def __init__(self, m, B, M, D, goal=True, seed=0):
        from soundspaces_b200 import smt
        self.ops = _ops()
        self.m = _cuda(m)
        d = m.transformer.d_model
        pi = m._pose_indices[0] if m._use_pose_encoding and m._pose_indices[0] + 4 <= D else None
        x, memory, masks, g = make_inputs(B, M, D=D, d_model=d, pose_index=pi, seed=seed, goal=goal)
        self.B, self.M = B, M
        self.x, self.memory, self.masks = x.to(DEV), memory.to(DEV), masks.to(DEV)
        self.goal = None if g is None else g.to(DEV)
        self.out = torch.empty(max(B, 1), d, device=DEV)
        self.params = smt.smt_params(self.m, D)
        n = int(self.ops.lib.ssb_smt_scratch_bytes(B, M, C.byref(self.params)))
        self.scratch = torch.empty(max(n, 16) + 64, dtype=torch.uint8, device=DEV)

    def ptrs(self):
        def p(t):
            return None if t is None or t.numel() == 0 else t.data_ptr()
        return dict(x=p(self.x), memory=p(self.memory), masks=p(self.masks), goal=p(self.goal),
                    scratch=p(self.scratch), out=p(self.out))

    def call(self, B=None, M=None, params=None, **ptrs):
        a = self.ptrs()
        a.update(ptrs)
        ops = self.ops
        return ops.lib.ssb_smt_state_encoder_batch(
            ops.ctx.handle, self.B if B is None else B, self.M if M is None else M, a["x"], a["memory"], a["masks"],
            a["goal"], C.byref(self.params if params is None else params), a["scratch"], a["out"], ops._stream())

    def params_with(self, **fields):
        from soundspaces_b200 import _lib
        q = _lib.SmtParams.from_buffer_copy(self.params)
        for k, v in fields.items():
            setattr(q, k, v)
        return q

    def refused(self, code, fragment, **kw):
        """The call returns ``code``, its message holds ``fragment`` and nothing is launched.  A refusal with another
        message goes first, so the message checked is this call's."""
        ops = self.ops
        assert self.call(B=-7) == SSB_E_INVALID_ARG
        assert "B=-7" in ops.lib.ssb_last_error(ops.ctx.handle).decode()
        before = ops.ctx.launch_count
        rc = self.call(**kw)
        msg = ops.lib.ssb_last_error(ops.ctx.handle).decode()
        assert rc == code and fragment in msg, (kw, rc, msg)
        assert ops.ctx.launch_count == before

    def runs(self, **kw):
        ops = self.ops
        before = ops.ctx.launch_count
        rc = self.call(**kw)
        assert rc == 0, ops.lib.ssb_last_error(ops.ctx.handle).decode()
        assert ops.ctx.launch_count - before == LAUNCHES
        torch.cuda.synchronize()
        assert torch.isfinite(self.out[:self.B if kw.get("B") is None else kw["B"]]).all()


def test_entry_refuses_bad_pointers():
    e = Entry(make_smt(D=40, pose_index=36, d_model=64, nhead=4, seed=120), 3, 5, 40)
    args = "bad arguments (B=3 M=5)"
    p = e.ptrs()
    for name in ("x", "out", "scratch", "memory", "masks"):
        e.refused(SSB_E_INVALID_ARG, args, **{name: None})
        e.refused(SSB_E_INVALID_ARG, args, **{name: p[name] + 2})
    e.refused(SSB_E_INVALID_ARG, args, goal=p["goal"] + 2)
    e.refused(SSB_E_INVALID_ARG, args, scratch=p["scratch"] + 4)            # 4-byte but not 16-byte aligned
    e.refused(SSB_E_INVALID_ARG, args, scratch=p["scratch"] + 8)
    e.refused(SSB_E_INVALID_ARG, "bad arguments (B=3 M=-1)", M=-1)
    e.runs(scratch=p["scratch"] + 16)
    e.runs(goal=None)                                                        # NULL goal: no goal
    e.runs()


def test_entry_refuses_bad_parameters():
    e = Entry(make_smt(D=40, pose_index=36, d_model=64, nhead=4, seed=121), 3, 5, 40)
    e.refused(SSB_E_INVALID_ARG, "n_heads=3", params=e.params_with(n_heads=3))             # 64 % 3 != 0
    e.refused(SSB_E_INVALID_ARG, "n_heads=0", params=e.params_with(n_heads=0))
    e.refused(SSB_E_INVALID_ARG, "pretraining=2", params=e.params_with(pretraining=2))
    e.refused(SSB_E_INVALID_ARG, "pose_index=-2", params=e.params_with(pose_index=-2))
    e.refused(SSB_E_INVALID_ARG, "d_in=0", params=e.params_with(d_in=0))
    from soundspaces_b200 import _lib
    for i, name in enumerate(("fuse1", "fuse2", "enc_qkv", "enc_out", "enc_ff1", "enc_ff2", "dec_sa_qkv",
                              "dec_sa_out", "dec_ca_qkv", "dec_ca_out", "dec_ff1", "dec_ff2", "pose")):
        e.refused(SSB_E_INVALID_ARG, f"linear parameter {i}", params=e.params_with(**{name: _lib.Linear()}))
    for i, name in enumerate(("enc_norm1", "enc_norm2", "enc_norm", "dec_norm1", "dec_norm2", "dec_norm3", "dec_norm")):
        for eps in (0.0, -1e-5, float("nan")):
            ln = getattr(e.params, name)
            bad = _lib.LayerNorm(ln.d_gamma, ln.d_beta, eps, 0)
            e.refused(SSB_E_INVALID_ARG, f"bad LayerNorm {i} (eps=", params=e.params_with(**{name: bad}))
    e.runs()


def test_entry_limits():
    """One past each limit is refused with SSB_E_SHAPE before any launch; the limit itself runs."""
    def nopose(D, d=64, h=4, seed=0):
        return make_smt(D=D, pose_index=None, d_model=d, nhead=h, seed=seed)

    small = make_smt(D=40, pose_index=36, d_model=64, nhead=4, seed=130)
    # B: memory and masks NULL with M = 0
    Entry(small, 1025, 0, 40).refused(SSB_E_SHAPE, "B=1025 M=0")
    Entry(small, 1024, 0, 40).runs()
    # M + 1
    Entry(small, 1, 1024, 40).refused(SSB_E_SHAPE, "B=1 M=1024")
    Entry(small, 1, 1023, 40).runs()
    # d_model and head dim
    Entry(make_smt(D=40, pose_index=36, d_model=513, nhead=27, seed=131), 2, 3, 40).refused(SSB_E_SHAPE, "d_model=513")
    Entry(make_smt(D=40, pose_index=36, d_model=512, nhead=4, seed=132), 2, 3, 40).runs()
    Entry(make_smt(D=40, pose_index=36, d_model=258, nhead=2, seed=133), 2, 3, 40).refused(SSB_E_SHAPE, "head dim=129")
    Entry(make_smt(D=40, pose_index=36, d_model=128, nhead=1, seed=134), 2, 3, 40).runs()
    # D
    Entry(nopose(1025, seed=135), 2, 3, 1025).refused(SSB_E_SHAPE, "d_in=1025")
    Entry(nopose(1024, seed=136), 2, 3, 1024).runs()
    # pose index + 4 <= D
    Entry(make_smt(D=40, pose_index=37, d_model=64, nhead=4, seed=137), 2, 3, 40).refused(SSB_E_SHAPE, "pose_index=37")
    Entry(make_smt(D=40, pose_index=36, d_model=64, nhead=4, seed=138), 2, 3, 40).runs()
    # without pose encoding D = 1 and 2 run (pose index -1 has no D limit)
    for D in (1, 2):
        Entry(nopose(D, seed=139 + D), 3, 4, D).runs()


def test_width_mismatch_is_refused_before_any_launch():
    """Without pose encoding x must be as wide as fusion_encoder[0]'s input: ValueError, nothing launched."""
    ops = _ops()
    mc = _cuda(make_smt(D=64, pose_index=None, d_model=64, nhead=4, seed=150))
    for D in (40, 100):
        x, memory, masks, goal = (t.to(DEV) for t in make_inputs(3, 5, D=D, d_model=64, pose_index=None, seed=D))
        before = ops.ctx.launch_count
        with pytest.raises(ValueError, match="fusion_encoder"):
            ops.smt_state_encoder(mc, x, memory, masks, goal)
        assert ops.ctx.launch_count == before
