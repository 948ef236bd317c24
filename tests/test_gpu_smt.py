"""SAVi's scene memory transformer on the GPU (``ssb_smt_state_encoder_batch``): accuracy per env against a float64
forward of the stand-in at SAVi's shapes and across the entry's limits, bit-identity across batch sizes, positions and
masked-slot contents, the golden reference cases, a fixed launch count, and the patched ``single_forward`` against the
original when it falls back."""
import copy

import pytest

from smt_models import SMTStandIn, episode_masks, make_inputs, make_smt, ring_masks
from test_smt_host import golden_cases

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

LAUNCHES = 6
DEV = torch.device("cuda", 0)


def _ops():
    from soundspaces_b200.renderer import WaveformOps
    return WaveformOps.get(DEV)


def _cuda(m):
    return copy.deepcopy(m).to(DEV)


def _run(m, x, memory, masks, goal=None):
    with torch.no_grad():
        return _ops().smt_state_encoder(m, x.to(DEV), memory.to(DEV), masks.to(DEV),
                                        None if goal is None else goal.to(DEV))


def _ref64(m, x, memory, masks, goal=None):
    ref = copy.deepcopy(m).cpu().double()
    with torch.no_grad():
        return ref.single_forward(x.double(), memory.double(), masks.double(), None if goal is None else goal.double())


def _check(got, want):
    """max|got_b - ref_b| <= 1e-4 max|ref_b| for every env b."""
    got = got.double().cpu()
    assert torch.isfinite(got).all()
    for b in range(want.shape[0]):
        err = (got[b] - want[b]).abs().max().item()
        scale = want[b].abs().max().item()
        assert err <= 1e-4 * scale, f"env {b}: max|d| {err:.3g} > 1e-4 * {scale:.3g}"


def _case(m, N, M, **kw):
    d = m.transformer.d_model
    D = m.fusion_encoder[0].in_features if not m._use_pose_encoding else kw.pop("D", 276)
    pi = m._pose_indices[0] if m._use_pose_encoding else None
    x, memory, masks, goal = make_inputs(N, M, D=D, d_model=d, pose_index=pi, **kw)
    _check(_run(_cuda(m), x, memory, masks, goal), _ref64(m, x, memory, masks, goal))


@pytest.mark.parametrize("B", [8, 16])
@pytest.mark.parametrize("M,fill", [(300, 150), (150, 75)])
@pytest.mark.parametrize("goal", [True, False])
def test_savi_shapes(B, M, fill, goal):
    """D 276, pose index 272, d 256, 8 heads: training (300 slots, 150 valid in a wrapped ring) and eval (150 slots,
    half valid)."""
    m = make_smt(seed=B + M)
    x, memory, _, g = make_inputs(B, M, seed=M, goal=goal)
    masks = ring_masks(B, M, [fill - (b % 3) for b in range(B)], start=[(37 * b + 11) % M for b in range(B)])
    _check(_run(_cuda(m), x, memory, masks, g), _ref64(m, x, memory, masks, g))


def test_pretraining_episodes_and_non_binary_masks():
    m = make_smt(pretraining=True, seed=3)
    _case(m, 8, 40, seed=1, goal=False)
    m = make_smt(seed=4)
    gen = torch.Generator().manual_seed(5)
    masks = episode_masks(8, 40, 97, 9, gen)
    masks[:, ::7] *= 2.0                      # 2 is valid, 0.5 is padding
    masks[:, 3::11] = 0.5
    _case(m, 8, 40, seed=2, masks=masks)


@pytest.mark.parametrize("d,nhead", [(64, 1), (64, 8), (128, 1), (128, 4), (256, 4), (256, 8), (512, 4), (512, 8)])
def test_widths_and_heads(d, nhead):
    _case(make_smt(D=70, pose_index=60, d_model=d, nhead=nhead, seed=d + nhead), 8, 33, D=70, seed=d)


def test_no_pose_encoding():
    _case(make_smt(D=100, pose_index=None, d_model=128, nhead=8, seed=9), 8, 50, seed=9)
    _case(make_smt(D=100, pose_index=None, d_model=128, nhead=8, seed=9), 8, 50, seed=9, goal=False)


def test_only_current_and_all_valid():
    m = make_smt(seed=11)
    _case(m, 8, 30, seed=11, masks=torch.zeros(8, 30))
    _case(m, 8, 30, seed=12, masks=torch.ones(8, 30))
    _case(m, 4, 0, seed=13)                                            # no memory at all


def test_token_limit():
    _case(make_smt(D=40, pose_index=36, d_model=64, nhead=4, seed=14), 2, 1023, D=40, seed=14,
          masks=torch.ones(2, 1023))


@pytest.mark.parametrize("B", [1, 8, 64, 1024])
def test_batch_sizes(B):
    _case(make_smt(D=40, pose_index=36, d_model=64, nhead=4, seed=15), B, 12, D=40, seed=B)


def test_bit_identity_across_batch_position_and_masked_content():
    m = _cuda(make_smt(seed=21))
    B, M = 16, 300
    x, memory, masks, goal = make_inputs(B, M, seed=21)
    full = _run(m, x, memory, masks, goal)
    for b in (0, 5, 15):
        one = _run(m, x[b:b + 1].contiguous(), memory[:, b:b + 1].contiguous(), masks[b:b + 1].contiguous(), goal[b:b + 1])
        assert torch.equal(one[0], full[b])
    perm = torch.randperm(B, generator=torch.Generator().manual_seed(0))
    shuffled = _run(m, x[perm].contiguous(), memory[:, perm].contiguous(), masks[perm].contiguous(), goal[perm].contiguous())
    assert torch.equal(shuffled, full[perm.to(DEV)])
    half = _run(m, x[:7].contiguous(), memory[:, :7].contiguous(), masks[:7].contiguous(), goal[:7].contiguous())
    assert torch.equal(half, full[:7])
    for fill in (float("nan"), float("inf"), 1e30):
        dirty = memory.clone()
        dirty[(masks == 0).t()] = fill
        assert torch.equal(_run(m, x, dirty, masks, goal), full)


def test_golden_cases_through_the_library():
    for name, (m, x, memory, masks, goal, want) in golden_cases().items():
        f32 = copy.deepcopy(m).float().to(DEV)
        got = _run(f32, x.float(), memory.float(), masks.float(), None if goal is None else goal.float())
        _check(got, want)


def test_launch_count_is_fixed():
    ops = _ops()
    small = dict(D=40, pose_index=36, d_model=64, nhead=4)
    for kw, N, M, masks in (({}, 8, 300, None), ({}, 16, 150, torch.zeros(16, 150)), (small, 1024, 3, torch.ones(1024, 3)),
                            (small, 1, 0, None)):
        m = make_smt(seed=31, **kw)
        x, memory, mk, _ = make_inputs(N, M, D=kw.get("D", 276), d_model=kw.get("d_model", 256),
                                       pose_index=kw.get("pose_index", 272), masks=masks)
        mc = _cuda(m)
        before = ops.ctx.launch_count
        _run(mc, x, memory, mk)
        assert ops.ctx.launch_count - before == LAUNCHES
    x, memory, mk, _ = make_inputs(0, 5)
    before = ops.ctx.launch_count
    assert _run(_cuda(make_smt()), x, memory, mk).shape == (0, 256)
    assert ops.ctx.launch_count == before


class Patched(SMTStandIn):
    pass


def test_patched_forward_paths():
    from soundspaces_b200.smt import patch_smt_state_encoder
    patch_smt_state_encoder(Patched)
    original = Patched.single_forward._ssb_original
    ops = _ops()
    m = make_smt(seed=41)
    m.__class__ = Patched
    m = _cuda(m)
    m.train()                                          # the trainer's rollouts: training mode, dropout 0
    x, memory, masks, goal = (t.to(DEV) for t in make_inputs(8, 300, seed=41))
    before = ops.ctx.launch_count
    with torch.no_grad():
        fused = m.single_forward(x, memory, masks, goal)
    assert ops.ctx.launch_count - before == LAUNCHES
    _check(fused, _ref64(m, x.cpu(), memory.cpu(), masks.cpu(), goal.cpu()))
    # grad enabled (the PPO update): the original, bit for bit
    before = ops.ctx.launch_count
    got = m.single_forward(x, memory, masks, goal)
    want = original(m, x, memory, masks, goal)
    assert ops.ctx.launch_count == before and torch.equal(got, want) and got.requires_grad
    # a refused shape (M + 1 > 1024) falls back to the original
    x2, memory2, masks2, _ = (t.to(DEV) if t is not None else None for t in make_inputs(2, 1024, seed=42, goal=False))
    with torch.no_grad():
        before = ops.ctx.launch_count
        got = m.single_forward(x2, memory2, masks2)
        assert ops.ctx.launch_count == before
        assert torch.equal(got, original(m, x2, memory2, masks2))
    # dropout > 0 in training mode falls back too
    m.transformer.encoder.layers[0].dropout.p = 0.1
    with torch.no_grad():
        before = ops.ctx.launch_count
        m.single_forward(x, memory, masks, goal)
        assert ops.ctx.launch_count == before


def test_live_parameters():
    m = _cuda(make_smt(seed=51))
    x, memory, masks, goal = make_inputs(8, 60, seed=51)
    a = _run(m, x, memory, masks, goal)
    with torch.no_grad():
        m.transformer.decoder.layers[0].linear2.weight.mul_(1.5)
        m.fusion_encoder[0].bias.add_(0.2)
    b = _run(m, x, memory, masks, goal)
    assert not torch.equal(a, b)
    _check(b, _ref64(m, x, memory, masks, goal))
