"""SAVi's scene memory transformer trained in the PPO update through the library (ssb_smt_state_encoder_train_*,
SmtFunction and ``patch_smt_state_encoder(..., training=True)``): forward bits against the rollout entry, gradients
against float64, determinism, silent rows, masked NaN, launch counts, host syncs, a PPO round on the patched rollout
storage (also under DDP), and refused and fallback calls."""
import copy
import ctypes
import os

import numpy as np
import pytest

from smt_models import episode_masks, make_inputs, make_smt
from smt_train_models import CASES, case_inputs, case_module, SMTStandIn

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

FWD, BWD = 6, 10
GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "smt_train_golden.npz")


@pytest.fixture(scope="module")
def ops():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    from soundspaces_b200.renderer import WaveformOps
    return WaveformOps.get("cuda:0")


def _cuda(*ts):
    return [None if t is None else t.cuda() for t in ts]


def _savi(N, M, seed=0, goal=True, steps=None):
    """SAVi's shape: D 276, pose index 272, d_model 256, 8 heads; episode masks."""
    m = make_smt(seed=seed).cuda()
    x, memory, _, g = make_inputs(N, M, seed=seed, goal=goal)
    masks = episode_masks(N, M, steps or M, 40, torch.Generator().manual_seed(seed))
    return m, _cuda(x, memory, masks, g)


def _fused(m, x, memory, masks, goal):
    from soundspaces_b200.smt import SmtFunction, smt_train_parameters
    return SmtFunction.apply(True, m, x, memory, masks, goal, *smt_train_parameters(m))


def _fused_grads(m, x, memory, masks, goal, g):
    from soundspaces_b200.smt import smt_train_parameters
    x = x.clone().requires_grad_(True)
    goal = goal.clone().requires_grad_(True) if goal is not None else None
    ps = smt_train_parameters(m)
    out = _fused(m, x, memory, masks, goal)
    ins = ps + [x] + ([goal] if goal is not None else [])
    return out, torch.autograd.grad((out * g).sum(), ins)


def _ref_grads(m, x, memory, masks, goal, g):
    from soundspaces_b200.smt import smt_train_parameters
    m64 = copy.deepcopy(m).double()
    m64.__class__ = SMTStandIn
    x = x.double().requires_grad_(True)
    goal = goal.double().requires_grad_(True) if goal is not None else None
    out = m64.single_forward(x, memory.double(), masks.double(), goal)
    ins = smt_train_parameters(m64) + [x] + ([goal] if goal is not None else [])
    return out, torch.autograd.grad((out * g.double()).sum(), ins)


def _rel(a, b):
    return (a.double() - b.double()).abs().max().item() / max(b.abs().max().item(), 1e-30)


@pytest.mark.parametrize("B,M", [(1, 150), (16, 150), (600, 300), (1024, 150)])
def test_forward_bits_match_rollout(ops, B, M):
    m, (x, memory, masks, goal) = _savi(B, M, seed=B)
    for gl in (goal, None):
        want = ops.smt_state_encoder(m, x, memory, masks, gl)
        got, _ = ops.smt_train_forward(m, x, memory, masks, gl)
        assert torch.equal(got, want)


def test_forward_bits_above_the_rollout_limit(ops):
    B = 1100
    m, (x, memory, masks, goal) = _savi(B, 60, seed=5)
    got, _ = ops.smt_train_forward(m, x, memory, masks, goal)
    want = torch.cat([ops.smt_state_encoder(m, x[i:i + 1024], memory[:, i:i + 1024].contiguous(),
                                            masks[i:i + 1024], goal[i:i + 1024]) for i in (0, 1024)])
    assert torch.equal(got, want)


@pytest.mark.parametrize("name", sorted(CASES))
def test_gradients_match_float64_golden_cases(ops, name):
    z = np.load(GOLDEN)
    m = case_module(SMTStandIn, name, torch.float32).cuda()
    x, memory, masks, goal, g = _cuda(*case_inputs(name))
    out, grads = _fused_grads(m, x, memory, masks, goal, g)
    assert _rel(out.cpu(), torch.from_numpy(z[f"{name}/out"])) <= 1e-4
    n = len(grads) - (2 if goal is not None else 1)
    for j in range(n):
        ref = torch.from_numpy(z[f"{name}/g{j}"])
        assert _rel(grads[j].cpu(), ref) <= 1e-4 or ref.abs().max() == 0 and grads[j].abs().max() == 0, j
    assert _rel(grads[n].cpu(), torch.from_numpy(z[f"{name}/dx"])) <= 1e-4
    if goal is not None:
        assert _rel(grads[n + 1].cpu(), torch.from_numpy(z[f"{name}/dgoal"])) <= 1e-4
    if name == "current_only":
        assert (grads[n][:, 16:19] == 0).all()


def test_gradients_match_float64_at_savi_shape(ops):
    """600 rows, 300 slots, episode masks: the decoder's gradients and dgoal within 1e-4 of float64 (relative to the
    tensor's maximum); the encoder's other gradients and dx within 1e-3, and its linear1's within 1e-2.  Of the ~6.7M
    ReLU inputs of the encoder FF on valid tokens at this shape, a few lie within FP32 rounding of 0; where the
    library's forward (k-ascending FMA chains) rounds one to the other side of 0 than float64, that (token, unit) moves
    linear1's weight and bias gradient by its whole term: 1.5e-4 and 5.6e-3 of the maximum at this seed with and
    without a goal (measured on an H100), and the encoder's other gradients, through that token, by up to 3e-5."""
    from soundspaces_b200.smt import smt_train_parameters
    m, (x, memory, masks, goal) = _savi(600, 300, seed=7, steps=600)
    g = torch.randn(600, 256, generator=torch.Generator().manual_seed(7)).cuda()
    n_enc = 20                        # pose_encoder .. encoder.norm in smt_train_parameters order
    n_par = len(smt_train_parameters(m))
    for gl in (goal, None):
        out, grads = _fused_grads(m, x, memory, masks, gl, g)
        r_out, ref = _ref_grads(m, x, memory, masks, gl, g)
        assert _rel(out, r_out) <= 1e-4
        errs = [_rel(a, r) if r.abs().max() > 0 else a.abs().max().item() for a, r in zip(grads, ref)]
        bounds = [1e-2 if j in (10, 11) else 1e-3 if j < n_enc or j == n_par else 1e-4 for j in range(len(errs))]
        bad = [f"{j}: {e:.3g} > {b:.3g}" for j, (e, b) in enumerate(zip(errs, bounds)) if e > b]
        assert not bad, bad


def test_deterministic_silent_rows_and_masked_nan(ops):
    m, (x, memory, masks, goal) = _savi(64, 80, seed=9)
    g = torch.randn(64, 256, generator=torch.Generator().manual_seed(9)).cuda()
    g[::3] = 0
    o1, g1 = _fused_grads(m, x, memory, masks, goal, g)
    o2, g2 = _fused_grads(m, x, memory, masks, goal, g)
    assert torch.equal(o1, o2) and all(torch.equal(a, b) for a, b in zip(g1, g2))
    # rows with zero upstream gradient add nothing, whatever their inputs hold
    x2, mem2 = x.clone(), memory.clone()
    x2[::3] = torch.randn_like(x2[::3])
    mem2[:, ::3] = torch.randn_like(mem2[:, ::3])
    _, g3 = _fused_grads(m, x2, mem2, masks, goal, g)
    for j, (a, b) in enumerate(zip(g1[:-2], g3[:-2])):
        assert torch.equal(a, b), j
    # a NaN in a masked memory slot changes no output and no gradient bit
    mem3 = memory.clone()
    mem3[masks.t() == 0] = float("nan")
    o4, g4 = _fused_grads(m, x, mem3, masks, goal, g)
    assert torch.equal(o1, o4) and all(torch.equal(a, b) for a, b in zip(g1, g4))


@pytest.mark.parametrize("B,M,pre", [(3, 9, False), (40, 200, False), (130, 17, True)])
def test_launch_counts(ops, B, M, pre):
    m, (x, memory, masks, goal) = _savi(B, M, seed=B)
    m._pretraining = pre
    g = torch.randn(B, 256, device="cuda")
    n0 = ops.ctx.launch_count
    out, ws = ops.smt_train_forward(m, x, memory, masks, goal)
    n1 = ops.ctx.launch_count
    ops.smt_train_backward(m, x, memory, masks, goal, ws, g)
    n2 = ops.ctx.launch_count
    assert (n1 - n0, n2 - n1) == (FWD, BWD)


def test_no_host_sync_in_the_patched_step(ops):
    from soundspaces_b200.smt import patch_smt_state_encoder
    P = patch_smt_state_encoder(type("PatchedSMT", (SMTStandIn,), {}), training=True)
    m = P(276, 8, 256, 0.0, 272, False).cuda()
    _, (x, memory, masks, goal) = _savi(32, 50, seed=3)
    g = torch.randn(32, 256, device="cuda")
    torch.cuda.synchronize()
    n0 = ops.ctx.launch_count
    torch.cuda.set_sync_debug_mode("error")
    try:
        (m.single_forward(x, memory, masks, goal) * g).sum().backward()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert ops.ctx.launch_count - n0 == FWD + BWD
    assert all(p.grad is not None for p in m.parameters())


def _rollout_minibatch(T=150, N=4, M=150):
    """The one recurrent_generator minibatch (T x N = 600 rows) of SAVi's rollout storage under
    patch_rollout_storage, with an external memory of M + T slots holding M per env (SAVi's memory_size and
    num_steps) of pose trajectories -> (memory (M + T, 600, 276), masks (600, M + T))."""
    import rollout_models as rm
    from soundspaces_b200 import rollout as ro
    storage_cls = ro.patch_rollout_storage(type("PatchedSavi", (rm.SaviRolloutStorage,), {}))
    st = storage_cls(T, N, rm.spaces({"depth": (2, 2, 1)}), rm.ActionSpace(), 16, True, M + T, M, 276, 1)
    st.to("cuda")
    dev = torch.device("cuda")
    gen = torch.Generator().manual_seed(41)
    pos = torch.zeros(N, 4)
    for t in range(T):
        done = (torch.rand(N, generator=gen) < 0.02).float()
        pos = pos * (1 - done[:, None])
        pos[:, :2] += torch.randn(N, 2, generator=gen) * 0.5
        pos[:, 2] += torch.randn(N, generator=gen) * 0.4
        pos[:, 3] += 1.0
        feat = torch.randn(N, 276, generator=gen)
        feat[:, 272:] = pos
        st.insert({"depth": torch.zeros(N, 2, 2, 1, device=dev)}, torch.zeros((1, N, 16), device=dev),
                  torch.zeros((N, 1), dtype=torch.long, device=dev), torch.zeros((N, 1), device=dev),
                  torch.zeros((N, 1), device=dev), torch.zeros((N, 1), device=dev),
                  (1 - done)[:, None].to(dev), feat.to(dev))
    st.compute_returns(torch.zeros(N, 1, device=dev), True, 0.99, 0.95)
    batch = next(iter(st.recurrent_generator(torch.zeros_like(st.returns[:-1]), 1)))
    return batch[-2].contiguous(), batch[-1].contiguous()


def test_ppo_round_matches_eager_fp32_and_float64(ops):
    """Three Adam steps of the patched SMT on a 600-row rollout minibatch: after the steps, the fused parameters
    are within 1e-4 of float64's (relative to each tensor's maximum) or within twice eager FP32's distance."""
    from soundspaces_b200.smt import patch_smt_state_encoder
    memory, masks = _rollout_minibatch()
    B = masks.shape[0]
    assert B == 600 and memory.shape == (300, 600, 276)
    gen = torch.Generator().manual_seed(31)
    x = torch.randn(B, 276, generator=gen).cuda()
    x[:, 272:] = memory[-1, :, 272:]
    goal = torch.randn(B, 256, generator=gen).cuda()
    g = torch.randn(B, 256, generator=gen).cuda()
    P = patch_smt_state_encoder(type("PatchedSMT", (SMTStandIn,), {}), training=True)
    fused = make_smt(seed=31)
    fused.__class__ = P
    fused = fused.cuda()
    eager = copy.deepcopy(fused)
    eager.__class__ = SMTStandIn
    ref = copy.deepcopy(eager).double()
    opts = [torch.optim.Adam(m.parameters(), lr=1e-3) for m in (fused, eager, ref)]
    prev = torch.backends.cuda.matmul.allow_tf32
    try:
        for _ in range(3):
            for o in opts:
                o.zero_grad()
            n0 = ops.ctx.launch_count
            (fused.single_forward(x, memory, masks, goal) * g).sum().backward()
            assert ops.ctx.launch_count - n0 == FWD + BWD
            torch.backends.cuda.matmul.allow_tf32 = False
            (eager.single_forward(x, memory, masks, goal) * g).sum().backward()
            (ref.single_forward(x.double(), memory.double(), masks.double(), goal.double()) * g.double()).sum().backward()
            for o in opts:
                o.step()
    finally:
        torch.backends.cuda.matmul.allow_tf32 = prev
    pf, pe, pr = (list(m.parameters()) for m in (fused, eager, ref))
    bound = max(1e-4, 2 * max(_rel(e, r) for e, r in zip(pe, pr)))
    for i, (a, r) in enumerate(zip(pf, pr)):
        assert _rel(a, r) <= bound, f"parameter {i}: {_rel(a, r):.3g}, bound {bound:.3g}"


def test_ddp_world_size_one(ops, tmp_path):
    import torch.distributed as dist
    from soundspaces_b200.smt import patch_smt_state_encoder
    P = patch_smt_state_encoder(type("PatchedSMT", (SMTStandIn,), {}), training=True)
    dist.init_process_group("gloo", init_method=f"file://{tmp_path / 'store'}", rank=0, world_size=1)
    try:
        _, (x, memory, masks, goal) = _savi(32, 40, seed=12)
        g = torch.randn(32, 256, generator=torch.Generator().manual_seed(12)).cuda()
        m = make_smt(seed=12)
        m.__class__ = P
        m = m.cuda()
        ref = copy.deepcopy(m)
        ddp = torch.nn.parallel.DistributedDataParallel(m, device_ids=[0], output_device=0,
                                                        find_unused_parameters=True)
        (ddp(x, memory, masks, goal) * g).sum().backward()
        (ref(x, memory, masks, goal) * g).sum().backward()
        for (name, a), b in zip(m.named_parameters(), ref.parameters()):
            assert a.grad is not None, name
            assert torch.equal(a.grad, b.grad), name
    finally:
        dist.destroy_process_group()


def test_refusals_launch_nothing(ops):
    from soundspaces_b200.smt import smt_params
    m, (x, memory, masks, goal) = _savi(4, 10, seed=2)
    p = smt_params(m, 276)
    ws = torch.empty(int(ops.lib.ssb_smt_train_workspace_bytes(4, 10, ctypes.byref(p))), dtype=torch.uint8,
                     device="cuda")
    out = torch.empty(4, 256, device="cuda")
    h = ops.ctx.handle
    P = ctypes.byref(p)
    fwd = ops.lib.ssb_smt_state_encoder_train_forward_batch
    bwd = ops.lib.ssb_smt_state_encoder_train_backward_batch
    grads = [torch.empty_like(t) for t in __import__("soundspaces_b200.smt", fromlist=["x"]).smt_train_parameters(m)]
    table = (ctypes.c_void_p * len(grads))(*[t.data_ptr() for t in grads])
    assert ops.lib.ssb_smt_train_workspace_bytes(65536, 10, P) == -1
    assert ops.lib.ssb_smt_train_workspace_bytes(4, 1024, P) == -1
    cases = [
        lambda: fwd(h, 65536, 10, x.data_ptr(), memory.data_ptr(), masks.data_ptr(), None, P, ws.data_ptr(),
                    out.data_ptr(), None),
        lambda: fwd(h, 4, 1024, x.data_ptr(), memory.data_ptr(), masks.data_ptr(), None, P, ws.data_ptr(),
                    out.data_ptr(), None),
        lambda: fwd(h, 4, 10, x.data_ptr(), memory.data_ptr(), masks.data_ptr(), None, P, None, out.data_ptr(), None),
        lambda: fwd(h, 4, 10, x.data_ptr(), memory.data_ptr(), masks.data_ptr(), None, P, ws.data_ptr() + 4,
                    out.data_ptr(), None),
        lambda: bwd(h, 4, 10, x.data_ptr(), memory.data_ptr(), masks.data_ptr(), None, P, out.data_ptr(), 255,
                    ws.data_ptr(), table, None, None, None),
        lambda: bwd(h, 4, 10, x.data_ptr(), memory.data_ptr(), masks.data_ptr(), None, P, out.data_ptr(), 256,
                    ws.data_ptr(), None, None, None, None),
        lambda: bwd(h, 4, 10, x.data_ptr(), memory.data_ptr(), masks.data_ptr(), None, P, out.data_ptr(), 256,
                    ws.data_ptr(), table, None, out.data_ptr(), None),
    ]
    for i, c in enumerate(cases):
        n0 = ops.ctx.launch_count
        assert c() != 0 and ops.ctx.launch_count == n0, i
    n0 = ops.ctx.launch_count
    assert fwd(h, 4, 10, x.data_ptr(), memory.data_ptr(), masks.data_ptr(), None, P, ws.data_ptr(), out.data_ptr(),
               None) == 0
    assert bwd(h, 4, 10, x.data_ptr(), memory.data_ptr(), masks.data_ptr(), None, P, out.data_ptr(), 256,
               ws.data_ptr(), table, None, None, None) == 0
    assert ops.ctx.launch_count - n0 == FWD + BWD


def test_fallback_reasons_run_the_original(ops):
    from soundspaces_b200.smt import patch_smt_state_encoder, smt_train_error
    P = patch_smt_state_encoder(type("PatchedSMT", (SMTStandIn,), {}), training=True)
    m = make_smt(seed=4)
    m.__class__ = P
    m = m.cuda()
    _, (x, memory, masks, goal) = _savi(8, 20, seed=4)
    refused = {
        "not a contiguous float32": (x.t().contiguous().t(), memory, masks, goal),
        "memory or masks require grad": (x, memory.clone().requires_grad_(True), masks, goal),
        "M + 1 = 1025": (x, torch.zeros(1024, 8, 276, device="cuda"), torch.zeros(8, 1024, device="cuda"), goal),
    }
    for why, args in refused.items():
        assert why in smt_train_error(m, *args), why
        n0 = ops.ctx.launch_count
        out = m.single_forward(*args)
        assert ops.ctx.launch_count == n0 and out.grad_fn is not None, why
    assert "disagree" in smt_train_error(m, x, memory, masks[:, :5].contiguous(), goal)
    assert smt_train_error(m, x.cpu(), memory, masks, goal) == "x is not a CUDA tensor"
    big = torch.zeros(65536, 276, device="cuda")
    assert "65536 rows" in smt_train_error(m, big, torch.zeros(0, 65536, 276, device="cuda"),
                                           torch.zeros(65536, 0, device="cuda"), None)
    with torch.autocast("cuda"):
        assert smt_train_error(m, x, memory, masks, goal) == "autocast is on"
    m64 = copy.deepcopy(m).double()
    assert "parameters" in smt_train_error(m64, x, memory, masks, goal)
    n0 = ops.ctx.launch_count
    assert m.single_forward(x, memory, masks, goal).grad_fn is not None and ops.ctx.launch_count - n0 == FWD
