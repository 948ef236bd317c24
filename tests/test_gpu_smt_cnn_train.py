"""SAVi's visual encoder trained in the PPO update through the library (ssb_smt_cnn_train_*, SmtCnnFunction and
``patch_smt_cnn(..., training=True)``): forward bits against the rollout entry, gradients against float64,
determinism, silent rows, launch counts, host syncs, the frozen second stage, a PPO round on the patched rollout
storage (also under DDP), and refused and fallback calls."""
import copy
import ctypes

import pytest

from smt_cnn_models import SMTCNN, observations, set_params
from smt_cnn_train_models import CASES, PARAM_SEED, case_grad, case_observations

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

FWD = {1: 39, 2: 77}      # 1 + 38 n_inputs
BWD = {1: 80, 2: 160}     # 80 n_inputs, every gradient requested


@pytest.fixture(scope="module")
def ops():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    from soundspaces_b200.renderer import WaveformOps
    return WaveformOps.get("cuda:0")


def _patched():
    from soundspaces_b200.encoder import patch_smt_cnn
    return patch_smt_cnn(type("PatchedSMTCNN", (SMTCNN,), {}), training=True)


def _module(mods=("rgb", "depth"), seed=PARAM_SEED, cls=SMTCNN):
    return set_params(cls({m: 3 if m == "rgb" else 1 for m in mods}), seed).cuda()


def _obs(B, H=128, W=128, seed=0, mods=("rgb", "depth")):
    o = observations(B, H, W, seed, rgb=3 if "rgb" in mods else 0, depth=1 if "depth" in mods else 0)
    return {k: v.cuda() for k, v in o.items()}


def _eps(m):
    from soundspaces_b200.belief_nets import conv_norm_pairs
    return tuple(float(n.eps) for k in ("rgb", "depth") if k in m.input_modalities
                 for _, n in conv_norm_pairs(getattr(m, f"{k}_encoder")))


def _train_fwd(ops, m, obs):
    from soundspaces_b200.encoder import smt_cnn_params
    return ops.smt_cnn_train_forward(obs.get("rgb"), obs.get("depth"), smt_cnn_params(m), _eps(m), True)


def _train_bwd(ops, m, obs, ws, g, need=None):
    from soundspaces_b200.encoder import smt_cnn_params
    return ops.smt_cnn_train_backward(obs.get("rgb"), obs.get("depth"), smt_cnn_params(m), _eps(m), True, ws,
                                      g.contiguous(), need)


def _rollout(ops, m, obs):
    return ops.smt_cnn(obs.get("rgb"), obs.get("depth"), getattr(m, "rgb_encoder", None),
                       getattr(m, "depth_encoder", None), resize=True)


@pytest.mark.parametrize("B", [1, 16, 600, 1024])
def test_forward_bits_match_rollout(ops, B):
    m = _module()
    obs = _obs(B, seed=B)
    with torch.no_grad():
        want = _rollout(ops, m, obs)
    got, _ = _train_fwd(ops, m, obs)
    assert torch.equal(got, want)
    if B == 600:
        perm = torch.randperm(B, generator=torch.Generator().manual_seed(5)).cuda()
        got_p, _ = _train_fwd(ops, m, {k: v[perm].contiguous() for k, v in obs.items()})
        assert torch.equal(got_p, want[perm])


@pytest.mark.parametrize("mods", [("rgb", "depth"), ("rgb",), ("depth",)])
def test_forward_bits_above_the_rollout_limit(ops, mods):
    m = _module(mods)
    obs = _obs(1200, seed=3, mods=mods)
    with torch.no_grad():
        want = torch.cat([_rollout(ops, m, {k: v[:1024] for k, v in obs.items()}),
                          _rollout(ops, m, {k: v[1024:] for k, v in obs.items()})])
    got, _ = _train_fwd(ops, m, obs)
    assert torch.equal(got, want)


def test_frozen_stage_is_the_rollout(ops):
    P = _patched()
    m = _module(cls=P).requires_grad_(False)
    obs = _obs(1200, seed=4)
    with torch.no_grad():
        want = torch.cat([_rollout(ops, m, {k: v[:1024] for k, v in obs.items()}),
                          _rollout(ops, m, {k: v[1024:] for k, v in obs.items()})])
    n0 = ops.ctx.launch_count
    got = m(obs)                         # grad mode, every parameter frozen: 1024 + 176 rows
    assert ops.ctx.launch_count - n0 == 2 * 39
    assert torch.equal(got, want) and not got.requires_grad and got.grad_fn is None


def _rel(a, b):
    return (a.double() - b).abs().max().item() / b.abs().max().item()


def _grads_three_ways(m32, obs, g):
    """(fused, eager FP32 with TF32 off, float64) parameter gradients of sum(out * g) and the outputs."""
    from soundspaces_b200.encoder import SmtCnnFunction, smt_cnn_params
    ps = smt_cnn_params(m32)
    out = SmtCnnFunction.apply(True, _eps(m32), True, obs.get("rgb"), obs.get("depth"), *ps)
    fused = torch.autograd.grad((out * g).sum(), [p for p in ps if p is not None])
    prev = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    try:
        e_out = m32(obs)
        eager = torch.autograd.grad((e_out * g).sum(), [p for p in ps if p is not None])
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = prev
    m64 = copy.deepcopy(m32).double()
    ps64 = [p for p in smt_cnn_params(m64) if p is not None]
    r_out = m64({k: v.double() for k, v in obs.items()})
    ref = torch.autograd.grad((r_out * g.double()).sum(), ps64)
    return fused, eager, ref, out, r_out


def _check_grads(fused, eager, ref):
    bound = max(1e-4, 2 * max(_rel(e, r) for e, r in zip(eager, ref)))
    for i, (a, r) in enumerate(zip(fused, ref)):
        assert _rel(a, r) <= bound, f"gradient {i}: {_rel(a, r):.3g}, bound {bound:.3g}"


@pytest.mark.parametrize("name", sorted(CASES))
def test_gradients_match_float64_golden_cases(ops, name):
    B, H, W, mods, _ = CASES[name]
    m = set_params(SMTCNN({k: 3 if k == "rgb" else 1 for k in mods}), PARAM_SEED).cuda()
    obs = {k: v.cuda() for k, v in case_observations(name).items()}
    g = case_grad(name, 64 * len(mods)).float().cuda()
    fused, eager, ref, out, r_out = _grads_three_ways(m, obs, g)
    assert _rel(out, r_out) <= 1e-4
    _check_grads(fused, eager, ref)


def test_gradients_match_float64_at_600_rows(ops):
    m = _module()
    obs = _obs(600, seed=6)
    g = torch.randn((600, 128), generator=torch.Generator().manual_seed(6)).cuda()
    fused, eager, ref, _, _ = _grads_three_ways(m, obs, g)
    _check_grads(fused, eager, ref)


def test_deterministic_and_silent_rows_cost_no_bits(ops):
    m = _module()
    B = 96
    obs = _obs(B, seed=7)
    g = torch.randn((B, 128), generator=torch.Generator().manual_seed(7)).cuda()
    silent = torch.arange(B, device="cuda") % 3 == 1
    g[silent] = 0.0
    g[torch.arange(B, device="cuda") % 5 == 2, 64:] = 0.0     # the depth network alone drops these
    out, ws = _train_fwd(ops, m, obs)
    a = _train_bwd(ops, m, obs, ws, g)
    out2, ws2 = _train_fwd(ops, m, obs)
    b = _train_bwd(ops, m, obs, ws2, g)
    assert torch.equal(out, out2) and all(torch.equal(x, y) for x, y in zip(a, b))
    keep = ~silent
    obs_k = {k: v[keep].contiguous() for k, v in obs.items()}
    _, ws3 = _train_fwd(ops, m, obs_k)
    c = _train_bwd(ops, m, obs_k, ws3, g[keep])
    assert all(torch.equal(x, y) for x, y in zip(a, c))


@pytest.mark.parametrize("mods", [("rgb", "depth"), ("depth",)])
def test_launch_counts(ops, mods):
    m = _module(mods)
    n = len(mods)
    for B in (1, 600, 1200):
        obs = _obs(B, seed=8, mods=mods)
        g = torch.randn((B, 64 * n), generator=torch.Generator().manual_seed(B)).cuda()
        g[: B // 2] = 0.0
        n0 = ops.ctx.launch_count
        _, ws = _train_fwd(ops, m, obs)
        n1 = ops.ctx.launch_count
        _train_bwd(ops, m, obs, ws, g)
        n2 = ops.ctx.launch_count
        assert (n1 - n0, n2 - n1) == (FWD[n], BWD[n]), B
        del ws


def test_no_host_sync_in_the_patched_step(ops):
    P = _patched()
    m = _module(cls=P)
    obs = _obs(64, seed=9)
    m(obs).sum().backward()                        # warm up the allocator
    m.zero_grad()
    n0 = ops.ctx.launch_count
    torch.cuda.set_sync_debug_mode("error")
    try:
        out = m(obs)
        (out * out).sum().backward()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert ops.ctx.launch_count - n0 == FWD[2] + BWD[2]
    assert all(p.grad is not None for p in m.parameters())


def _rollout_minibatch(T=150, N=4):
    """The one recurrent_generator minibatch (T x N = 600 rows) of SAVi's rollout storage under
    patch_rollout_storage, holding 128 x 128 RGB-D observations."""
    import numpy as np
    import rollout_models as rm
    from soundspaces_b200 import rollout as ro
    storage_cls = ro.patch_rollout_storage(type("PatchedSavi", (rm.SaviRolloutStorage,), {}))
    st = storage_cls(T, N, rm.spaces({"rgb": (128, 128, 3), "depth": (128, 128, 1)}), rm.ActionSpace(), 16, False, 1,
                     1, 1)
    st.to("cuda")
    dev = torch.device("cuda")
    for t in range(T):
        o = _obs(N, seed=1000 + t)
        st.insert(o, torch.zeros((1, N, 16), device=dev), torch.zeros((N, 1), dtype=torch.long, device=dev),
                  torch.zeros((N, 1), device=dev), torch.zeros((N, 1), device=dev), torch.zeros((N, 1), device=dev),
                  torch.ones((N, 1), device=dev), None)
    st.compute_returns(torch.zeros(N, 1, device=dev), True, 0.99, 0.95)
    batch = next(iter(st.recurrent_generator(torch.zeros_like(st.returns[:-1]), 1)))
    return batch[0]


def test_ppo_round_matches_eager_fp32_and_float64(ops):
    """Three Adam steps of the patched SMTCNN on a 600-row rollout minibatch: at every step, on the same parameters,
    the fused gradients are within the float64 bound of the gradient tests; after the steps, the fused parameters
    are within 1e-4 of float64's (relative to each tensor's maximum) or within eager FP32's distance from float64."""
    obs = _rollout_minibatch()
    B = obs["rgb"].shape[0]
    assert B == 600
    P = _patched()
    fused = _module(cls=P, seed=31)
    eager = _module(seed=31)
    ref = copy.deepcopy(eager).double()
    g = torch.randn((B, 128), generator=torch.Generator().manual_seed(31)).cuda()
    opts = [torch.optim.Adam(x.parameters(), lr=1e-3) for x in (fused, eager, ref)]
    prev = torch.backends.cudnn.allow_tf32
    try:
        for _ in range(3):
            for o in opts:
                o.zero_grad()
            (fused(obs) * g).sum().backward()
            torch.backends.cudnn.allow_tf32 = False
            (eager(obs) * g).sum().backward()
            torch.backends.cudnn.allow_tf32 = prev
            (ref({k: v.double() for k, v in obs.items()}) * g.double()).sum().backward()
            for o in opts:
                o.step()
    finally:
        torch.backends.cudnn.allow_tf32 = prev
    pf, pe, pr = (list(x.parameters()) for x in (fused, eager, ref))
    bound = max(1e-4, 2 * max(_rel(e, r) for e, r in zip(pe, pr)))
    for i, (a, r) in enumerate(zip(pf, pr)):
        assert _rel(a, r) <= bound, f"parameter {i}: {_rel(a, r):.3g}, bound {bound:.3g}"


def test_ddp_world_size_one(ops, tmp_path):
    import torch.distributed as dist
    P = _patched()
    dist.init_process_group("gloo", init_method=f"file://{tmp_path / 'store'}", rank=0, world_size=1)
    try:
        obs = _obs(32, seed=12)
        g = torch.randn((32, 128), generator=torch.Generator().manual_seed(12)).cuda()
        m = _module(cls=P, seed=12)
        ref = _module(cls=P, seed=12)
        ddp = torch.nn.parallel.DistributedDataParallel(m, device_ids=[0], output_device=0,
                                                        find_unused_parameters=True)
        (ddp(obs) * g).sum().backward()
        (ref(obs) * g).sum().backward()
        for (name, a), b in zip(m.named_parameters(), ref.parameters()):
            assert a.grad is not None, name
            assert torch.equal(a.grad, b.grad), name
    finally:
        dist.destroy_process_group()


def _table(ops, m, obs):
    from soundspaces_b200.encoder import smt_cnn_params
    return ops._smt_cnn_train_table(obs.get("rgb"), obs.get("depth"), smt_cnn_params(m), _eps(m), True)


def test_refusals_launch_nothing(ops):
    from soundspaces_b200 import _lib
    lib = ops.lib
    m = _module()
    obs = _obs(4, seed=13)
    B, table, n, ld = _table(ops, m, obs)
    nbytes = lib.ssb_smt_cnn_train_workspace_bytes(B, n, table)
    assert nbytes > 0 and lib.ssb_smt_cnn_train_workspace_bytes(65536, n, table) == -1
    assert lib.ssb_smt_cnn_train_workspace_bytes(65535, n, table) > 0
    ws = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    out = torch.empty((B, ld), device="cuda")
    h = ops.ctx.handle

    def bad_table(**kw):
        t = (_lib.SmtCnnInput * 2)()
        ctypes.memmove(t, table, ctypes.sizeof(t))
        for k, v in kw.items():
            setattr(t[0], k, v)
        return t

    fwd_cases = [
        (B, n, table, None, ws.data_ptr()),                        # NULL output
        (B, n, table, out.data_ptr(), None),                       # NULL workspace
        (B, n, table, out.data_ptr(), ws.data_ptr() + 4),          # misaligned workspace
        (B, n, table, ws.data_ptr(), ws.data_ptr()),               # output inside the workspace
        (B, n, table, obs["rgb"].data_ptr(), ws.data_ptr()),       # output over an observation
        (B, 3, table, out.data_ptr(), ws.data_ptr()),              # n_inputs outside 1..2
        (B, 0, table, out.data_ptr(), ws.data_ptr()),
        (65536, n, table, out.data_ptr(), ws.data_ptr()),          # B past 65535
        (B, n, bad_table(crop_y=70), out.data_ptr(), ws.data_ptr()),   # crop outside the resize
        (B, n, bad_table(fc_in=4096), out.data_ptr(), ws.data_ptr()),  # fc_in mismatch
        (B, n, bad_table(d_obs=None), out.data_ptr(), ws.data_ptr()),
    ]
    for args in fwd_cases:
        n0 = ops.ctx.launch_count
        rc = lib.ssb_smt_cnn_train_forward_batch(h, *args, None)
        assert rc != 0 and ops.ctx.launch_count == n0, args
    assert lib.ssb_smt_cnn_train_forward_batch(h, B, n, table, out.data_ptr(), ws.data_ptr(), None) == 0
    from soundspaces_b200.encoder import smt_cnn_params
    grads = [torch.empty_like(p) for p in smt_cnn_params(m)]
    ptrs = lambda gs: (ctypes.c_void_p * 124)(*[x.data_ptr() for x in gs])   # noqa: E731
    dout = torch.randn((B, ld), device="cuda")
    alias = list(grads)
    alias[70] = grads[3]                                            # two networks' gradients overlap
    over_obs = list(grads)
    over_obs[0] = obs["depth"]                                      # a gradient over an observation
    bwd_cases = [
        (dout.data_ptr(), ws.data_ptr(), None),
        (None, ws.data_ptr(), ptrs(grads)),
        (dout.data_ptr(), ws.data_ptr(), ptrs(alias)),
        (dout.data_ptr(), ws.data_ptr(), ptrs(over_obs)),
    ]
    for args in bwd_cases:
        n0 = ops.ctx.launch_count
        rc = lib.ssb_smt_cnn_train_backward_batch(h, B, n, table, *args, None)
        assert rc != 0 and ops.ctx.launch_count == n0, args
    n0 = ops.ctx.launch_count
    assert lib.ssb_smt_cnn_train_backward_batch(h, B, n, table, dout.data_ptr(), ws.data_ptr(), ptrs(grads), None) == 0
    assert ops.ctx.launch_count - n0 == BWD[2]
    torch.cuda.synchronize()


def test_fallback_reasons_run_the_original(ops):
    from soundspaces_b200.encoder import smt_cnn_train_error
    P = _patched()
    m = _module(cls=P)
    obs = _obs(4, seed=14)
    cases = {
        "requires grad": {"rgb": obs["rgb"].clone().requires_grad_(), "depth": obs["depth"]},
        "contiguous": {"rgb": obs["rgb"].transpose(1, 2), "depth": obs["depth"].transpose(1, 2)},
        "CUDA": {"rgb": obs["rgb"].cpu(), "depth": obs["depth"].cpu()},
        "rows": {k: v[:0] for k, v in obs.items()},
    }
    for word, o in cases.items():
        err = smt_cnn_train_error(m, o)
        assert word in err, (word, err)
        if word in ("CUDA", "rows"):
            continue                                    # the module lives on the GPU; the original needs rows
        n0 = ops.ctx.launch_count
        out = m(o)
        assert ops.ctx.launch_count == n0 and out.shape == (o["rgb"].shape[0], 128)
    with torch.autocast("cuda"):
        assert smt_cnn_train_error(m, obs) == "autocast is on"
        n0 = ops.ctx.launch_count
        m(obs)
        assert ops.ctx.launch_count == n0
    sem = _module(cls=P)
    sem.input_modalities = ["rgb", "depth", "semantic"]
    assert "only 'rgb' and / or 'depth'" in smt_cnn_train_error(sem, obs)
    # training=False keeps grad-mode calls on the original
    from soundspaces_b200.encoder import patch_smt_cnn
    Q = patch_smt_cnn(type("Q", (SMTCNN,), {}))
    q = _module(cls=Q)
    n0 = ops.ctx.launch_count
    assert q(obs).grad_fn is not None and ops.ctx.launch_count == n0
