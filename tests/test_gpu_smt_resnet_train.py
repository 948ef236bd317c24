"""SAVi's SMT location predictor trained online through the library (ssb_smt_resnet18_train_*, SmtResNetFunction and
``patch_belief_predictor(..., training=True)``): forward bits against the inference entry, gradients against float64,
determinism, silent rows, launch counts, host syncs, frozen, refused and fallback calls, and a train_belief_predictor
round on the patched rollout storage against eager FP32 and float64 at every epoch."""
import copy
import ctypes

import pytest

from belief_nets_models import network_input, smt_net

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

HW = (65, 26)
FWD_LAUNCHES = 38
BWD_LAUNCHES = {0: 80, 21: 82}


@pytest.fixture(scope="module")
def ops():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    from soundspaces_b200.renderer import WaveformOps
    return WaveformOps.get("cuda:0")


def _obs(B, seed=0, silent=()):
    g = torch.Generator().manual_seed(seed)
    x = torch.rand((B, HW[0], HW[1], 2), generator=g) * 3.0
    for i in silent:
        x[i] = 0.0
    return x.cuda()


def _labels(B, n, seed=1):
    if not n:
        return None
    g = torch.Generator().manual_seed(seed)
    return torch.nn.functional.one_hot(torch.randint(0, n, (B,), generator=g), n).float().cuda()


def _net(n_labels, seed=0):
    return smt_net(2 + n_labels, HW, 2, seed).cuda()


def _forward(net, x, labels):
    from soundspaces_b200.belief_nets import SmtResNetFunction, conv_norm_pairs, smt_resnet18_params
    eps = tuple(float(n.eps) for _, n in conv_norm_pairs(net))
    return SmtResNetFunction.apply(torch.is_grad_enabled(), eps, x, labels, *smt_resnet18_params(net))


def _masked_mse(pred, x, gts):
    """train_belief_predictor's loss: rows whose spectrogram sums to 0 are masked out of prediction and target."""
    masks = (torch.sum(torch.reshape(x, (x.shape[0], -1)), dim=1, keepdim=True) != 0).float()
    return torch.nn.functional.mse_loss(masks.expand_as(pred) * pred, masks.expand_as(gts) * gts)


def _grads(net):
    from soundspaces_b200.belief_nets import smt_resnet18_params
    return [p.grad.detach().clone() for p in smt_resnet18_params(net)]


def _fused_grads(net, x, labels, gts):
    net.zero_grad(set_to_none=True)
    _masked_mse(_forward(net, x, labels), x, gts).backward()
    return _grads(net)


@pytest.mark.parametrize("n_labels", [0, 21])
@pytest.mark.parametrize("B", [1, 8, 1024])
def test_forward_bits_match_inference(ops, B, n_labels):
    net = _net(n_labels)
    x, labels = _obs(B), _labels(B, n_labels)
    with torch.no_grad():
        want = ops.smt_resnet18(x, net, labels)
        got = _forward(net, x, labels)
    assert torch.equal(got, want)


@pytest.mark.parametrize("n_labels", [0, 21])
def test_forward_bits_above_the_inference_limit_and_permuted(ops, n_labels):
    net = _net(n_labels, seed=3)
    B = 1200
    x, labels = _obs(B, seed=4), _labels(B, n_labels, seed=5)
    with torch.no_grad():
        got = _forward(net, x, labels)
        want = torch.cat([ops.smt_resnet18(x[:1024].contiguous(), net, None if labels is None else labels[:1024]),
                          ops.smt_resnet18(x[1024:].contiguous(), net, None if labels is None else labels[1024:])])
        perm = torch.randperm(B, generator=torch.Generator().manual_seed(6)).cuda()
        got_p = _forward(net, x[perm].contiguous(), None if labels is None else labels[perm].contiguous())
    assert torch.equal(got, want)
    assert torch.equal(got_p, got[perm])


def _check_grads(net, x, labels, gts, tol=1e-4):
    """Each fused gradient against float64, within ``tol`` of its tensor's maximum or, where FP32 itself cannot get
    that close, within twice the worst error of eager FP32 (cuDNN, TF32 off) over the call's tensors: the error comes
    from the ill-conditioned forward, and how it lands on a single tensor differs between two FP32 evaluations by up
    to 16x (DESIGN.md §4).  test_gradients_match_float64_well_conditioned holds every tensor to 1e-4."""
    got = _fused_grads(net, x, labels, gts)
    prev = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    try:
        e32 = copy.deepcopy(net)
        e32.zero_grad(set_to_none=True)
        _masked_mse(e32(network_input(x, labels)), x, gts).backward()
    finally:
        torch.backends.cudnn.allow_tf32 = prev
    eager = _grads(e32)
    ref = copy.deepcopy(net).double()
    ref.zero_grad(set_to_none=True)
    xd = x.double()
    pred = ref(network_input(xd, None if labels is None else labels.double()))
    _masked_mse(pred, xd, gts.double()).backward()
    want = _grads(ref)
    rel = lambda a, b: (a.double() - b).abs().max().item() / max(b.abs().max().item(), 1e-30)   # noqa: E731
    bound = max(tol, 2 * max(rel(e, b) for e, b in zip(eager, want)))
    for i, (a, b) in enumerate(zip(got, want)):
        assert rel(a, b) <= bound, f"parameter {i}: relative error {rel(a, b):.3g}, bound {bound:.3g}"


@pytest.mark.parametrize("n_labels", [0, 21])
@pytest.mark.parametrize("B", [3, 1200])
def test_gradients_match_float64(ops, B, n_labels):
    net = _net(n_labels, seed=7)
    silent = [i for i in range(B) if i % 3 == 1]
    x = _obs(B, seed=8, silent=silent)
    x[0] *= 1e-3
    labels = _labels(B, n_labels, seed=9)
    gts = torch.randn((B, 2), generator=torch.Generator().manual_seed(10)).cuda() * 5
    _check_grads(net, x, labels, gts)


@pytest.mark.parametrize("n_labels", [0, 21])
def test_gradients_match_float64_well_conditioned(ops, n_labels):
    """No row near the GroupNorm eps: every gradient within 1e-4 of its tensor's maximum against float64."""
    net = _net(n_labels, seed=30)
    B = 8
    x = _obs(B, seed=31, silent=[5])
    labels = _labels(B, n_labels, seed=32)
    gts = torch.randn((B, 2), generator=torch.Generator().manual_seed(33)).cuda() * 5
    got = _fused_grads(net, x, labels, gts)
    ref = copy.deepcopy(net).double()
    ref.zero_grad(set_to_none=True)
    xd = x.double()
    _masked_mse(ref(network_input(xd, None if labels is None else labels.double())), xd, gts.double()).backward()
    for i, (a, b) in enumerate(zip(got, _grads(ref))):
        err = (a.double() - b).abs().max().item()
        assert err <= 1e-4 * b.abs().max().item(), f"parameter {i}: error {err:.3g}"


@pytest.mark.parametrize("n_labels", [0, 21])
def test_deterministic_and_silent_rows_cost_no_bits(ops, n_labels):
    net = _net(n_labels, seed=11)
    B = 300
    silent = [i for i in range(B) if i % 4 != 0]
    x = _obs(B, seed=12, silent=silent)
    labels = _labels(B, n_labels, seed=13)
    gts = torch.randn((B, 2), generator=torch.Generator().manual_seed(14)).cuda()
    a = _fused_grads(net, x, labels, gts)
    b = _fused_grads(net, x, labels, gts)
    assert all(torch.equal(u, v) for u, v in zip(a, b))
    # the same live rows without the silent ones: an upstream gradient scaled to match MSE's 1 / (2 B)
    keep = torch.tensor([i for i in range(B) if i not in set(silent)]).cuda()
    xs, ls = x[keep].contiguous(), None if labels is None else labels[keep].contiguous()

    def grads_from(xx, ll, g):
        net.zero_grad(set_to_none=True)
        _forward(net, xx, ll).backward(g)
        return _grads(net)

    pred = _forward(net, x, labels).detach()
    g_full = torch.zeros_like(pred)
    g_full[keep] = 2.0 * (pred[keep] - gts[keep]) / (2 * B)
    full = grads_from(x, labels, g_full)
    removed = grads_from(xs, ls, g_full[keep].contiguous())
    for i, (u, v) in enumerate(zip(full, removed)):
        assert torch.equal(u, v), f"parameter {i}"


@pytest.mark.parametrize("n_labels", [0, 21])
def test_launch_counts(ops, n_labels):
    net = _net(n_labels, seed=15)
    for B, every in ((1, 1), (64, 3), (1100, 1), (1100, 1000000)):
        x = _obs(B, seed=B, silent=[i for i in range(B) if i % every])
        labels = _labels(B, n_labels)
        n0 = ops.ctx.launch_count
        pred = _forward(net, x, labels)
        n1 = ops.ctx.launch_count
        pred.backward(torch.where(x.reshape(B, -1).sum(1, keepdim=True) != 0, 1.0, 0.0).expand(B, 2).contiguous())
        torch.cuda.synchronize()
        n2 = ops.ctx.launch_count
        assert (n1 - n0, n2 - n1) == (FWD_LAUNCHES, BWD_LAUNCHES[n_labels]), (B, every)


class _Predictor(torch.nn.Module):
    """The parts of SAVi's BeliefPredictor that train_belief_predictor touches (belief_predictor.py:55-134)."""

    def __init__(self, n_labels, seed=0):
        super().__init__()
        self.has_distractor_sound = bool(n_labels)
        self.predictor = _net(n_labels, seed)

    def cnn_forward(self, observations):
        spectrograms = observations["spectrogram"].permute(0, 3, 1, 2)
        if self.has_distractor_sound:
            labels = observations["category"]
            expanded = labels.reshape(labels.shape + (1, 1)).expand(labels.shape + spectrograms.shape[-2:])
            inputs = torch.cat([spectrograms, expanded], dim=1)
        else:
            inputs = spectrograms
        return self.predictor(inputs)


def _patched_class():
    from soundspaces_b200.belief import patch_belief_predictor

    class P(_Predictor):
        def update(self, observations, dones):
            raise NotImplementedError
    patch_belief_predictor(P, networks=True, training=True)
    return P


def test_patched_cnn_forward_paths(ops):
    P = _patched_class()
    orig = P.cnn_forward._ssb_original
    from soundspaces_b200.belief import patch_belief_predictor
    patch_belief_predictor(P, networks=True, training=True)
    assert P.cnn_forward._ssb_original is orig
    m = P(0, seed=16)
    obs = {"spectrogram": _obs(16)}
    n0 = ops.ctx.launch_count
    with torch.no_grad():
        m.cnn_forward(obs)
    assert ops.ctx.launch_count == n0            # no-grad calls keep the module
    out = m.cnn_forward(obs)
    assert ops.ctx.launch_count == n0 + FWD_LAUNCHES and out.grad_fn is not None
    out_bits = out.detach().clone()
    del out
    torch.cuda.synchronize()
    from soundspaces_b200.belief_nets import smt_resnet18_train_forward
    base = torch.cuda.memory_allocated()
    held = smt_resnet18_train_forward(m, obs)                    # grad: the workspace stays with the graph
    torch.cuda.synchronize()
    assert torch.cuda.memory_allocated() - base >= ops.lib.ssb_smt_resnet18_train_workspace_bytes(16, 65, 26, 0, 2)
    del held
    for p in m.parameters():
        p.requires_grad_(False)
    base = torch.cuda.memory_allocated()
    frozen = smt_resnet18_train_forward(m, obs)
    torch.cuda.synchronize()
    assert frozen.grad_fn is None                # a frozen predictor saves nothing: only the output stays allocated
    assert torch.cuda.memory_allocated() - base <= 4096
    assert torch.equal(frozen, out_bits)


def test_no_host_sync_in_the_patched_step(ops):
    P = _patched_class()
    m = P(21, seed=17)
    B = 200
    obs = {"spectrogram": _obs(B, silent=range(0, B, 2)), "category": _labels(B, 21)}
    gts = torch.randn((B, 2), device="cuda")
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        pred = m.cnn_forward(obs)
        _masked_mse(pred, obs["spectrogram"], gts).backward()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert m.predictor.fc.weight.grad is not None


def _rollout_minibatch(n_labels, T=150, N=8):
    """One recurrent_generator minibatch (T x N rows) of SAVi's rollout storage under patch_rollout_storage, with
    silent steps: every fifth step of every env, and env 3 from step 100 on."""
    import numpy as np
    import rollout_models as rm
    from soundspaces_b200 import rollout as ro
    storage_cls = ro.patch_rollout_storage(type("PatchedSavi", (rm.SaviRolloutStorage,), {}))
    shapes = {"spectrogram": (65, 26, 2), "pointgoal": (2,)}
    if n_labels:
        shapes["category"] = (n_labels,)
    st = storage_cls(T, N, rm.spaces(shapes), rm.ActionSpace(), 16, False, 1, 1, 1)
    st.to("cuda")
    g = np.random.default_rng(40 + n_labels)
    dev = torch.device("cuda")
    for t in range(T):
        spec = g.random((N, 65, 26, 2), dtype=np.float32) * 3
        spec[:, :, :, :] *= np.array([t % 5 != 3 and not (e == 3 and t >= 100) for e in range(N)],
                                     np.float32)[:, None, None, None]
        obs = {"spectrogram": torch.from_numpy(spec).to(dev),
               "pointgoal": torch.from_numpy(g.standard_normal((N, 2), dtype=np.float32) * 3).to(dev)}
        if n_labels:
            obs["category"] = torch.from_numpy(np.eye(n_labels, dtype=np.float32)[g.integers(0, n_labels, N)]).to(dev)
        st.insert(obs, torch.zeros((1, N, 16), device=dev), torch.zeros((N, 1), dtype=torch.long, device=dev),
                  torch.zeros((N, 1), device=dev), torch.zeros((N, 1), device=dev), torch.zeros((N, 1), device=dev),
                  torch.ones((N, 1), device=dev), None)
    st.compute_returns(torch.zeros(N, 1, device=dev), True, 0.99, 0.95)
    batch = next(iter(st.recurrent_generator(torch.zeros_like(st.returns[:-1]), 1)))
    return batch[0]


@pytest.mark.parametrize("n_labels", [0, 21])
def test_train_round_matches_the_module(ops, n_labels):
    """train_belief_predictor's body (ppo_trainer.py:342-400) on a minibatch of the patched SAVi rollout storage: 5
    epochs of masked MSE, backward and Adam through the patched cnn_forward.  At every epoch, on the same parameters,
    the fused loss matches eager FP32's within 1e-5 and every fused gradient is within 1e-4 of its tensor's maximum
    against float64, or within twice eager FP32's worst error over the tensors where FP32 cannot get that close."""
    P = _patched_class()
    obs = _rollout_minibatch(n_labels)
    x = obs["spectrogram"]
    B = x.shape[0]
    assert B == 1200 and (x.reshape(B, -1).sum(1) == 0).sum() > 200
    gts = torch.stack([obs["pointgoal"][:, 1], -obs["pointgoal"][:, 0]], dim=1)
    fused = P(n_labels, seed=21)
    opt = torch.optim.Adam(fused.predictor.parameters(), lr=1e-3)
    prev = torch.backends.cudnn.allow_tf32
    n_launch = 0
    try:
        for _ in range(5):
            start = copy.deepcopy(fused.predictor.state_dict())
            opt.zero_grad()
            n0 = ops.ctx.launch_count
            loss = _masked_mse(fused.cnn_forward(obs), x, gts)
            loss.backward()
            n_launch += ops.ctx.launch_count - n0
            got = [p.grad.clone() for p in fused.predictor.parameters()]
            torch.backends.cudnn.allow_tf32 = False
            eager = _Predictor(n_labels)
            eager.predictor.load_state_dict(start)
            e_loss = _masked_mse(eager.cnn_forward(obs), x, gts)
            e_loss.backward()
            e_grads = [p.grad for p in eager.predictor.parameters()]
            torch.backends.cudnn.allow_tf32 = prev
            ref = _Predictor(n_labels).double()
            ref.predictor.load_state_dict(start)
            obs64 = {k: v.double() for k, v in obs.items()}
            _masked_mse(ref.cnn_forward(obs64), obs64["spectrogram"], gts.double()).backward()
            assert abs(loss.item() - e_loss.item()) <= 1e-5 * abs(e_loss.item())
            rel = lambda a, b: (a.double() - b).abs().max().item() / b.abs().max().item()   # noqa: E731
            want = [p64.grad for p64 in ref.predictor.parameters()]
            bound = max(1e-4, 2 * max(rel(e, b) for e, b in zip(e_grads, want)))
            for i, (a, b) in enumerate(zip(got, want)):
                assert rel(a, b) <= bound, f"gradient {i}: {rel(a, b):.3g}, bound {bound:.3g}"
            opt.step()
    finally:
        torch.backends.cudnn.allow_tf32 = prev
    assert n_launch == 5 * (FWD_LAUNCHES + BWD_LAUNCHES[n_labels])


def _abi_args(net, x, labels, out, ws):
    from soundspaces_b200.belief_nets import conv_table
    B, H, W = x.shape[:3]
    L = labels.shape[1] if labels is not None else 0
    return [B, x.data_ptr(), H, W, labels.data_ptr() if L else None, L, L, conv_table(net, False),
            net.fc.weight.data_ptr(), net.fc.bias.data_ptr(), net.fc.in_features, 2, out.data_ptr(), ws.data_ptr()]


def test_refusals_launch_nothing(ops):
    lib = ops.lib
    assert lib.ssb_smt_resnet18_train_workspace_bytes(65536, 65, 26, 0, 2) == -1
    assert lib.ssb_smt_resnet18_train_workspace_bytes(65535, 65, 26, 0, 2) > 0
    assert lib.ssb_smt_resnet18_train_workspace_bytes(4, 257, 26, 0, 2) == -1
    net = _net(0, seed=22)
    B = 4
    x = _obs(B)
    out = torch.empty((B, 2), device="cuda")
    ws = ops.smt_resnet18_train_workspace(B, 65, 26, 0, 2)
    good = _abi_args(net, x, None, out, ws)

    def call(args):
        n0 = ops.ctx.launch_count
        rc = lib.ssb_smt_resnet18_train_forward_batch(ops.ctx.handle, *args, None)
        assert ops.ctx.launch_count == n0
        return rc

    cases = []
    a = list(good); a[1] = None; cases.append(a)                       # NULL spectrogram
    a = list(good); a[1] = x.data_ptr() + 2; cases.append(a)           # misaligned
    a = list(good); a[13] = x.data_ptr(); cases.append(a)              # workspace over the input
    a = list(good); a[12] = ws.data_ptr(); cases.append(a)             # output inside the workspace
    a = list(good); a[10] = 4607; cases.append(a)                      # bad fc_in
    a = list(good); a[0] = 65536; cases.append(a)                      # B past the limit
    a = list(good); a[5] = 3; cases.append(a)                          # labels without a pointer
    for a in cases:
        assert call(a) != 0
    n0 = ops.ctx.launch_count
    assert lib.ssb_smt_resnet18_train_forward_batch(ops.ctx.handle, *good, None) == 0
    assert ops.ctx.launch_count == n0 + FWD_LAUNCHES
    # backward: a gradient buffer over the workspace
    grads = [torch.empty_like(p) for p in net.parameters()]
    dpred = torch.ones((B, 2), device="cuda")
    arr = (ctypes.c_void_p * 20)(*([ws.data_ptr()] + [None] * 19))
    none = (ctypes.c_void_p * 20)()
    n0 = ops.ctx.launch_count
    rc = lib.ssb_smt_resnet18_train_backward_batch(
        ops.ctx.handle, B, x.data_ptr(), 65, 26, None, 0, 0, good[7], net.fc.weight.data_ptr(), 4608, 2,
        dpred.data_ptr(), ws.data_ptr(), arr, none, none, None, None, None)
    assert rc != 0 and ops.ctx.launch_count == n0
    del grads


def test_ddp_world_size_one(ops, tmp_path):
    import torch.distributed as dist

    class Mixin:
        def init_distributed(self, find_unused_params=True):
            class Guard:
                def __init__(self, model, device):
                    self.ddp = torch.nn.parallel.DistributedDataParallel(model, device_ids=[device],
                                                                         output_device=device)
            self._ddp_hooks = Guard(self, 0)
            self.reducer = self._ddp_hooks.ddp.reducer
            self.find_unused_params = find_unused_params

        def before_backward(self, loss):
            self.reducer.prepare_for_backward([loss] if self.find_unused_params else [])

    P = _patched_class()

    class DDPPredictor(Mixin, P):
        pass

    dist.init_process_group("gloo", init_method=f"file://{tmp_path / 'store'}", rank=0, world_size=1)
    try:
        B = 64
        obs = {"spectrogram": _obs(B, seed=23, silent=range(0, B, 3))}
        gts = torch.randn((B, 2), device="cuda")
        m = DDPPredictor(0, seed=24)
        ref = P(0, seed=24)
        ref.load_state_dict(m.state_dict())
        m.init_distributed(find_unused_params=True)
        loss = _masked_mse(m.cnn_forward(obs), obs["spectrogram"], gts)
        m.before_backward(loss)
        loss.backward()
        _masked_mse(ref.cnn_forward(obs), obs["spectrogram"], gts).backward()
        for (name, a), b in zip(m.predictor.named_parameters(), ref.predictor.parameters()):
            assert a.grad is not None, name
            assert torch.equal(a.grad, b.grad), name       # the same fused step without DDP
    finally:
        dist.destroy_process_group()


def test_fallback_reasons(ops):
    """Every reason smt_resnet18_train_error gives, and that the patched cnn_forward then runs the original (no
    library launch) with the same result as the unpatched module."""
    from soundspaces_b200.belief_nets import smt_resnet18_train_error as why
    P = _patched_class()
    m, ml = P(0, seed=50), P(21, seed=51)
    B = 6
    x, lab = _obs(B, seed=52), _labels(B, 21, seed=53)
    cases = [
        (m, {"spectrogram": x.cpu()}, "not a CUDA tensor"),
        (m, {"spectrogram": x.double()}, "not float32"),
        (m, {"spectrogram": x.permute(0, 2, 1, 3).contiguous().permute(0, 2, 1, 3)}, "not contiguous"),
        (m, {"spectrogram": x.clone().requires_grad_(True)}, "spectrogram requires grad"),
        (m, {"spectrogram": torch.zeros((65536, 1, 1, 2), device="cuda")}, "65536 rows"),
        (ml, {"spectrogram": x, "category": lab.clone().requires_grad_(True)}, "category requires grad"),
        (ml, {"spectrogram": x, "category": lab.double()}, "category is not a float32"),
        (ml, {"spectrogram": x, "category": lab[:, ::2]}, "category is not a float32"),
        (ml, {"spectrogram": x}, "without a (B, L) category"),
        (ml, {"spectrogram": x, "category": lab[:, :20].contiguous()}, "not the SMT custom_resnet18"),
    ]
    for model, obs, reason in cases:
        assert reason in why(model, obs), (reason, why(model, obs))
    # a predictor with other widths, parameters on another device, autocast
    other = P(0, seed=54)
    other.predictor.layer2[0].conv1 = torch.nn.Conv2d(16, 32, 3, 1, 1, bias=False).cuda()
    assert "not the SMT custom_resnet18" in why(other, {"spectrogram": x})
    cpu = P(0, seed=55)
    cpu.predictor.fc.cpu()
    assert "parameters are not contiguous float32 tensors" in why(cpu, {"spectrogram": x})
    with torch.autocast("cuda"):
        assert why(m, {"spectrogram": x}) == "autocast is on"
    assert why(m, {"spectrogram": x}) == "" and why(ml, {"spectrogram": x, "category": lab}) == ""
    # the patched cnn_forward runs the original for a call that does not qualify
    obs = {"spectrogram": x.permute(0, 2, 1, 3).contiguous().permute(0, 2, 1, 3)}
    n0 = ops.ctx.launch_count
    got = m.cnn_forward(obs)
    assert ops.ctx.launch_count == n0
    assert torch.allclose(got, _Predictor.cnn_forward(m, obs), rtol=1e-6, atol=0)
