"""The fused ``RNNStateEncoder.seq_forward`` and its backward (``ssb_gru_seq_*``, ``WaveformOps.gru_seq_forward`` /
``gru_seq_backward``, ``patch_rnn_state_encoder(cls, sequence=True)``) on the GPU: out and h_last within
1e-4 max|ref_b| of float64 per env, every gradient within 1e-4 max|g64|, at the reference's golden cases and at
AV-Nav's shape; deterministic gradients and per-env bit-identity across N and positions; launch counts fixed across
T, N and done patterns; no host synchronisation; refusals that launch nothing; and one PPO-style update of an
AV-Nav-shaped net over a minibatch of the patched rollout storage against the unpatched modules."""
import copy
import os

import numpy as np
import pytest

import gru_seq_models as gm

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
nn = torch.nn

DEV = "cuda:0"
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "gru_seq_golden.npz")
GRADS = ("dx", "dh0", "dw_ih", "dw_hh", "db_ih", "db_hh")


def _ops():
    from soundspaces_b200.renderer import WaveformOps
    return WaveformOps.get(DEV)


def _patched():
    from soundspaces_b200.rnn import patch_rnn_state_encoder
    return patch_rnn_state_encoder(type("PatchedRNNStateEncoder", (gm.RNNStateEncoder,), {}), sequence=True)


@pytest.fixture
def no_tf32():
    saved = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = saved


@pytest.fixture(scope="module")
def golden():
    with np.load(GOLDEN) as z:
        return {k: z[k] for k in z.files}


def _case(golden, name):
    return {k.split("/", 1)[1]: v for k, v in golden.items() if k.startswith(name + "/")}


def _run(enc_cls, I, Hd, params, x, h0, masks, g_out, g_h):
    """(out, h_last, grads) of ``enc_cls`` in float32 on the device with upstream gradients g_out / g_h."""
    enc = gm.make_encoder(I, Hd, params, torch.float32)
    enc.__class__ = enc_cls
    enc = enc.to(DEV)
    x = torch.as_tensor(x, dtype=torch.float32, device=DEV).requires_grad_(True)
    h0 = torch.as_tensor(h0, dtype=torch.float32, device=DEV).requires_grad_(True)
    masks = torch.as_tensor(masks, dtype=torch.float32, device=DEV)
    out, h_last = enc(x, h0, masks)
    loss = (out * torch.as_tensor(g_out, dtype=torch.float32, device=DEV)).sum()
    loss = loss + (h_last * torch.as_tensor(g_h, dtype=torch.float32, device=DEV)).sum()
    loss.backward()
    return out.detach(), h_last.detach(), [x.grad, h0.grad] + [p.grad for p in gm.gru_params(enc)]


def _per_env(got, ref, N, Hd):
    got = got.detach().cpu().double().numpy().reshape(-1, N, Hd)
    ref = np.asarray(ref, np.float64).reshape(-1, N, Hd)
    for e in range(N):
        scale = np.abs(ref[:, e]).max()
        err = np.abs(got[:, e] - ref[:, e]).max()
        assert err <= 1e-4 * scale, f"env {e}: max err {err:.3g} > 1e-4 * {scale:.3g}"


def _whole(got, ref, what):
    got = got.detach().cpu().double().numpy()
    ref = ref.detach().cpu().double().numpy() if isinstance(ref, torch.Tensor) else np.asarray(ref, np.float64)
    assert got.shape == ref.shape, what
    scale = np.abs(ref).max()
    err = np.abs(got - ref).max()
    assert err <= 1e-4 * scale, f"{what}: max err {err:.3g} > 1e-4 * {scale:.3g}"


@pytest.mark.parametrize("name", list(gm.CASES))
def test_golden_cases_against_float64(golden, name):
    c = _case(golden, name)
    T, N, I, Hd = gm.CASES[name]
    ops = _ops()
    before = ops.ctx.launch_count
    out, h_last, grads = _run(_patched(), I, Hd, (c["w_ih"], c["w_hh"], c["b_ih"], c["b_hh"]), c["x"], c["h0"],
                              c["masks"], c["g_out"], c["g_h_last"])
    assert ops.ctx.launch_count - before == 2 + 4            # the fused path ran, forward and backward
    assert not h_last.data_ptr() == out[-N:].data_ptr()
    _per_env(out, c["out"], N, Hd)
    _per_env(h_last, c["h_last"], N, Hd)
    for k, g in zip(GRADS, grads):
        _whole(g, c[k], k)


def _avnav_inputs(T=150, N=10, I=1024, Hd=512, seed=0, done_p=0.02):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(T * N, I, generator=g)
    h0 = torch.randn(1, N, Hd, generator=g)
    masks = (torch.rand(T * N, 1, generator=g) >= done_p).float()
    g_out = torch.randn(T * N, Hd, generator=g)
    g_h = torch.randn(1, N, Hd, generator=g)
    enc = gm.RNNStateEncoder(I, Hd)                          # torch's default GRU init
    params = [p.detach().clone() for p in gm.gru_params(enc)]
    return params, x, h0, masks, g_out, g_h


def test_avnav_shape_against_float64():
    T, N, I, Hd = 150, 10, 1024, 512
    params, x, h0, masks, g_out, g_h = _avnav_inputs()
    ref = gm.make_encoder(I, Hd, params)
    xr, hr = x.double().requires_grad_(True), h0.double().requires_grad_(True)
    y, hl = ref(xr, hr, masks.double())
    ((y * g_out.double()).sum() + (hl * g_h.double()).sum()).backward()
    want = [xr.grad, hr.grad] + [p.grad for p in gm.gru_params(ref)]
    out, h_last, grads = _run(_patched(), I, Hd, params, x, h0, masks, g_out, g_h)
    _per_env(out, y.detach(), N, Hd)
    _per_env(h_last, hl.detach(), N, Hd)
    for k, a, b in zip(GRADS, grads, want):
        _whole(a, b, k)


def test_gradients_are_deterministic():
    params, x, h0, masks, g_out, g_h = _avnav_inputs(T=40, N=6, I=96, Hd=72, seed=3, done_p=0.1)
    first = _run(_patched(), 96, 72, params, x, h0, masks, g_out, g_h)
    second = _run(_patched(), 96, 72, params, x, h0, masks, g_out, g_h)
    assert torch.equal(first[0], second[0]) and torch.equal(first[1], second[1])
    for a, b in zip(first[2], second[2]):
        assert torch.equal(a, b)


@pytest.mark.parametrize("N, pos", [(1, 0), (5, 3), (17, 16)])
def test_an_env_is_bit_identical_at_any_n_and_position(N, pos):
    """Every env has the same masks, so the segment starts (which depend on all envs) are the same at every N."""
    T, I, Hd = 12, 40, 36
    g = torch.Generator().manual_seed(11)
    params = [p.detach().clone() for p in gm.gru_params(gm.RNNStateEncoder(I, Hd))]
    x0, h00 = torch.randn(T, 1, I, generator=g), torch.randn(1, 1, Hd, generator=g)
    go0, gh0 = torch.randn(T, 1, Hd, generator=g), torch.randn(1, 1, Hd, generator=g)
    col = torch.tensor([0.5, 1, 1, 0, 1, 1, 1, 0, 0, 1, 1, 0.25])[:, None, None]

    def place(N, pos):
        x, h0 = torch.randn(T, N, I, generator=g), torch.randn(1, N, Hd, generator=g)
        go, gh = torch.randn(T, N, Hd, generator=g), torch.randn(1, N, Hd, generator=g)
        x[:, pos:pos + 1], h0[:, pos:pos + 1], go[:, pos:pos + 1], gh[:, pos:pos + 1] = x0, h00, go0, gh0
        masks = col.expand(T, N, 1).reshape(T * N, 1).contiguous()
        out, h_last, grads = _run(_patched(), I, Hd, params, x.reshape(T * N, I), h0, masks, go.reshape(T * N, Hd), gh)
        return (out.view(T, N, Hd)[:, pos], h_last[0, pos], grads[0].view(T, N, I)[:, pos], grads[1][0, pos])

    base = place(1, 0)
    for a, b in zip(place(N, pos), base):
        assert torch.equal(a, b)


def test_nan_in_a_masked_state_propagates_as_reference(no_tf32):
    params, x, h0, masks, g_out, g_h = _avnav_inputs(T=5, N=3, I=16, Hd=8, seed=4, done_p=0.0)
    h0[0, 1, 2] = float("nan")
    masks.view(5, 3)[0, 1] = 0.0
    ref = gm.make_encoder(16, 8, params, torch.float32).to(DEV)
    want, hw = ref(x.to(DEV), h0.to(DEV), masks.to(DEV))
    with torch.no_grad():
        out, h_last, _ = _ops().gru_seq_forward(x.to(DEV), h0.to(DEV), masks.to(DEV),
                                                 [p.to(DEV) for p in params])
    assert torch.equal(out.isnan(), want.isnan()) and torch.equal(h_last.isnan(), hw.isnan())
    assert out.isnan().any()


NEEDS = {  # (dx, dh0, dw_ih, dw_hh, db_ih, db_hh): backward launches
    (True, True, True, True, True, True): 4,
    (True, False, False, False, False, False): 2,
    (False, True, False, False, False, False): 1,
    (False, False, True, False, False, False): 2,
    (False, False, False, False, True, False): 2,
    (False, False, False, True, False, True): 2,
    (False, False, False, False, False, False): 0,
}


@pytest.mark.parametrize("need", list(NEEDS))
def test_launch_counts_are_fixed(need):
    ops = _ops()
    for T, N, done_p in ((2, 1, 0.0), (30, 7, 0.5), (150, 10, 0.02), (64, 4, 1.0)):
        params, x, h0, masks, g_out, g_h = _avnav_inputs(T=T, N=N, I=48, Hd=32, seed=T, done_p=done_p)
        params = [p.to(DEV) for p in params]
        x, h0, masks, g_out, g_h = (t.to(DEV) for t in (x, h0, masks, g_out, g_h))
        before = ops.ctx.launch_count
        _, _, saved = ops.gru_seq_forward(x, h0, masks, params, save=True)
        assert ops.ctx.launch_count - before == 2
        before = ops.ctx.launch_count
        got = ops.gru_seq_backward(x, N, masks, params[0], params[1], saved, g_out, None, need=need)
        assert ops.ctx.launch_count - before == NEEDS[need]
        assert [g is not None for g in got] == list(need)


def test_autograd_requests_only_the_needed_gradients():
    """x frozen and h0 without grad: the backward computes the four parameter gradients only (3 launches)."""
    params, x, h0, masks, g_out, g_h = _avnav_inputs(T=20, N=3, I=24, Hd=16, seed=9, done_p=0.1)
    enc = gm.make_encoder(24, 16, params, torch.float32)
    enc.__class__ = _patched()
    enc = enc.to(DEV)
    ops = _ops()
    out, h_last = enc(x.to(DEV), h0.to(DEV), masks.to(DEV))
    before = ops.ctx.launch_count
    out.sum().backward()                                      # h_last's gradient is None
    assert ops.ctx.launch_count - before == 3
    assert all(p.grad is not None for p in enc.parameters())
    with torch.no_grad():
        before = ops.ctx.launch_count
        enc(x.to(DEV), h0.to(DEV), masks.to(DEV))
        assert ops.ctx.launch_count - before == 2


def test_no_grad_and_frozen_calls_save_nothing(monkeypatch):
    """The saved state is allocated only when a backward can follow: grad mode on and some input requiring grad."""
    from soundspaces_b200.renderer import WaveformOps
    params, x, h0, masks, g_out, g_h = _avnav_inputs(T=10, N=3, I=24, Hd=16, seed=6, done_p=0.1)
    enc = gm.make_encoder(24, 16, params, torch.float32)
    enc.__class__ = _patched()
    enc = enc.to(DEV)
    saves = []
    orig = WaveformOps.gru_seq_forward

    def spy(self, *args, save=False):
        saves.append(save)
        return orig(self, *args, save=save)

    monkeypatch.setattr(WaveformOps, "gru_seq_forward", spy)
    args = (x.to(DEV), h0.to(DEV), masks.to(DEV))
    with torch.no_grad():
        out, h_last = enc(*args)
    assert not out.requires_grad
    enc.requires_grad_(False)
    enc(*args)
    enc.requires_grad_(True)
    out, _ = enc(*args)
    assert saves == [False, False, True] and out.requires_grad


def test_no_host_synchronisation():
    params, x, h0, masks, g_out, g_h = _avnav_inputs(T=50, N=8, I=64, Hd=48, seed=2, done_p=0.1)
    enc = gm.make_encoder(64, 48, params, torch.float32)
    enc.__class__ = _patched()
    enc = enc.to(DEV)
    x, h0, masks = x.to(DEV).requires_grad_(True), h0.to(DEV).requires_grad_(True), masks.to(DEV)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        out, h_last = enc(x, h0, masks)
        loss = out.square().mean() + h_last.sum()
        loss.backward()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert x.grad is not None and h0.grad is not None


def test_not_qualifying_calls_run_the_original(no_tf32):
    from soundspaces_b200.rnn import gru_seq_error
    params, x, h0, masks, g_out, g_h = _avnav_inputs(T=6, N=2, I=8, Hd=4, seed=1, done_p=0.3)
    enc = gm.make_encoder(8, 4, params, torch.float32)
    enc.__class__ = _patched()
    enc = enc.to(DEV)
    ops = _ops()
    xd, hd, md = x.to(DEV), h0.to(DEV), masks.to(DEV)
    for args, why in (((xd, hd, md.requires_grad_(True)), "masks require grad"),
                      ((xd.t().contiguous().t(), hd, md.detach()), "x is not")):
        assert why in gru_seq_error(enc, *args)
        before = ops.ctx.launch_count
        enc(*args)
        assert ops.ctx.launch_count == before
    with torch.autocast("cuda"):
        assert gru_seq_error(enc, xd, hd, md.detach()) == "autocast is on"
    lstm = type("P", (gm.RNNStateEncoder,), {})
    from soundspaces_b200.rnn import patch_rnn_state_encoder
    patch_rnn_state_encoder(lstm, sequence=True)
    m = lstm(8, 4, rnn_type="LSTM").to(DEV)
    assert "LSTM" in gru_seq_error(m, xd, hd, md.detach())


def test_refusals_launch_nothing():
    ops = _ops()
    lib, h = ops.lib, ops.ctx.handle
    T, N, I, Hd = 4, 3, 8, 6
    f = lambda *s: torch.randn(*s, device=DEV)               # noqa: E731
    x, h0, m, wi, wh, bi, bh = f(T * N, I), f(N, Hd), torch.ones(T * N, device=DEV), f(3 * Hd, I), f(3 * Hd, Hd), \
        f(3 * Hd), f(3 * Hd)
    out, hl, sv = f(T * N, Hd), f(N, Hd), f(5, T * N, Hd)
    ws = torch.empty(int(lib.ssb_gru_seq_workspace_bytes(T, N, I, Hd)), dtype=torch.uint8, device=DEV)
    gx, gh0, gwi, gwh, gbi, gbh = f(T * N, I), f(N, Hd), f(3 * Hd, I), f(3 * Hd, Hd), f(3 * Hd), f(3 * Hd)
    p = lambda t: t.data_ptr()                                 # noqa: E731
    st = ops._stream()

    def fwd(T=T, N=N, I=I, Hd=Hd, **kw):
        a = dict(x=p(x), h0=p(h0), m=p(m), wi=p(wi), wh=p(wh), bi=p(bi), bh=p(bh), out=p(out), hl=p(hl), sv=p(sv),
                 ws=p(ws))
        a.update(kw)
        return lib.ssb_gru_seq_forward_batch(h, T, N, I, Hd, *a.values(), st)

    def bwd(T=T, N=N, I=I, Hd=Hd, **kw):
        a = dict(x=p(x), m=p(m), wi=p(wi), wh=p(wh), sv=p(sv), go=p(out), gh=p(hl), ws=p(ws), dx=p(gx), dh0=p(gh0),
                 dwi=p(gwi), dwh=p(gwh), dbi=p(gbi), dbh=p(gbh))
        a.update(kw)
        return lib.ssb_gru_seq_backward_batch(h, T, N, I, Hd, *a.values(), st)

    before = ops.ctx.launch_count
    for call in (lambda: fwd(T=0), lambda: fwd(T=4097), lambda: fwd(N=0), lambda: fwd(N=257), lambda: fwd(I=0),
                 lambda: fwd(Hd=0), lambda: fwd(Hd=1025), lambda: fwd(x=None), lambda: fwd(ws=None),
                 lambda: fwd(out=p(out) + 2), lambda: fwd(ws=p(ws) + 4), lambda: fwd(out=p(x)),
                 lambda: fwd(hl=p(h0)), lambda: fwd(out=p(out), hl=p(out) + 8), lambda: fwd(sv=p(wi)),
                 lambda: bwd(T=0), lambda: bwd(N=257), lambda: bwd(Hd=1025), lambda: bwd(sv=None),
                 lambda: bwd(dx=p(x)), lambda: bwd(dwh=p(wh)), lambda: bwd(dh0=p(gh0) + 2),
                 lambda: bwd(dbi=p(gbh), dbh=p(gbh)), lambda: bwd(ws=p(sv))):
        assert call() == -1
        assert b"bad arguments" in lib.ssb_last_error(h)
    assert ops.ctx.launch_count == before
    assert lib.ssb_gru_seq_workspace_bytes(0, 1, 1, 1) == -1
    assert lib.ssb_gru_seq_workspace_bytes(1, 257, 1, 1) == -1
    assert lib.ssb_gru_seq_workspace_bytes(4096, 256, 1, 1024) == 2 * 4096 * 256 * 3 * 1024 * 4
    assert fwd() == 0 and bwd() == 0
    assert ops.ctx.launch_count - before == 6
    with pytest.raises(RuntimeError, match="outside the library's limits"):
        ops.gru_seq_forward(f(2 * 300, I), f(1, 300, Hd), torch.ones(600, device=DEV), [wi, wh, bi, bh])


# end to end: one PPO update of an AV-Nav-shaped net -----------------------------------------------------------------

class _Net(nn.Module):
    """avnav_models.AudioNavBaselineNet with the sequence stand-in as its state encoder, plus actor and critic."""

    def __init__(self, hidden=512, n_actions=4):
        super().__init__()
        from avnav_models import VisualCNN
        from test_encoder_host import reference_classes
        self.audio_encoder = reference_classes()[0]((65, 26, 2), hidden, audiogoal_sensor="spectrogram")
        self.visual_encoder = VisualCNN(0, 1, 64, 64, hidden)
        self.state_encoder = gm.RNNStateEncoder(2 * hidden, hidden)
        self.actor = nn.Linear(hidden, n_actions)
        self.critic = nn.Linear(hidden, 1)

    def forward(self, obs, h, masks):
        x = torch.cat([self.audio_encoder(obs), self.visual_encoder(obs)], dim=1)
        return self.state_encoder(x, h, masks)


def _ppo_update(net, batch):
    obs, h, actions, _, value_preds, returns, masks, old_lp, adv = batch[:9]
    feats, _ = net(obs, h, masks)
    dist = torch.distributions.Categorical(logits=net.actor(feats))
    lp = dist.log_prob(actions.view(-1)).unsqueeze(-1)
    ratio = torch.exp(lp - old_lp)
    action_loss = -torch.min(ratio * adv, torch.clamp(ratio, 0.8, 1.2) * adv).mean()
    value_loss = 0.5 * (returns - net.critic(feats)).pow(2).mean()
    loss = value_loss * 0.5 + action_loss - dist.entropy().mean() * 0.01
    opt = torch.optim.Adam(net.parameters(), lr=2.5e-4, eps=1e-5)
    opt.zero_grad()
    loss.backward()
    nn.utils.clip_grad_norm_(net.parameters(), 0.5)
    grads = [p.grad.detach().clone() for p in net.parameters()]
    opt.step()
    return grads, [p.detach().clone() for p in net.parameters()]


def test_ppo_update_matches_unpatched(no_tf32):
    import rollout_models as rm
    from soundspaces_b200 import rollout as ro
    S, N, hidden = 150, 10, 512
    storage_cls = ro.patch_rollout_storage(type("PatchedStorage", (rm.CommonRolloutStorage,), {}))
    sp = rm.spaces({"spectrogram": (65, 26, 2), "depth": (64, 64, 1)})
    st = storage_cls(S, N, sp, rm.ActionSpace(), hidden, 1)
    st.to(DEV)
    g = np.random.default_rng(21)
    for _ in range(S):
        obs = {"spectrogram": torch.from_numpy(g.random((N, 65, 26, 2), dtype=np.float32) * 3).to(DEV),
               "depth": torch.from_numpy(g.random((N, 64, 64, 1), dtype=np.float32)).to(DEV)}
        st.insert(obs, torch.from_numpy(g.standard_normal((1, N, hidden), dtype=np.float32)).to(DEV),
                  torch.from_numpy(g.integers(0, 4, (N, 1))).to(DEV),
                  -torch.from_numpy(g.random((N, 1), dtype=np.float32)).to(DEV) - 1.0,
                  torch.from_numpy(g.standard_normal((N, 1), dtype=np.float32)).to(DEV),
                  torch.from_numpy(g.standard_normal((N, 1), dtype=np.float32)).to(DEV),
                  torch.from_numpy((g.random((N, 1)) >= 0.02).astype(np.float32)).to(DEV))
    st.compute_returns(torch.zeros(N, 1, device=DEV), True, 0.99, 0.95)
    adv = st.returns[:-1] - st.value_preds[:-1]
    batch = next(iter(st.recurrent_generator(adv.contiguous(), 1)))
    torch.manual_seed(5)
    plain = _Net(hidden).to(DEV)
    fused = copy.deepcopy(plain)
    fused.state_encoder.__class__ = _patched()
    ops = _ops()
    before = ops.ctx.launch_count
    g_fused, p_fused = _ppo_update(fused, batch)
    assert ops.ctx.launch_count - before == 2 + 4
    g_plain, p_plain = _ppo_update(plain, batch)
    for (name, _), a, b in zip(plain.named_parameters(), g_fused, g_plain):
        _whole(a, b, "grad " + name)
    for (name, _), a, b in zip(plain.named_parameters(), p_fused, p_plain):
        _whole(a, b, "param " + name)
