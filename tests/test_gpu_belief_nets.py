"""SAVi's belief-predictor ResNet-18s on the GPU (``ssb_resnet18_batch``, ``ssb_smt_resnet18_batch``): accuracy against
a float64 forward of the same module, bit-identity across batch sizes and positions, live parameters, every refusal,
the fallbacks, and a patched rollout with ``networks=True`` against the unpatched reference-shaped class."""
import copy
import ctypes as C

import numpy as np
import pytest

import belief_oracle as bo
from belief_nets_models import make_net, network_input
from test_belief_host import make_reference_class

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
pytest.importorskip("torchvision")

LAUNCHES = {"tv": 39, "smt": 38}


def _ops():
    from soundspaces_b200.renderer import WaveformOps
    return WaveformOps.get("cuda:0")


def _inputs(B, shape=(65, 26), seed=0):
    """Spectrogram-like rows (log1p magnitudes >= 0), row 0 silent, row 1 scaled by 1e-3; labels one-hot-ish rows."""
    g = torch.Generator().manual_seed(seed)
    x = torch.log1p(torch.rand((B,) + shape + (2,), generator=g) * 20.0)
    x[0] = 0
    if B > 1:
        x[1] *= 1e-3
    labels = torch.softmax(torch.randn(B, 21, generator=g) * 3.0, dim=1)
    return x.cuda(), labels.cuda()


def _run(net, kind, x, labels):
    ops = _ops()
    if kind.startswith("tv"):
        return ops.resnet18(x, net)
    return ops.smt_resnet18(x, net, labels if kind == "smt23" else None)


def _ref64(net, x, labels, kind):
    ref = copy.deepcopy(net).double()
    with torch.no_grad():
        return ref(network_input(x.double(), labels.double() if kind == "smt23" else None))


def _check(got, want):
    err = (got.double() - want).abs().max().item()
    scale = want.abs().max().item()
    assert err <= 1e-4 * scale, f"max|d| {err:.3g} > 1e-4 * {scale:.3g}"


@pytest.mark.parametrize("kind,shape", [("tv21", (65, 26)), ("tv23", (65, 69)), ("smt2", (65, 26)),
                                        ("smt23", (65, 26))])
def test_accuracy_and_batch_invariance(kind, shape):
    """Within 1e-4 max|ref| of float64 at B = 1, 8, 16, 64; each env's outputs bit-identical across B and positions."""
    net = make_net(kind, seed=3).cuda()
    x, labels = _inputs(64, shape, seed=5)
    ref = _ref64(net, x, labels, kind)
    full = _run(net, kind, x, labels)
    _check(full, ref)
    for B in (1, 8, 16):
        out = _run(net, kind, x[:B].contiguous(), labels[:B].contiguous())
        _check(out, ref[:B])
        assert torch.equal(out, full[:B]), B
    perm = torch.randperm(64, generator=torch.Generator().manual_seed(1)).cuda()
    out = _run(net, kind, x[perm].contiguous(), labels[perm].contiguous())
    assert torch.equal(out, full[perm])
    torch.cuda.synchronize()


def test_live_parameters():
    """An in-place Adam step on the SMT predictor, a replaced parameter tensor and a changed BatchNorm running
    statistic each change the next call's output to the new float64 forward."""
    x, labels = _inputs(8, seed=9)
    smt = make_net("smt23", seed=4).cuda()
    before = _run(smt, "smt23", x, labels)
    opt = torch.optim.Adam(smt.parameters(), lr=1e-2)
    loss = smt(network_input(x, labels)).square().mean()
    loss.backward()
    opt.step()
    after = _run(smt, "smt23", x, labels)
    assert not torch.equal(before, after)
    _check(after, _ref64(smt, x, labels, "smt23"))
    smt.layer2[0].conv1.weight = torch.nn.Parameter(torch.randn_like(smt.layer2[0].conv1.weight) * 0.1)
    _check(_run(smt, "smt23", x, labels), _ref64(smt, x, labels, "smt23"))
    tv = make_net("tv21", seed=6).cuda()
    before = _run(tv, "tv21", x, labels)
    tv.layer3[1].bn2.running_var.mul_(3.0)
    tv.layer1[0].bn1.running_mean.add_(0.5)
    after = _run(tv, "tv21", x, labels)
    assert not torch.equal(before, after)
    _check(after, _ref64(tv, x, labels, "tv21"))


def test_refusals_launch_nothing():
    from soundspaces_b200 import _lib
    from soundspaces_b200.belief_nets import conv_table
    ops = _ops()
    tv, smt = make_net("tv21").cuda(), make_net("smt23").cuda()
    x, labels = _inputs(4)
    out = torch.zeros(2048 * 32, device="cuda")
    tv_tab, smt_tab = conv_table(tv, True), conv_table(smt, False)

    def tv_call(B=4, spec=x.data_ptr(), H=65, W=26, table=tv_tab, fcw=tv.fc.weight.data_ptr(), fcb=tv.fc.bias.data_ptr(),
                fc_in=512, n_out=21, o=out.data_ptr()):
        return ops.lib.ssb_resnet18_batch(ops.ctx.handle, B, spec, H, W, table, fcw, fcb, fc_in, n_out, o, ops._stream())

    def smt_call(B=4, spec=x.data_ptr(), H=65, W=26, lab=labels.data_ptr(), nl=21, ls=21, table=smt_tab,
                 fcw=smt.fc.weight.data_ptr(), fcb=smt.fc.bias.data_ptr(), fc_in=4608, n_out=2, o=out.data_ptr()):
        return ops.lib.ssb_smt_resnet18_batch(ops.ctx.handle, B, spec, H, W, lab, nl, ls, table, fcw, fcb, fc_in, n_out,
                                              o, ops._stream())

    def edited(tab, i, **kw):
        t = (_lib.ResnetConv * 20)()
        C.memmove(t, tab, C.sizeof(t))
        for k, v in kw.items():
            setattr(t[i], k, v)
        return t

    assert tv_call() == 0 and smt_call() == 0
    torch.cuda.synchronize()
    before = ops.ctx.launch_count
    cases = [
        (tv_call, dict(B=-1), -1), (tv_call, dict(spec=None), -1), (tv_call, dict(spec=x.data_ptr() + 2), -1),
        (tv_call, dict(H=0), -1), (tv_call, dict(W=0), -1), (tv_call, dict(table=None), -1),
        (tv_call, dict(fcw=None), -1), (tv_call, dict(fcb=tv.fc.bias.data_ptr() + 1), -1), (tv_call, dict(n_out=0), -1),
        (tv_call, dict(o=None), -1), (tv_call, dict(o=out.data_ptr() + 3), -1),
        (tv_call, dict(table=edited(tv_tab, 7, d_weight=None)), -1),
        (tv_call, dict(table=edited(tv_tab, 19, d_var=None)), -1),
        (tv_call, dict(table=edited(tv_tab, 3, d_mean=tv_tab[3].d_mean + 2)), -1),
        (tv_call, dict(table=edited(tv_tab, 0, eps=0.0)), -1), (tv_call, dict(table=edited(tv_tab, 5, eps=-1e-5)), -1),
        (tv_call, dict(B=1025), -4), (tv_call, dict(H=257), -4), (tv_call, dict(fc_in=4608), -4),
        (smt_call, dict(nl=-1), -1), (smt_call, dict(ls=20), -1), (smt_call, dict(lab=None), -1),
        (smt_call, dict(lab=labels.data_ptr() + 1), -1), (smt_call, dict(table=edited(smt_tab, 12, d_gamma=None)), -1),
        (smt_call, dict(table=edited(smt_tab, 1, eps=0.0)), -1),
        (smt_call, dict(B=1025), -4), (smt_call, dict(W=69), -4), (smt_call, dict(fc_in=512), -4),
    ]
    for fn, kw, code in cases:
        assert fn(**kw) == code, (fn.__name__, kw)
        assert ops.ctx.launch_count == before, (fn.__name__, kw)
    assert tv_call(B=0) == 0 and smt_call(B=0) == 0 and ops.ctx.launch_count == before
    assert tv_call() == 0 and ops.ctx.launch_count == before + LAUNCHES["tv"]
    assert smt_call(nl=0, lab=None, ls=0, table=conv_table(make_net("smt2").cuda(), False)) == 0
    assert ops.ctx.launch_count == before + LAUNCHES["tv"] + LAUNCHES["smt"]
    torch.cuda.synchronize()


def test_fallbacks_run_the_module():
    """Grad enabled, BatchNorm in training mode, CPU tensors and the SMT network at (65, 69, 2): no launch."""
    from soundspaces_b200.belief_nets import fused_forward
    ops = _ops()
    tv, smt = make_net("tv21").cuda(), make_net("smt2").cuda()
    x, _ = _inputs(4)
    before = ops.ctx.launch_count
    assert fused_forward(tv, x) is None                              # grad enabled
    with torch.no_grad():
        train = copy.deepcopy(tv)
        train.layer2[1].bn1.train()
        assert fused_forward(train, x) is None
        assert fused_forward(make_net("tv21"), x) is None             # CPU parameters
        assert fused_forward(tv, x.cpu()) is None                     # CPU observation
        assert fused_forward(smt, _inputs(4, (65, 69))[0]) is None
        assert ops.ctx.launch_count == before
        assert fused_forward(tv, x) is not None
        assert ops.ctx.launch_count == before + LAUNCHES["tv"]


def _reference_classes():
    """The unpatched and the patched reference-shaped class, with ``cnn_forward`` concatenating the category like
    belief_predictor.py:123-134 when ``has_distractor_sound``."""
    out = []
    for _ in range(2):
        Base = make_reference_class()

        class BeliefPredictor(Base):
            has_distractor_sound = False

            def cnn_forward(self, observations):
                labels = observations["category"] if self.has_distractor_sound else None
                return self.predictor(network_input(observations["spectrogram"], labels))

        out.append(BeliefPredictor)
    return out


@pytest.mark.parametrize("pair", ["offline", "online", "online_distractor"])
def test_patched_update_with_networks(pair):
    """A 50-step rollout written into (T + 1, B, .) rollout slots with networks=True against the unpatched class
    (cuDNN TF32 off): location within belief_oracle.location_bound plus the network tolerance, category within the
    network tolerance, the silent / reset decisions identical, a fixed launch count per call, no host sync."""
    from soundspaces_b200.belief import patch_belief_predictor
    T, B, shape = 50, 8, (65, 26, 2)
    kinds = {"offline": ("tv23", "tv21"), "online": ("smt2", "tv21"), "online_distractor": ("smt23", "tv21")}[pair]
    predictor, classifier = make_net(kinds[0], seed=11).cuda(), make_net(kinds[1], seed=12).cuda()
    Ref, Patched = _reference_classes()
    patch_belief_predictor(Patched, networks=True)
    ref = Ref(B, w=0.5, predictor=predictor, classifier=classifier)
    pat = Patched(B, w=0.5, predictor=predictor, classifier=classifier)
    ref.has_distractor_sound = pat.has_distractor_sound = pair == "online_distractor"
    per_call = LAUNCHES[kinds[0][:-2] if kinds[0].startswith("tv") else "smt"] + LAUNCHES["tv"] + 1
    peak = [0.0]
    hooks = [m.register_forward_hook(lambda m, i, o: peak.__setitem__(0, max(peak[0], o.abs().max().item())))
             for m in (predictor, classifier)]
    seq = bo.make_sequence(31, T, B, p_done=0.08)
    dims = {"spectrogram": shape, "pose": (4,), "location_belief": (2,), "category_belief": (21,), "category": (21,)}
    g = torch.Generator().manual_seed(2)
    cats = torch.softmax(torch.randn(T, B, 21, generator=g) * 3.0, dim=-1)
    storage = {}
    for side in ("ref", "pat"):
        storage[side] = {k: torch.zeros((T + 1, B) + d, device="cuda") for k, d in dims.items()}
        s = storage[side]
        for t in range(T):
            s["spectrogram"][t + 1] = torch.from_numpy(bo.make_spectrograms(seq["silent"][t], shape, t)).cuda() * 4.0
            s["pose"][t + 1] = torch.from_numpy(seq["pose"][t]).cuda()
            s["category"][t + 1] = cats[t].cuda()
    prev = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    ops = _ops()
    try:
        for t in range(T):
            dones = [bool(d) for d in seq["dones"][t]]
            ref.update({k: v[t + 1] for k, v in storage["ref"].items()}, dones)
            obs = {k: v[t + 1] for k, v in storage["pat"].items()}
            before = ops.ctx.launch_count
            torch.cuda.synchronize()
            torch.cuda.set_sync_debug_mode("error")
            try:
                pat.update(obs, dones)
            finally:
                torch.cuda.set_sync_debug_mode(0)
            assert ops.ctx.launch_count == before + per_call
        for h in hooks:
            h.remove()
        obs = {k: v[T] for k, v in storage["pat"].items()}
        loc_before, cat_before = obs["location_belief"].clone(), obs["category_belief"].clone()
        torch.cuda.synchronize()
        torch.cuda._sleep(200_000_000)
        busy = torch.cuda.Event()
        busy.record()
        pat.update(obs, [False] * B)
        assert not busy.query()
        torch.cuda.synchronize()
        obs["location_belief"].copy_(loc_before)
        obs["category_belief"].copy_(cat_before)
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = prev
    r, p = storage["ref"], storage["pat"]
    net_tol = 2e-4 * peak[0]
    assert (p["category_belief"] - r["category_belief"]).abs().max().item() <= net_tol
    assert torch.equal(p["location_belief"] == 10, r["location_belief"] == 10)
    assert torch.equal(p["category_belief"] == np.float32(1 / 21), r["category_belief"] == np.float32(1 / 21))
    scale = max(r["location_belief"].abs().max().item(), r["pose"][..., :2].abs().max().item())
    err = (p["location_belief"] - r["location_belief"]).abs().max().item()
    assert err <= bo.location_bound(scale) + net_tol, err
    assert (r["category_belief"][1:] == np.float32(1 / 21)).all(-1).any()
