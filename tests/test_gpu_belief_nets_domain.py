"""SAVi's belief-predictor ResNet-18s on the GPU across the inputs their entries accept: every spatial size class of
H, W in 1..256, label widths whose stem K leaves tails of several lengths, strided labels, heads of 1..300 outputs with
and without a bias, norm edges (tiny running variances, eps away from 1e-5, constant, zero and badly scaled envs) and
the 1024-env limit.  Each env's outputs are compared with a float64 forward of the same module on their own scale:
``max|got_b - ref_b| <= TOL * max|ref_b|`` for every env b, so a wrong env with small outputs cannot hide behind a
loud one.  Outside the entries' limits ``fused_forward`` and the patched ``update`` run the module instead.

``sweep()`` lists every launch this file makes; tests/test_belief_nets_host.py checks through a restatement of the
host's K-split rule that it reaches every convolution kernel instance's edges."""
import copy

import pytest

from belief_nets_models import make_net, network_input, smt_net
from test_gpu_belief_nets import LAUNCHES, _reference_classes

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
pytest.importorskip("torchvision")

# Per-env tolerance, relative to the env's largest float64 output.  The kernels stay within 3e-5 at every input here
# (H100).  For comparison, torch's float32 forward on a CPU stays within 1.2e-6 on the torchvision net and 4e-5 on
# the SMT net with category channels, but misses by up to 5e-4 (1 x 1), 1e-2 (the all-zero env at 256 x 256) and 0.29
# (1 x 1, eps = 1e-8) on the SMT net without them: there GroupNorm subtracts a group mean that sits very close to
# every element (a zero env is constant per channel after the stem; a 1 x 1 map has groups of 1 to 8 elements).  The
# kernels lose far less to that cancellation than the CPU forward does, so these envs are held to TOL like the others.
TOL = 1e-4

# (H, W): B.  1 x 1 runs every layer on one pixel (P4 = 1, stride-2 convs on a 1-pixel map); 1 x 256 / 256 x 1 and
# 2 x 3 give the maxpool odd and even inputs; 65 x 35 / 65 x 76 are the 22.05 and 48 kHz observations; 256 x 256 is
# the largest input, with the most K ranges per layer and the largest GroupNorm groups.
TV_SHAPES = {(1, 1): 8, (1, 256): 8, (256, 1): 8, (2, 3): 8, (7, 7): 8, (8, 9): 8, (17, 17): 8, (31, 33): 8,
             (65, 35): 8, (65, 76): 8, (256, 256): 2}
# The SMT fc is 128 H4 W4 wide: 128 at 1 x 1 (whose stem GroupNorm groups hold one pixel), 10368 at 65 x 69, 131072
# at 256 x 256.  Each runs without and with the 21 category channels.
SMT_SHAPES = {(1, 1): 8, (8, 8): 8, (65, 69): 8, (33, 200): 4, (256, 256): 2}
SMT_LABELS = (0, 21)
# (2 + n) 49 = 147, 196, 343, 1127, 2058: K tails of 3, 4, 7, 7 and 10 rows past the last 16-row tile
LABEL_WIDTHS = (1, 2, 5, 21, 40)
HEAD_WIDTHS = (1, 8, 9, 300)          # the head runs one warp per output, 8 warps per env
NORM_EDGES = ("tiny_var", "eps_1e-3", "eps_1e-8")
NORM_SHAPES = ((65, 26), (1, 1))
LIMIT = 1024                          # RN_MAX_ENVS
HW = (65, 26)
B = 8


def sweep():
    """Every (smt, H, W, B, n_labels) this file launches, for the host's coverage check."""
    out = []
    for (h, w), b in TV_SHAPES.items():
        out += [(False, h, w, b, 0), (False, h, w, 1, 0)]
    for (h, w), b in SMT_SHAPES.items():
        for n in SMT_LABELS:
            out += [(True, h, w, b, n), (True, h, w, 1, n)]
    out += [(True, *HW, B, n) for n in LABEL_WIDTHS]
    out += [(True, *HW, b, 21) for b in (B, 1)]                            # strided labels
    out += [(smt, *HW, B, 0) for smt in (False, True)]                     # heads
    for hw in NORM_SHAPES:
        out += [(smt, *hw, B, 0) for smt in (False, True)]                 # norm edges
    for smt, n in ((False, 0), (True, 21)):
        out += [(smt, *HW, b, n) for b in (LIMIT, LIMIT - 1, 1)]
    return out


def _ops():
    from soundspaces_b200.renderer import WaveformOps
    return WaveformOps.get("cuda:0")


def _obs(B, hw=HW, seed=0):
    """Spectrogram-like rows (log1p magnitudes >= 0); row 0 silent and row 1 scaled by 1e-3 when there are several."""
    g = torch.Generator().manual_seed(seed)
    x = torch.log1p(torch.rand((B,) + tuple(hw) + (2,), generator=g) * 20.0)
    if B > 1:
        x[0] = 0
        x[1] *= 1e-3
    return x


def _edge_obs(hw, seed=0):
    """Eight envs in one batch: all zero, constant over the pixels (0.7 left, 1.3 right), and spectrogram rows
    scaled by 1e-6, 1e-4, 1e-2, 1, 10 and 1e3."""
    x = _obs(8, hw, seed)
    x[0] = 0
    x[1] = torch.tensor([0.7, 1.3])
    for b, s in enumerate((1e-6, 1e-4, 1e-2, 1.0, 10.0, 1e3)):
        x[2 + b] = _obs(1, hw, seed + 1 + b)[0] * s
    return x


def _labels(B, n, seed=0):
    g = torch.Generator().manual_seed(seed)
    return torch.softmax(torch.randn(B, n, generator=g) * 3.0, dim=1)


def _run(net, x, labels=None):
    ops = _ops()
    if hasattr(net, "avgpool"):
        return ops.resnet18(x, net)
    return ops.smt_resnet18(x, net, labels)


def _ref64(net, x, labels=None):
    ref = copy.deepcopy(net).double()
    with torch.no_grad():
        return ref(network_input(x.double(), None if labels is None else labels.double()))


def check_envs(got, want):
    """max|got_b - want_b| <= TOL max|want_b| for every env b."""
    err = (got.double() - want).abs().amax(dim=1)
    scale = want.abs().amax(dim=1)
    bad = (err > TOL * scale).nonzero().flatten().tolist()
    assert not bad, f"envs {bad}: max|d| / max|ref| = {(err[bad] / scale[bad]).tolist()} > {TOL}"


def _accuracy(net, x, labels=None):
    """Per-env accuracy of a batch, and its last env alone bit-identical to its row."""
    out = _run(net, x, labels)
    check_envs(out, _ref64(net, x, labels))
    one = _run(net, x[-1:].contiguous(), None if labels is None else labels[-1:].contiguous())
    assert torch.equal(one, out[-1:])
    return out


# ---------------------------------------------------------------------------
# spatial shapes
# ---------------------------------------------------------------------------
@pytest.mark.parametrize("hw", list(TV_SHAPES), ids=lambda hw: f"{hw[0]}x{hw[1]}")
def test_tv_shapes(hw):
    net = make_net("tv21", seed=31).cuda()
    _accuracy(net, _obs(TV_SHAPES[hw], hw, seed=32).cuda())
    torch.cuda.synchronize()


@pytest.mark.parametrize("n_labels", SMT_LABELS)
@pytest.mark.parametrize("hw", list(SMT_SHAPES), ids=lambda hw: f"{hw[0]}x{hw[1]}")
def test_smt_shapes(hw, n_labels):
    B = SMT_SHAPES[hw]
    net = smt_net(2 + n_labels, hw, seed=33).cuda()
    _accuracy(net, _obs(B, hw, seed=34).cuda(), _labels(B, n_labels, seed=35).cuda() if n_labels else None)
    torch.cuda.synchronize()


# ---------------------------------------------------------------------------
# label channels
# ---------------------------------------------------------------------------
@pytest.mark.parametrize("n_labels", LABEL_WIDTHS)
def test_label_widths(n_labels):
    net = smt_net(2 + n_labels, HW, seed=36).cuda()
    _accuracy(net, _obs(B, seed=37).cuda(), _labels(B, n_labels, seed=38).cuda())
    torch.cuda.synchronize()


def test_label_row_strides():
    """Labels as columns 5..25 of a (B, 40) tensor (row stride 40) give the contiguous copy's outputs bit for bit; so
    does one env whose (1, 21) label view reports a row stride of 1."""
    from soundspaces_b200.belief_nets import fused_forward
    net = smt_net(23, HW, seed=39).cuda()
    x = _obs(B, seed=40).cuda()
    wide = _labels(B, 40, seed=41).cuda()
    labels = wide[:, 5:26]
    assert labels.stride() == (40, 1)
    dense = _run(net, x, labels.contiguous())
    check_envs(dense, _ref64(net, x, labels))
    assert torch.equal(_run(net, x, labels), dense)
    with torch.no_grad():
        assert torch.equal(fused_forward(net, x, labels), dense)
    one = wide[0, 5:26].contiguous().as_strided((1, 21), (1, 1))
    assert one.stride(0) == 1
    x1 = x[:1].contiguous()
    want = _run(net, x1, one.contiguous())
    assert torch.equal(_run(net, x1, one), want)
    with torch.no_grad():
        assert torch.equal(fused_forward(net, x1, one), want)
    torch.cuda.synchronize()


# ---------------------------------------------------------------------------
# heads
# ---------------------------------------------------------------------------
@pytest.mark.parametrize("bias", [True, False], ids=["bias", "no_bias"])
@pytest.mark.parametrize("n_out", HEAD_WIDTHS)
@pytest.mark.parametrize("kind", ["tv", "smt"])
def test_heads(kind, n_out, bias):
    net = make_net(f"tv{n_out}", seed=42) if kind == "tv" else smt_net(2, HW, n_out=n_out, seed=42)
    if not bias:
        net.fc.bias = None
    net = net.cuda()
    out = _accuracy(net, _obs(B, seed=43).cuda())
    assert out.shape == (B, n_out)
    torch.cuda.synchronize()


# ---------------------------------------------------------------------------
# norm edges
# ---------------------------------------------------------------------------
def _norm_edge(net, edge):
    norms = [m for m in net.modules() if isinstance(m, (torch.nn.BatchNorm2d, torch.nn.GroupNorm))]
    if edge == "tiny_var":
        # every fourth channel of the stem norm and of one norm per stage: (x - mean) / sqrt(1e-8 + eps)
        with torch.no_grad():
            for m in (net.bn1, net.layer1[0].bn2, net.layer2[0].bn1, net.layer3[1].bn1, net.layer4[0].downsample[1]):
                m.running_var[::4] = 1e-8
    else:
        for m in norms:
            m.eps = float(edge.split("_")[1])
    return net


@pytest.mark.parametrize("hw", NORM_SHAPES, ids=lambda hw: f"{hw[0]}x{hw[1]}")
@pytest.mark.parametrize("kind,edge", [("tv", e) for e in NORM_EDGES] + [("smt", e) for e in NORM_EDGES[1:]])
def test_norm_edges(kind, edge, hw):
    """Zero, constant and 1e-6 .. 1e3-scaled envs in one batch under each norm edge."""
    net = make_net("tv21", seed=44) if kind == "tv" else smt_net(2, hw, seed=44)
    net = _norm_edge(net, edge).cuda()
    _accuracy(net, _edge_obs(hw, seed=45).cuda())
    torch.cuda.synchronize()


# ---------------------------------------------------------------------------
# the 1024-env limit
# ---------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["tv", "smt"])
def test_batch_limit(kind):
    """At B = 1024 every env passes the float64 check; envs 0, 1, 511 and 1023 alone, a permuted batch and the first
    1023 envs (whose last N tiles end elsewhere) give the same rows bit for bit."""
    net = (make_net("tv21", seed=46) if kind == "tv" else make_net("smt23", seed=46)).cuda()
    x = _obs(LIMIT, seed=47).cuda()
    labels = _labels(LIMIT, 21, seed=48).cuda() if kind == "smt" else None

    def sub(idx):
        return x[idx].contiguous(), None if labels is None else labels[idx].contiguous()

    full = _run(net, x, labels)
    check_envs(full, _ref64(net, x, labels))
    for b in (0, 1, 511, 1023):
        assert torch.equal(_run(net, *sub(slice(b, b + 1))), full[b:b + 1]), b
    perm = torch.randperm(LIMIT, generator=torch.Generator().manual_seed(49)).cuda()
    assert torch.equal(_run(net, *sub(perm))[torch.argsort(perm)], full)
    assert torch.equal(_run(net, *sub(slice(0, LIMIT - 1))), full[:LIMIT - 1])
    torch.cuda.synchronize()


# ---------------------------------------------------------------------------
# outside the limits: the module runs
# ---------------------------------------------------------------------------
def test_fused_forward_falls_back_outside_the_limits():
    """B = 1025, a 257-wide torchvision input and a 257-tall SMT input: None, no launch, no error."""
    from soundspaces_b200.belief_nets import MAX_ENVS, MAX_HW, fused_forward
    assert (MAX_ENVS, MAX_HW) == (LIMIT, 256)
    ops = _ops()
    tv, smt = make_net("tv21").cuda(), make_net("smt23").cuda()
    tall = smt_net(2, (MAX_HW + 1, 26)).cuda()
    x = _obs(MAX_ENVS + 1, seed=50).cuda()
    labels = _labels(MAX_ENVS + 1, 21, seed=51).cuda()
    with torch.no_grad():
        before = ops.ctx.launch_count
        assert fused_forward(tv, x) is None
        assert fused_forward(smt, x, labels) is None
        assert fused_forward(tv, _obs(2, (65, MAX_HW + 1)).cuda()) is None
        assert fused_forward(tall, _obs(2, (MAX_HW + 1, 26)).cuda()) is None
        assert ops.ctx.launch_count == before
        assert fused_forward(tv, _obs(2, (65, MAX_HW)).cuda()) is not None
        assert fused_forward(smt, x[:MAX_ENVS], labels[:MAX_ENVS]) is not None
        assert ops.ctx.launch_count == before + LAUNCHES["tv"] + LAUNCHES["smt"]
    torch.cuda.synchronize()


def test_patched_update_falls_back_above_1024_envs():
    """1025 envs with networks=True: the original update runs, networks included, and writes the unpatched class's
    beliefs bit for bit over two steps; nothing is launched in the library."""
    from soundspaces_b200.belief import patch_belief_predictor
    n = LIMIT + 1
    predictor, classifier = make_net("tv23", seed=52).cuda(), make_net("tv21", seed=53).cuda()
    Ref, Patched = _reference_classes()
    patch_belief_predictor(Patched, networks=True)
    ref = Ref(n, w=0.5, predictor=predictor, classifier=classifier)
    pat = Patched(n, w=0.5, predictor=predictor, classifier=classifier)
    ops = _ops()
    before = ops.ctx.launch_count
    beliefs = {}
    for side, model in (("ref", ref), ("pat", pat)):
        obs = {"location_belief": torch.zeros(n, 2, device="cuda"), "category_belief": torch.zeros(n, 21, device="cuda")}
        for t in range(2):
            obs["spectrogram"] = _obs(n, seed=55 + t).cuda()
            obs["spectrogram"][3::7] = 0                              # silent envs
            obs["pose"] = torch.randn(n, 4, generator=torch.Generator().manual_seed(57 + t)).cuda()
            dones = [t == 1 and i % 5 == 0 for i in range(n)]
            model.update(obs, dones)
        beliefs[side] = (obs["location_belief"], obs["category_belief"])
    assert ops.ctx.launch_count == before
    for r, p in zip(beliefs["ref"], beliefs["pat"]):
        assert torch.equal(r, p)
    assert (beliefs["ref"][0] == 10).all(1).any()                      # silent on the first step
    assert pat.last_pointgoal[1] is not None and pat.last_label[1] is not None   # the device path leaves the lists
