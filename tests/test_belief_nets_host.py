"""Host side of the belief-predictor ResNets: the structural layout checks of ``soundspaces_b200.belief_nets`` on
torchvision's resnet18 and an independent restatement of the SMT network, every single deviation they refuse, the
parameter table's order and the entries' arguments (with the library replaced by a recorder), and the dispatch of
``fused_forward``.  No GPU."""
import copy
import ctypes as C
from types import SimpleNamespace

import pytest

torch = pytest.importorskip("torch")
pytest.importorskip("torchvision")
nn = torch.nn

from belief_nets_models import make_net, smt_net  # noqa: E402
from soundspaces_b200 import belief_nets as bn  # noqa: E402

CPU = torch.device("cpu")


def test_accepts_both_topologies():
    assert bn.resnet18_layout_error(make_net("tv21")) == ""
    assert bn.resnet18_layout_error(make_net("tv23"), CPU) == ""
    assert bn.smt_resnet18_layout_error(make_net("smt2"), 2, (65, 26), CPU) == ""
    assert bn.smt_resnet18_layout_error(make_net("smt23"), 23, (65, 26), CPU) == ""
    # each topology is refused by the other's check
    assert bn.resnet18_layout_error(make_net("smt2")) != ""
    assert bn.smt_resnet18_layout_error(make_net("tv21"), 2) != ""
    assert bn.smt_resnet18_layout_error(make_net("smt23"), 2) != ""


def _set(net, path, value):
    *parent, last = path.split(".")
    m = net
    for p in parent:
        m = m[int(p)] if p.isdigit() else getattr(m, p)
    if last.isdigit():
        m[int(last)] = value
    else:
        setattr(m, last, value)


TV_DEVIATIONS = {
    "stem_padding": lambda n: _set(n, "conv1", nn.Conv2d(2, 64, 7, 2, 2, bias=False)),
    "stem_stride": lambda n: _set(n, "conv1", nn.Conv2d(2, 64, 7, 1, 3, bias=False)),
    "stem_bias": lambda n: _set(n, "conv1", nn.Conv2d(2, 64, 7, 2, 3, bias=True)),
    "stem_channels": lambda n: _set(n, "conv1", nn.Conv2d(3, 64, 7, 2, 3, bias=False)),
    "block_stride": lambda n: _set(n, "layer3.1.conv1", nn.Conv2d(256, 256, 3, 2, 1, bias=False)),
    "block_padding": lambda n: _set(n, "layer2.0.conv2", nn.Conv2d(128, 128, 3, 1, 0, bias=False)),
    "block_dilation": lambda n: _set(n, "layer1.0.conv1", nn.Conv2d(64, 64, 3, 1, 1, dilation=2, bias=False)),
    "width": lambda n: _set(n, "layer4.1.bn2", nn.BatchNorm2d(256)),
    "ds_stride": lambda n: _set(n, "layer2.0.downsample.0", nn.Conv2d(64, 128, 1, 1, bias=False)),
    "bn_training": lambda n: n.layer3[0].bn1.train(),
    "bn_no_stats": lambda n: _set(n, "layer1.1.bn2", nn.BatchNorm2d(64, track_running_stats=False).eval()),
    "bn_not_affine": lambda n: _set(n, "bn1", nn.BatchNorm2d(64, affine=False).eval()),
    "group_norm": lambda n: _set(n, "bn1", nn.GroupNorm(16, 64)),
    "extra_module": lambda n: n.layer2[1].add_module("extra", nn.Identity()),
    "extra_top_module": lambda n: n.add_module("dropout", nn.Dropout()),
    "missing_downsample": lambda n: _set(n, "layer3.0.downsample", None),
    "maxpool": lambda n: _set(n, "maxpool", nn.MaxPool2d(2, 2)),
    "avgpool": lambda n: _set(n, "avgpool", nn.AdaptiveAvgPool2d((2, 1))),
    "fc_width": lambda n: _set(n, "fc", nn.Linear(256, 21)),
    "relu": lambda n: _set(n, "layer1.0.relu", nn.GELU()),
}

SMT_DEVIATIONS = {      # (network, its input channels)
    "stem_padding": lambda n, c: _set(n, "conv1", nn.Conv2d(c, 16, 7, 1, 2, bias=False)),
    "stem_stride": lambda n, c: _set(n, "conv1", nn.Conv2d(c, 16, 7, 2, 3, bias=False)),
    "stem_bias": lambda n, c: _set(n, "conv1", nn.Conv2d(c, 16, 7, 1, 3, bias=True)),
    "stem_channels": lambda n, c: _set(n, "conv1", nn.Conv2d(c + 1, 16, 7, 1, 3, bias=False)),
    "block_stride": lambda n, c: _set(n, "layer2.1.conv1", nn.Conv2d(32, 32, 3, 2, 1, bias=False)),
    "block_padding": lambda n, c: _set(n, "layer1.0.conv2", nn.Conv2d(16, 16, 3, 1, 0, bias=False)),
    "width": lambda n, c: _set(n, "layer3.1.conv2", nn.Conv2d(64, 48, 3, 1, 1, bias=False)),
    "groups_8": lambda n, c: _set(n, "layer2.0.bn1", nn.GroupNorm(8, 32)),
    "groups_32": lambda n, c: _set(n, "layer4.0.downsample.1", nn.GroupNorm(32, 128)),
    "gn_not_affine": lambda n, c: _set(n, "bn1", nn.GroupNorm(16, 16, affine=False)),
    "batch_norm": lambda n, c: _set(n, "layer1.1.bn1", nn.BatchNorm2d(16).eval()),
    "grouped_conv": lambda n, c: _set(n, "layer3.0.conv2", nn.Conv2d(64, 64, 3, 1, 1, groups=2, bias=False)),
    "extra_module": lambda n, c: n.layer4[0].add_module("extra", nn.ReLU()),
    "extra_top_module": lambda n, c: n.add_module("avgpool", nn.AdaptiveAvgPool2d(1)),
    "ds_kernel": lambda n, c: _set(n, "layer2.0.downsample.0", nn.Conv2d(16, 32, 3, 2, 1, bias=False)),
    "fc_width": lambda n, c: _set(n, "fc", nn.Linear(4096, 2)),
}


@pytest.mark.parametrize("name", sorted(TV_DEVIATIONS))
def test_resnet18_refuses_each_deviation(name):
    net = make_net("tv21")
    TV_DEVIATIONS[name](net)
    assert bn.resnet18_layout_error(net) != "", name


@pytest.mark.parametrize("channels", [2, 23])
@pytest.mark.parametrize("name", sorted(SMT_DEVIATIONS))
def test_smt_refuses_each_deviation(name, channels):
    net = make_net(f"smt{channels}")
    SMT_DEVIATIONS[name](net, channels)
    assert bn.smt_resnet18_layout_error(net, channels, (65, 26)) != "", name


def test_smt_fc_width_follows_the_observation():
    net = make_net("smt2")
    assert bn.smt_out_hw(65, 26) == (9, 4)
    assert bn.smt_resnet18_layout_error(net, 2, (65, 26)) == ""
    assert "fc takes 4608" in bn.smt_resnet18_layout_error(net, 2, (65, 69))     # 44.1 kHz: 128 * 9 * 9
    assert bn.smt_resnet18_layout_error(net, 2) == ""                          # shape not given: not checked


def test_parameters_must_be_float32_contiguous_on_the_device():
    net = make_net("tv21")
    assert bn.resnet18_layout_error(net, torch.device("cuda", 0)) != ""        # CPU parameters
    net.layer2[0].conv1.weight.data = net.layer2[0].conv1.weight.data.transpose(2, 3).contiguous().transpose(2, 3)
    assert "contiguous" in bn.resnet18_layout_error(net, CPU)
    smt = make_net("smt2").double()
    assert "float32" in bn.smt_resnet18_layout_error(smt, 2, (65, 26), CPU)


# ---------------------------------------------------------------------------
# the parameter table and the entries' arguments, the library replaced by a recorder
# ---------------------------------------------------------------------------
class FakeLib:
    def __init__(self):
        self.calls = []

    def _record(self, name, args):
        table = args[5] if name == "ssb_resnet18_batch" else args[8]
        rows = [(t.d_weight, t.d_gamma, t.d_beta, t.d_mean, t.d_var, t.eps) for t in table]
        self.calls.append((name, args, rows))
        return 0

    def ssb_resnet18_batch(self, *args):
        return self._record("ssb_resnet18_batch", args)

    def ssb_smt_resnet18_batch(self, *args):
        return self._record("ssb_smt_resnet18_batch", args)


def _cpu_ops():
    from soundspaces_b200.renderer import WaveformOps
    ops = object.__new__(WaveformOps)
    ops.device = CPU
    ops.lib = FakeLib()
    ops.ctx = SimpleNamespace(handle=None, check=lambda rc, what: None)
    ops._stream = lambda: None
    return ops


def _documented_order(net):
    order = ["conv1/bn1"]
    for s in range(1, 5):
        for j in range(2):
            order += [f"layer{s}.{j}.conv1/bn1", f"layer{s}.{j}.conv2/bn2"]
            if s > 1 and j == 0:
                order.append(f"layer{s}.{j}.downsample.0/1")
    mods = dict(net.named_modules())
    pairs = []
    for entry in order:
        conv, norm = entry.split("/")
        base = conv.rsplit(".", 1)[0] if "." in conv else ""
        pairs.append((mods[conv], mods[(base + "." if base else "") + norm]))
    return pairs


def test_resnet18_table_in_module_order():
    ops = _cpu_ops()
    net = make_net("tv23")
    x = torch.rand(3, 65, 69, 2)
    out = ops.resnet18(x, net)
    assert out.shape == (3, 23)
    ((name, args, rows),) = ops.lib.calls
    assert name == "ssb_resnet18_batch"
    assert args[1:5] == (3, x.data_ptr(), 65, 69)
    assert args[6:11] == (net.fc.weight.data_ptr(), net.fc.bias.data_ptr(), 512, 23, out.data_ptr())
    pairs = _documented_order(net)
    assert len(rows) == len(pairs) == 20
    for row, (conv, norm) in zip(rows, pairs):
        assert row[:5] == (conv.weight.data_ptr(), norm.weight.data_ptr(), norm.bias.data_ptr(),
                           norm.running_mean.data_ptr(), norm.running_var.data_ptr())
        assert row[5] == pytest.approx(norm.eps)


@pytest.mark.parametrize("channels", [2, 23])
def test_smt_table_in_module_order(channels):
    ops = _cpu_ops()
    net = make_net(f"smt{channels}")
    x = torch.rand(4, 65, 26, 2)
    labels = torch.rand(4, 30)[:, :21] if channels == 23 else None         # row stride 30
    ops.smt_resnet18(x, net, labels)
    ((name, args, rows),) = ops.lib.calls
    assert name == "ssb_smt_resnet18_batch"
    assert args[1:5] == (4, x.data_ptr(), 65, 26)
    if labels is None:
        assert args[5:8] == (None, 0, 0)
    else:
        assert args[5:8] == (labels.data_ptr(), 21, 30)
    assert args[9:13] == (net.fc.weight.data_ptr(), net.fc.bias.data_ptr(), 4608, 2)
    for row, (conv, norm) in zip(rows, _documented_order(net)):
        assert row[:5] == (conv.weight.data_ptr(), norm.weight.data_ptr(), norm.bias.data_ptr(), None, None)


def test_replaced_parameter_is_read_at_call_time():
    ops = _cpu_ops()
    net = make_net("smt2")
    x = torch.rand(2, 65, 26, 2)
    ops.smt_resnet18(x, net)
    old = net.layer3[1].conv2.weight                    # kept alive so the new tensor cannot reuse its address
    net.layer3[1].conv2.weight = nn.Parameter(torch.randn(64, 64, 3, 3))
    ops.smt_resnet18(x, net)
    a, b = ops.lib.calls
    k = 14                                              # stem, layer1 (4), layer2 (5), layer3.0 (3), layer3.1.conv1
    assert a[2][k][0] == old.data_ptr() and b[2][k][0] == net.layer3[1].conv2.weight.data_ptr() != old.data_ptr()


def _refused(fn):
    with pytest.raises(ValueError):
        fn()


def test_wrappers_refuse_bad_inputs():
    ops = _cpu_ops()
    tv, smt = make_net("tv21"), make_net("smt23")
    x = torch.rand(2, 65, 26, 2)
    _refused(lambda: ops.resnet18(x.double(), tv))
    _refused(lambda: ops.resnet18(x.permute(0, 3, 1, 2), tv))
    _refused(lambda: ops.resnet18(x, smt))
    _refused(lambda: ops.smt_resnet18(x, smt))                                # 23 channels without labels
    _refused(lambda: ops.smt_resnet18(x, smt, torch.rand(2, 21).double()))
    _refused(lambda: ops.smt_resnet18(x, smt, torch.rand(21, 2).t()))        # column stride 2
    _refused(lambda: ops.smt_resnet18(x, smt, torch.rand(3, 21)))
    _refused(lambda: ops.smt_resnet18(torch.rand(2, 65, 69, 2), smt, torch.rand(2, 21)))   # fc width
    bad = copy.deepcopy(tv)
    bad.layer1[0].bn1.train()
    _refused(lambda: ops.resnet18(x, bad))
    assert not ops.lib.calls


def test_abi_prototypes():
    from soundspaces_b200 import _lib
    assert C.sizeof(_lib.ResnetConv) == 48
    r, a = _lib.EXPORTS["ssb_resnet18_batch"]
    assert r is C.c_int and len(a) == 12
    r, a = _lib.EXPORTS["ssb_smt_resnet18_batch"]
    assert r is C.c_int and len(a) == 15 and a[7] is C.c_int64


# ---------------------------------------------------------------------------
# fused_forward: what takes the library path
# ---------------------------------------------------------------------------
class FakeCuda(torch.Tensor):
    @property
    def is_cuda(self):
        return True


@pytest.fixture
def device_calls(monkeypatch):
    from soundspaces_b200.renderer import WaveformOps
    calls = []

    class Recorder:
        def resnet18(self, x, net):
            calls.append(("resnet18", x, net, None))
            return "fused"

        def smt_resnet18(self, x, net, labels=None):
            calls.append(("smt_resnet18", x, net, labels))
            return "fused"

    monkeypatch.setattr(WaveformOps, "get", classmethod(lambda cls, device="cuda:0": Recorder()))
    return calls


def test_fused_forward_dispatch(device_calls):
    x = torch.rand(3, 65, 26, 2).as_subclass(FakeCuda)
    labels = torch.rand(3, 21).as_subclass(FakeCuda)
    tv, smt2, smt23 = make_net("tv21"), make_net("smt2"), make_net("smt23")
    with torch.no_grad():
        assert bn.fused_forward(tv, x) == "fused"
        assert bn.fused_forward(smt2, x) == "fused"
        assert bn.fused_forward(smt23, x, labels) == "fused"
        assert bn.fused_forward(smt23, x) is None                      # 23 channels need the labels
        assert bn.fused_forward(tv, x, labels) is None                  # the torchvision stem takes 2 channels
        assert bn.fused_forward(smt2, torch.rand(3, 65, 69, 2).as_subclass(FakeCuda)) is None     # fc width
        assert bn.fused_forward(tv, torch.rand(3, 65, 26, 2)) is None   # not CUDA
        assert bn.fused_forward(tv, x.double()) is None
    assert bn.fused_forward(tv, x) is None                              # grad enabled
    assert [c[0] for c in device_calls] == ["resnet18", "smt_resnet18", "smt_resnet18"]
    assert device_calls[2][3] is labels


def test_fused_forward_outside_the_entries_limits(device_calls):
    """More than MAX_ENVS envs, or an observation taller or wider than MAX_HW: None (the entries would refuse them)."""
    big = torch.rand(bn.MAX_ENVS + 1, 65, 26, 2).as_subclass(FakeCuda)
    labels = torch.rand(bn.MAX_ENVS + 1, 21).as_subclass(FakeCuda)
    tall = smt_net(2, (bn.MAX_HW + 1, 26))
    with torch.no_grad():
        assert bn.fused_forward(make_net("tv21"), big) is None
        assert bn.fused_forward(make_net("smt23"), big, labels) is None
        assert bn.fused_forward(make_net("tv21"), torch.rand(2, 65, bn.MAX_HW + 1, 2).as_subclass(FakeCuda)) is None
        assert bn.fused_forward(tall, torch.rand(2, bn.MAX_HW + 1, 26, 2).as_subclass(FakeCuda)) is None
        assert not device_calls
        edge = smt_net(2, (bn.MAX_HW, 26))
        assert bn.fused_forward(edge, torch.rand(2, bn.MAX_HW, 26, 2).as_subclass(FakeCuda)) == "fused"
        assert bn.fused_forward(make_net("tv21"), big[:bn.MAX_ENVS]) == "fused"


# ---------------------------------------------------------------------------
# the K split of every conv, restated, against the GPU sweep of tests/test_gpu_belief_nets_domain.py
# ---------------------------------------------------------------------------
RN_TK = 16


def rn_layer(ic, oc, ks, stride, pad, h, w):
    """rn_layer of ssb200.cu (static RnLayer rn_layer, just above rn_launch_conv): output size, the M tile tm and
    the K split (S ranges of kps rows, kps a multiple of RN_TK), chosen from the layer's shape alone."""
    ho, wo = (h + 2 * pad - ks) // stride + 1, (w + 2 * pad - ks) // stride + 1
    tm = 16 if oc <= 16 else 32 if oc <= 32 else 64
    K = ic * ks * ks
    kt, tn = (K + RN_TK - 1) // RN_TK, 4096 // tm
    tiles = (oc + tm - 1) // tm * ((8 * ho * wo + tn - 1) // tn)
    s0 = max(1, min(max(1, kt // 4), 512 // tiles))
    kps = (kt + s0 - 1) // s0 * RN_TK
    return dict(ks=ks, ho=ho, wo=wo, tm=tm, K=K, kps=kps, S=(K + kps - 1) // kps, h=h, w=w, stride=stride)


def rn_layers(smt, H, W, n_labels):
    """The 20 layers of resnet18() in ssb200.cu (the geometry loop after the shape checks), and the stem's output."""
    width = (16, 32, 64, 128) if smt else (64, 128, 256, 512)
    L = [rn_layer(2 + n_labels if smt else 2, width[0], 7, 1 if smt else 2, 3, H, W)]
    h, w = L[0]["ho"], L[0]["wo"]
    if not smt:
        h, w = (h - 1) // 2 + 1, (w - 1) // 2 + 1                      # MaxPool2d(3, 2, 1)
    ic = width[0]
    for s in range(4):
        for blk in range(2):
            stride = 2 if s > 0 and blk == 0 else 1
            a = rn_layer(ic, width[s], 3, stride, 1, h, w)
            L += [a, rn_layer(width[s], width[s], 3, 1, 1, a["ho"], a["wo"])]
            if stride == 2:
                L.append(rn_layer(ic, width[s], 1, 2, 0, h, w))
            h, w, ic = a["ho"], a["wo"], width[s]
    return L


# rn_conv_kernel<KS, OBS, TM> instances rn_launch_conv launches, by (KS, TM)
INSTANCES = {(7, 16), (7, 64), (3, 16), (3, 32), (3, 64), (1, 32), (1, 64)}
# What rn_layer never produces for H, W <= 256:
# - S > 1 for the torchvision stem (K = 98, kt = 7, so kt / 4 = 1) and the SMT layer2 downsample (K = 16, kt = 1);
# - a last K range shorter than kps for the 1x1 TM = 64 convs (K = 32, 64, 128 or 256: wherever S > 1, kps divides K);
# - a partial 16-row K tile for any 3x3 or 1x1 conv (K = 9 IC or IC, IC a multiple of 16): only the stems have one.
ONLY_S1 = {(7, 64), (1, 32)}
NO_SHORT_RANGE = ONLY_S1 | {(1, 64)}


def test_rn_layer_mirror_matches_the_entries_geometry():
    """The mirror's final maps give the fc widths the layout checks expect, and its K splits cover K exactly."""
    for H, W in ((1, 1), (65, 26), (65, 69), (256, 256), (2, 255)):
        tv, smt = rn_layers(False, H, W, 0), rn_layers(True, H, W, 21)
        assert (smt[-3]["ho"], smt[-3]["wo"]) == bn.smt_out_hw(H, W)
        for L in (tv, smt):
            assert len(L) == bn.N_CONVS and {(l["ks"], l["tm"]) for l in L} <= INSTANCES
            for l in L:
                assert l["kps"] % RN_TK == 0 and (l["S"] - 1) * l["kps"] < l["K"] <= l["S"] * l["kps"]


def test_gpu_sweep_reaches_every_conv_instance_edge():
    """Every rn_conv_kernel instance meets S = 1 and S > 1 (where rn_layer allows both), a last K range shorter than
    kps, and an exactly full and a partial last N tile (N = B HO WO columns of 4096 / TM); both stems meet a partial
    K tile.  Also the network-level edges: a 1 x 1 and a larger final map, odd and even maxpool inputs, a stride-2
    conv on a 1-pixel map, SMT heads of 128 and 131072 features, and stem GroupNorm groups of one pixel."""
    from test_gpu_belief_nets_domain import sweep
    seen = {i: set() for i in INSTANCES}
    smt_stem_tails, net_edges = set(), set()
    for smt, H, W, B, n in sweep():
        L = rn_layers(smt, H, W, n)
        for l in L:
            i = (l["ks"], l["tm"])
            seen[i].add("S=1" if l["S"] == 1 else "S>1")
            if l["S"] > 1 and l["K"] % l["kps"]:
                seen[i].add("short last range")
            seen[i].add("partial N" if B * l["ho"] * l["wo"] % (4096 // l["tm"]) else "full N")
            if l["K"] % RN_TK:
                seen[i].add("K tail")
            if l["stride"] == 2 and l["h"] * l["w"] == 1:
                net_edges.add("stride 2 on 1 pixel")
        p4 = L[-3]["ho"] * L[-3]["wo"]
        if smt:
            smt_stem_tails.add(L[0]["K"] % RN_TK)
            net_edges.add(f"smt fc {128 * p4}")
            if H * W == 1:
                net_edges.add("smt stem group of 1 pixel")
        else:
            net_edges.add("tv P4 = 1" if p4 == 1 else "tv P4 > 1")
            net_edges.add({0: "even", 1: "odd"}[L[0]["ho"] % 2] + " maxpool rows")
            net_edges.add({0: "even", 1: "odd"}[L[0]["wo"] % 2] + " maxpool columns")
    for i in INSTANCES:
        want = {"S=1", "partial N", "full N"} | (set() if i in ONLY_S1 else {"S>1"})
        want |= (set() if i in NO_SHORT_RANGE else {"short last range"}) | ({"K tail"} if i[0] == 7 else set())
        assert want <= seen[i], (i, want - seen[i])
    assert ONLY_S1.isdisjoint(i for i in INSTANCES if "S>1" in seen[i])
    assert len(smt_stem_tails - {0}) >= 4, smt_stem_tails
    assert {"stride 2 on 1 pixel", "smt fc 128", "smt fc 131072", "smt stem group of 1 pixel", "tv P4 = 1",
            "tv P4 > 1", "even maxpool rows", "odd maxpool rows", "even maxpool columns",
            "odd maxpool columns"} <= net_edges, net_edges
