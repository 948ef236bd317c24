"""AV-WaN's fused map encoder (``ssb_map_encoder_batch``) on the GPU across the layouts its entry accepts, not only
``MapCNN``'s: non-square kernels and strides in every layer, each of the three conv kernel instances on non-reference
parameters, every conv3 kernel instance at sh != sw, idle cluster ranks and partial conv1 rows, conv2 slices and
conv3-gather owners, map channels 1 to 8, bias=False, F and hidden off the Linear's tiles, the shared-memory limit
through each branch of its formula, every combination of the relu flags, 65535 envs, and NaN / Inf / badly scaled /
all-zero maps.  The entry is also called directly: each refusal returns its code and message and launches nothing, and
more than 2^31 - 1 conv3 features are refused (in the visual entry too).  The cases are listed in
tests/map_cnn_domain_cases.py; tests/test_map_cnn_domain_host.py checks that they reach every tile edge.

Accuracy: each env is compared with a float64 forward of the same module on the CPU,
``max|got_b - ref_b| <= 1e-4 * max|ref_b|`` over the finite values, and the NaN, +Inf and -Inf positions must equal
float64's exactly.  It is checked on the conv3 features and on the Linear's pre-activation (the entry called with
lin_relu = 0); lin_relu = 1 must then be torch's ReLU of it bit for bit, which keeps the check meaningful where the
ReLU zeroes a whole env.

Calibration (tests/test_map_cnn_domain_host.py: torch's float32 forward on a CPU against float64 on every case and
input here, max over envs of the error over max|ref_b|): 0 .. 3.7e-6, that is at most 0.037 of the bar; the worst is
the conv3-phase limit case (117504 features), then H1 = 1 (3.0e-6).
"""
import copy
import itertools

import pytest

import map_cnn_domain_cases as cases
from map_cnn_models import MapCNN, map_obs

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
nn = torch.nn

DEV = "cuda:0"
SSB_E_INVALID_ARG, SSB_E_SHAPE = -1, -4


def _ops():
    from soundspaces_b200.renderer import WaveformOps
    return WaveformOps.get(DEV)


def _ptr(t):
    return t.data_ptr() if t is not None else None


def same(a, b):
    """Equal values, NaN at the same positions."""
    return (a.shape == b.shape and torch.equal(a.isnan(), b.isnan())
            and torch.equal(torch.where(a.isnan(), 0.0, a), torch.where(b.isnan(), 0.0, b)))


def check_env(got, ref):
    """Per env b: the NaN / +Inf / -Inf pattern of float64's, and max|got_b - ref_b| <= 1e-4 max|ref_b| over the
    finite values."""
    got = got.detach().cpu().double()
    assert got.shape == ref.shape
    for b in range(ref.shape[0]):
        g, r = got[b], ref[b]
        for f in (torch.isnan, torch.isposinf, torch.isneginf):
            assert torch.equal(f(g), f(r)), f"env {b}: {f.__name__} pattern differs from float64"
        fin = torch.isfinite(r)
        if fin.any():
            scale = r[fin].abs().max().item()
            err = (g[fin] - r[fin]).abs().max().item()
            assert err <= 1e-4 * scale, f"env {b}: max err {err:.3g} > 1e-4 * {scale:.3g}"


def map_cnn(c, seed=0):
    return cases.make_cnn(c, seed).to(DEV)


def map_input(c, B, seed=1, kind="dense", scale=1.0):
    """(B, H, W, C) on the GPU: 'gm' 0 / 1 occupancy, 'am' sparse non-negative, 'dense' standard normal (the inputs of
    the host file's calibration)."""
    return (map_obs(B, c["H"], c["W"], c["C"], seed=seed, kind=kind) * scale).to(DEV)


def conv_layers(cnn, relu=(1, 1, 0)):
    from soundspaces_b200 import _lib
    layers = (_lib.Conv2dLayer * 3)()
    for i, (conv, r) in enumerate(zip((cnn[0], cnn[2], cnn[4]), relu)):
        layers[i] = _lib.Conv2dLayer(conv.weight.data_ptr(), _ptr(conv.bias), conv.out_channels, *conv.kernel_size,
                                     *conv.stride, r)
    return layers


_DEFAULT = object()


def map_entry(ops, cnn, x, lin_relu=1, relu=(1, 1, 0), layers=None, B=None, C=None, H=None, W=None, hidden=None,
              lin_weight=None, lin_bias=_DEFAULT, feats=None, out=None, map_ptr=_DEFAULT):
    """ssb_map_encoder_batch called directly -> (rc, features, out); any argument can be overridden."""
    n, h, w, ch = x.shape
    lin = cnn[6]
    f = torch.full((max(n, 1), lin.in_features), float("nan"), device=DEV)
    o = torch.full((max(n, 1), lin.out_features), float("nan"), device=DEV)
    rc = ops.lib.ssb_map_encoder_batch(
        ops.ctx.handle, n if B is None else B, x.data_ptr() if map_ptr is _DEFAULT else map_ptr,
        ch if C is None else C, h if H is None else H, w if W is None else W,
        conv_layers(cnn, relu) if layers is None else layers,
        lin.weight.data_ptr() if lin_weight is None else lin_weight, _ptr(lin.bias) if lin_bias is _DEFAULT else lin_bias,
        lin.out_features if hidden is None else hidden, lin_relu, f.data_ptr() if feats is None else feats,
        o.data_ptr() if out is None else out, ops._stream())
    return rc, f[:n], o[:n]


def run_map(cnn, x, lin_relu, relu=(1, 1, 0)):
    ops = _ops()
    before = ops.ctx.launch_count
    rc, f, o = map_entry(ops, cnn, x, lin_relu, relu)
    assert rc == 0, ops.lib.ssb_last_error(ops.ctx.handle)
    assert ops.ctx.launch_count - before == 2
    return f, o


def ref64(cnn, x, idx=None, relu=(1, 1, 0)):
    """(features, pre-activation) of ``cnn`` with the given conv relu flags in float64 on the CPU for the envs ``idx``
    (all when None)."""
    m = copy.deepcopy(cnn).cpu().double()
    y = (x if idx is None else x[idx]).cpu().double().permute(0, 3, 1, 2)
    with torch.no_grad():
        for conv, r in zip((m[0], m[2], m[4]), relu):
            y = conv(y)
            if r:
                y = torch.relu(y)
        feats = y.flatten(1)
        return feats, m[6](feats)


def check_map(cnn, x, idx=None, relu=(1, 1, 0)):
    """Features and pre-activation against float64 per env; lin_relu = 1 is relu of lin_relu = 0 bit for bit.
    -> (features, pre-activation, output) of the whole batch."""
    f, pre = run_map(cnn, x, 0, relu)
    f1, out = run_map(cnn, x, 1, relu)
    assert same(f1, f) and same(out, torch.relu(pre))
    f_ref, pre_ref = ref64(cnn, x, idx, relu)
    sel = slice(None) if idx is None else torch.tensor(idx, device=DEV)
    check_env(f[sel], f_ref)
    check_env(pre[sel], pre_ref)
    return f, pre, out


def _names(cs):
    return [c["name"] for c in cs]


@pytest.mark.parametrize("name", _names(cases.LAYOUTS + cases.LIMIT))
def test_layouts(name):
    """Every layout on dense normal maps, 17 envs (a partial 16-env tile in the Linear); the shared-memory limit cases
    with 3.  The features buffer, filled with NaN beforehand, receives every conv3 value."""
    c = {x["name"]: x for x in cases.LAYOUTS + cases.LIMIT}[name]
    B = 3 if c in cases.LIMIT else 17
    f, _, _ = check_map(map_cnn(c, seed=len(name)), map_input(c, B, seed=len(name) + 1))
    assert bool(torch.isfinite(f).all())


@pytest.mark.parametrize("relu", list(itertools.product((0, 1), repeat=3)), ids=lambda r: "relu" + "".join(map(str, r)))
def test_relu_flags(relu):
    """Each combination of the three conv relu flags (and both lin_relu values, in check_map) through the entry."""
    c = cases.RELU_LAYOUT
    check_map(map_cnn(c, seed=2), map_input(c, 17, seed=3), relu=relu)


@pytest.mark.parametrize("kind", ["gm", "am", "dense"])
def test_input_values_and_a_zero_env(kind):
    """Reference-like 0 / 1 geometric maps, sparse non-negative acoustic maps and dense normal maps; env 2 is all zero
    (its outputs are the biases carried through the layers)."""
    c = cases.INPUT_LAYOUT
    x = map_input(c, 5, seed=4, kind=kind)
    x[2] = 0.0
    check_map(map_cnn(c, seed=5), x)


@pytest.mark.parametrize("scale", cases.SCALES)
def test_scaled_inputs(scale):
    for c in (cases.INPUT_LAYOUT, cases.IDENTITY_LAYOUT):
        check_map(map_cnn(c, seed=6), map_input(c, 5, seed=7, scale=scale))


@pytest.mark.parametrize("value", ["nan", "inf", "-inf"])
@pytest.mark.parametrize("where", ["shared_row", "unread"])
def test_one_nonfinite_pixel(where, value):
    """One NaN / +Inf / -Inf pixel in env 3.  In an input row that conv1 rows of two ranks read: env 3's NaN / Inf
    pattern equals float64's and its finite values are within tolerance.  In a column conv1 never reads: env 3 is
    bit-identical to the clean run.  Every other env is bit-identical to the clean run either way."""
    c = cases.INPUT_LAYOUT
    cnn = map_cnn(c, seed=8)
    x = map_input(c, 5, seed=9, kind="gm")
    f0, pre0 = run_map(cnn, x, 0)
    _, out0 = run_map(cnn, x, 1)
    bad = x.clone()
    r, col = cases.SHARED_ROW_PIXEL if where == "shared_row" else cases.UNREAD_PIXEL
    bad[3, r, col, -1] = float(value)
    f, pre, out = check_map(cnn, bad)
    keep = torch.tensor([0, 1, 2, 4] if where == "shared_row" else [0, 1, 2, 3, 4], device=DEV)
    assert torch.equal(f[keep], f0[keep]) and torch.equal(pre[keep], pre0[keep]) and torch.equal(out[keep], out0[keep])
    if where == "shared_row":
        assert not bool(torch.isfinite(f[3]).all())
        if value == "nan":
            assert bool(out[3].isnan().all())


def test_bit_identical_across_batches_and_positions():
    """On a layout of the generic instance with idle ranks in conv1 and conv3: each env's features and outputs are
    the same bits at B = 1, 16, 17 and 129, at any offset, and under a permutation of the batch."""
    c = cases.IDENTITY_LAYOUT
    cnn = map_cnn(c, seed=10)
    x = map_input(c, 129, seed=11)
    f_all, out_all = run_map(cnn, x, 1)
    for B in cases.IDENTITY_BATCHES:
        for k in sorted({0, 1, 129 - B}):
            f, o = run_map(cnn, x[k:k + B].contiguous(), 1)
            assert torch.equal(f, f_all[k:k + B]) and torch.equal(o, out_all[k:k + B]), (B, k)
    perm = torch.randperm(129, generator=torch.Generator().manual_seed(12)).to(DEV)
    f, o = run_map(cnn, x[perm].contiguous(), 1)
    assert torch.equal(f, f_all[perm]) and torch.equal(o, out_all[perm])


class CaseMapCNN(MapCNN):
    """A MapCNN whose ``cnn`` is a case's (``make_cnn``), on the geometric map."""

    def __init__(self, c, seed=0):
        nn.Module.__init__(self)
        self._map_type, self._n_input_gm = "gm", c["C"]
        self.cnn = cases.make_cnn(c, seed)


def _patched():
    from soundspaces_b200.encoder import patch_map_cnn

    class Patched(CaseMapCNN):
        pass
    return patch_map_cnn(Patched)


@pytest.fixture
def no_tf32():
    saved = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = saved


def test_65535_envs_and_65536_refused(no_tf32):
    c = cases.BIG_B_LAYOUT
    cnn = map_cnn(c, seed=13)
    x = map_input(c, cases.MAX_ENVS, seed=14, kind="am")
    idx = [0, 1, 16, 32767, 65534]
    f, pre, _ = check_map(cnn, x, idx)
    for k in idx:
        f1, pre1 = run_map(cnn, x[k:k + 1].contiguous(), 0)
        assert torch.equal(f1[0], f[k]) and torch.equal(pre1[0], pre[k]), k
    del x, f, pre
    ops = _ops()
    cls = _patched()
    m = cls(c, seed=15).to(DEV).eval()
    big = {"gm": map_input(c, cases.MAX_ENVS + 1, seed=16, kind="am")}
    before = ops.ctx.launch_count
    rc, _, _ = map_entry(ops, m.cnn, big["gm"][:1], B=cases.MAX_ENVS + 1)
    assert rc == SSB_E_INVALID_ARG and b"bad arguments" in ops.lib.ssb_last_error(ops.ctx.handle)
    with torch.no_grad():
        got = m(big)
        assert ops.ctx.launch_count == before                  # the original ran
        assert torch.equal(got, cls.forward._ssb_original(m, big))


@pytest.mark.parametrize("name", _names(cases.LIMIT + cases.OVER_LIMIT))
def test_shared_memory_limit(no_tf32, name):
    """At the limit the patched forward runs fused (2 launches; test_layouts checks its accuracy) and equals the
    direct call; past it the entry refuses with the byte count encoder.map_encoder_smem_bytes computes, and the patched
    forward runs the original bit for bit (0 launches)."""
    from soundspaces_b200.encoder import map_encoder_smem_bytes
    c = {x["name"]: x for x in cases.LIMIT + cases.OVER_LIMIT}[name]
    cls = _patched()
    m = cls(c, seed=17).to(DEV).eval()
    obs = {"gm": map_input(c, 3, seed=18)}
    ops = _ops()
    nbytes = map_encoder_smem_bytes(m.cnn, c["C"], c["H"], c["W"])[0]
    before = ops.ctx.launch_count
    with torch.no_grad():
        got = m(obs)
    if c in cases.LIMIT:
        assert nbytes == cases.SMEM_LIMIT and ops.ctx.launch_count - before == 2
        assert torch.equal(got, run_map(m.cnn, obs["gm"], 1)[1])
        return
    assert nbytes > cases.SMEM_LIMIT and ops.ctx.launch_count == before
    with torch.no_grad():
        assert torch.equal(got, cls.forward._ssb_original(m, obs))
    rc, _, _ = map_entry(ops, m.cnn, obs["gm"])
    assert rc == SSB_E_SHAPE and f"({nbytes} bytes of shared memory".encode() in ops.lib.ssb_last_error(ops.ctx.handle)
    assert ops.ctx.launch_count == before


def test_refusals_launch_nothing():
    c = cases.INPUT_LAYOUT
    cnn = map_cnn(c, seed=19)
    x = map_input(c, 2, seed=20)
    ops = _ops()

    def layers_with(i, **kw):
        layers = conv_layers(cnn)
        for k, v in kw.items():
            setattr(layers[i], k, v)
        return layers

    feats = torch.zeros(2, cnn[6].in_features + 1, device=DEV)
    out = torch.zeros(2, cnn[6].out_features + 1, device=DEV)
    lin_w, lin_b = cnn[6].weight.data_ptr(), cnn[6].bias.data_ptr()
    cases_ = [
        (dict(B=-1), SSB_E_INVALID_ARG, b"bad arguments"), (dict(B=65536), SSB_E_INVALID_ARG, b"bad arguments"),
        (dict(C=0), SSB_E_INVALID_ARG, b"bad arguments"), (dict(H=0), SSB_E_INVALID_ARG, b"bad arguments"),
        (dict(W=0), SSB_E_INVALID_ARG, b"bad arguments"), (dict(hidden=0), SSB_E_INVALID_ARG, b"bad arguments"),
        (dict(lin_relu=2), SSB_E_INVALID_ARG, b"bad arguments"), (dict(lin_relu=-1), SSB_E_INVALID_ARG, b"bad arguments"),
        (dict(map_ptr=None), SSB_E_INVALID_ARG, b"bad arguments"),
        (dict(map_ptr=x.data_ptr() + 2), SSB_E_INVALID_ARG, b"bad arguments"),
        (dict(lin_weight=lin_w + 2), SSB_E_INVALID_ARG, b"bad arguments"),
        (dict(lin_bias=lin_b + 2), SSB_E_INVALID_ARG, b"bad arguments"),
        (dict(feats=feats.data_ptr() + 2), SSB_E_INVALID_ARG, b"bad arguments"),
        (dict(out=out.data_ptr() + 2), SSB_E_INVALID_ARG, b"bad arguments"),
        (dict(H=7), SSB_E_SHAPE, b"layer 1 output is empty (7x66 input, 8x8 kernel)"),
        (dict(W=7), SSB_E_SHAPE, b"layer 1 output is empty (64x7 input, 8x8 kernel)"),
        (dict(layers=layers_with(1, kh=16)), SSB_E_SHAPE, b"layer 2 output is empty (15x15 input, 16x4 kernel)"),
        (dict(layers=layers_with(2, kw=7)), SSB_E_SHAPE, b"layer 3 output is empty (6x6 input, 3x7 kernel)"),
        (dict(H=35), SSB_E_SHAPE, b"layer 3 output is empty"),
    ]
    for i in range(3):
        conv = cnn[2 * i]
        msg = f"bad layer {i + 1}".encode()
        cases_ += [(dict(layers=layers_with(i, **{k: v})), SSB_E_INVALID_ARG, msg)
                   for k, v in (("kh", 0), ("kw", 0), ("sh", 0), ("sw", 0), ("kh", -1), ("sw", -2), ("out_channels", 0),
                                ("relu", 2), ("d_weight", None), ("d_weight", conv.weight.data_ptr() + 2),
                                ("d_bias", conv.bias.data_ptr() + 2))]
    before = ops.ctx.launch_count
    for kw, rc_want, msg in cases_:
        rc, _, _ = map_entry(ops, cnn, x, **kw)
        err = ops.lib.ssb_last_error(ops.ctx.handle)
        assert rc == rc_want and msg in err, (kw, rc, err)
    assert map_entry(ops, cnn, x, B=0)[0] == 0                  # B = 0
    assert ops.ctx.launch_count == before
    assert map_entry(ops, cnn, x, lin_bias=None)[0] == 0         # a NULL bias is allowed
    assert ops.ctx.launch_count - before == 2


def test_more_than_int32_max_features_refused():
    """A 120 x 120 x 1 input through three 1 x 1 convs to 149131 channels fits the shared-memory limit of both the map
    and the visual entry but has 2147486400 conv3 features: both refuse it with SSB_E_SHAPE and the count, at B = 1
    and B = 0, before reading any buffer (the Linear weight, features and output here are 16 floats) or launching."""
    c = cases.HUGE_F
    H, W = c["H"], c["W"]
    C3 = c["Cs"][2]
    ops = _ops()
    from soundspaces_b200 import _lib
    w = [torch.ones(1, device=DEV), torch.ones(1, device=DEV), torch.ones(C3, device=DEV)]
    layers = (_lib.Conv2dLayer * 3)()
    for i, (oc, r) in enumerate(zip(c["Cs"], (1, 1, 0))):
        layers[i] = _lib.Conv2dLayer(w[i].data_ptr(), None, oc, 1, 1, 1, 1, r)
    x = torch.zeros(1, H, W, 1, device=DEV)
    small = [torch.zeros(16, device=DEV) for _ in range(3)]
    want = f"{cases.HUGE_F_FEATURES} features".encode()
    before = ops.ctx.launch_count
    for B in (1, 0):
        rc = ops.lib.ssb_map_encoder_batch(ops.ctx.handle, B, x.data_ptr(), 1, H, W, layers, small[0].data_ptr(), None,
                                           1, 1, small[1].data_ptr(), small[2].data_ptr(), ops._stream())
        assert rc == SSB_E_SHAPE and want in ops.lib.ssb_last_error(ops.ctx.handle), B
        rc = ops.lib.ssb_visual_encoder_batch(ops.ctx.handle, B, None, 0, x.data_ptr(), 1, H, W, layers,
                                              small[0].data_ptr(), None, 1, 1, small[1].data_ptr(),
                                              small[2].data_ptr(), ops._stream())
        assert rc == SSB_E_SHAPE and want in ops.lib.ssb_last_error(ops.ctx.handle), B
    assert ops.ctx.launch_count == before
    torch.cuda.synchronize()
    assert all(bool((t == 0).all()) for t in small)
