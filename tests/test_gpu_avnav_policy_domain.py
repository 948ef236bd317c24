"""AV-Nav's fused visual encoder (``ssb_visual_encoder_batch``) and GRU step (``ssb_gru_step_batch``) on the GPU across
the inputs their entries accept: non-square kernels and strides, every conv2 / conv3 kernel instance at sh != sw, idle
cluster ranks, the conv1 row tails, odd channel counts, bias=False, F and hidden off the Linear's tiles, the
shared-memory limit through both of its branches, 65535 envs, NaN / Inf / badly scaled inputs, every kind of GRU mask
value and saturated gates.  The entries are also called directly: each refusal returns its code and message and
launches nothing.  The cases are listed in tests/avnav_domain_cases.py; tests/test_avnav_domain_host.py checks that
they reach every tile edge.

Accuracy: each env is compared with a float64 forward of the same module on the CPU,
``max|got_b - ref_b| <= 1e-4 * scale_b`` over the finite values, and the NaN, +Inf and -Inf positions must equal
float64's exactly.  For the visual encoder ``scale_b = max|ref_b|``, checked on the conv3 features and on the Linear's
pre-activation (the entry called with lin_relu = 0); lin_relu = 1 must then be torch's ReLU of it bit for bit, which
keeps the check meaningful where the ReLU zeroes a whole env.  For the GRU ``scale_b = max(max|ref_b|, 1, max|m_b h_b|)``:
h' = (1 - z) n + z m h with |n| <= 1, so the rounding of the output is bounded relative to that floor even where the
output itself is small (a mask of 0.5 at I = Hd = 1 came within 9.7e-5 of the bar without it).

Calibration (torch's float32 forward on a CPU against float64, max over envs of the error over scale_b): visual layouts
1e-8 .. 6e-7, including inputs scaled by 1e-6 and 1e3; GRU cases 3e-8 .. 5.6e-6, 1.2e-5 with weights x 30.  x scaled
by 1e3 at I = 255 reached 1.8e-4 (gate sums of ~1e4 where a tanh argument crosses 0), so that case runs at I = 1.
"""
import copy

import pytest

import avnav_domain_cases as cases
from avnav_models import AudioNavBaselineNet, RNNStateEncoder, VisualCNN
from test_encoder_host import make_cnn as make_audio_cnn, reference_classes

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


def check_env(got, ref, floor=None):
    """Per env b: the NaN / +Inf / -Inf pattern of float64's, and max|got_b - ref_b| <= 1e-4 scale_b over the finite
    values, scale_b = max(max|ref_b|, floor[b])."""
    got = got.detach().cpu().double()
    assert got.shape == ref.shape
    for b in range(ref.shape[0]):
        g, r = got[b], ref[b]
        for f in (torch.isnan, torch.isposinf, torch.isneginf):
            assert torch.equal(f(g), f(r)), f"env {b}: {f.__name__} pattern differs from float64"
        fin = torch.isfinite(r)
        if fin.any():
            scale = max(r[fin].abs().max().item(), 0.0 if floor is None else floor[b])
            err = (g[fin] - r[fin]).abs().max().item()
            assert err <= 1e-4 * scale, f"env {b}: max err {err:.3g} > 1e-4 * {scale:.3g}"


# ------------------------------------------------------------------------------------------------ visual encoder
def visual_cnn(c, seed=0):
    return cases.make_cnn(c, seed).to(DEV)


def visual_obs(c, B, seed=1, scale=1.0):
    """RGB integers in 0..255 and depth in [0, 1), both times ``scale``."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    obs = {}
    if c["n_rgb"]:
        obs["rgb"] = torch.randint(0, 256, (B, c["H"], c["W"], c["n_rgb"]), device=DEV, generator=g).float() * scale
    if c["n_depth"]:
        obs["depth"] = torch.rand((B, c["H"], c["W"], c["n_depth"]), device=DEV, generator=g) * scale
    return obs


def conv_layers(cnn):
    from soundspaces_b200 import _lib
    layers = (_lib.Conv2dLayer * 3)()
    for i, (conv, relu) in enumerate(zip((cnn[0], cnn[2], cnn[4]), (1, 1, 0))):
        layers[i] = _lib.Conv2dLayer(conv.weight.data_ptr(), _ptr(conv.bias), conv.out_channels, *conv.kernel_size,
                                     *conv.stride, relu)
    return layers


def visual_entry(ops, cnn, obs, lin_relu=1, layers=None, B=None, H=None, W=None, hidden=None, lin_bias=None,
                 feats=None, out=None):
    """ssb_visual_encoder_batch called directly -> (rc, features, out); any argument can be overridden."""
    rgb, depth = obs.get("rgb"), obs.get("depth")
    first = rgb if rgb is not None else depth
    n, h, w = first.shape[:3]
    lin = cnn[6]
    f = torch.full((max(n, 1), lin.in_features), float("nan"), device=DEV)
    o = torch.full((max(n, 1), lin.out_features), float("nan"), device=DEV)
    rc = ops.lib.ssb_visual_encoder_batch(
        ops.ctx.handle, n if B is None else B, _ptr(rgb), rgb.shape[3] if rgb is not None else 0, _ptr(depth),
        depth.shape[3] if depth is not None else 0, h if H is None else H, w if W is None else W,
        conv_layers(cnn) if layers is None else layers, lin.weight.data_ptr(),
        _ptr(lin.bias) if lin_bias is None else lin_bias, lin.out_features if hidden is None else hidden, lin_relu,
        f.data_ptr() if feats is None else feats, o.data_ptr() if out is None else out, ops._stream())
    return rc, f[:n], o[:n]


def run_visual(cnn, obs, lin_relu):
    ops = _ops()
    before = ops.ctx.launch_count
    rc, f, o = visual_entry(ops, cnn, obs, lin_relu)
    assert rc == 0, ops.lib.ssb_last_error(ops.ctx.handle)
    assert ops.ctx.launch_count - before == 2
    return f, o


def visual_ref64(cnn, obs, idx=None):
    """(features, pre-activation) of ``cnn`` in float64 on the CPU for the envs ``idx`` (all when None)."""
    m = copy.deepcopy(cnn).cpu().double()
    o = {k: (v if idx is None else v[idx]).cpu().double() for k, v in obs.items()}
    x = []
    if "rgb" in o:
        x.append(o["rgb"].permute(0, 3, 1, 2) / 255.0)
    if "depth" in o:
        x.append(o["depth"].permute(0, 3, 1, 2))
    with torch.no_grad():
        feats = m[:6](torch.cat(x, 1))
        return feats, m[6](feats)


def check_visual(cnn, obs, idx=None):
    """Features and pre-activation against float64 per env; lin_relu = 1 is relu of lin_relu = 0 bit for bit.
    -> (features, pre-activation, output) of the whole batch."""
    f, pre = run_visual(cnn, obs, 0)
    f1, out = run_visual(cnn, obs, 1)
    assert same(f1, f) and same(out, torch.relu(pre))
    f_ref, pre_ref = visual_ref64(cnn, obs, idx)
    sel = slice(None) if idx is None else torch.tensor(idx, device=DEV)
    check_env(f[sel], f_ref)
    check_env(pre[sel], pre_ref)
    return f, pre, out


def _names(cs):
    return [c["name"] for c in cs]


@pytest.mark.parametrize("name", _names(cases.VISUAL + cases.LIMIT))
def test_visual_layouts(name):
    """Every layout, 17 envs (a partial 16-env tile in the Linear); the shared-memory limit cases with 3."""
    c = {x["name"]: x for x in cases.VISUAL + cases.LIMIT}[name]
    B = 3 if c in cases.LIMIT else 17
    check_visual(visual_cnn(c, seed=len(name)), visual_obs(c, B, seed=len(name) + 1))


def test_rgb_outside_the_sensor_range_and_a_zero_depth_env():
    """RGB that is not an integer, negative and above 255; env 2's depth is all zero."""
    c = cases.INPUT_LAYOUT
    g = torch.Generator(device=DEV).manual_seed(5)
    obs = visual_obs(c, 5, seed=6)
    obs["rgb"] = torch.randn(obs["rgb"].shape, device=DEV, generator=g) * 300 + 100
    obs["depth"][2] = 0.0
    assert bool((obs["rgb"] < 0).any()) and bool((obs["rgb"] > 255).any())
    check_visual(visual_cnn(c, seed=7), obs)


@pytest.mark.parametrize("scale", cases.SCALES)
def test_scaled_inputs(scale):
    for c in (cases.INPUT_LAYOUT, cases.VISUAL[2]):
        check_visual(visual_cnn(c, seed=8), visual_obs(c, 5, seed=9, scale=scale))


@pytest.mark.parametrize("value", ["nan", "inf", "-inf"])
@pytest.mark.parametrize("where", ["rgb", "depth"])
def test_one_nonfinite_pixel(where, value):
    """One NaN / +Inf / -Inf pixel in env 3: its NaN / Inf pattern equals float64's (torch's ReLU keeps NaN), its
    finite values are within tolerance, and every other env is bit-identical to the clean run."""
    c = cases.INPUT_LAYOUT
    cnn = visual_cnn(c, seed=10)
    obs = visual_obs(c, 5, seed=11)
    f0, pre0 = run_visual(cnn, obs, 0)
    _, out0 = run_visual(cnn, obs, 1)
    bad = {k: v.clone() for k, v in obs.items()}
    bad[where][3, 21, 30, -1] = float(value)
    f, pre, out = check_visual(cnn, bad)
    keep = torch.tensor([0, 1, 2, 4], device=DEV)
    assert torch.equal(f[keep], f0[keep]) and torch.equal(pre[keep], pre0[keep]) and torch.equal(out[keep], out0[keep])
    assert not bool(torch.isfinite(f[3]).all())
    if value == "nan":
        assert bool(out[3].isnan().all())


def _patched_visual():
    from soundspaces_b200.encoder import patch_visual_cnn

    class Patched(VisualCNN):
        pass
    return patch_visual_cnn(Patched)


@pytest.fixture
def no_tf32():
    saved = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = saved


def test_visual_65535_envs_and_65536_refused(no_tf32):
    c = cases.BIG_B_LAYOUT
    cnn = visual_cnn(c, seed=12)
    obs = visual_obs(c, cases.MAX_ENVS, seed=13)
    idx = [0, 1, 16, 32767, 65534]
    f, pre, _ = check_visual(cnn, obs, idx)
    for k in idx:
        f1, pre1 = run_visual(cnn, {"depth": obs["depth"][k:k + 1].contiguous()}, 0)
        assert torch.equal(f1[0], f[k]) and torch.equal(pre1[0], pre[k]), k
    del obs, f, pre
    ops = _ops()
    cls = _patched_visual()
    torch.manual_seed(14)
    m = cls(0, 1, c["H"], c["W"], c["hidden"]).to(DEV)
    big = visual_obs(c, cases.MAX_ENVS + 1, seed=15)
    before = ops.ctx.launch_count
    rc, _, _ = visual_entry(ops, m.cnn, {"depth": big["depth"][:1]}, B=cases.MAX_ENVS + 1)
    assert rc == SSB_E_INVALID_ARG and b"bad arguments" in ops.lib.ssb_last_error(ops.ctx.handle)
    with torch.no_grad():
        got = m(big)
        assert ops.ctx.launch_count == before                  # the original ran
        assert torch.equal(got, cls.forward._ssb_original(m, big))


@pytest.mark.parametrize("name", _names(cases.LIMIT + cases.OVER_LIMIT))
def test_shared_memory_limit(no_tf32, name):
    """At the limit the patched forward runs fused (2 launches; test_visual_layouts checks its accuracy); past it the
    entry refuses with the byte count encoder.visual_encoder_smem_bytes computes, and the patched forward runs the
    original (0 launches)."""
    from soundspaces_b200.encoder import visual_encoder_smem_bytes
    c = {x["name"]: x for x in cases.LIMIT + cases.OVER_LIMIT}[name]
    cls = _patched_visual()
    torch.manual_seed(16)
    m = cls(c["n_rgb"], c["n_depth"], c["H"], c["W"], c["hidden"]).to(DEV).eval()
    obs = visual_obs(c, 2, seed=17)
    ops = _ops()
    nbytes = visual_encoder_smem_bytes(m.cnn, c["IC"], c["H"], c["W"])[0]
    before = ops.ctx.launch_count
    with torch.no_grad():
        got = m(obs)
    if c in cases.LIMIT:
        assert nbytes == cases.SMEM_LIMIT and ops.ctx.launch_count - before == 2
        assert torch.equal(got, run_visual(m.cnn, obs, 1)[1])
        return
    assert ops.ctx.launch_count == before
    with torch.no_grad():
        assert torch.equal(got, cls.forward._ssb_original(m, obs))
    rc, _, _ = visual_entry(ops, m.cnn, obs)
    assert rc == SSB_E_SHAPE and f"({nbytes} bytes".encode() in ops.lib.ssb_last_error(ops.ctx.handle)
    assert ops.ctx.launch_count == before


def test_visual_refusals_launch_nothing():
    c = cases.INPUT_LAYOUT
    cnn = visual_cnn(c, seed=18)
    obs = visual_obs(c, 2, seed=19)
    ops = _ops()

    def layers_with(i, **kw):
        layers = conv_layers(cnn)
        for k, v in kw.items():
            setattr(layers[i], k, v)
        return layers

    feats = torch.zeros(2, cnn[6].in_features + 1, device=DEV)
    out = torch.zeros(2, cnn[6].out_features + 1, device=DEV)
    lin_b = cnn[6].bias.data_ptr()
    cases_ = [
        (dict(layers=layers_with(1, relu=2)), SSB_E_INVALID_ARG, b"bad layer 2"),
        (dict(lin_relu=2), SSB_E_INVALID_ARG, b"bad arguments"),
        (dict(layers=layers_with(0, sh=0)), SSB_E_INVALID_ARG, b"bad layer 1"),
        (dict(layers=layers_with(2, sw=0)), SSB_E_INVALID_ARG, b"bad layer 3"),
        (dict(layers=layers_with(2, kw=0)), SSB_E_INVALID_ARG, b"bad layer 3"),
        (dict(layers=layers_with(0, kh=0)), SSB_E_INVALID_ARG, b"bad layer 1"),
        (dict(hidden=0), SSB_E_INVALID_ARG, b"bad arguments"),
        (dict(layers=layers_with(1, d_bias=cnn[2].bias.data_ptr() + 2)), SSB_E_INVALID_ARG, b"bad layer 2"),
        (dict(lin_bias=lin_b + 2), SSB_E_INVALID_ARG, b"bad arguments"),
        (dict(feats=feats.data_ptr() + 2), SSB_E_INVALID_ARG, b"bad arguments"),
        (dict(out=out.data_ptr() + 2), SSB_E_INVALID_ARG, b"bad arguments"),
        (dict(H=7), SSB_E_SHAPE, b"layer 1 output is empty"),
        (dict(layers=layers_with(1, kh=c["H"] // 4)), SSB_E_SHAPE, b"layer 2 output is empty"),
    ]
    before = ops.ctx.launch_count
    for kw, rc_want, msg in cases_:
        rc, _, _ = visual_entry(ops, cnn, obs, **kw)
        assert rc == rc_want, kw
        assert msg in ops.lib.ssb_last_error(ops.ctx.handle), kw
    assert ops.ctx.launch_count == before


def test_audio_encoder_nan_propagates_as_torch():
    """The conv stack kernels are shared with the audio encoder: one NaN bin in env 2 makes its output NaN as in
    torch's forward; the other envs are bit-identical to the clean run."""
    torch.manual_seed(20)
    cnn = make_audio_cnn((65, 26, 2)).to(DEV).eval()
    g = torch.Generator(device=DEV).manual_seed(21)
    spec = torch.rand(4, 65, 26, 2, device=DEV, generator=g) * 3
    ops = _ops()
    clean = ops.audio_encoder(spec, cnn)
    bad = spec.clone()
    bad[2, 30, 10, 1] = float("nan")
    F = cnn[6].in_features
    feats = torch.empty(4, F, device=DEV)
    out = ops.audio_encoder(bad, cnn, features=feats)
    ref = copy.deepcopy(cnn).cpu().double()
    with torch.no_grad():
        x = bad.cpu().double().permute(0, 3, 1, 2)
        check_env(feats, ref[:6](x))
        check_env(out, ref(x))
    assert bool(out[2].isnan().all())
    keep = torch.tensor([0, 1, 3], device=DEV)
    assert torch.equal(out[keep], clean[keep])


# ------------------------------------------------------------------------------------------------ GRU
def gru_module(I, Hd, scales=(1, 1, 1), seed=0):
    w_scale, _, b_scale = scales
    torch.manual_seed(seed)
    r = nn.GRU(I, Hd)
    with torch.no_grad():
        for name, p in r.named_parameters():
            if "bias" in name:
                p.uniform_(-0.3, 0.3).mul_(b_scale)
            else:
                p.mul_(w_scale)
    return r.to(DEV)


def gru_inputs(I, Hd, B, masks="mixed", x_scale=1.0, seed=1):
    g = torch.Generator(device=DEV).manual_seed(seed)
    x = torch.randn(B, I, device=DEV, generator=g) * x_scale
    h = torch.randn(B, Hd, device=DEV, generator=g)
    if masks == "mixed":
        m = (torch.arange(B, device=DEV) % 3 != 0).float()[:, None]
    else:
        m = torch.tensor([masks[b % len(masks)] for b in range(B)], device=DEV)[:, None]
    return x, h, m


def gru_ref64(r, x, h, m):
    ref = copy.deepcopy(r).cpu().double()
    mh = m.cpu().double() * h.cpu().double()
    with torch.no_grad():
        y, _ = ref(x.cpu().double()[None], mh[None])
    floor = [max([1.0] + [v for v in mh[b].abs().tolist() if v == v and v != float("inf")]) for b in range(len(mh))]
    return y[0], floor


def _gru_id(case):
    I, Hd, B, masks, scales = case
    return f"I{I}-Hd{Hd}-B{B}-{'mixed' if masks == 'mixed' else 'values'}-{'x'.join(f'{s:g}' for s in scales)}"


@pytest.mark.parametrize("case", cases.GRU, ids=_gru_id)
def test_gru_against_float64(case):
    """Each case against float64 nn.GRU on m * h; the masks passed as (n, 1) and as (n,) give the same bits."""
    I, Hd, B, masks, scales = case
    r = gru_module(I, Hd, scales, seed=I + 3 * Hd)
    x, h, m = gru_inputs(I, Hd, B, masks, scales[1], seed=B)
    ops = _ops()
    before = ops.ctx.launch_count
    out, h_out = ops.gru_step(x, h, m, r)
    assert ops.ctx.launch_count - before == 1
    y_ref, floor = gru_ref64(r, x, h, m)
    check_env(out, y_ref, floor)
    assert same(out, h_out) and out.data_ptr() != h_out.data_ptr()
    out1, _ = ops.gru_step(x, h, m[:, 0].contiguous(), r)
    assert same(out1, out)


def test_gru_nan_in_last_env_of_a_partial_tile():
    """The kernel fills the unused lanes of the last 16-env tile with env ne - 1; NaN in x of env 16 of 17 stays in
    env 16, and envs 0-15 are bit-identical to the clean run."""
    r = gru_module(257, 31, seed=22)
    x, h, m = gru_inputs(257, 31, 17, seed=23)
    ops = _ops()
    clean, _ = ops.gru_step(x, h, m, r)
    x = x.clone()
    x[16, 100] = float("nan")
    out, _ = ops.gru_step(x, h, m, r)
    assert torch.equal(out[:16], clean[:16]) and bool(out[16].isnan().all())
    y_ref, floor = gru_ref64(r, x, h, m)
    check_env(out, y_ref, floor)


def test_gru_bit_identical_across_batches_at_odd_widths():
    ops = _ops()
    r = gru_module(257, 31, seed=24)
    x, h, m = gru_inputs(257, 31, 129, masks=cases.MASK_VALUES[:3] + (1.0, 0.0), seed=25)
    out_all, _ = ops.gru_step(x, h, m, r)
    out_rev, _ = ops.gru_step(x.flip(0).contiguous(), h.flip(0).contiguous(), m.flip(0).contiguous(), r)
    assert torch.equal(out_rev.flip(0), out_all)
    for k in (0, 15, 16, 17, 128):
        o1, _ = ops.gru_step(x[k:k + 1].contiguous(), h[k:k + 1].contiguous(), m[k:k + 1].contiguous(), r)
        assert torch.equal(o1[0], out_all[k])
    for j in (0, 1, 16, 127, 128):
        idx = torch.arange(129, device=DEV)
        idx[j], idx[7] = 7, j
        o, _ = ops.gru_step(x[idx].contiguous(), h[idx].contiguous(), m[idx].contiguous(), r)
        assert torch.equal(o[j], out_all[7])


def _patched_rnn():
    from soundspaces_b200.rnn import patch_rnn_state_encoder

    class Patched(RNNStateEncoder):
        pass
    return patch_rnn_state_encoder(Patched)


def test_gru_65535_envs_and_65536_refused(no_tf32):
    I, Hd = cases.GRU_BIG_B
    ops = _ops()
    r = gru_module(I, Hd, seed=26)
    x, h, m = gru_inputs(I, Hd, cases.MAX_ENVS, seed=27)
    out, _ = ops.gru_step(x, h, m, r)
    idx = [0, 1, 16, 32767, 65534]
    sel = torch.tensor(idx, device=DEV)
    y_ref, floor = gru_ref64(r, x[sel], h[sel], m[sel])
    check_env(out[sel], y_ref, floor)
    for k in idx:
        o1, _ = ops.gru_step(x[k:k + 1].contiguous(), h[k:k + 1].contiguous(), m[k:k + 1].contiguous(), r)
        assert torch.equal(o1[0], out[k])
    cls = _patched_rnn()
    torch.manual_seed(28)
    enc = cls(I, Hd).to(DEV)
    x, h, m = gru_inputs(I, Hd, cases.MAX_ENVS + 1, seed=29)
    p = [q.data_ptr() for q in (enc.rnn.weight_ih_l0, enc.rnn.weight_hh_l0, enc.rnn.bias_ih_l0, enc.rnn.bias_hh_l0)]
    o = torch.empty_like(h)
    before = ops.ctx.launch_count
    rc = ops.lib.ssb_gru_step_batch(ops.ctx.handle, cases.MAX_ENVS + 1, I, Hd, x.data_ptr(), h.data_ptr(), m.data_ptr(),
                                    *p, o.data_ptr(), o.data_ptr(), ops._stream())
    assert rc == SSB_E_INVALID_ARG and b"bad arguments" in ops.lib.ssb_last_error(ops.ctx.handle)
    with torch.no_grad():
        got, h_got = enc(x, h[None].contiguous(), m)
        assert ops.ctx.launch_count == before                  # the original ran
        want, h_want = cls.single_forward._ssb_original(enc, x, h[None].contiguous(), m)
    assert torch.equal(got, want) and torch.equal(h_got, h_want)


# ------------------------------------------------------------------------------------------------ zero envs
def test_patched_classes_at_zero_envs():
    """N = 0: the patched VisualCNN, RNNStateEncoder and AudioNavBaselineNet return what the unpatched ones return
    (shapes and dtype; they run on the CPU here), with no launch.  The network's audio encoder flattens with
    nn.Flatten: with the reference's ``Flatten`` the unpatched forward raises on an empty batch."""
    from soundspaces_b200.encoder import patch_audio_cnn, patch_visual_cnn
    from soundspaces_b200.rnn import patch_rnn_state_encoder
    ops = _ops()
    vis_cls = _patched_visual()
    for n_rgb, n_depth in ((0, 1), (3, 1)):
        torch.manual_seed(30)
        m = vis_cls(n_rgb, n_depth, 64, 64, 32).to(DEV)
        obs = {k: torch.zeros(0, 64, 64, ch, device=DEV) for k, ch in (("rgb", n_rgb), ("depth", n_depth)) if ch}
        before = ops.ctx.launch_count
        with torch.no_grad():
            got = m(obs)
            want = vis_cls.forward._ssb_original(copy.deepcopy(m).cpu(), {k: v.cpu() for k, v in obs.items()})
        assert ops.ctx.launch_count == before
        assert got.is_cuda and got.shape == want.shape == (0, 32) and got.dtype == want.dtype

    rnn_cls = _patched_rnn()
    enc = rnn_cls(40, 24).to(DEV)
    x, h, m = torch.zeros(0, 40, device=DEV), torch.zeros(1, 0, 24, device=DEV), torch.zeros(0, 1, device=DEV)
    before = ops.ctx.launch_count
    with torch.no_grad():
        got = enc(x, h, m)
        want = rnn_cls.single_forward._ssb_original(copy.deepcopy(enc).cpu(), x.cpu(), h.cpu(), m.cpu())
    assert ops.ctx.launch_count == before
    assert [t.shape for t in got] == [t.shape for t in want] == [(0, 24), (1, 0, 24)]
    assert [t.dtype for t in got] == [t.dtype for t in want] and got[0].is_cuda

    AudioCNN = reference_classes()[0]

    class PAudio(AudioCNN):
        pass

    class PVisual(VisualCNN):
        pass

    class PRnn(RNNStateEncoder):
        pass

    torch.manual_seed(31)
    audio = AudioCNN((65, 26, 2), 512, audiogoal_sensor="spectrogram")
    audio.cnn[5] = nn.Flatten()          # the reference's x.reshape(x.size(0), -1) cannot reshape an empty batch
    plain = AudioNavBaselineNet(audio, VisualCNN(3, 1, 64, 64, 512))
    fused = copy.deepcopy(plain).to(DEV)
    fused.audio_encoder.__class__ = patch_audio_cnn(PAudio)
    fused.visual_encoder.__class__ = patch_visual_cnn(PVisual)
    fused.state_encoder.__class__ = patch_rnn_state_encoder(PRnn)
    obs = {"spectrogram": torch.zeros(0, 65, 26, 2), "rgb": torch.zeros(0, 64, 64, 3), "depth": torch.zeros(0, 64, 64, 1)}
    h = torch.zeros(1, 0, 512)
    masks = torch.zeros(0, 1)
    before = ops.ctx.launch_count
    with torch.no_grad():
        got = fused({k: v.to(DEV) for k, v in obs.items()}, h.to(DEV), masks.to(DEV))
        want = plain(obs, h, masks)
    assert ops.ctx.launch_count == before
    assert [t.shape for t in got] == [t.shape for t in want] == [(0, 512), (1, 0, 512)]
    assert [t.dtype for t in got] == [t.dtype for t in want] and got[0].is_cuda
