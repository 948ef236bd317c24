"""The fused audio encoder (``ssb_audio_encoder_batch``, ``ssb_audio_encoder_category_batch``, ``patch_audio_cnn``) on the
GPU across the inputs its entries accept: idle cluster ranks and odd, partial per-rank chunks in every layer, non-square
kernels and strides, strides larger than the kernel, a conv1 kernel that covers the whole input, a one-column
observation, every conv2 / conv3 kernel instance at sh != sw, 1, 21 and 222 labels of every kind and scale with conv1's
bias present or not, bias=False on every layer, F and hidden off the Linear's tiles, every combination of the ReLU
flags, one NaN / +Inf / -Inf bin or NaN label, an all-zero env, 65535 envs, and the shared-memory limit through each of
its terms.  The entries are also called directly: each refusal returns its code and message and launches nothing, and
the patched ``forward`` runs the original wherever the entries refuse.  The cases are listed in
tests/audio_encoder_domain_cases.py; tests/test_audio_encoder_domain_host.py checks that they reach every tile edge.

Accuracy, as in test_gpu_encoder.py: per element ``|got - ref64| <= 1e-5 * bound``, where ref64 is the same network in
float64 on the CPU and ``bound`` is that network with |x|, |labels|, |W| and |b| and no ReLU.  It is checked on the
conv3 features and on the Linear's pre-activation (the entry called with lin_relu = 0); lin_relu = 1 must then be
torch's ReLU of it bit for bit.  The non-finite cases check instead that the NaN, +Inf and -Inf positions equal
float64's and that every other env is bit-identical to the clean run.

Calibration: torch's float32 forward on a CPU against float64, the largest err / bound over features and
pre-activation, on the same inputs and weights:

    AUDIO layouts                               8e-10 .. 3.9e-8 (c1_17_kernel_is_input)
    LABELS, each of the six label kinds         9e-11 .. 1.8e-8 (lab21_kk192_no_conv1_bias, zero labels)
    LIMIT and REF_FITS                          9e-11 .. 9.5e-9 (limit_observation)
    every ReLU flag combination                 5.3e-10 .. 1.3e-8
    the five sampled envs of 65535              8.8e-10 .. 9.9e-10

The worst case is 3.9e-8, 250x under the 1e-5 bar.
"""
import copy
import itertools

import pytest

import audio_encoder_domain_cases as cases
from test_encoder_host import reference_classes

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
nn = torch.nn

DEV = "cuda:0"
SSB_E_INVALID_ARG, SSB_E_SHAPE = -1, -4
NAN = float("nan")


def _ops():
    from soundspaces_b200.renderer import WaveformOps
    return WaveformOps.get(DEV)


def _ptr(t):
    return t.data_ptr() if t is not None else None


def same(a, b):
    """Equal values, NaN at the same positions."""
    return (a.shape == b.shape and torch.equal(a.isnan(), b.isnan())
            and torch.equal(torch.where(a.isnan(), 0.0, a), torch.where(b.isnan(), 0.0, b)))


def conv_layers(cnn, relus=(1, 1, 0)):
    from soundspaces_b200 import _lib
    layers = (_lib.Conv2dLayer * 3)()
    for i, (conv, relu) in enumerate(zip((cnn[0], cnn[2], cnn[4]), relus)):
        layers[i] = _lib.Conv2dLayer(conv.weight.data_ptr(), _ptr(conv.bias), conv.out_channels, *conv.kernel_size,
                                     *conv.stride, relu)
    return layers


def entry(ops, cnn, x, lab=None, category=False, relus=(1, 1, 0), lin_relu=1, B=None, spec=None, layers=None,
          lin_weight=None, lin_bias=None, feats=None, out=None):
    """ssb_audio_encoder_batch, or ssb_audio_encoder_category_batch when ``lab`` is given or ``category`` is set,
    called directly -> (rc, features, out); any argument can be overridden."""
    n, H, W = x.shape[:3]
    lin = cnn[6]
    f = torch.full((max(n, 1), lin.in_features), NAN, device=DEV)
    o = torch.full((max(n, 1), lin.out_features), NAN, device=DEV)
    args = (ops.ctx.handle, n if B is None else B, x.data_ptr() if spec is None else spec, H, W,
            conv_layers(cnn, relus) if layers is None else layers)
    tail = (lin.weight.data_ptr() if lin_weight is None else lin_weight, _ptr(lin.bias) if lin_bias is None else lin_bias,
            lin.out_features, lin_relu, f.data_ptr() if feats is None else feats,
            o.data_ptr() if out is None else out, ops._stream())
    if lab is None and not category:
        rc = ops.lib.ssb_audio_encoder_batch(*args, *tail)
    else:
        NL = 0 if lab is None else lab.shape[1]
        rc = ops.lib.ssb_audio_encoder_category_batch(*args, _ptr(lab) if NL else None, NL,
                                                      lab.stride(0) if NL else 0, *tail)
    return rc, f[:n], o[:n]


def run(cnn, x, lab=None, category=False, relus=(1, 1, 0), lin_relu=1):
    ops = _ops()
    before = ops.ctx.launch_count
    rc, f, o = entry(ops, cnn, x, lab, category, relus, lin_relu)
    assert rc == 0, ops.lib.ssb_last_error(ops.ctx.handle)
    assert ops.ctx.launch_count - before == 2
    return f, o


def float64_runs(cnn, x, lab=None, relus=(1, 1, 0)):
    """(features, pre-activation) of ``cnn`` with the given conv ReLU flags on cat(permute(x), expand(lab)) in float64
    on the CPU, and the same pair for the bound network: |x|, |labels|, |W|, |b|, no ReLU."""
    x64 = x.detach().cpu().double().permute(0, 3, 1, 2)
    inp = x64
    if lab is not None:
        l64 = lab.detach().cpu().double()
        inp = torch.cat([x64, l64[:, :, None, None].expand(l64.shape + x64.shape[-2:])], dim=1)
    ref = copy.deepcopy(cnn).cpu().double()
    acts = [nn.ReLU() if r else nn.Identity() for r in relus]
    net = nn.Sequential(ref[0], acts[0], ref[2], acts[1], ref[4], acts[2], ref[5])
    bnd = copy.deepcopy(nn.Sequential(ref[0], ref[2], ref[4], ref[5], ref[6]))
    with torch.no_grad():
        for p in bnd.parameters():
            p.abs_()
        feats, fb = net(inp), bnd[:4](inp.abs())
        return feats, ref[6](feats), fb, bnd[4](fb)


def check_bound(got, ref, bound):
    """|got - ref| <= 1e-5 bound wherever ref is finite, and the NaN / +Inf / -Inf positions of ref."""
    got = got.detach().cpu().double()
    assert got.shape == ref.shape
    for f in (torch.isnan, torch.isposinf, torch.isneginf):
        assert torch.equal(f(got), f(ref)), f"{f.__name__} pattern differs from float64"
    fin = torch.isfinite(ref)
    err = (got[fin] - ref[fin]).abs()
    ok = err <= 1e-5 * bound[fin]
    assert bool(ok.all()), f"max err / bound {(err / bound[fin].clamp_min(1e-300)).max().item():.3g}"


def check(cnn, x, lab=None, category=False, relus=(1, 1, 0), idx=None):
    """Features and pre-activation against float64; lin_relu = 1 is torch's ReLU of lin_relu = 0 bit for bit.
    ``idx``: check only these envs against float64.  -> (features, pre-activation, output) of the whole batch."""
    f, pre = run(cnn, x, lab, category, relus, 0)
    f1, out = run(cnn, x, lab, category, relus, 1)
    assert same(f1, f) and same(out, torch.relu(pre))
    sel = slice(None) if idx is None else torch.tensor(idx, device=DEV)
    f_ref, pre_ref, f_bnd, pre_bnd = float64_runs(cnn, x[sel], None if lab is None else lab[sel], relus)
    check_bound(f[sel], f_ref, f_bnd)
    check_bound(pre[sel], pre_ref, pre_bnd)
    return f, pre, out


def _names(cs):
    return [c["name"] for c in cs]


BY_NAME = {c["name"]: c for c in cases.AUDIO + cases.LIMIT + cases.REF_FITS}


@pytest.mark.parametrize("name", _names(cases.AUDIO + cases.LIMIT + cases.REF_FITS))
def test_layouts(name):
    """Every layout at its batch size (the limit cases at 3 envs) through both entries: the category entry with no
    labels is bit-identical to ssb_audio_encoder_batch, and WaveformOps.audio_encoder to the entry."""
    c = BY_NAME[name]
    cnn = cases.make_cnn(c, seed=len(name)).to(DEV)
    x, lab = cases.make_inputs(c, c["B"], seed=len(name) + 1, kind=("soft", 1.0), device=DEV)
    f, _, out = check(cnn, x, lab)
    if lab is None:
        f0, out0 = run(cnn, x, category=True)
        assert same(f0, f) and same(out0, out)
    feats = torch.empty_like(f)
    assert same(_ops().audio_encoder(x, cnn, features=feats, category=lab), out) and same(feats, f)


@pytest.mark.parametrize("kind", cases.LABEL_KINDS, ids=lambda k: f"{k[0]}{k[1]:g}")
@pytest.mark.parametrize("name", _names(cases.LABELS))
def test_labels(name, kind):
    c = {x["name"]: x for x in cases.LABELS}[name]
    cnn = cases.make_cnn(c, seed=len(name)).to(DEV)
    x, lab = cases.make_inputs(c, c["B"], seed=len(name) + 1, kind=kind, device=DEV)
    _, _, out = check(cnn, x, lab)
    assert same(_ops().audio_encoder(x, cnn, category=lab), out)


@pytest.mark.parametrize("labels", [False, True])
def test_relu_flags(labels):
    """Every combination of the three conv ReLU flags and lin_relu, called through the ABI."""
    c = cases.INPUT_LABELS if labels else cases.INPUT_LAYOUT
    cnn = cases.make_cnn(c, seed=3).to(DEV)
    x, lab = cases.make_inputs(c, c["B"], seed=4, device=DEV)
    for relus in itertools.product((0, 1), repeat=3):
        check(cnn, x, lab, relus=relus)


def _nonfinite_check(cnn, x, lab, bad_x, bad_lab):
    """Env 3 of the bad inputs against float64 (NaN / Inf pattern, finite values within the bound), every other env
    bit-identical to the clean run.  -> (features, pre-activation, output) of the bad run."""
    f0, pre0 = run(cnn, x, lab, lin_relu=0)
    _, out0 = run(cnn, x, lab, lin_relu=1)
    f, pre, out = check(cnn, bad_x, bad_lab)
    keep = torch.tensor([0, 1, 2, 4], device=DEV)
    assert torch.equal(f[keep], f0[keep]) and torch.equal(pre[keep], pre0[keep]) and torch.equal(out[keep], out0[keep])
    return f, pre, out


@pytest.mark.parametrize("value", ["nan", "inf", "-inf"])
@pytest.mark.parametrize("labels", [False, True])
def test_one_nonfinite_bin(labels, value):
    """One NaN / +Inf / -Inf bin in env 3 (env 2 is all zero)."""
    c = cases.INPUT_LABELS if labels else cases.INPUT_LAYOUT
    cnn = cases.make_cnn(c, seed=5).to(DEV)
    x, lab = cases.make_inputs(c, c["B"], seed=6, device=DEV)
    bad = x.clone()
    bad[3, 30, 10, 1] = float(value)
    f, _, out = _nonfinite_check(cnn, x, lab, bad, lab)
    assert not bool(torch.isfinite(f[3]).all())
    if value == "nan":
        assert bool(out[3].isnan().all())


def test_one_nan_label():
    """A NaN label makes every output of its env NaN, as in torch; the other envs are unchanged."""
    c = cases.INPUT_LABELS
    cnn = cases.make_cnn(c, seed=7).to(DEV)
    x, lab = cases.make_inputs(c, c["B"], seed=8, device=DEV)
    bad = lab.clone()
    bad[3, 20] = NAN
    f, _, out = _nonfinite_check(cnn, x, lab, x, bad)
    assert bool(f[3].isnan().all()) and bool(out[3].isnan().all())


def _patched(c, cnn=None):
    """A patched stand-in AudioCNN (SAVi's, with a distractor sound when the case has labels) running ``cnn``."""
    from soundspaces_b200.encoder import patch_audio_cnn
    _, _, Savi = reference_classes()
    patch_audio_cnn(Savi, category=True)
    torch.manual_seed(9)
    m = Savi((65, 26, 2), hidden=c["hidden"], has_distractor_sound=c["NL"] > 0)
    if cnn is not None:
        m.cnn = cnn
    return Savi, m.to(DEV).eval()


def _obs(x, lab):
    return {"audiogoal": x} if lab is None else {"audiogoal": x, "category": lab}


@pytest.fixture
def no_tf32():
    saved = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = saved


@pytest.mark.parametrize("labels", [False, True])
def test_65535_envs_and_65536_refused(no_tf32, labels):
    """65535 envs: envs 0, 1, 16, 32767 and 65534 against float64 and against single-env calls bit for bit.  65536
    envs: the entry refuses and launches nothing, and the patched forward runs the original."""
    c = cases.BIG_B_LABELS if labels else cases.BIG_B_LAYOUT
    cnn = cases.make_cnn(c, seed=10).to(DEV)
    x, lab = cases.make_inputs(c, cases.MAX_ENVS + 1, seed=11, device=DEV)
    xs, ls = x[:cases.MAX_ENVS], None if lab is None else lab[:cases.MAX_ENVS]
    idx = [0, 1, 16, 32767, 65534]
    f, pre, _ = check(cnn, xs, ls, idx=idx)
    for k in idx:
        f1, pre1 = run(cnn, x[k:k + 1], None if lab is None else lab[k:k + 1], lin_relu=0)
        assert torch.equal(f1[0], f[k]) and torch.equal(pre1[0], pre[k]), k
    del f, pre
    ops = _ops()
    cls, m = _patched(c, cnn)
    before = ops.ctx.launch_count
    rc, _, _ = entry(ops, cnn, x[:1], None if lab is None else lab[:1], B=cases.MAX_ENVS + 1)
    assert rc == SSB_E_INVALID_ARG and b"bad arguments" in ops.lib.ssb_last_error(ops.ctx.handle)
    with torch.no_grad():
        got = m(_obs(x, lab))
        assert ops.ctx.launch_count == before                  # the original ran
        assert torch.equal(got, cls.forward._ssb_original(m, _obs(x, lab)))


def _limit_model(c):
    """The patched model of a limit or reference-boundary case: the reference classes' own networks for the
    reference shapes (av_wan's for C3 = 32), the case's network in SAVi's stand-in otherwise."""
    from soundspaces_b200.encoder import patch_audio_cnn
    if c in cases.REF_FITS + cases.REF_OVER:
        AvNav, AvWan, Savi = reference_classes()
        torch.manual_seed(12)
        if c["NL"]:
            m = Savi((c["H"], c["W"], 2), hidden=c["hidden"], has_distractor_sound=True)
            cls = patch_audio_cnn(Savi, category=True)
        else:
            cls = patch_audio_cnn(AvWan if c["C"][2] == 32 else AvNav)
            m = cls((c["H"], c["W"], 2), hidden=c["hidden"])
        return cls, m.to(DEV).eval()
    return _patched(c, cases.make_cnn(c, seed=13).to(DEV))


@pytest.mark.parametrize("name", _names(cases.LIMIT + cases.OVER_LIMIT + cases.REF_FITS + cases.REF_OVER))
def test_shared_memory_limit(no_tf32, name):
    """Within the limit the patched forward runs fused (2 launches; test_layouts checks its accuracy) and equals the
    entry bit for bit; past it the entry refuses with the byte count encoder.audio_encoder_smem_bytes computes and
    launches nothing, and the patched forward runs the original."""
    from soundspaces_b200.encoder import audio_encoder_smem_bytes
    c = {x["name"]: x for x in cases.LIMIT + cases.OVER_LIMIT + cases.REF_FITS + cases.REF_OVER}[name]
    cls, m = _limit_model(c)
    x, lab = cases.make_inputs(c, 2, seed=14, kind=("one_hot", 1.0), device=DEV)
    obs = {getattr(m, "_audiogoal_sensor", "spectrogram"): x}
    if lab is not None:
        obs["category"] = lab
    nbytes = audio_encoder_smem_bytes(m.cnn, c["NL"], c["H"], c["W"])[0]
    ops = _ops()
    before = ops.ctx.launch_count
    with torch.no_grad():
        got = m(obs)
    fits = c in cases.LIMIT + cases.REF_FITS
    if fits:
        assert nbytes <= cases.SMEM_LIMIT and ops.ctx.launch_count - before == 2
        assert torch.equal(got, run(m.cnn, x, lab)[1])
        return
    assert nbytes > cases.SMEM_LIMIT and ops.ctx.launch_count == before
    with torch.no_grad():
        assert torch.equal(got, cls.forward._ssb_original(m, obs))
    rc, _, _ = entry(ops, m.cnn, x, lab)
    msg = ops.lib.ssb_last_error(ops.ctx.handle)
    assert rc == SSB_E_SHAPE and b"too large" in msg and f"({nbytes} bytes".encode() in msg
    assert ops.ctx.launch_count == before


@pytest.mark.parametrize("labels", [False, True])
def test_misaligned_pointers_refused(labels):
    """Every pointer the kernels read or write as floats must be 4-byte aligned: SSB_E_INVALID_ARG, nothing launched."""
    c = cases.INPUT_LABELS if labels else cases.INPUT_LAYOUT
    cnn = cases.make_cnn(c, seed=15).to(DEV)
    x, lab = cases.make_inputs(c, 2, seed=16, device=DEV)
    ops = _ops()
    fn = b"ssb_audio_encoder_category_batch" if labels else b"ssb_audio_encoder_batch"

    def layers_with(i, **kw):
        layers = conv_layers(cnn)
        for k, v in kw.items():
            setattr(layers[i], k, v)
        return layers

    spec = torch.zeros(x.numel() + 1, device=DEV)
    feats = torch.zeros(2, cnn[6].in_features + 1, device=DEV)
    out = torch.zeros(2, cnn[6].out_features + 1, device=DEV)
    refusals = [(dict(spec=spec.data_ptr() + 2), b"bad arguments"),
                (dict(lin_weight=cnn[6].weight.data_ptr() + 2), b"bad arguments"),
                (dict(lin_bias=cnn[6].bias.data_ptr() + 2), b"bad arguments"),
                (dict(feats=feats.data_ptr() + 2), b"bad arguments"),
                (dict(out=out.data_ptr() + 2), b"bad arguments")]
    for i, conv in enumerate((cnn[0], cnn[2], cnn[4])):
        refusals.append((dict(layers=layers_with(i, d_weight=conv.weight.data_ptr() + 2)), b"bad layer %d" % (i + 1)))
        refusals.append((dict(layers=layers_with(i, d_bias=conv.bias.data_ptr() + 2)), b"bad layer %d" % (i + 1)))
    before = ops.ctx.launch_count
    for kw, msg in refusals:
        rc, _, _ = entry(ops, cnn, x, lab, **kw)
        assert rc == SSB_E_INVALID_ARG, kw
        err = ops.lib.ssb_last_error(ops.ctx.handle)
        assert err.startswith(fn + b": ") and msg in err, (kw, err)
    assert ops.ctx.launch_count == before
