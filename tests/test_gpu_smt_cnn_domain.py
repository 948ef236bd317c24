"""SAVi's visual encoder (``ssb_smt_cnn_batch``) across the observation shapes, channel counts, heads, crops and batch
sizes its entry accepts (tests/smt_cnn_domain_cases.py).

The input stage has an exact oracle: the float32 image the header documents (tests/smt_cnn_models.py:
prep_image_f32), replayed through the same encoder as a 64 x 64 observation without a resize, where the input stage
is the identity.  The features of the two calls must be bit-identical.  Every case is also held to 1e-4 of each env's
largest float64 output, and the file checks NaN / Inf containment, batch identity up to B = 1024, the heads' columns
and biases, the scratch shared with ``ssb_smt_resnet18_batch``, and the patched module at other channel counts."""
import copy

import numpy as np
import pytest

import smt_cnn_domain_cases as cases
from smt_cnn_models import CROP, SMTCNN, bins, observations, prep_image_f32, resize_crop64, set_params

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

LAUNCHES = 39
TOL = 1e-4
RGB_MUL = np.float32(1) / np.float32(255)
NAMES = ("rgb", "depth")


def _ops():
    from soundspaces_b200.renderer import WaveformOps
    return WaveformOps.get("cuda:0")


def _model(c, seed=7):
    """The SMTCNN of a case: input 0 is RGB, input 1 depth, each with its channels, fc width and bias."""
    ms = dict(zip(NAMES, c["inputs"]))
    m = SMTCNN({k: v["C"] for k, v in ms.items()}, n_out={k: v["n_out"] for k, v in ms.items()},
               no_bias=[k for k, v in ms.items() if not v["bias"]])
    return set_params(m, seed).cuda().eval()


def _obs(c, seed=1, B=None):
    """Seeded observations of a case on the device, (B, H, W, C) each."""
    out = []
    for k, m in enumerate(c["inputs"]):
        o = observations(B or c["B"], m["H"], m["W"], seed + 17 * k, rgb=m["C"] if m["scale"] else 0,
                         depth=0 if m["scale"] else m["C"])
        out.append(o["rgb" if m["scale"] else "depth"].cuda())
    return out


def _nets(model, c):
    return [getattr(model, f"{n}_encoder") for n in NAMES[:len(c["inputs"])]]


def _geom(m):
    return m["rh"], m["rw"], m["cy"], m["cx"]


def _fused(c, model, xs):
    """One ssb_smt_cnn_batch call with the case's geometries: through WaveformOps.smt_cnn where they are the
    reference's, else through the C entry with a table built here."""
    from soundspaces_b200 import _lib
    from soundspaces_b200.belief_nets import conv_table
    from soundspaces_b200.encoder import resize_center_crop_geometry
    nets, ops = _nets(model, c), _ops()
    if all(_geom(m) == resize_center_crop_geometry(m["H"], m["W"]) for m in c["inputs"]) and \
            [m["scale"] for m in c["inputs"]] == [1, 0][:len(xs)]:
        return ops.smt_cnn(xs[0], xs[1] if len(xs) > 1 else None, nets[0], nets[1] if len(xs) > 1 else None)
    table = (_lib.SmtCnnInput * len(xs))()
    for k, (m, x, net) in enumerate(zip(c["inputs"], xs, nets)):
        fc = net.fc
        table[k] = _lib.SmtCnnInput(x.data_ptr(), m["C"], m["H"], m["W"], m["scale"], *_geom(m),
                                    conv_table(net, False), fc.weight.data_ptr(),
                                    fc.bias.data_ptr() if fc.bias is not None else None, fc.in_features,
                                    fc.out_features)
    out = torch.empty(xs[0].shape[0], sum(m["n_out"] for m in c["inputs"]), device="cuda")
    ops.ctx.check(ops.lib.ssb_smt_cnn_batch(ops.ctx.handle, xs[0].shape[0], len(xs), table, out.data_ptr(),
                                            ops._stream()), "ssb_smt_cnn_batch")
    return out


def _image(m, x):
    """The documented float32 image of one input, (B, 64, 64, C) on the device: a 64 x 64 observation."""
    img = prep_image_f32(x.cpu().numpy(), RGB_MUL if m["scale"] else 1, *_geom(m))
    return torch.from_numpy(img.transpose(0, 2, 3, 1).copy()).cuda()


def _replay(c, model, xs, out):
    """Each input's documented image through its encoder with the input stage as the identity (depth, no resize)
    gives bit for bit the features of the full call."""
    col = 0
    for m, x, net in zip(c["inputs"], xs, _nets(model, c)):
        got = _ops().smt_cnn(None, _image(m, x), None, net, resize=False)
        assert torch.equal(got, out[:, col:col + m["n_out"]]), (c["name"], m, (got - out[:, col:col + m["n_out"]])
                                                               .abs().max().item())
        col += m["n_out"]


def _ref64(c, model, xs, resize=None):
    """float64 forward on the device: the float64 area-matrix crop (or ``resize``) and each encoder in float64."""
    feats = []
    for m, x, net in zip(c["inputs"], xs, _nets(model, c)):
        x64 = x.permute(0, 3, 1, 2).double() / (255.0 if m["scale"] else 1.0)
        img = (resize or resize_crop64)(x64, *_geom(m))
        with torch.no_grad():
            feats.append(copy.deepcopy(net).double()(img))
    return torch.cat(feats, dim=1)


def _check(got, want, what=""):
    """Every env within TOL max|ref_b| of float64; returns the worst ratio to the bar."""
    got, want = got.double(), want.double()
    err = (got - want).abs().amax(dim=1)
    scale = want.abs().amax(dim=1)
    ratio = (err / (TOL * scale)).max().item()
    assert ratio <= 1.0, f"{what}: worst env at {ratio:.3f} of the bar"
    return ratio


# ------------------------------------------------------------------------------------------------ every case
@pytest.mark.parametrize("c", cases.fused_cases(), ids=lambda c: c["name"])
def test_identity_replay_and_accuracy(c):
    """The input stage computes exactly the documented image, and the features are within the float64 bar."""
    model = _model(c, seed=len(c["name"]))
    xs = _obs(c, seed=len(c["name"]) + 1)
    out = _fused(c, model, xs)
    assert out.shape == (c["B"], sum(m["n_out"] for m in c["inputs"]))
    _replay(c, model, xs, out)
    _check(out, _ref64(c, model, xs), c["name"])


def _interpolate64(x64, rh, rw, cy, cx):
    return torch.nn.functional.interpolate(x64, size=(rh, rw), mode="area")[..., cy:cy + CROP, cx:cx + CROP]


@pytest.mark.parametrize("hw", [(480, 640), (17, 900), (1, 1024), (255, 255)])
def test_accuracy_against_float64_interpolate(hw):
    """The area-matrix stand-in agrees with torch's own float64 area resize, and the features meet the bar against a
    float64 forward built on the latter."""
    c = cases.case("interp", cases.modality(*hw, 3, 1), cases.modality(*hw, 2, 0), B=3)
    model = _model(c, seed=3)
    xs = _obs(c, seed=5)
    a, b = _ref64(c, model, xs), _ref64(c, model, xs, resize=_interpolate64)
    assert (a - b).abs().max().item() <= 1e-12 * b.abs().max().item()
    _check(_fused(c, model, xs), b, str(hw))


# ------------------------------------------------------------------------------------------------ NaN / Inf
def _unread_mask(m):
    h0, h1 = bins(m["H"], m["rh"], m["cy"])
    w0, w1 = bins(m["W"], m["rw"], m["cx"])
    mask = torch.ones(m["H"], m["W"], dtype=torch.bool)
    mask[int(h0[0]):int(h1[-1]), int(w0[0]):int(w1[-1])] = False
    return mask.cuda()


@pytest.mark.parametrize("hw", cases.UNREAD_SHAPES)
def test_unread_pixels_never_reach_the_features(hw):
    """Every input pixel that no bin of the crop reads set to NaN, then to +Inf: the features are the clean run's bit
    for bit."""
    c = cases.case("unread", cases.modality(*hw, 3, 1), cases.modality(*hw, 2, 0), B=3)
    model = _model(c)
    xs = _obs(c, seed=2)
    clean = _fused(c, model, xs)
    masks = [_unread_mask(m) for m in c["inputs"]]
    assert all(mk.any() for mk in masks)
    for v in (float("nan"), float("inf")):
        bad = [x.clone() for x in xs]
        for x, mk in zip(bad, masks):
            x[:, mk, :] = v
        assert torch.equal(_fused(c, model, bad), clean), v


def test_nan_in_a_pixel_two_upsampling_bins_share():
    """A NaN in an input pixel two overlapping bins read (along rows and columns) changes only that env's features of
    that modality."""
    H, W = cases.SHARED_PIXEL_SHAPE
    c = cases.case("shared", cases.modality(H, W, 3, 1), cases.modality(H, W, 1, 0), B=4)
    m = c["inputs"][0]
    shared = []
    for n_in, n_out, c0 in ((H, m["rh"], m["cy"]), (W, m["rw"], m["cx"])):
        lo, hi = bins(n_in, n_out, c0)
        i = int(np.nonzero(lo[1:] < hi[:-1])[0][0])
        assert lo[i + 1] == hi[i] - 1
        shared.append(int(lo[i + 1]))
    model = _model(c)
    xs = _obs(c, seed=4)
    clean = _fused(c, model, xs)
    bad = [x.clone() for x in xs]
    bad[0][2, shared[0], shared[1], 1] = float("nan")
    out = _fused(c, model, bad)
    keep = [b for b in range(4) if b != 2]
    assert torch.equal(out[keep], clean[keep]) and torch.equal(out[2, 64:], clean[2, 64:])
    assert not torch.equal(out[2, :64], clean[2, :64])


# ------------------------------------------------------------------------------------------------ batch
def test_batch_identity_mixed_geometry_and_channels():
    """RGB 130 x 70 with 5 channels (four K ranges) beside depth 17 x 900 with 2 (one): an env's features are bit-identical
    at B = 1, 3, 129 and under a permutation of the full batch, and whether its modality runs alone."""
    c = cases.IDENTITY_CASE
    model = _model(c, seed=9)
    xs = _obs(c, seed=6)
    full = _fused(c, model, xs)
    _check(full, _ref64(c, model, xs), "identity")
    for B in cases.IDENTITY_BATCHES:
        assert torch.equal(_fused(c, model, [x[:B].contiguous() for x in xs]), full[:B]), B
    perm = torch.randperm(c["B"], generator=torch.Generator().manual_seed(2)).cuda()
    assert torch.equal(_fused(c, model, [x[perm].contiguous() for x in xs]), full[perm])
    n0 = c["inputs"][0]["n_out"]
    assert torch.equal(_fused(cases.case("alone", c["inputs"][0], B=c["B"]), model, xs[:1]), full[:, :n0])
    assert torch.equal(_ops().smt_cnn(None, xs[1], None, model.depth_encoder), full[:, n0:])


def test_largest_batch():
    """B = 1024 (RGB-D at 96 x 128, about 3 GB of scratch): every env within the float64 bar."""
    c = cases.MAX_B_CASE
    model = _model(c, seed=10)
    xs = _obs(c, seed=7)
    out = _fused(c, model, xs)
    for s in range(0, c["B"], 256):
        part = [x[s:s + 256] for x in xs]
        _check(out[s:s + 256], _ref64(c, model, part), f"envs {s}..")
    assert torch.equal(_fused(c, model, [x[-3:].contiguous() for x in xs]), out[-3:])
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------------ heads
def test_heads_land_in_their_columns():
    """n_out 257 + 1 and 100 + 64: each input's features at its own column offset with the summed row stride, equal to
    the input run alone; a bias-less fc gives the biased fc's result minus its bias to float32 rounding."""
    for c in cases.PAIR_CASES[:2]:
        model = _model(c, seed=12)
        xs = _obs(c, seed=8)
        out = _fused(c, model, xs)
        n0 = c["inputs"][0]["n_out"]
        assert out.shape == (c["B"], n0 + c["inputs"][1]["n_out"])
        assert torch.equal(_fused(cases.case("a", c["inputs"][0], B=c["B"]), model, xs[:1]), out[:, :n0])
        assert torch.equal(_ops().smt_cnn(None, xs[1], None, model.depth_encoder), out[:, n0:])
    c = cases.PAIR_CASES[1]                                         # RGB's fc without a bias
    model = _model(c, seed=12)
    xs = _obs(c, seed=8)
    plain = _fused(c, model, xs)
    biased = copy.deepcopy(model)
    biased.rgb_encoder.fc = torch.nn.Linear(8192, 100).cuda()
    with torch.no_grad():
        biased.rgb_encoder.fc.weight.copy_(model.rgb_encoder.fc.weight)
        biased.rgb_encoder.fc.bias.copy_(torch.linspace(-3, 3, 100))
    with_bias = _fused(c, biased, xs)
    assert torch.equal(with_bias[:, 100:], plain[:, 100:])
    d = with_bias[:, :100] - plain[:, :100] - biased.rgb_encoder.fc.bias
    assert d.abs().max().item() <= 1e-6 * (plain[:, :100].abs().max().item() + 3)


# ------------------------------------------------------------------------------------------------ scratch
def test_shared_scratch():
    """A call repeated after a larger call (more channels, larger B) and after ssb_smt_resnet18_batch on the same
    context (they share its scratch) gives bit-identical features."""
    from belief_nets_models import make_net
    small = cases.PAIR_CASES[0]
    model = _model(small, seed=13)
    xs = _obs(small, seed=9)
    first = _fused(small, model, xs)
    big = cases.case("big", cases.modality(100, 100, 8, 1), cases.modality(640, 480, 8, 0), B=64)
    bmodel = _model(big, seed=14)
    _fused(big, bmodel, _obs(big, seed=10))
    assert torch.equal(_fused(small, model, xs), first)
    net = make_net("smt2", seed=1).cuda()
    spec = torch.log1p(torch.rand(129, 65, 26, 2, generator=torch.Generator().manual_seed(3)) * 20).cuda()
    _ops().smt_resnet18(spec, net, None)
    assert torch.equal(_fused(small, model, xs), first)
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------ module level
@pytest.mark.parametrize("channels,no_bias", [({"rgb": 4, "depth": 2}, ()), ({"rgb": 3, "depth": 1}, ("rgb",)),
                                              ({"depth": 2}, ("depth",))])
def test_patched_module_other_channels(channels, no_bias):
    """Patched SMTCNNs with RGB C = 4 and depth C = 2, and with a bias-less fc, run fused in 39 launches and match the
    unpatched module's float64 forward."""
    from soundspaces_b200.encoder import patch_smt_cnn
    cls = type("SMTCNN", (SMTCNN,), {})
    patch_smt_cnn(cls)
    plain = set_params(SMTCNN(channels, no_bias=no_bias), 15).eval()
    patched = cls(channels, no_bias=no_bias)
    patched.load_state_dict(plain.state_dict())
    patched = patched.cuda().eval()
    obs = {k: v.cuda() for k, v in observations(6, 96, 128, 11, rgb=channels.get("rgb", 0),
                                                  depth=channels.get("depth", 0)).items()}
    ops = _ops()
    with torch.no_grad():
        before = ops.ctx.launch_count
        got = patched(obs)
        assert ops.ctx.launch_count == before + LAUNCHES
        want = copy.deepcopy(plain).double()({k: v.cpu().double() for k, v in obs.items()})
    assert got.shape == want.shape == (6, 64 * len(channels))
    _check(got.cpu(), want, str(channels))
