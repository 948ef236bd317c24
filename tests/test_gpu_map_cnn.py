"""The fused AV-WaN map encoder (``ssb_map_encoder_batch``, ``WaveformOps.map_encoder``, ``patch_map_cnn``) on the GPU:
per-env accuracy against float64 runs of the same module (max|got_b - ref_b| <= 1e-4 max|ref_b|) and against the
reference recording, bit-identity across batch sizes and positions, NaN / Inf containment, refusals, launch counts,
and the patched stand-ins against their original forward, alone and inside AV-WaN's rollout-time ``Net.forward``."""
import copy

import numpy as np
import pytest

from avnav_models import RNNStateEncoder, VisualCNN, set_params
from map_cnn_models import REFERENCE_SHAPES, AudioNavBaselineNet, MapCNN, map_obs
from test_encoder_host import reference_classes

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
nn = torch.nn

GEO_200, GEO_400, GEO_AM = ((8, 4, 3), (4, 2, 1)), ((8, 4, 3), (5, 4, 2)), ((5, 3, 3), (2, 1, 1))


def _ops():
    from soundspaces_b200.renderer import WaveformOps
    return WaveformOps.get("cuda:0")


def _map_cnn(H, W, C, map_type="gm", hidden=512, seed=0, layers=None):
    torch.manual_seed(seed)
    m = MapCNN(H, W, C, hidden, map_type, layers=layers)
    with torch.no_grad():
        for layer in m.cnn:
            if isinstance(layer, (nn.Conv2d, nn.Linear)):
                layer.bias.uniform_(-0.1, 0.1)             # non-zero biases so that every ReLU clips something
    return m.cuda().eval()


def _ref_map(name, B, kind, seed):
    map_type, H, W, C = REFERENCE_SHAPES[name]
    return map_obs(B, H, W, C, seed=seed, kind=map_type if kind == "like" else "dense").cuda()


def _float64(m, x, idx=None):
    """(features, out) of ``m.cnn`` in float64 on the CPU for the envs ``idx`` (all when None)."""
    ref = copy.deepcopy(m).cpu().double()
    xx = (x if idx is None else x[idx]).cpu().double().permute(0, 3, 1, 2)
    with torch.no_grad():
        return ref.cnn[:6](xx), ref.cnn(xx)


def _check_per_env(got, ref):
    got = got.detach().cpu().double()
    assert got.shape == ref.shape
    for b in range(ref.shape[0]):
        scale = ref[b].abs().max().item()
        assert scale > 0
        err = (got[b] - ref[b]).abs().max().item()
        assert err <= 1e-4 * scale, f"env {b}: max err {err:.3g} > 1e-4 * {scale:.3g}"


def _run(ops, m, x, features=True):
    feats = torch.full((x.shape[0], m.cnn[6].in_features), float("nan"), device="cuda") if features else None
    out = ops.map_encoder(x, m.cnn, features=feats)
    return feats, out


@pytest.mark.parametrize("kind", ["like", "dense"])
@pytest.mark.parametrize("name", sorted(REFERENCE_SHAPES))
def test_against_float64(name, kind):
    """Reference-like maps (0 / 1 geometric, sparse non-negative acoustic) and dense random ones; the features buffer
    (filled with NaN beforehand) receives every conv3 value."""
    map_type, H, W, C = REFERENCE_SHAPES[name]
    m = _map_cnn(H, W, C, map_type, seed=H + C)
    x = _ref_map(name, 16, kind, seed=3)
    feats, out = _run(_ops(), m, x)
    assert not bool(torch.isnan(feats).any())
    f_ref, o_ref = _float64(m, x)
    _check_per_env(feats, f_ref)
    _check_per_env(out, o_ref)


@pytest.mark.parametrize("name", sorted(REFERENCE_SHAPES))
def test_against_reference_golden(name):
    """The parameters and maps of tests/golden/map_cnn_golden.npz, regenerated from their seeds, in float32 on the
    GPU against the reference MapCNN's float64 outputs."""
    from test_map_cnn_host import GOLDEN
    g = np.load(GOLDEN)
    H, W, C, hidden, N, pseed, xseed = (int(v) for v in g[f"{name}/config"])
    map_type = REFERENCE_SHAPES[name][0]
    m = set_params(MapCNN(H, W, C, hidden, map_type), pseed).cuda().eval()
    x = map_obs(N, H, W, C, seed=xseed, kind=map_type).cuda()
    _check_per_env(_ops().map_encoder(x, m.cnn), torch.from_numpy(g[f"{name}/out"]))


@pytest.mark.parametrize("H,W,C,layers", [
    (120, 200, 2, GEO_200), (200, 96, 3, GEO_200), (36, 36, 1, GEO_200),          # 36 x 36: conv3 is 1 x 1
    (400, 250, 1, GEO_400), (63, 63, 3, GEO_400), (70, 130, 2, GEO_400),          # 63 x 63: conv3 is 1 x 1
    (13, 13, 1, GEO_AM), (20, 37, 2, GEO_AM), (31, 17, 3, GEO_AM),                # 13 x 13: conv3 is 1 x 1
    (50, 61, 2, ((6, 3, 2), (3, 2, 1))),
])
def test_other_shapes(H, W, C, layers):
    """Non-square maps, one to three channels and the smallest input each geometry accepts; the last geometry is
    none of the reference's, so the kernel reads its kernel sizes at run time."""
    m = _map_cnn(H, W, C, hidden=100, seed=H + W + C, layers=layers)
    x = map_obs(19, H, W, C, seed=5, kind="dense").cuda()
    feats, out = _run(_ops(), m, x)
    f_ref, o_ref = _float64(m, x)
    _check_per_env(feats, f_ref)
    _check_per_env(out, o_ref)


@pytest.mark.parametrize("B", [1, 16, 128, 1024])
def test_batch_sizes(B):
    m = _map_cnn(200, 200, 2, seed=11)
    x = _ref_map("gm200", B, "like", seed=B)
    feats, out = _run(_ops(), m, x)
    idx = sorted({0, B // 3, B // 2, B - 1, min(15, B - 1), min(16, B - 1)})
    f_ref, o_ref = _float64(m, x, idx)
    _check_per_env(feats[idx], f_ref)
    _check_per_env(out[idx], o_ref)


@pytest.mark.parametrize("name", sorted(REFERENCE_SHAPES))
def test_bit_identical_across_batches(name):
    ops = _ops()
    map_type, H, W, C = REFERENCE_SHAPES[name]
    m = _map_cnn(H, W, C, map_type, seed=21)
    x = _ref_map(name, 129, "dense", seed=22)
    f_all, out_all = _run(ops, m, x)
    f_rev, out_rev = _run(ops, m, x.flip(0).contiguous())
    assert torch.equal(out_rev.flip(0), out_all) and torch.equal(f_rev.flip(0), f_all)
    for k in (0, 15, 16, 17, 128):
        f1, o1 = _run(ops, m, x[k:k + 1].contiguous())
        assert torch.equal(o1[0], out_all[k]) and torch.equal(f1[0], f_all[k])
    for j in (0, 1, 16, 127, 128):
        idx = torch.arange(129, device="cuda")
        idx[j], idx[7] = 7, j
        _, o = _run(ops, m, x[idx].contiguous(), features=False)
        assert torch.equal(o[j], out_all[7])


@pytest.mark.parametrize("name", ["gm200", "am20"])
def test_nan_and_inf_stay_in_their_env(name):
    """NaN in env 3 and +Inf in env 5 give those envs float64's NaN / Inf pattern (the ReLUs keep NaN); every other env
    is bit for bit what it is without them."""
    ops = _ops()
    map_type, H, W, C = REFERENCE_SHAPES[name]
    m = _map_cnn(H, W, C, map_type, seed=41)
    x = _ref_map(name, 8, "dense", seed=42)
    f_clean, o_clean = _run(ops, m, x)
    bad = x.clone()
    bad[3, H // 2, W // 3, 0] = float("nan")
    bad[5, H // 3, W // 2, C - 1] = float("inf")
    f_bad, o_bad = _run(ops, m, bad)
    keep = [b for b in range(8) if b not in (3, 5)]
    assert torch.equal(f_bad[keep], f_clean[keep]) and torch.equal(o_bad[keep], o_clean[keep])
    f_ref, o_ref = _float64(m, bad, [3, 5])
    for got, ref in ((f_bad[[3, 5]].cpu(), f_ref), (o_bad[[3, 5]].cpu(), o_ref)):
        assert torch.equal(torch.isnan(got), torch.isnan(ref))
        assert torch.equal(torch.isposinf(got), torch.isposinf(ref))
        assert torch.equal(torch.isneginf(got), torch.isneginf(ref))
    assert bool(torch.isnan(o_bad[3]).any())


def test_launch_count_is_fixed():
    ops = _ops()
    for name in sorted(REFERENCE_SHAPES):
        map_type, H, W, C = REFERENCE_SHAPES[name]
        m = _map_cnn(H, W, C, map_type, seed=3)
        for B in (1, 16, 1024):
            x = _ref_map(name, B, "like", seed=B)
            before = ops.ctx.launch_count
            _run(ops, m, x)
            assert ops.ctx.launch_count - before == 2, (name, B)


def _abi(ops, m, x, C, H, W, B, relu=(1, 1, 0), hidden=None, lin_relu=1):
    from soundspaces_b200 import _lib
    cnn = m.cnn
    layers = (_lib.Conv2dLayer * 3)()
    for i, (conv, r) in enumerate(zip((cnn[0], cnn[2], cnn[4]), relu)):
        layers[i] = _lib.Conv2dLayer(conv.weight.data_ptr(), conv.bias.data_ptr(), conv.out_channels,
                                     *conv.kernel_size, *conv.stride, r)
    lin = cnn[6]
    feats = torch.zeros(max(B, 1), lin.in_features, device="cuda")
    out = torch.zeros(max(B, 1), lin.out_features, device="cuda")
    rc = ops.lib.ssb_map_encoder_batch(ops.ctx.handle, B, x, C, H, W, layers, lin.weight.data_ptr(),
                                       lin.bias.data_ptr(), lin.out_features if hidden is None else hidden, lin_relu,
                                       feats.data_ptr(), out.data_ptr(), ops._stream())
    return rc, ops.lib.ssb_last_error(ops.ctx.handle)


def test_refusals_launch_nothing():
    from soundspaces_b200.encoder import map_encoder_smem_bytes
    ops = _ops()
    m = _map_cnn(200, 200, 2, seed=4)
    x = _ref_map("gm200", 2, "like", seed=1)
    p = x.data_ptr()
    big = _map_cnn(1000, 1000, 2, hidden=8, seed=5, layers=GEO_400)
    big_bytes = map_encoder_smem_bytes(big.cnn, 2, 1000, 1000)[0]
    assert big_bytes > 232448
    before = ops.ctx.launch_count
    cases = [
        (dict(B=-1), -1, b"bad arguments"), (dict(B=65536), -1, b"bad arguments"),
        (dict(C=0), -1, b"bad arguments"), (dict(H=0), -1, b"bad arguments"), (dict(W=0), -1, b"bad arguments"),
        (dict(x=None), -1, b"bad arguments"), (dict(x=p + 2), -1, b"bad arguments"),
        (dict(hidden=0), -1, b"bad arguments"), (dict(lin_relu=2), -1, b"bad arguments"),
        (dict(relu=(1, 2, 0)), -1, b"bad layer 2"),
        (dict(H=35), -4, b"layer 3 output is empty"), (dict(W=7), -4, b"layer 1 output is empty"),
    ]
    for kw, rc_want, msg in cases:
        args = dict(x=p, C=2, H=200, W=200, B=2)
        args.update(kw)
        rc, err = _abi(ops, m, args.pop("x"), args.pop("C"), args.pop("H"), args.pop("W"), args.pop("B"), **args)
        assert rc == rc_want and msg in err, (kw, rc, err)
    rc, err = _abi(ops, big, p, 2, 1000, 1000, 1)
    assert rc == -4 and f"{big_bytes} bytes of shared memory".encode() in err, err
    assert _abi(ops, m, p, 2, 200, 200, 0)[0] == 0                                  # B = 0
    assert ops.ctx.launch_count == before
    with pytest.raises(RuntimeError, match="shared memory"):
        ops.map_encoder(torch.zeros(1, 1000, 1000, 2, device="cuda"), big.cnn)
    assert ops.ctx.launch_count == before
    with pytest.raises(ValueError):
        ops.map_encoder(x.permute(0, 3, 1, 2), m.cnn)                               # not channels-last contiguous
    with pytest.raises(ValueError):
        ops.map_encoder(x[..., :1].contiguous(), m.cnn)                             # conv1 takes 2 channels
    assert ops.map_encoder(x[:0], m.cnn).shape == (0, 512) and ops.ctx.launch_count == before


# ------------------------------------------------------------------------------------------------ patched classes
@pytest.fixture
def no_tf32():
    saved = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = saved


def _patched():
    from soundspaces_b200.encoder import patch_map_cnn

    class Patched(MapCNN):
        pass
    return patch_map_cnn(Patched)


@pytest.mark.parametrize("name", sorted(REFERENCE_SHAPES))
def test_patched_matches_original(no_tf32, name):
    map_type, H, W, C = REFERENCE_SHAPES[name]
    cls = _patched()
    torch.manual_seed(31)
    m = cls(H, W, C, 512, map_type).cuda()
    obs = {map_type: _ref_map(name, 16, "like", seed=32)}
    ops = _ops()
    with torch.no_grad():
        before = ops.ctx.launch_count
        got = m(obs)
        assert ops.ctx.launch_count - before == 2             # the fused path ran
        want = cls.forward._ssb_original(m, obs)
    _check_per_env(got, want.double().cpu())


def test_patched_grad_runs_original_bit_for_bit():
    cls = _patched()
    torch.manual_seed(33)
    m = cls(200, 200, 2, 512).cuda()
    obs = {"gm": _ref_map("gm200", 4, "like", seed=34)}
    ops = _ops()
    before = ops.ctx.launch_count
    got = m(obs)
    assert got.requires_grad and ops.ctx.launch_count == before
    assert torch.equal(got, cls.forward._ssb_original(m, obs))


@pytest.mark.parametrize("gm_size", [200, 400])
def test_patched_policy_net_matches_unpatched(no_tf32, gm_size):
    """AV-WaN's rollout-time Net.forward (audio, gm, am, depth visual and state encoders) with every patch against
    the same modules without them, in 9 library launches: audio 2, gm 2, am 2, visual 2, GRU 1."""
    from soundspaces_b200.encoder import patch_audio_cnn, patch_map_cnn, patch_visual_cnn
    from soundspaces_b200.rnn import patch_rnn_state_encoder
    AudioCNN = reference_classes()[1]

    class PAudio(AudioCNN):
        pass

    class PMap(MapCNN):
        pass

    class PVisual(VisualCNN):
        pass

    class PRnn(RNNStateEncoder):
        pass

    torch.manual_seed(7)
    plain = AudioNavBaselineNet(AudioCNN((65, 26, 2), 512), MapCNN(gm_size, gm_size, 2, 512, "gm"),
                                MapCNN(20, 20, 1, 512, "am"), VisualCNN(0, 1, 128, 128, 512, "av_wan")).cuda()
    fused = copy.deepcopy(plain)
    fused.audio_encoder.__class__ = patch_audio_cnn(PAudio)
    fused.gm_encoder.__class__ = patch_map_cnn(PMap)
    fused.am_encoder.__class__ = PMap
    fused.visual_encoder.__class__ = patch_visual_cnn(PVisual)
    fused.state_encoder.__class__ = patch_rnn_state_encoder(PRnn)
    g = torch.Generator(device="cuda").manual_seed(8)
    obs = {"spectrogram": torch.rand(16, 65, 26, 2, device="cuda", generator=g) * 3,
           "gm": (torch.rand(16, gm_size, gm_size, 2, device="cuda", generator=g) < 0.3).float(),
           "am": torch.rand(16, 20, 20, 1, device="cuda", generator=g)
           * (torch.rand(16, 20, 20, 1, device="cuda", generator=g) < 0.125).float(),
           "depth": torch.rand(16, 128, 128, 1, device="cuda", generator=g)}
    h = torch.randn(1, 16, 512, device="cuda", generator=g)
    masks = (torch.arange(16, device="cuda") % 4 != 0).float()[:, None]
    ops = _ops()
    with torch.no_grad():
        before = ops.ctx.launch_count
        out, h_out = fused(obs, h, masks)
        assert ops.ctx.launch_count - before == 9
        want, h_want = plain(obs, h, masks)
    assert not bool(torch.isnan(out).any())
    _check_per_env(out, want.double().cpu())
    _check_per_env(h_out[0], h_want[0].double().cpu())
