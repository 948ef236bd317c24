"""The fused audio encoder (``ssb_audio_encoder_batch``, ``WaveformOps.audio_encoder``, ``patch_audio_cnn``) on the GPU:
against a float64 run of the same ``nn.Sequential``, bit-identity across batch sizes and positions, the shape limits,
and the patched reference-shaped ``AudioCNN`` classes against their original forward."""
import copy

import pytest

from test_encoder_host import make_cnn, reference_classes

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
nn = torch.nn

# observation shapes (65, ceil((1 + sr // 160) / 4), 2)
SHAPES = {16000: (65, 26, 2), 44100: (65, 69, 2), 48000: (65, 76, 2), 22050: (65, 35, 2)}


def _ops():
    from soundspaces_b200.renderer import WaveformOps
    return WaveformOps.get("cuda:0")


def _random_cnn(shape, c3, hidden, seed):
    torch.manual_seed(seed)
    cnn = make_cnn(shape, c3, hidden)
    with torch.no_grad():
        for m in cnn:
            if isinstance(m, (nn.Conv2d, nn.Linear)):
                m.bias.uniform_(-0.2, 0.2)                # non-zero biases so that every ReLU clips something
    return cnn


def _float64_runs(cnn, x):
    """(features, out) of ``cnn`` in float64 on the CPU, and the same pair for the bound network: |x|, |W|, |b|, no ReLU."""
    x64 = x.detach().cpu().double().permute(0, 3, 1, 2)
    ref = copy.deepcopy(cnn).cpu().double()
    bnd = copy.deepcopy(ref)
    with torch.no_grad():
        for i, m in enumerate(bnd):
            if isinstance(m, nn.ReLU):
                bnd[i] = nn.Identity()
            for p in m.parameters():
                p.abs_()
        return ref[:6](x64), ref(x64), bnd[:6](x64.abs()), bnd(x64.abs())


def _check(got, ref, bound):
    got = got.detach().cpu().double()
    assert got.shape == ref.shape
    err = (got - ref).abs()
    assert bool((err <= 1e-5 * bound).all()), f"max err / bound {(err / bound.clamp_min(1e-30)).max().item():.3g}"


@pytest.mark.parametrize("hidden", [512, 100])
@pytest.mark.parametrize("c3", [64, 32])                  # av_nav / savi, av_wan
@pytest.mark.parametrize("sr", [16000, 44100, 48000])
def test_encoder_against_float64(sr, c3, hidden):
    shape = SHAPES[sr]
    cnn = _random_cnn(shape, c3, hidden, seed=sr + c3 + hidden).cuda()
    x = torch.rand((129,) + shape, device="cuda") * 3.0
    f_ref, o_ref, f_bnd, o_bnd = _float64_runs(cnn, x)
    ops = _ops()
    for b in (1, 16, 129):
        feats = torch.full((b, f_ref.shape[1]), float("nan"), device="cuda")
        out = ops.audio_encoder(x[:b].contiguous(), cnn, features=feats)
        torch.cuda.synchronize()
        _check(feats, f_ref[:b], f_bnd[:b])
        _check(out, o_ref[:b], o_bnd[:b])


@pytest.mark.parametrize("sr", [16000, 44100])
def test_encoder_bit_identical_across_batches(sr):
    shape = SHAPES[sr]
    cnn = _random_cnn(shape, 64, 512, seed=5).cuda()
    x = torch.rand((129,) + shape, device="cuda") * 3.0
    ops = _ops()
    F = cnn[6].in_features
    f_all = torch.empty((129, F), device="cuda")
    out_all = ops.audio_encoder(x, cnn, features=f_all)
    f_rev = torch.empty((129, F), device="cuda")
    out_rev = ops.audio_encoder(x.flip(0).contiguous(), cnn, features=f_rev)
    assert torch.equal(out_rev.flip(0), out_all) and torch.equal(f_rev.flip(0), f_all)
    for k in (0, 15, 16, 17, 77, 128):
        f1 = torch.empty((1, F), device="cuda")
        out1 = ops.audio_encoder(x[k:k + 1].contiguous(), cnn, features=f1)
        assert torch.equal(out1[0], out_all[k]) and torch.equal(f1[0], f_all[k])
    # env 7 at every position j of a 129-env batch filled with other envs
    for j in (0, 1, 15, 16, 63, 127, 128):
        idx = torch.arange(129, device="cuda")
        idx[j], idx[7] = 7, j
        assert torch.equal(ops.audio_encoder(x[idx].contiguous(), cnn)[j], out_all[7])


def _layers(cnn, relus=(1, 1, 0)):
    from soundspaces_b200 import _lib
    layers = (_lib.Conv2dLayer * 3)()
    for i, (conv, relu) in enumerate(zip((cnn[0], cnn[2], cnn[4]), relus)):
        layers[i] = _lib.Conv2dLayer(conv.weight.data_ptr(), conv.bias.data_ptr(), conv.out_channels,
                                     *conv.kernel_size, *conv.stride, relu)
    return layers


def _abi(ops, cnn, x, F, relus=(1, 1, 0), lin_relu=1):
    lin = cnn[6]
    feats = torch.zeros((x.shape[0], max(F, 1)), device="cuda")
    out = torch.zeros((x.shape[0], lin.out_features), device="cuda")
    rc = ops.lib.ssb_audio_encoder_batch(ops.ctx.handle, x.shape[0], x.data_ptr(), x.shape[1], x.shape[2],
                                         _layers(cnn, relus), lin.weight.data_ptr(), lin.bias.data_ptr(), lin.out_features,
                                         lin_relu, feats.data_ptr(), out.data_ptr(), ops._stream())
    return rc, feats, out


def test_empty_conv3_is_refused():
    """22.05 kHz: 8x8/4 -> 32x15x7, 4x4/2 -> 64x6x2, 3x3/1 -> empty (the reference cannot build this model either)."""
    ops = _ops()
    shape = SHAPES[22050]
    torch.manual_seed(1)
    cnn = nn.Sequential(nn.Conv2d(2, 32, 8, 4), nn.ReLU(), nn.Conv2d(32, 64, 4, 2), nn.ReLU(), nn.Conv2d(64, 64, 3, 1),
                        nn.Flatten(), nn.Linear(64, 512), nn.ReLU()).cuda()
    x = torch.rand((16,) + shape, device="cuda")
    before = ops.ctx.launch_count
    rc, _, _ = _abi(ops, cnn, x, 0)
    assert rc == -4                                        # SSB_E_SHAPE
    assert b"layer 3 output is empty" in ops.lib.ssb_last_error(ops.ctx.handle)
    assert ops.ctx.launch_count == before                  # decided on the host: nothing launched
    with pytest.raises(ValueError, match="layer 3 output is empty"):
        ops.audio_encoder(x, cnn)


def _limit_cnn(c2):
    """(32, 8, 2) observation, 1x1 convolutions: 32*8*2 + 96*256 + c2*256 floats of activations plus the largest
    per-rank weight slice, conv2's ceil(c2 / 8) * 96 floats; c2 = 123 is exactly 232448 bytes (227 KB)."""
    torch.manual_seed(2)
    return nn.Sequential(nn.Conv2d(2, 96, 1), nn.ReLU(), nn.Conv2d(96, c2, 1), nn.ReLU(), nn.Conv2d(c2, 4, 1),
                         nn.Flatten(), nn.Linear(4 * 32 * 8, 33), nn.ReLU()).cuda()


def test_shared_memory_limit():
    ops = _ops()
    assert (32 * 8 * 2 + 96 * 256 + 123 * 256 + 16 * 96) * 4 == 232448
    x = torch.rand((3, 32, 8, 2), device="cuda") * 3.0
    cnn = _limit_cnn(123)
    feats = torch.empty((3, 1024), device="cuda")
    out = ops.audio_encoder(x, cnn, features=feats)
    f_ref, o_ref, f_bnd, o_bnd = _float64_runs(cnn, x)
    _check(feats, f_ref, f_bnd)
    _check(out, o_ref, o_bnd)
    before = ops.ctx.launch_count
    rc, _, _ = _abi(ops, _limit_cnn(124), x, 1024)
    assert rc == -4
    assert b"too large" in ops.lib.ssb_last_error(ops.ctx.handle)
    assert ops.ctx.launch_count == before


def test_abi_flags_and_bad_arguments():
    """Per-layer ReLU flags and the identity output activation follow the arguments; malformed arguments are refused."""
    ops = _ops()
    shape = SHAPES[16000]
    cnn = _random_cnn(shape, 64, 100, seed=9).cuda()
    x = torch.rand((5,) + shape, device="cuda") * 3.0
    rc, feats, out = _abi(ops, cnn, x, cnn[6].in_features, relus=(0, 1, 1), lin_relu=0)
    assert rc == 0
    plain = copy.deepcopy(nn.Sequential(cnn[0], cnn[2], nn.ReLU(), cnn[4], nn.ReLU(), cnn[5], cnn[6])).cpu().double()
    with torch.no_grad():
        ref = plain(x.cpu().double().permute(0, 3, 1, 2))
    assert (out.cpu().double() - ref).abs().max().item() <= 1e-4 * ref.abs().max().item()
    assert (out < 0).any()                                  # identity output activation
    for kw in ({"lin_relu": 2}, {"relus": (1, 2, 0)}):
        rc, _, _ = _abi(ops, cnn, x, cnn[6].in_features, **kw)
        assert rc == -1                                     # SSB_E_INVALID_ARG
    with pytest.raises(ValueError):
        ops.audio_encoder(x.permute(0, 2, 1, 3), cnn)       # not contiguous
    with pytest.raises(ValueError):
        ops.audio_encoder(x, _random_cnn(SHAPES[44100], 64, 100, seed=9).cuda())   # Linear.in_features mismatch


def _bad_cnns():
    base = lambda: make_cnn(SHAPES[16000])                  # noqa: E731
    out = []
    m = base(); m[0] = nn.Conv2d(2, 32, 5, 2, padding=1); out.append(m)
    m = base(); m[2] = nn.Conv2d(32, 64, 3, 2, dilation=2); out.append(m)
    m = base(); m[4] = nn.Conv2d(64, 64, 3, 1, groups=2); out.append(m)
    m = base(); m[0] = nn.Conv2d(3, 32, 5, 2); out.append(m)
    m = base(); out.append(nn.Sequential(*[m[i] for i in (0, 2, 3, 4, 5, 6, 7)]))
    m = base(); out.append(nn.Sequential(*[m[i] for i in (0, 1, 2, 3, 4, 6, 5, 7)]))
    return out


def test_audio_encoder_refuses_other_layouts():
    ops = _ops()
    x = torch.rand((2,) + SHAPES[16000], device="cuda")
    for cnn in _bad_cnns():
        with pytest.raises(ValueError):
            ops.audio_encoder(x, cnn.cuda())


@pytest.mark.parametrize("sr", [16000, 44100])
def test_patched_audio_cnn_matches_original(sr):
    from soundspaces_b200.encoder import patch_audio_cnn
    shape = SHAPES[sr]
    prev = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    try:
        for cls in reference_classes():
            torch.manual_seed(sr)
            model = cls(shape).cuda()
            key = getattr(model, "_audiogoal_sensor", "spectrogram")
            obs = {key: torch.rand((16,) + shape, device="cuda") * 3.0}
            with torch.no_grad():
                ref = model(obs)
                patch_audio_cnn(cls)
                launches = _ops().ctx.launch_count
                got = model(obs)
                assert _ops().ctx.launch_count == launches + 2          # the fused path ran
            assert torch.allclose(got, ref, rtol=1e-4, atol=1e-4)
            grad = model(obs)                                          # grad enabled: the original forward
            assert grad.requires_grad and torch.allclose(grad, ref, rtol=1e-4, atol=1e-4)
    finally:
        torch.backends.cudnn.allow_tf32 = prev
