"""The fused audio encoder for SAVi with a distractor sound (``ssb_audio_encoder_category_batch``,
``WaveformOps.audio_encoder(..., category=)``, ``patch_audio_cnn(cls, category=True)``) on the GPU: against a float64
run of the same 23-channel ``nn.Sequential`` on the concatenated input, bit-identity across batch sizes, positions and
label row strides, the shape limits and refusals, and the patched SAVi-shaped ``AudioCNN`` against its original
forward."""
import copy

import pytest

from test_encoder_host import make_cnn, reference_classes

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
nn = torch.nn

# observation shapes (65, ceil((1 + sr // 160) / 4), 2)
SHAPES = {16000: (65, 26, 2), 44100: (65, 69, 2), 48000: (65, 76, 2)}
N_CAT = 21


def _ops():
    from soundspaces_b200.renderer import WaveformOps
    return WaveformOps.get("cuda:0")


def _random_cnn(shape, c3, hidden, seed, n_cat=N_CAT):
    torch.manual_seed(seed)
    cnn = make_cnn(shape, c3, hidden, in_ch=2 + n_cat)
    with torch.no_grad():
        for m in cnn:
            if isinstance(m, (nn.Conv2d, nn.Linear)):
                m.bias.uniform_(-0.2, 0.2)                # non-zero biases so that every ReLU clips something
    return cnn.cuda()


def _labels(kind, n, n_cat=N_CAT, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    if kind == "one_hot":
        idx = torch.randint(0, n_cat, (n,), device="cuda", generator=g)
        return nn.functional.one_hot(idx, n_cat).float()
    if kind == "zero":
        return torch.zeros((n, n_cat), device="cuda")
    return torch.rand((n, n_cat), device="cuda", generator=g) * 2.0 - 1.0             # signed soft values


def _float64_runs(cnn, x, lab):
    """(features, out) of ``cnn`` on cat(permute(x), expand(lab)) in float64 on the CPU, and the same pair for the
    bound network: |x|, |labels|, |W|, |b|, no ReLU."""
    x64 = x.detach().cpu().double().permute(0, 3, 1, 2)
    l64 = lab.detach().cpu().double()
    inp = torch.cat([x64, l64[:, :, None, None].expand(l64.shape + x64.shape[-2:])], dim=1)
    ref = copy.deepcopy(cnn).cpu().double()
    bnd = copy.deepcopy(ref)
    with torch.no_grad():
        for i, m in enumerate(bnd):
            if isinstance(m, nn.ReLU):
                bnd[i] = nn.Identity()
            for p in m.parameters():
                p.abs_()
        return ref[:6](inp), ref(inp), bnd[:6](inp.abs()), bnd(inp.abs())


def _check(got, ref, bound):
    got = got.detach().cpu().double()
    assert got.shape == ref.shape
    err = (got - ref).abs()
    assert bool((err <= 1e-5 * bound).all()), f"max err / bound {(err / bound.clamp_min(1e-30)).max().item():.3g}"


@pytest.mark.parametrize("hidden", [128, 512])
@pytest.mark.parametrize("c3", [64, 32])
@pytest.mark.parametrize("sr", [16000, 44100, 48000])
def test_category_encoder_against_float64(sr, c3, hidden):
    shape = SHAPES[sr]
    cnn = _random_cnn(shape, c3, hidden, seed=sr + c3 + hidden)
    x = torch.rand((129,) + shape, device="cuda") * 3.0
    ops = _ops()
    for kind in ("one_hot", "zero", "soft"):
        lab = _labels(kind, 129, seed=sr + hidden)
        f_ref, o_ref, f_bnd, o_bnd = _float64_runs(cnn, x, lab)
        for b in (1, 16, 129):
            feats = torch.full((b, f_ref.shape[1]), float("nan"), device="cuda")
            out = ops.audio_encoder(x[:b].contiguous(), cnn, features=feats, category=lab[:b].contiguous())
            torch.cuda.synchronize()
            _check(feats, f_ref[:b], f_bnd[:b])
            _check(out, o_ref[:b], o_bnd[:b])


@pytest.mark.parametrize("sr", [16000, 44100])
def test_category_encoder_bit_identical_across_batches(sr):
    shape = SHAPES[sr]
    cnn = _random_cnn(shape, 64, 128, seed=5)
    x = torch.rand((129,) + shape, device="cuda") * 3.0
    lab = _labels("soft", 129, seed=6)
    ops = _ops()
    F = cnn[6].in_features
    f_all = torch.empty((129, F), device="cuda")
    out_all = ops.audio_encoder(x, cnn, features=f_all, category=lab)
    f_rev = torch.empty((129, F), device="cuda")
    out_rev = ops.audio_encoder(x.flip(0).contiguous(), cnn, features=f_rev, category=lab.flip(0).contiguous())
    assert torch.equal(out_rev.flip(0), out_all) and torch.equal(f_rev.flip(0), f_all)
    for k in (0, 15, 16, 17, 77, 128):
        f1 = torch.empty((1, F), device="cuda")
        out1 = ops.audio_encoder(x[k:k + 1].contiguous(), cnn, features=f1, category=lab[k:k + 1].contiguous())
        assert torch.equal(out1[0], out_all[k]) and torch.equal(f1[0], f_all[k])
    # env 7 at every position j of a 129-env batch filled with other envs, its labels moved with it
    for j in (0, 1, 15, 16, 63, 127, 128):
        idx = torch.arange(129, device="cuda")
        idx[j], idx[7] = 7, j
        assert torch.equal(ops.audio_encoder(x[idx].contiguous(), cnn, category=lab[idx].contiguous())[j], out_all[7])


@pytest.mark.parametrize("sr", [16000, 44100])
def test_label_row_stride(sr):
    """Labels as a column slice of a wider tensor, NaN in the other columns: bit-identical to contiguous labels."""
    shape = SHAPES[sr]
    cnn = _random_cnn(shape, 64, 128, seed=7)
    x = torch.rand((17,) + shape, device="cuda") * 3.0
    lab = _labels("soft", 17, seed=8)
    ops = _ops()
    ref = ops.audio_encoder(x, cnn, category=lab)
    for width, col in ((22, 1), (37, 0), (64, 40)):
        wide = torch.full((17, width), float("nan"), device="cuda")
        wide[:, col:col + N_CAT] = lab
        view = wide[:, col:col + N_CAT]
        assert view.stride() == (width, 1)
        assert torch.equal(ops.audio_encoder(x, cnn, category=view), ref)
        assert torch.equal(ops.audio_encoder(x[3:4], cnn, category=view[3:4]), ref[3:4])


def _layers(cnn, relus=(1, 1, 0)):
    from soundspaces_b200 import _lib
    layers = (_lib.Conv2dLayer * 3)()
    for i, (conv, relu) in enumerate(zip((cnn[0], cnn[2], cnn[4]), relus)):
        layers[i] = _lib.Conv2dLayer(conv.weight.data_ptr(), conv.bias.data_ptr(), conv.out_channels,
                                     *conv.kernel_size, *conv.stride, relu)
    return layers


def _abi(ops, cnn, x, labels_ptr, n_labels, label_stride):
    lin = cnn[6]
    feats = torch.zeros((x.shape[0], lin.in_features), device="cuda")
    out = torch.zeros((x.shape[0], lin.out_features), device="cuda")
    rc = ops.lib.ssb_audio_encoder_category_batch(
        ops.ctx.handle, x.shape[0], x.data_ptr(), x.shape[1], x.shape[2], _layers(cnn), labels_ptr, n_labels,
        label_stride, lin.weight.data_ptr(), lin.bias.data_ptr(), lin.out_features, 1, feats.data_ptr(),
        out.data_ptr(), ops._stream())
    return rc, feats, out


@pytest.mark.parametrize("sr", [16000, 44100])
def test_no_labels_matches_ear_only_entry(sr):
    """n_labels = 0 (d_labels NULL) is bit-identical to ssb_audio_encoder_batch."""
    shape = SHAPES[sr]
    cnn = _random_cnn(shape, 64, 512, seed=11, n_cat=0)
    x = torch.rand((33,) + shape, device="cuda") * 3.0
    ops = _ops()
    feats = torch.empty((33, cnn[6].in_features), device="cuda")
    ref = ops.audio_encoder(x, cnn, features=feats)
    rc, f0, out0 = _abi(ops, cnn, x, None, 0, 0)
    assert rc == 0
    assert torch.equal(out0, ref) and torch.equal(f0, feats)
    empty = torch.empty((33, 0), device="cuda")
    assert torch.equal(ops.audio_encoder(x, cnn, category=empty), ref)


def _limit_cnn(c2, n_cat=222):
    """(16, 16, 2) observation, conv1 16x16 over the whole input, then 1x1 convolutions: 512 + 8 + c2 floats of
    observation and activations plus the largest per-rank weight slice, conv1's 1 * (2 + 222) * 256 floats; c2 = 248 is
    exactly 232448 bytes (227 KB)."""
    torch.manual_seed(12)
    return nn.Sequential(nn.Conv2d(2 + n_cat, 8, 16), nn.ReLU(), nn.Conv2d(8, c2, 1), nn.ReLU(), nn.Conv2d(c2, 4, 1),
                         nn.Flatten(), nn.Linear(4, 33), nn.ReLU()).cuda()


def test_shared_memory_limit_with_conv1_slice_largest():
    ops = _ops()
    assert (512 + 8 + 248 + 224 * 256) * 4 == 232448
    assert 224 * 256 > max(31 * 8, 248)                    # conv1's slice is the largest of the three
    assert (512 + 8 + 249 + 224 * 256) * 4 == 232448 + 4 and 224 * 256 > max(32 * 8, 249)
    x = torch.rand((3, 16, 16, 2), device="cuda") * 3.0
    lab = _labels("soft", 3, n_cat=222, seed=13)
    cnn = _limit_cnn(248)
    feats = torch.empty((3, 4), device="cuda")
    out = ops.audio_encoder(x, cnn, features=feats, category=lab)
    f_ref, o_ref, f_bnd, o_bnd = _float64_runs(cnn, x, lab)
    _check(feats, f_ref, f_bnd)
    _check(out, o_ref, o_bnd)
    before = ops.ctx.launch_count
    rc, _, _ = _abi(ops, _limit_cnn(249), x, lab.data_ptr(), 222, 222)
    assert rc == -4                                        # SSB_E_SHAPE
    msg = ops.lib.ssb_last_error(ops.ctx.handle)
    assert b"ssb_audio_encoder_category_batch" in msg and b"too large" in msg and b"232452 bytes" in msg
    assert ops.ctx.launch_count == before                  # decided on the host: nothing launched


def test_label_refusals():
    ops = _ops()
    shape = SHAPES[16000]
    cnn = _random_cnn(shape, 64, 128, seed=14)
    x = torch.rand((4,) + shape, device="cuda")
    lab = _labels("one_hot", 4, seed=15)
    buf = torch.zeros(4 * N_CAT + 1, device="cuda")
    rc, _, _ = _abi(ops, cnn, x, lab.data_ptr(), N_CAT, N_CAT)
    assert rc == 0
    torch.cuda.synchronize()
    before = ops.ctx.launch_count
    for ptr, n_labels, stride in ((lab.data_ptr(), -1, N_CAT),          # negative label count
                                  (None, N_CAT, N_CAT),                  # labels without a pointer
                                  (lab.data_ptr(), N_CAT, N_CAT - 1),    # rows overlap
                                  (None, 0, -1),                         # negative stride
                                  (buf.data_ptr() + 2, N_CAT, N_CAT)):   # not 4-byte aligned
        rc, _, _ = _abi(ops, cnn, x, ptr, n_labels, stride)
        assert rc == -1, (n_labels, stride)                # SSB_E_INVALID_ARG
        assert b"ssb_audio_encoder_category_batch: bad labels" in ops.lib.ssb_last_error(ops.ctx.handle)
    assert ops.ctx.launch_count == before                  # decided on the host: nothing launched
    # the Python side: bad category tensors
    for bad in (lab.cpu(), lab.double(), lab[:3], lab.t().contiguous().t(), lab[:, :20], _labels("soft", 4, 22)):
        with pytest.raises(ValueError):
            ops.audio_encoder(x, cnn, category=bad)
    with pytest.raises(ValueError):                        # category given for an ears-only network
        ops.audio_encoder(x, _random_cnn(shape, 64, 128, seed=14, n_cat=0), category=lab)
    with pytest.raises(ValueError):                        # no category for a 23-channel network
        ops.audio_encoder(x, cnn)
    assert ops.ctx.launch_count == before


@pytest.mark.parametrize("sr", [16000, 44100])
def test_patched_savi_with_distractor_matches_original(sr):
    from soundspaces_b200.encoder import patch_audio_cnn
    shape = SHAPES[sr]
    prev = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    try:
        _, _, Savi = reference_classes()
        torch.manual_seed(sr)
        model = Savi(shape, hidden=128, has_distractor_sound=True).cuda()
        obs = {"audiogoal": torch.rand((16,) + shape, device="cuda") * 3.0, "category": _labels("one_hot", 16, seed=1)}
        with torch.no_grad():
            ref = model(obs)
            patch_audio_cnn(Savi, category=True)
            launches = _ops().ctx.launch_count
            got = model(obs)
            assert _ops().ctx.launch_count == launches + 2          # the fused path ran
        assert torch.allclose(got, ref, rtol=1e-4, atol=1e-4)
        launches = _ops().ctx.launch_count
        grad = model(obs)                                          # grad enabled: the original forward
        assert grad.requires_grad and torch.allclose(grad, ref, rtol=1e-4, atol=1e-4)
        assert _ops().ctx.launch_count == launches
    finally:
        torch.backends.cudnn.allow_tf32 = prev


def test_patched_loop_does_not_synchronise():
    from soundspaces_b200.encoder import patch_audio_cnn
    shape = SHAPES[16000]
    _, _, Savi = reference_classes()
    patch_audio_cnn(Savi, category=True)
    torch.manual_seed(0)
    model = Savi(shape, hidden=128, has_distractor_sound=True).cuda()
    xs = torch.rand((50, 16) + shape, device="cuda")
    labs = _labels("one_hot", 50 * 16, seed=2).view(50, 16, N_CAT)
    outs = torch.empty((50, 16, 128), device="cuda")
    with torch.no_grad():
        model({"audiogoal": xs[0], "category": labs[0]})          # first call: context and module set-up
        launches = _ops().ctx.launch_count
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            for t in range(50):
                outs[t] = model({"audiogoal": xs[t], "category": labs[t]})
        finally:
            torch.cuda.set_sync_debug_mode(0)
        assert _ops().ctx.launch_count == launches + 100
        ref = model({"audiogoal": xs[49], "category": labs[49]})
    assert torch.equal(outs[49], ref)
