"""The fused AV-Nav visual encoder (``ssb_visual_encoder_batch``, ``WaveformOps.visual_encoder``, ``patch_visual_cnn``)
and GRU state encoder (``ssb_gru_step_batch``, ``WaveformOps.gru_step``, ``patch_rnn_state_encoder``) on the GPU:
per-env accuracy against float64 runs of the same modules (max|got_b - ref_b| <= 1e-4 max|ref_b|), bit-identity across
batch sizes and positions, refusals, launch counts, and the patched stand-ins of the reference classes against their
original forward."""
import copy

import pytest

from avnav_models import AudioNavBaselineNet, RNNStateEncoder, VisualCNN
from test_encoder_host import reference_classes

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
nn = torch.nn

VARIANTS = ("av_nav", "av_wan", "savi")
INPUTS = {"rgb": (3, 0), "depth": (0, 1), "rgbd": (3, 1)}


def _ops():
    from soundspaces_b200.renderer import WaveformOps
    return WaveformOps.get("cuda:0")


def _visual(variant, n_rgb, n_depth, H=128, W=128, hidden=512, seed=0):
    torch.manual_seed(seed)
    m = VisualCNN(n_rgb, n_depth, H, W, hidden, variant)
    with torch.no_grad():
        for layer in m.cnn:
            if isinstance(layer, (nn.Conv2d, nn.Linear)):
                layer.bias.uniform_(-0.1, 0.1)             # non-zero biases so that every ReLU clips something
    return m.cuda().eval()


def _obs(N, H, W, n_rgb, n_depth, seed=1):
    g = torch.Generator(device="cuda").manual_seed(seed)
    obs = {}
    if n_rgb:
        obs["rgb"] = torch.randint(0, 256, (N, H, W, n_rgb), device="cuda", generator=g).float()
    if n_depth:
        obs["depth"] = torch.rand((N, H, W, n_depth), device="cuda", generator=g)
    return obs


def _float64(m, obs, idx=None):
    """(features, out) of ``m`` in float64 on the CPU for the envs ``idx`` (all when None)."""
    ref = copy.deepcopy(m).cpu().double()
    o = {k: (v if idx is None else v[idx]).cpu().double() for k, v in obs.items()}
    x = []
    if "rgb" in o:
        x.append(o["rgb"].permute(0, 3, 1, 2) / 255.0)
    if "depth" in o:
        x.append(o["depth"].permute(0, 3, 1, 2))
    x = torch.cat(x, 1)
    with torch.no_grad():
        return ref.cnn[:6](x), ref.cnn(x)


def _check_per_env(got, ref):
    got = got.detach().cpu().double()
    assert got.shape == ref.shape
    for b in range(ref.shape[0]):
        scale = ref[b].abs().max().item()
        assert scale > 0
        err = (got[b] - ref[b]).abs().max().item()
        assert err <= 1e-4 * scale, f"env {b}: max err {err:.3g} > 1e-4 * {scale:.3g}"


def _run_visual(ops, m, obs, features=True):
    first = obs.get("rgb", obs.get("depth"))
    feats = torch.full((first.shape[0], m.cnn[6].in_features), float("nan"), device="cuda") if features else None
    out = ops.visual_encoder(obs.get("rgb"), obs.get("depth"), m.cnn, features=feats)
    return feats, out


def test_rgb_scaling_is_torch_cuda_division():
    """The kernel multiplies RGB by float32(1 / 255); torch's CUDA x / 255.0 computes exactly that."""
    x = torch.cat([torch.arange(256, device="cuda", dtype=torch.float32),
                   torch.rand(1 << 20, device="cuda") * 255, torch.randn(1 << 16, device="cuda") * 1e4])
    assert torch.equal(x / 255.0, x * torch.tensor(1.0 / 255.0, dtype=torch.float32, device="cuda"))


@pytest.mark.parametrize("inputs", sorted(INPUTS))
@pytest.mark.parametrize("variant", VARIANTS)
def test_visual_against_float64(variant, inputs):
    n_rgb, n_depth = INPUTS[inputs]
    m = _visual(variant, n_rgb, n_depth, seed=len(variant) + n_rgb + 7 * n_depth)
    obs = _obs(16, 128, 128, n_rgb, n_depth, seed=3)
    feats, out = _run_visual(_ops(), m, obs)
    f_ref, o_ref = _float64(m, obs)
    _check_per_env(feats, f_ref)
    _check_per_env(out, o_ref)


@pytest.mark.parametrize("B", [1, 16, 128, 1024])
def test_visual_batch_sizes(B):
    m = _visual("av_nav", 3, 1, seed=11)
    obs = _obs(B, 128, 128, 3, 1, seed=B)
    feats, out = _run_visual(_ops(), m, obs)
    idx = sorted({0, B // 3, B // 2, B - 1, min(15, B - 1), min(16, B - 1)})
    f_ref, o_ref = _float64(m, obs, idx)
    _check_per_env(feats[idx], f_ref)
    _check_per_env(out[idx], o_ref)


@pytest.mark.parametrize("variant,inputs,H,W", [("av_nav", "rgbd", 96, 128), ("av_wan", "depth", 128, 72),
                                                ("savi", "rgb", 36, 36), ("av_wan", "rgbd", 36, 36),
                                                ("av_nav", "depth", 37, 39)])
def test_visual_other_shapes(variant, inputs, H, W):
    """Non-square inputs and the smallest accepted input (36 x 36: conv3 is 1 x 1 at strides 4/2/2)."""
    n_rgb, n_depth = INPUTS[inputs]
    m = _visual(variant, n_rgb, n_depth, H, W, hidden=100, seed=H + W)
    obs = _obs(19, H, W, n_rgb, n_depth, seed=5)
    feats, out = _run_visual(_ops(), m, obs)
    f_ref, o_ref = _float64(m, obs)
    _check_per_env(feats, f_ref)
    _check_per_env(out, o_ref)


@pytest.mark.parametrize("variant", ["av_nav", "av_wan"])
def test_visual_bit_identical_across_batches(variant):
    ops = _ops()
    m = _visual(variant, 3, 1, seed=21)
    obs = _obs(129, 128, 128, 3, 1, seed=22)
    f_all, out_all = _run_visual(ops, m, obs)
    f_rev, out_rev = _run_visual(ops, m, {k: v.flip(0).contiguous() for k, v in obs.items()})
    assert torch.equal(out_rev.flip(0), out_all) and torch.equal(f_rev.flip(0), f_all)
    for k in (0, 15, 16, 17, 128):
        f1, o1 = _run_visual(ops, m, {n: v[k:k + 1].contiguous() for n, v in obs.items()})
        assert torch.equal(o1[0], out_all[k]) and torch.equal(f1[0], f_all[k])
    for j in (0, 1, 16, 127, 128):
        idx = torch.arange(129, device="cuda")
        idx[j], idx[7] = 7, j
        _, o = _run_visual(ops, m, {n: v[idx].contiguous() for n, v in obs.items()}, features=False)
        assert torch.equal(o[j], out_all[7])


def test_visual_launch_count_is_fixed():
    ops = _ops()
    m = _visual("av_nav", 3, 1, seed=3)
    for B in (1, 16, 1024):
        obs = _obs(B, 128, 128, 3, 1)
        before = ops.ctx.launch_count
        _run_visual(ops, m, obs)
        assert ops.ctx.launch_count - before == 2


def _vis_abi(ops, m, rgb, n_rgb, depth, n_depth, H, W, B, feats=None, out=None):
    from soundspaces_b200 import _lib
    cnn = m.cnn
    layers = (_lib.Conv2dLayer * 3)()
    for i, (conv, relu) in enumerate(zip((cnn[0], cnn[2], cnn[4]), (1, 1, 0))):
        layers[i] = _lib.Conv2dLayer(conv.weight.data_ptr(), conv.bias.data_ptr(), conv.out_channels,
                                     *conv.kernel_size, *conv.stride, relu)
    lin = cnn[6]
    feats = feats if feats is not None else torch.zeros(max(B, 1), max(lin.in_features, 1), device="cuda").data_ptr()
    out = out if out is not None else torch.zeros(max(B, 1), lin.out_features, device="cuda").data_ptr()
    return ops.lib.ssb_visual_encoder_batch(ops.ctx.handle, B, rgb, n_rgb, depth, n_depth, H, W, layers,
                                            lin.weight.data_ptr(), lin.bias.data_ptr(), lin.out_features, 1, feats,
                                            out, ops._stream())


def test_visual_refusals_launch_nothing():
    ops = _ops()
    m = _visual("av_nav", 3, 1, seed=4)
    obs = _obs(2, 128, 128, 3, 1)
    rgb, depth = obs["rgb"].data_ptr(), obs["depth"].data_ptr()
    before = ops.ctx.launch_count
    cases = [
        (dict(rgb=None, n_rgb=0, depth=None, n_depth=0), -1, b"bad arguments"),        # no input channel
        (dict(rgb=rgb, n_rgb=0, depth=None, n_depth=1), -1, b"bad arguments"),         # counts 0 / NULL: none left
        (dict(rgb=rgb + 2, n_rgb=3, depth=depth, n_depth=1), -1, b"bad arguments"),    # misaligned
        (dict(rgb=rgb, n_rgb=-1, depth=depth, n_depth=1), -1, b"bad channel counts"),
        (dict(rgb=rgb, n_rgb=3, depth=depth, n_depth=1, B=-1), -1, b"bad arguments"),
        (dict(rgb=rgb, n_rgb=3, depth=depth, n_depth=1, H=35, W=128), -4, b"layer 3 output is empty"),
        (dict(rgb=rgb, n_rgb=3, depth=depth, n_depth=1, H=1024, W=1024), -4, b"bytes of shared memory"),
    ]
    for kw, rc_want, msg in cases:
        args = dict(H=128, W=128, B=2)
        args.update(kw)
        rc = _vis_abi(ops, m, args["rgb"], args["n_rgb"], args["depth"], args["n_depth"], args["H"], args["W"],
                      args["B"])
        assert rc == rc_want, kw
        assert msg in ops.lib.ssb_last_error(ops.ctx.handle), kw
    # the 1024 x 1024 interactive_demo sensor: the byte count is in the message
    big = _visual("av_nav", 3, 1, 1024, 1024, hidden=8, seed=5)
    rc = _vis_abi(ops, big, rgb, 3, depth, 1, 1024, 1024, 1)
    assert rc == -4 and b"12405888 bytes" in ops.lib.ssb_last_error(ops.ctx.handle)
    assert _vis_abi(ops, m, rgb, 3, depth, 1, 128, 128, 0) == 0                        # B = 0
    assert ops.ctx.launch_count == before
    with pytest.raises(RuntimeError, match="shared memory"):
        ops.visual_encoder(torch.zeros(1, 1024, 1024, 3, device="cuda"), torch.zeros(1, 1024, 1024, 1, device="cuda"),
                           big.cnn)


# ------------------------------------------------------------------------------------------------ GRU
def _gru(I, Hd, seed):
    torch.manual_seed(seed)
    r = nn.GRU(I, Hd)
    with torch.no_grad():
        for name, p in r.named_parameters():
            if "bias" in name:
                p.uniform_(-0.3, 0.3)
    return r.cuda()


def _gru_inputs(B, I, Hd, seed, masks="mixed"):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(B, I, device="cuda", generator=g)
    h = torch.randn(B, Hd, device="cuda", generator=g)
    if masks == "mixed":
        m = (torch.rand(B, 1, device="cuda", generator=g) > 0.3).float()
    else:
        m = torch.full((B, 1), float(masks), device="cuda")
    return x, h, m


def _gru_float64(r, x, h, m):
    ref = copy.deepcopy(r).cpu().double()
    with torch.no_grad():
        y, hn = ref(x.cpu().double()[None], (m.cpu().double() * h.cpu().double())[None])
    return y[0], hn[0]


GRU_WIDTHS = [(1024, 512), (1026, 512), (1068, 512), (1024, 64), (1024, 1024), (33, 100), (1, 1)]


@pytest.mark.parametrize("I,Hd", GRU_WIDTHS)
def test_gru_against_float64(I, Hd):
    r = _gru(I, Hd, seed=I + Hd)
    x, h, m = _gru_inputs(37, I, Hd, seed=1)
    out, h_out = _ops().gru_step(x, h, m, r)
    y_ref, h_ref = _gru_float64(r, x, h, m)
    _check_per_env(out, y_ref)
    assert torch.equal(out, h_out) and out.data_ptr() != h_out.data_ptr()


@pytest.mark.parametrize("B", [1, 16, 128, 1024])
@pytest.mark.parametrize("masks", ["mixed", 0.0, 1.0])
def test_gru_batch_sizes_and_masks(B, masks):
    r = _gru(1024, 512, seed=3)
    x, h, m = _gru_inputs(B, 1024, 512, seed=B, masks=masks)
    out, _ = _ops().gru_step(x, h, m, r)
    y_ref, _ = _gru_float64(r, x, h, m)
    _check_per_env(out, y_ref)


def test_gru_bit_identical_across_batches():
    ops = _ops()
    r = _gru(1068, 512, seed=4)
    x, h, m = _gru_inputs(129, 1068, 512, seed=5)
    out_all, _ = ops.gru_step(x, h, m, r)
    out_rev, _ = ops.gru_step(x.flip(0).contiguous(), h.flip(0).contiguous(), m.flip(0).contiguous(), r)
    assert torch.equal(out_rev.flip(0), out_all)
    for k in (0, 15, 16, 17, 128):
        o1, _ = ops.gru_step(x[k:k + 1].contiguous(), h[k:k + 1].contiguous(), m[k:k + 1].contiguous(), r)
        assert torch.equal(o1[0], out_all[k])
    for j in (0, 1, 16, 127, 128):
        idx = torch.arange(129, device="cuda")
        idx[j], idx[7] = 7, j
        o, _ = ops.gru_step(x[idx].contiguous(), h[idx].contiguous(), m[idx].contiguous(), r)
        assert torch.equal(o[j], out_all[7])


def test_gru_nan_in_masked_state_propagates_as_reference():
    """masks * hidden is a multiply: 0 * NaN is NaN, so a done env with NaN state gets NaN, as in the reference;
    the other envs are untouched."""
    r = _gru(64, 32, seed=6)
    x, h, _ = _gru_inputs(20, 64, 32, seed=7)
    m = torch.ones(20, 1, device="cuda")
    m[3] = 0.0
    h[3, 5] = float("nan")
    out, h_out = _ops().gru_step(x, h, m, r)
    with torch.no_grad():
        y_ref, _ = r(x[None], (m * h)[None])
    assert torch.equal(torch.isnan(out), torch.isnan(y_ref[0])) and bool(torch.isnan(out[3]).all())
    keep = torch.arange(20, device="cuda") != 3
    assert not bool(torch.isnan(out[keep]).any())


def test_gru_launch_count_and_refusals():
    ops = _ops()
    r = _gru(1024, 512, seed=8)
    for B in (1, 16, 1024):
        x, h, m = _gru_inputs(B, 1024, 512, seed=B)
        before = ops.ctx.launch_count
        ops.gru_step(x, h, m, r)
        assert ops.ctx.launch_count - before == 1
    x, h, m = _gru_inputs(4, 1024, 512, seed=9)
    out = torch.empty(4, 512, device="cuda")
    params = [p.data_ptr() for p in (r.weight_ih_l0, r.weight_hh_l0, r.bias_ih_l0, r.bias_hh_l0)]
    before = ops.ctx.launch_count
    for args, what in [((4, 1024, 512, x.data_ptr(), h.data_ptr(), m.data_ptr(), *params, out.data_ptr(), h.data_ptr()),
                        "in place"),
                       ((4, 1024, 512, x.data_ptr(), h.data_ptr(), None, *params, out.data_ptr(), out.data_ptr()),
                        "NULL masks"),
                       ((4, 1024, 512, x.data_ptr() + 1, h.data_ptr(), m.data_ptr(), *params, out.data_ptr(),
                         out.data_ptr()), "misaligned"),
                       ((4, 0, 512, x.data_ptr(), h.data_ptr(), m.data_ptr(), *params, out.data_ptr(), out.data_ptr()),
                        "I = 0")]:
        assert ops.lib.ssb_gru_step_batch(ops.ctx.handle, *args, ops._stream()) == -1, what
        assert b"ssb_gru_step_batch: bad arguments" in ops.lib.ssb_last_error(ops.ctx.handle)
    assert ops.lib.ssb_gru_step_batch(ops.ctx.handle, 0, 1024, 512, x.data_ptr(), h.data_ptr(), m.data_ptr(), *params,
                                      out.data_ptr(), out.data_ptr(), ops._stream()) == 0
    assert ops.ctx.launch_count == before


# ------------------------------------------------------------------------------------------------ patched classes
@pytest.fixture
def no_tf32():
    saved = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = saved


def _patched_visual():
    from soundspaces_b200.encoder import patch_visual_cnn

    class Patched(VisualCNN):
        pass
    return patch_visual_cnn(Patched)


def _patched_rnn():
    from soundspaces_b200.rnn import patch_rnn_state_encoder

    class Patched(RNNStateEncoder):
        pass
    return patch_rnn_state_encoder(Patched)


@pytest.mark.parametrize("inputs", sorted(INPUTS))
@pytest.mark.parametrize("variant", VARIANTS)
def test_patched_visual_matches_original(no_tf32, variant, inputs):
    n_rgb, n_depth = INPUTS[inputs]
    cls = _patched_visual()
    torch.manual_seed(31)
    m = cls(n_rgb, n_depth, 128, 128, 512, variant).cuda()
    obs = _obs(16, 128, 128, n_rgb, n_depth, seed=32)
    ops = _ops()
    with torch.no_grad():
        before = ops.ctx.launch_count
        got = m(obs)
        assert ops.ctx.launch_count - before == 2             # the fused path ran
        want = cls.forward._ssb_original(m, obs)
    _check_per_env(got, want.double().cpu())


def test_patched_visual_grad_runs_original_bit_for_bit():
    cls = _patched_visual()
    torch.manual_seed(33)
    m = cls(3, 1, 128, 128, 512, "av_nav").cuda()
    obs = _obs(4, 128, 128, 3, 1)
    ops = _ops()
    before = ops.ctx.launch_count
    got = m(obs)
    assert got.requires_grad and ops.ctx.launch_count == before
    assert torch.equal(got, cls.forward._ssb_original(m, obs))


@pytest.mark.parametrize("I,Hd", [(1024, 512), (1026, 512), (1068, 512)])
def test_patched_rnn_matches_original(no_tf32, I, Hd):
    cls = _patched_rnn()
    torch.manual_seed(I)
    m = cls(I, Hd).cuda()
    x, h, masks = _gru_inputs(16, I, Hd, seed=2)
    h = h[None].contiguous()
    ops = _ops()
    with torch.no_grad():
        before = ops.ctx.launch_count
        out, h_out = m(x, h, masks)
        assert ops.ctx.launch_count - before == 1
        want, h_want = cls.single_forward._ssb_original(m, x, h, masks)
    assert out.shape == want.shape and h_out.shape == h_want.shape == (1, 16, Hd)
    assert out.dtype == want.dtype and h_out.dtype == h_want.dtype
    _check_per_env(out, want.double().cpu())
    _check_per_env(h_out[0], h_want[0].double().cpu())


def test_patched_rnn_grad_and_lstm_run_original_bit_for_bit():
    cls = _patched_rnn()
    torch.manual_seed(5)
    ops = _ops()
    m = cls(64, 32).cuda()
    x, h, masks = _gru_inputs(8, 64, 32, seed=3)
    h = h[None].contiguous()
    before = ops.ctx.launch_count
    out, h_out = m(x, h, masks)
    assert out.requires_grad and ops.ctx.launch_count == before
    want, h_want = cls.single_forward._ssb_original(m, x, h, masks)
    assert torch.equal(out, want) and torch.equal(h_out, h_want)
    lstm = cls(64, 32, rnn_type="LSTM").cuda()
    with torch.no_grad():
        hh = torch.cat([h, h])
        out, h_out = lstm(x, hh, masks)
        want, h_want = cls.single_forward._ssb_original(lstm, x, hh, masks)
    assert ops.ctx.launch_count == before and torch.equal(out, want) and torch.equal(h_out, h_want)


def test_patched_policy_net_matches_unpatched(no_tf32):
    """The rollout-time Net.forward of av_nav (audio, depth visual and state encoders) with all three patches
    against the same modules without them."""
    from soundspaces_b200.encoder import patch_audio_cnn
    from soundspaces_b200.rnn import patch_rnn_state_encoder
    from soundspaces_b200.encoder import patch_visual_cnn
    AudioCNN = reference_classes()[0]

    class PAudio(AudioCNN):
        pass

    class PVisual(VisualCNN):
        pass

    class PRnn(RNNStateEncoder):
        pass

    torch.manual_seed(7)
    audio, visual = AudioCNN((65, 26, 2), 512, audiogoal_sensor="spectrogram"), VisualCNN(0, 1, 128, 128, 512)
    plain = AudioNavBaselineNet(audio, visual).cuda()
    fused = copy.deepcopy(plain)
    fused.audio_encoder.__class__ = patch_audio_cnn(PAudio)
    fused.visual_encoder.__class__ = patch_visual_cnn(PVisual)
    fused.state_encoder.__class__ = patch_rnn_state_encoder(PRnn)
    g = torch.Generator(device="cuda").manual_seed(8)
    obs = {"spectrogram": torch.rand(16, 65, 26, 2, device="cuda", generator=g) * 3,
           "depth": torch.rand(16, 128, 128, 1, device="cuda", generator=g)}
    h = torch.randn(1, 16, 512, device="cuda", generator=g)
    masks = (torch.arange(16, device="cuda") % 4 != 0).float()[:, None]
    ops = _ops()
    with torch.no_grad():
        before = ops.ctx.launch_count
        out, h_out = fused(obs, h, masks)
        assert ops.ctx.launch_count - before == 5
        want, h_want = plain(obs, h, masks)
    _check_per_env(out, want.double().cpu())
    _check_per_env(h_out[0], h_want[0].double().cpu())
