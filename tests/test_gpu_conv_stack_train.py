"""The CNN encoders' conv stack for PPO's update (``ssb_conv_stack_train_*``, ``ConvStackFunction``, the
``training=True`` patches) on the GPU: features and out bit-identical to the inference entries at any B and env
order, gradients against float64, determinism, launch counts, no host synchronisation, frozen encoders, refusals,
fallbacks and one PPO-style optimiser step against the unpatched modules."""
import copy
import ctypes as C

import pytest

from avnav_models import VisualCNN, visual_obs
from map_cnn_models import MapCNN, map_obs
from test_encoder_host import reference_classes

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
nn = torch.nn

AUDIO = {16000: (65, 26, 2), 44100: (65, 69, 2)}


def _ops():
    from soundspaces_b200.renderer import WaveformOps
    return WaveformOps.get("cuda:0")


def _dead_units(module, seed):
    """Biases that leave some ReLU units dead, so the masks matter."""
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for m in module.cnn:
            if isinstance(m, (nn.Conv2d, nn.Linear)):
                m.bias.copy_(torch.rand(m.bias.shape, generator=g) * 0.4 - 0.25)
    return module


def _case(name, B, seed=0):
    """(module, observations) of a named configuration on the GPU."""
    torch.manual_seed(seed)
    if name.startswith("audio"):
        sr = 44100 if name.endswith("44k") else 16000
        _, _, Savi = reference_classes()
        cat = "cat" in name
        m = Savi(AUDIO[sr], hidden=128, has_distractor_sound=cat)
        obs = {"audiogoal": torch.rand((B,) + AUDIO[sr]) * 3.0}
        if cat:
            obs["category"] = nn.functional.one_hot(torch.randint(0, 21, (B,)), 21).float()
    elif name.startswith("visual"):
        n_rgb, n_depth = {"visual_rgbd": (3, 1), "visual_depth": (0, 1), "visual_rgb": (3, 0)}[name]
        m = VisualCNN(n_rgb, n_depth, 64, 64, 128)
        obs = visual_obs(B, 64, 64, n_rgb, n_depth, seed)
    else:
        kind, H, C_ = {"map_gm": ("gm", 200, 2), "map_am": ("am", 20, 1)}[name]
        m = MapCNN(H, H, C_, 128, map_type=kind)
        obs = {kind: map_obs(B, H, H, C_, seed, kind)}
    _dead_units(m, seed)
    return m.cuda(), {k: v.cuda() for k, v in obs.items()}


CASES = ["audio16k", "audio44k", "audio16k_cat", "visual_rgbd", "visual_depth", "visual_rgb", "map_gm", "map_am"]


def _train(m, obs):
    from soundspaces_b200.encoder import _train_inputs, _params
    kind, x, depth, labels = _train_inputs(m, obs)
    cnn = m.cnn
    strides = tuple(tuple(c.stride) for c in (cnn[0], cnn[2], cnn[4]))
    return kind, x, depth, labels, [p.detach() for p in _params(cnn)], strides


def _inference(m, obs, features):
    ops = _ops()
    with torch.no_grad():
        if "rgb" in obs or "depth" in obs:
            return ops.visual_encoder(obs.get("rgb"), obs.get("depth"), m.cnn, features=features)
        if hasattr(m, "_map_type"):
            return ops.map_encoder(obs[m._map_type], m.cnn, features=features)
        return ops.audio_encoder(obs["audiogoal"], m.cnn, features=features, category=obs.get("category"))


@pytest.mark.parametrize("name", CASES)
@pytest.mark.parametrize("B", [1, 16, 1500])
def test_forward_bit_identical_to_inference(name, B):
    if B == 1500 and name == "map_gm":
        B = 750
    m, obs = _case(name, B)
    kind, x, depth, labels, params, strides = _train(m, obs)
    out, feat, _ = _ops().conv_stack_train_forward(kind, x, depth, labels, params, strides)
    ref_feat = torch.empty_like(feat)
    ref = _inference(m, obs, ref_feat)
    assert torch.equal(feat, ref_feat) and torch.equal(out, ref)
    if B > 1:                                        # a permuted batch gives each env the same bits
        perm = torch.randperm(B, device="cuda")
        pobs = {k: v[perm].contiguous() for k, v in obs.items()}
        kind, x, depth, labels, params, strides = _train(m, pobs)
        pout, pfeat, _ = _ops().conv_stack_train_forward(kind, x, depth, labels, params, strides)
        assert torch.equal(pfeat, feat[perm]) and torch.equal(pout, out[perm])


def _grads_fused(m, obs, dout):
    kind, x, depth, labels, params, strides = _train(m, obs)
    ops = _ops()
    out, feat, saved = ops.conv_stack_train_forward(kind, x, depth, labels, params, strides)
    return out, ops.conv_stack_train_backward(kind, x, depth, labels, params, strides, feat, out, saved, dout)


def _grads_float64(m, obs, dout):
    ref = copy.deepcopy(m).cpu().double()
    out = ref({k: v.cpu().double() for k, v in obs.items()})
    out.backward(dout.cpu().double())
    cnn = ref.cnn
    return out, [p.grad for c in (cnn[0], cnn[2], cnn[4], cnn[6]) for p in (c.weight, c.bias)]


@pytest.mark.parametrize("name", CASES)
def test_gradients_against_float64(name):
    B = 24
    m, obs = _case(name, B, seed=3)
    dout = torch.randn((B, 128), device="cuda")
    out, got = _grads_fused(m, obs, dout)
    ref_out, ref = _grads_float64(m, obs, dout)
    assert (out.cpu().double() - ref_out).abs().max() <= 1e-5 * max(ref_out.abs().max(), 1.0)
    for i, (g, r) in enumerate(zip(got, ref)):
        err = (g.cpu().double() - r).abs().max().item()
        assert err <= 1e-5 * max(r.abs().max().item(), 1e-30), (name, i, err, r.abs().max().item())


def test_gradients_at_avnav_update_shape_deterministic():
    """AV-Nav's update minibatch (T 150 x N 10 = 1500 rows) on the 128 x 128 RGB-D encoder: two runs give the same
    bits, and the gradients match float64 on the CPU."""
    torch.manual_seed(5)
    m = _dead_units(VisualCNN(3, 1, 128, 128, 512), 5).cuda()
    obs = {k: v.cuda() for k, v in visual_obs(1500, 128, 128, 3, 1, 5).items()}
    dout = torch.randn((1500, 512), device="cuda")
    _, a = _grads_fused(m, obs, dout)
    _, b = _grads_fused(m, obs, dout)
    assert all(torch.equal(x, y) for x, y in zip(a, b))
    _, ref = _grads_float64(m, obs, dout)
    for g, r in zip(a, ref):
        assert (g.cpu().double() - r).abs().max() <= 1e-5 * r.abs().max()


@pytest.mark.parametrize("name,fwd,bwd", [("audio16k", 4, 11), ("audio16k_cat", 5, 13), ("visual_rgbd", 4, 11),
                                          ("map_am", 4, 11)])
def test_launch_counts(name, fwd, bwd):
    m, obs = _case(name, 8)
    kind, x, depth, labels, params, strides = _train(m, obs)
    ops = _ops()
    n0 = ops.ctx.launch_count
    out, feat, saved = ops.conv_stack_train_forward(kind, x, depth, labels, params, strides)
    assert ops.ctx.launch_count == n0 + fwd
    n0 = ops.ctx.launch_count
    dout = torch.randn_like(out)
    ops.conv_stack_train_backward(kind, x, depth, labels, params, strides, feat, out, saved, dout)
    assert ops.ctx.launch_count == n0 + bwd
    n0 = ops.ctx.launch_count                       # only the Linear: mask + one GEMM
    ops.conv_stack_train_backward(kind, x, depth, labels, params, strides, feat, out, saved, dout,
                                  need=(False,) * 6 + (True, True))
    assert ops.ctx.launch_count == n0 + 2


def _patch(m, training=True):
    from soundspaces_b200.encoder import patch_audio_cnn, patch_map_cnn, patch_visual_cnn
    cls = type(m)
    if hasattr(m, "_map_type"):
        patch_map_cnn(cls, training=training)
    elif hasattr(m, "_n_input_rgb"):
        patch_visual_cnn(cls, training=training)
    else:
        patch_audio_cnn(cls, category=True, training=training)
    return cls


@pytest.mark.parametrize("name", ["audio16k_cat", "visual_rgbd", "map_gm"])
def test_patched_training_path_no_sync_and_matches_original(name):
    m, obs = _case(name, 32, seed=7)
    orig = copy.deepcopy(m)
    cls = _patch(m)
    try:
        ops = _ops()
        out = m(obs)                                 # warm-up: context, workspaces
        out.sum().backward()
        m.zero_grad()
        torch.cuda.synchronize()
        n0 = ops.ctx.launch_count
        torch.cuda.set_sync_debug_mode("error")
        try:
            out = m(obs)
            (out * out).sum().backward()
        finally:
            torch.cuda.set_sync_debug_mode(0)
        assert ops.ctx.launch_count > n0             # the library ran
        with torch.no_grad():
            n0 = ops.ctx.launch_count
            m(obs)
            assert ops.ctx.launch_count == n0 + 2    # no-grad calls keep the inference entries
        ref64 = copy.deepcopy(orig).cpu().double()          # float64: cuDNN's FP32 algorithms are less accurate
        ref = cls.forward._ssb_original(ref64, {k: v.cpu().double() for k, v in obs.items()})
        (ref * ref).sum().backward()
        assert (out.cpu().double() - ref).abs().max() <= 1e-5 * ref.abs().max()
        for p, q in zip(m.parameters(), ref64.parameters()):
            # loose: the upstream gradient 2 out is itself FP32, and on binary maps a few ReLU inputs sit at zero
            # (test_gradients_against_float64 holds each gradient to 1e-5 with a fixed upstream gradient)
            assert (p.grad.cpu().double() - q.grad).abs().max() <= 1e-3 * q.grad.abs().max()
    finally:
        cls.forward = cls.forward._ssb_original


def test_frozen_encoder_saves_nothing():
    m, obs = _case("visual_rgbd", 16)
    cls = _patch(m)
    try:
        for p in m.parameters():
            p.requires_grad_(False)
        packed = []
        with torch.autograd.graph.saved_tensors_hooks(lambda t: packed.append(t) or t, lambda t: t):
            n0 = _ops().ctx.launch_count
            out = m(obs)
        assert _ops().ctx.launch_count == n0 + 4     # the training entry ran
        assert packed == [] and out.grad_fn is None
    finally:
        cls.forward = cls.forward._ssb_original


def test_fallback_reasons():
    from soundspaces_b200.encoder import conv_stack_train_error
    m, obs = _case("visual_rgbd", 4)
    assert conv_stack_train_error(m, obs) == ""
    with torch.autocast("cuda"):
        assert "autocast" in conv_stack_train_error(m, obs)
    assert "CUDA" in conv_stack_train_error(m, {k: v.cpu() for k, v in obs.items()})
    assert "float32" in conv_stack_train_error(m, {**obs, "rgb": obs["rgb"].double()})
    assert "contiguous" in conv_stack_train_error(m, {**obs, "rgb": obs["rgb"].transpose(1, 2)})
    assert "requires grad" in conv_stack_train_error(m, {**obs, "depth": obs["depth"].clone().requires_grad_()})
    m.cnn[0].padding = (1, 1)
    assert "unpadded" in conv_stack_train_error(m, obs)
    sem = VisualCNN(3, 1, 64, 64, 128, variant="savi", n_semantic=6).cuda()
    assert "semantic" in conv_stack_train_error(sem, obs)
    blind = VisualCNN(0, 0, 64, 64, 128)
    assert "blind" in conv_stack_train_error(blind, obs)
    a, aobs = _case("audio16k_cat", 4)
    assert "category" in conv_stack_train_error(a, {"audiogoal": aobs["audiogoal"]})
    assert "requires grad" in conv_stack_train_error(a, {**aobs, "category": aobs["category"].requires_grad_()})
    big, _ = _case("visual_rgb", 1)
    bobs = {"rgb": torch.zeros((65536, 64, 64, 3), device="cuda")}
    assert "refuses" in conv_stack_train_error(big, bobs)


def test_refusals_launch_nothing():
    from soundspaces_b200 import _lib
    m, obs = _case("map_am", 4)
    kind, x, depth, labels, params, strides = _train(m, obs)
    ops = _ops()
    B, inp, layers, F, hidden = ops._conv_stack_train_args(kind, x, depth, labels, params, strides)
    feat = torch.empty((B, F), device="cuda")
    out = torch.empty((B, hidden), device="cuda")
    ws = torch.empty(int(ops.lib.ssb_conv_stack_train_workspace_bytes(B, C.byref(inp), layers, F, hidden, 0)),
                     dtype=torch.uint8, device="cuda")
    lw = params[6].data_ptr()

    def fwd(inp=inp, layers=layers, F=F, feat=feat.data_ptr(), out=out.data_ptr(), ws=ws.data_ptr(), B=B):
        return ops.lib.ssb_conv_stack_train_forward_batch(ops.ctx.handle, B, C.byref(inp), layers, lw, None, F,
                                                          hidden, 1, feat, out, ws, None)
    n0 = ops.ctx.launch_count
    assert fwd() == 0 and ops.ctx.launch_count == n0 + 4
    n0 = ops.ctx.launch_count
    bad_inp = _lib.ConvStackInput.from_buffer_copy(inp)
    bad_inp.kind = 7
    assert fwd(inp=bad_inp) == -1                                  # SSB_E_INVALID_ARG
    assert fwd(F=F + 1) == -4 and "in_features" in ops.lib.ssb_last_error(ops.ctx.handle).decode()
    assert fwd(feat=None) == -1
    assert fwd(out=out.data_ptr() + 2) == -1                        # misaligned
    assert fwd(out=feat.data_ptr()) == -1                           # overlapping
    assert fwd(ws=x.data_ptr()) == -1                               # workspace over the input
    assert fwd(B=65536) == -1
    big = (_lib.Conv2dLayer * 3)(*layers)
    big[0].kh = big[0].kw = 30
    assert fwd(layers=big) == -4 and "empty" in ops.lib.ssb_last_error(ops.ctx.handle).decode()
    assert ops.ctx.launch_count == n0


def test_ppo_step_matches_unpatched():
    """One PPO update (clipped surrogate, value loss, entropy, backward, clip_grad_norm_, Adam) of an AV-Nav-shaped
    net on a minibatch of the patched rollout storage, with both encoders on the training path and the GRU on
    ``sequence=True``, against the unpatched modules: gradients and parameters agree within 1e-4 of each tensor's
    largest value, and the library makes exactly the launches of the three fused pieces."""
    import numpy as np
    import rollout_models as rm
    from soundspaces_b200 import rollout as ro
    from soundspaces_b200.encoder import patch_audio_cnn, patch_visual_cnn
    from test_gpu_gru_seq import _Net, _patched, _ppo_update, _whole
    S, N, hidden = 150, 10, 512
    storage_cls = ro.patch_rollout_storage(type("PatchedStorage", (rm.CommonRolloutStorage,), {}))
    sp = rm.spaces({"spectrogram": (65, 26, 2), "depth": (64, 64, 1)})
    st = storage_cls(S, N, sp, rm.ActionSpace(), hidden, 1)
    st.to("cuda")
    g = np.random.default_rng(31)
    dev = torch.device("cuda")
    for _ in range(S):
        obs = {"spectrogram": torch.from_numpy(g.random((N, 65, 26, 2), dtype=np.float32) * 3).to(dev),
               "depth": torch.from_numpy(g.random((N, 64, 64, 1), dtype=np.float32)).to(dev)}
        st.insert(obs, torch.from_numpy(g.standard_normal((1, N, hidden), dtype=np.float32)).to(dev),
                  torch.from_numpy(g.integers(0, 4, (N, 1))).to(dev),
                  -torch.from_numpy(g.random((N, 1), dtype=np.float32)).to(dev) - 1.0,
                  torch.from_numpy(g.standard_normal((N, 1), dtype=np.float32)).to(dev),
                  torch.from_numpy(g.standard_normal((N, 1), dtype=np.float32)).to(dev),
                  torch.from_numpy((g.random((N, 1)) >= 0.02).astype(np.float32)).to(dev))
    st.compute_returns(torch.zeros(N, 1, device=dev), True, 0.99, 0.95)
    adv = st.returns[:-1] - st.value_preds[:-1]
    batch = next(iter(st.recurrent_generator(adv.contiguous(), 1)))
    prev = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    try:
        torch.manual_seed(5)
        plain = _Net(hidden).cuda()
        fused = copy.deepcopy(plain)
        fused.state_encoder.__class__ = _patched()
        for m, patch in ((fused.audio_encoder, patch_audio_cnn), (fused.visual_encoder, patch_visual_cnn)):
            m.__class__ = patch(type("Patched" + type(m).__name__, (type(m),), {}), training=True)
        before = _ops().ctx.launch_count
        g_fused, p_fused = _ppo_update(fused, batch)
        assert _ops().ctx.launch_count - before == 2 * (4 + 11) + 2 + 4
        g_plain, p_plain = _ppo_update(plain, batch)
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = prev
    for (name, _), a, b in zip(plain.named_parameters(), g_fused, g_plain):
        _whole(a, b, "grad " + name)
    for (name, _), a, b in zip(plain.named_parameters(), p_fused, p_plain):
        _whole(a, b, "param " + name)
