"""SAVi's visual encoder SMTCNN on the GPU (``ssb_smt_cnn_batch``): accuracy against a float64 forward of the stand-in
and against the reference's recorded outputs, bit-identity across batch sizes, positions and modality sets, NaN
containment, every refusal, and the patched module inside a reference-shaped ``get_features``."""
import copy
import os

import numpy as np
import pytest

from smt_cnn_models import SMTCNN, observations, set_params

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
nn = torch.nn

LAUNCHES = 39
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "smt_cnn_golden.npz")
SHAPES = [(128, 128), (96, 128), (100, 100), (48, 48), (256, 256)]
MODALITIES = {"rgb": {"rgb": 3}, "depth": {"depth": 1}, "rgbd": {"rgb": 3, "depth": 1}}


def _ops():
    from soundspaces_b200.renderer import WaveformOps
    return WaveformOps.get("cuda:0")


def _model(channels, seed=3, obs_transform="default"):
    m = set_params(SMTCNN(channels, obs_transform=obs_transform), seed).eval()
    return m.cuda()


def _cuda(obs, keys):
    return {k: obs[k].cuda() for k in keys}


def _fused(model, obs):
    return _ops().smt_cnn(obs.get("rgb"), obs.get("depth"), getattr(model, "rgb_encoder", None),
                          getattr(model, "depth_encoder", None), resize=model.obs_transform is not None)


def _ref64(model, obs):
    ref = copy.deepcopy(model).cpu().double()
    with torch.no_grad():
        return ref({k: v.cpu().double() for k, v in obs.items()})


def _check(got, want):
    """Every env within 1e-4 max|ref_b| of float64."""
    got = got.cpu().double()
    for b in range(want.shape[0]):
        err = (got[b] - want[b]).abs().max().item()
        scale = want[b].abs().max().item()
        assert err <= 1e-4 * scale, f"env {b}: max|d| {err:.3g} > 1e-4 * {scale:.3g}"


@pytest.mark.parametrize("hw", SHAPES)
@pytest.mark.parametrize("mod", list(MODALITIES))
def test_parity(mod, hw):
    """Randomised weights and GroupNorm affines, 4 envs, against the float64 stand-in."""
    model = _model(MODALITIES[mod], seed=11 + SHAPES.index(hw))
    obs = _cuda(observations(4, *hw, seed=21), MODALITIES[mod])
    out = _fused(model, obs)
    assert out.shape == (4, 64 * len(MODALITIES[mod]))
    _check(out, _ref64(model, obs))


def test_parity_with_reference_recording():
    g = np.load(GOLDEN)
    for name in sorted({k.split("/")[0] for k in g.files if "/" in k}):
        B, H, W, seed = (int(v) for v in g[f"{name}/config"])
        model = _model({"rgb": 3, "depth": 1}, seed=int(g["param_seed"]))
        out = _fused(model, _cuda(observations(B, H, W, seed), ("rgb", "depth")))
        _check(out, torch.from_numpy(g[f"{name}/out"]))


def test_without_transform():
    model = _model({"rgb": 3, "depth": 1}, obs_transform=None)
    obs = _cuda(observations(5, 64, 64, seed=4), ("rgb", "depth"))
    _check(_fused(model, obs), _ref64(model, obs))


def test_batch_and_modality_invariance():
    """An env's features are bit-identical at B = 1, 8, 16, 64, under a permutation, and whether its modality runs
    alone or with the other; 128 x 128 RGB with 100 x 100 depth (each input keeps its own geometry)."""
    model = _model({"rgb": 3, "depth": 1}, seed=5)
    obs = {"rgb": observations(64, 128, 128, seed=8, depth=0)["rgb"].cuda(),
           "depth": observations(64, 100, 100, seed=9, rgb=0)["depth"].cuda()}
    full = _fused(model, obs)
    _check(full, _ref64(model, obs))
    for B in (1, 8, 16):
        out = _fused(model, {k: v[:B].contiguous() for k, v in obs.items()})
        assert torch.equal(out, full[:B]), B
    perm = torch.randperm(64, generator=torch.Generator().manual_seed(1)).cuda()
    assert torch.equal(_fused(model, {k: v[perm].contiguous() for k, v in obs.items()}), full[perm])
    ops = _ops()
    rgb = ops.smt_cnn(obs["rgb"], None, model.rgb_encoder, None)
    depth = ops.smt_cnn(None, obs["depth"], None, model.depth_encoder)
    assert torch.equal(rgb, full[:, :64]) and torch.equal(depth, full[:, 64:])
    torch.cuda.synchronize()


def test_nan_containment():
    model = _model({"rgb": 3, "depth": 1}, seed=6)
    obs = _cuda(observations(8, 128, 128, seed=3), ("rgb", "depth"))
    clean = _fused(model, obs)
    bad = {k: v.clone() for k, v in obs.items()}
    bad["rgb"][3, 40, 50, 1] = float("nan")
    bad["depth"][5, 7, 9, 0] = float("nan")
    out = _fused(model, bad)
    keep = [b for b in range(8) if b not in (3, 5)]
    assert torch.equal(out[keep], clean[keep])
    # the other modality of the same env is untouched too (what the NaN itself becomes is not pinned: the kernels'
    # ReLU is fmaxf, which maps a NaN GroupNorm group to 0 as in the belief-predictor ResNets)
    assert torch.equal(out[3, 64:], clean[3, 64:]) and not torch.equal(out[3, :64], clean[3, :64])
    assert torch.equal(out[5, :64], clean[5, :64]) and not torch.equal(out[5, 64:], clean[5, 64:])


def test_refusals_launch_nothing():
    from soundspaces_b200 import _lib
    from soundspaces_b200.belief_nets import conv_table
    ops = _ops()
    model = _model({"rgb": 3, "depth": 1})
    obs = _cuda(observations(4, 128, 128, seed=2), ("rgb", "depth"))
    out = torch.zeros(2048 * 128, device="cuda")

    def table(**kw):
        t = (_lib.SmtCnnInput * 2)()
        for k, (name, scale) in enumerate((("rgb", 1), ("depth", 0))):
            net, x = getattr(model, f"{name}_encoder"), obs[name]
            t[k] = _lib.SmtCnnInput(x.data_ptr(), x.shape[3], 128, 128, scale, 128, 128, 32, 32,
                                    conv_table(net, False), net.fc.weight.data_ptr(), net.fc.bias.data_ptr(), 8192, 64)
        for key, v in kw.items():
            k, field = key.split("__")
            if field.startswith("conv"):
                i, f = field[4:].split("_", 1)
                setattr(t[int(k)].convs[int(i)], f, v)
            else:
                setattr(t[int(k)], field, v)
        return t

    def call(B=4, n=2, tab=None, o=out.data_ptr(), **kw):
        return ops.lib.ssb_smt_cnn_batch(ops.ctx.handle, B, n, table(**kw) if tab is None else tab, o, ops._stream())

    assert call() == 0
    torch.cuda.synchronize()
    before = ops.ctx.launch_count
    cases = [
        (dict(B=-1), -1), (dict(n=0), -1), (dict(n=3), -1), (dict(o=None), -1), (dict(o=out.data_ptr() + 2), -1),
        (dict(_0__d_obs=None), -1), (dict(_1__d_obs=obs["depth"].data_ptr() + 1), -1), (dict(_0__C=0), -1),
        (dict(_1__scale=2), -1), (dict(_0__scale=-1), -1), (dict(_0__d_fc_weight=None), -1),
        (dict(_1__d_fc_bias=model.depth_encoder.fc.bias.data_ptr() + 1), -1), (dict(_0__n_out=0), -1),
        (dict(_0__conv7_d_weight=None), -1), (dict(_1__conv0_d_gamma=None), -1),
        (dict(_1__conv19_d_beta=model.depth_encoder.fc.bias.data_ptr() + 2), -1),
        (dict(_0__conv3_eps=0.0), -1), (dict(_1__conv12_eps=-1e-5), -1),
        (dict(B=1025), -4), (dict(_0__H=0), -4), (dict(_1__W=1025), -4), (dict(_0__H=1025), -4),
        (dict(_0__resized_h=63), -4), (dict(_1__resized_w=65537), -4), (dict(_0__crop_y=-1), -4),
        (dict(_1__crop_x=65), -4), (dict(_0__crop_y=64, _0__resized_h=127), -4), (dict(_1__fc_in=4608), -4),
    ]
    for kw, code in cases:
        kw = {k.lstrip("_"): v for k, v in kw.items()}
        assert call(**kw) == code, kw
        assert ops.ctx.launch_count == before, kw
    assert call(tab=None, B=0) == 0 and ops.ctx.launch_count == before
    assert ops.lib.ssb_smt_cnn_batch(ops.ctx.handle, 4, 1, None, out.data_ptr(), ops._stream()) == -1
    assert call(n=1) == 0 and ops.ctx.launch_count == before + LAUNCHES
    assert call() == 0 and ops.ctx.launch_count == before + 2 * LAUNCHES
    torch.cuda.synchronize()


def make_policy_class(smt_cnn_cls):
    """The visual / action half of AudioNavSMTNet.get_features (ss_baselines/savi/ppo/policy.py:439-451)."""

    class Policy(nn.Module):
        def __init__(self):
            super().__init__()
            self.visual_encoder = smt_cnn_cls({"rgb": 3, "depth": 1})
            self.action_encoder = nn.Linear(4, 16)

        def get_features(self, observations, prev_actions):
            x = [self.visual_encoder(observations),
                 self.action_encoder(torch.nn.functional.one_hot(prev_actions.long().squeeze(-1), 4).float())]
            return torch.cat(x, dim=1)

    return Policy


def test_patched_get_features():
    from soundspaces_b200.encoder import patch_smt_cnn
    patched_cls = type("SMTCNN", (SMTCNN,), {})
    patch_smt_cnn(patched_cls)
    ref = make_policy_class(SMTCNN)()
    set_params(ref, 12)
    ref = ref.cuda().eval()
    pol = make_policy_class(patched_cls)()
    pol.load_state_dict(ref.state_dict())
    pol = pol.cuda().eval()
    obs = _cuda(observations(16, 128, 128, seed=30), ("rgb", "depth"))
    prev = torch.randint(0, 4, (16, 1), generator=torch.Generator().manual_seed(0)).cuda()
    ops = _ops()
    tf32 = torch.backends.cudnn.allow_tf32
    try:
        torch.backends.cudnn.allow_tf32 = False            # the unpatched convolutions in FP32, as the kernels run
        with torch.no_grad():
            want = ref.get_features(obs, prev)
            before = ops.ctx.launch_count
            got = pol.get_features(obs, prev)
            assert ops.ctx.launch_count == before + LAUNCHES
    finally:
        torch.backends.cudnn.allow_tf32 = tf32
    assert got.shape == want.shape == (16, 144)
    _check(got, want.double().cpu())
    _check(got[:, :128], _ref64(ref.visual_encoder, obs))
    assert torch.equal(got[:, 128:], want[:, 128:])
    # grad enabled (the PPO update) runs the original
    before = ops.ctx.launch_count
    y = pol.get_features(obs, prev)
    assert y.requires_grad and ops.ctx.launch_count == before


def test_63_pixel_short_edge_raises_in_both():
    from soundspaces_b200.encoder import patch_smt_cnn
    patched_cls = type("SMTCNN", (SMTCNN,), {})
    patch_smt_cnn(patched_cls)
    plain = _model({"rgb": 3, "depth": 1})
    patched = set_params(patched_cls({"rgb": 3, "depth": 1}), 3).cuda().eval()
    obs = _cuda(observations(2, 98, 98, seed=1), ("rgb", "depth"))
    ops = _ops()
    before = ops.ctx.launch_count
    with torch.no_grad():
        with pytest.raises(RuntimeError):
            plain(obs)
        with pytest.raises(RuntimeError):
            patched(obs)
    assert ops.ctx.launch_count == before
    with pytest.raises(RuntimeError, match="does not lie inside"):
        ops.smt_cnn(obs["rgb"], obs["depth"], plain.rgb_encoder, plain.depth_encoder)
