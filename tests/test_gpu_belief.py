"""SAVi's belief update on the GPU (``ssb_belief_update_batch``, ``WaveformOps.belief_update``,
``patch_belief_predictor``): the recording of the real ``BeliefPredictor.update`` and seeded rollouts against the
float32 model, the silence test at the edges of a row, every refusal, and the patched update on a reference-shaped
stand-in with torchvision ResNets against the unpatched one, with no host synchronisation."""
import ctypes as C

import numpy as np
import pytest

import belief_oracle as bo
from test_belief_host import CONFIGS, golden_scale, load_golden, make_reference_class

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

SHAPES = [(65, 26, 2), (65, 69, 2)]       # 16 kHz, 44.1 kHz observations
EXTRA = 3                                 # state / output rows past B that must stay untouched


def _ops():
    from soundspaces_b200.renderer import WaveformOps
    return WaveformOps.get("cuda:0")


class Run:
    """Device state with EXTRA sentinel rows past num_env's first B, and outputs with EXTRA sentinel rows past B."""

    def __init__(self, B, num_env, loc, label):
        self.B, self.loc, self.label = B, loc, label
        self.last_pg = torch.full((num_env, 2), float("nan"), device="cuda")
        self.loc_valid = torch.full((num_env,), 0xAB, dtype=torch.uint8, device="cuda")
        self.last_label = torch.full((num_env, 21), float("nan"), device="cuda")
        self.label_valid = torch.full((num_env,), 0xAB, dtype=torch.uint8, device="cuda")
        for t in (self.last_pg, self.loc_valid, self.last_label, self.label_valid):
            t[:B] = 0
        self.loc_out = torch.full((B + EXTRA, 2), float("nan"), device="cuda")
        self.cat_out = torch.full((B + EXTRA, 21), float("nan"), device="cuda")

    def step(self, spec, pose, loc_pred, label_pred, dones, w, cpo):
        B = self.B
        _ops().belief_update(
            spec, dones, w, cpo, pose=pose if self.loc else None, loc_pred=loc_pred if self.loc else None,
            last_pg=self.last_pg, loc_valid=self.loc_valid, loc_out=self.loc_out[:B],
            label_pred=label_pred if self.label else None, last_label=self.last_label, label_valid=self.label_valid,
            cat_out=self.cat_out[:B])

    def check_untouched(self):
        B = self.B
        assert torch.isnan(self.last_pg[B:]).all() and (self.loc_valid[B:] == 0xAB).all()
        assert torch.isnan(self.last_label[B:]).all() and (self.label_valid[B:] == 0xAB).all()
        assert torch.isnan(self.loc_out[B:]).all() and torch.isnan(self.cat_out[B:]).all()
        if not self.loc:
            assert torch.isnan(self.loc_out).all() and (self.loc_valid[:B] == 0).all()
        if not self.label:
            assert torch.isnan(self.cat_out).all() and (self.label_valid[:B] == 0).all()


def _run_against_oracle(seq, shape, loc, label, w, cpo, num_env, seed):
    T, B = seq["silent"].shape
    run = Run(B, num_env, loc, label)
    st = bo.new_state(B)
    cuda = {k: torch.from_numpy(np.ascontiguousarray(seq[k])).cuda() for k in ("pose", "loc_pred", "label_pred")}
    worst, scale = 0.0, np.abs(seq["pose"][..., :2]).max()
    for t in range(T):
        spec = torch.from_numpy(bo.make_spectrograms(seq["silent"][t], shape, seed * 1000 + t)).cuda()
        dones = [bool(d) for d in seq["dones"][t]]
        run.step(spec, cuda["pose"][t], cuda["loc_pred"][t], cuda["label_pred"][t], dones, w, cpo)
        lo, co, _ = bo.step(st, seq["silent"][t], seq["pose"][t], seq["loc_pred"][t] if loc else None,
                            seq["label_pred"][t] if label else None, seq["dones"][t], w, cpo)
        if label:
            assert np.array_equal(run.cat_out[:B].cpu().numpy(), co), f"label belief, step {t}"
            assert np.array_equal(run.label_valid[:B].cpu().numpy().astype(bool), st["label_valid"])
            v = st["label_valid"]
            assert np.array_equal(run.last_label[:B].cpu().numpy()[v], st["last_label"][v])
        if loc:
            assert np.array_equal(run.loc_valid[:B].cpu().numpy().astype(bool), st["loc_valid"])
            v = st["loc_valid"]
            worst = max(worst, np.abs(run.loc_out[:B].cpu().numpy() - lo).max(),
                        np.abs(run.last_pg[:B].cpu().numpy()[v] - st["last_pg"][v]).max(initial=0.0))
            scale = max(scale, np.abs(lo).max(), np.abs(st["last_pg"][v]).max(initial=0.0))
    assert worst <= bo.location_bound(scale), f"location belief: {worst:.3g} > {bo.location_bound(scale):.3g}"
    run.check_untouched()


@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("name", CONFIGS)
def test_golden_sequences(name, shape):
    """The recording of the real class: label belief and state bit-identical, decisions identical, location within
    the bound of ``belief_oracle.location_bound``."""
    g = load_golden(name)
    T, B = g["silent"].shape
    run = Run(B, B + 5, bool(g["loc"]), bool(g["label"]))
    bound = bo.location_bound(golden_scale(g))
    w, cpo = float(g["w"]), bool(g["cpo"])
    pose, lp, cp = (torch.from_numpy(g[k]).cuda() for k in ("pose", "loc_pred", "label_pred"))
    for t in range(T):
        spec = torch.from_numpy(bo.make_spectrograms(g["silent"][t], shape, t)).cuda()
        run.step(spec, pose[t], lp[t], cp[t], list(g["dones"][t]), w, cpo)
        if g["label"]:
            assert np.array_equal(run.cat_out[:B].cpu().numpy(), g["cat_out"][t])
            v = g["label_valid"][t]
            assert np.array_equal(run.label_valid[:B].cpu().numpy().astype(bool), v)
            assert np.array_equal(run.last_label[:B].cpu().numpy()[v], g["last_label"][t][v])
        if g["loc"]:
            v = g["loc_valid"][t]
            assert np.array_equal(run.loc_valid[:B].cpu().numpy().astype(bool), v)
            assert np.abs(run.loc_out[:B].cpu().numpy() - g["loc_out"][t]).max() <= bound
            assert np.abs(run.last_pg[:B].cpu().numpy()[v] - g["last_pg"][t][v]).max(initial=0.0) <= bound
    run.check_untouched()


@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("B", [1, 8, 16, 129])
def test_seeded_sequences(B, shape):
    """Seeded rollouts at B = 1, 8, 16 and 129 (dones past bit 31 of the mask) with num_env > B, in four
    configurations, against the float32 model."""
    for k, (loc, label, w, cpo, cols) in enumerate([(True, True, 0.5, False, 2), (True, True, 0.5, True, 23),
                                                    (True, False, 0.3, False, 23), (False, True, 0.7, False, 2)]):
        seed = 100 * B + 10 * k + shape[1]
        seq = bo.make_sequence(seed, 20, B, loc_cols=cols, p_done=0.1)
        _run_against_oracle(seq, shape, loc, label, w, cpo, num_env=B + EXTRA + 4, seed=seed)


@pytest.mark.parametrize("shape", SHAPES)
def test_silence_test_at_row_edges(shape):
    """Rows that are all zero, or zero but for one element at the first, a middle or the last position (the scalar
    tail), at every alignment a row can start at; NaN and Inf count as sounding, -0.0 as silent."""
    n = shape[0] * shape[1] * shape[2]
    cases = [None, 0, n // 2 + 1, n - 1, n - 2, n - 4, 3]
    B = 4 * len(cases)
    for offset in range(4):                               # the batch starts 0..3 floats past a 16-byte boundary
        buf = torch.zeros(B * n + 4, device="cuda")
        spec = buf[offset:offset + B * n].view((B,) + shape)
        flat = spec.view(B, -1)
        for j, pos in enumerate(cases):
            for r in range(4):
                if pos is not None:
                    flat[4 * j + r, pos] = (1e-30, float("nan"), float("inf"), 3.0)[r]
                elif r == 1:
                    flat[4 * j + r, 5] = -0.0
        label_pred = torch.rand((B, 21), device="cuda")
        run = Run(B, B, False, True)
        run.step(spec, None, None, label_pred, None, 0.5, False)
        got = run.cat_out[:B].cpu()
        for j, pos in enumerate(cases):
            for r in range(4):
                i = 4 * j + r
                want = torch.full((21,), np.float32(1 / 21)) if pos is None else label_pred[i].cpu()
                assert torch.equal(got[i], want), (offset, pos, r)
        assert (run.label_valid[:B].cpu().numpy() == [0 if pos is None else 1 for pos in cases for _ in range(4)]).all()


def _abi(ops, B=4, num_env=8, H=65, W=26, spec=None, pose=None, pose_stride=4, loc_pred=None, loc_stride=2,
         label_pred=None, label_stride=21, dones=None, w=0.5, cpo=0, last_pg=None, loc_valid=None, last_label=None,
         label_valid=None, loc_out=None, cat_out=None):
    return ops.lib.ssb_belief_update_batch(ops.ctx.handle, B, num_env, spec, H, W, pose, pose_stride, loc_pred,
                                           loc_stride, label_pred, label_stride, dones, w, cpo, last_pg, loc_valid,
                                           last_label, label_valid, loc_out, cat_out, ops._stream())


def test_refusals_launch_nothing():
    ops = _ops()
    n = 2048
    buf = torch.zeros(n * 65 * 26 * 2 + 8, device="cuda")
    f = torch.zeros(n * 32, device="cuda")
    u8 = torch.zeros(n, dtype=torch.uint8, device="cuda")
    p = buf.data_ptr()
    good = dict(spec=p, pose=f.data_ptr(), loc_pred=f.data_ptr(), label_pred=f.data_ptr(), last_pg=f.data_ptr(),
                loc_valid=u8.data_ptr(), last_label=f.data_ptr(), label_valid=u8.data_ptr(), loc_out=f.data_ptr(),
                cat_out=f.data_ptr())
    assert _abi(ops, **good) == 0
    torch.cuda.synchronize()
    bad = [dict(B=9), dict(B=-1), dict(num_env=0), dict(spec=None), dict(spec=p + 2), dict(H=0), dict(W=0), dict(cpo=2),
           dict(loc_stride=1), dict(pose_stride=2), dict(pose=None), dict(pose=f.data_ptr() + 1), dict(loc_pred=p + 1),
           dict(last_pg=None), dict(last_pg=f.data_ptr() + 2), dict(loc_valid=None), dict(loc_out=None),
           dict(loc_out=f.data_ptr() + 3), dict(label_stride=20), dict(label_pred=p + 2), dict(last_label=None),
           dict(label_valid=None), dict(cat_out=None), dict(cat_out=f.data_ptr() + 1)]
    for kw in bad:
        before = ops.ctx.launch_count
        assert _abi(ops, **{**good, **kw}) == -1, kw                  # SSB_E_INVALID_ARG
        assert ops.ctx.launch_count == before, kw
    before = ops.ctx.launch_count
    assert _abi(ops, **{**good, "B": 1025, "num_env": n}) == -4      # SSB_E_SHAPE: the dones bitmask holds 1024
    assert b"1024" in ops.lib.ssb_last_error(ops.ctx.handle)
    assert _abi(ops, **{**good, "loc_pred": None, "label_pred": None}) == 0      # nothing asked: nothing launched
    assert _abi(ops, **{**good, "B": 0}) == 0
    assert ops.ctx.launch_count == before
    # without the belief they belong to, the other belief's pointers are not needed
    assert _abi(ops, **{**good, "loc_pred": None, "pose": None, "last_pg": None, "loc_out": None, "pose_stride": 0}) == 0
    assert _abi(ops, **{**good, "label_pred": None, "last_label": None, "cat_out": None, "label_stride": 0}) == 0
    dones = (C.c_uint8 * 1024)(*([1] * 1024))
    assert _abi(ops, **{**good, "B": 1024, "num_env": n, "dones": dones}) == 0
    assert ops.ctx.launch_count == before + 3
    torch.cuda.synchronize()


def _resnet(n_out):
    import torchvision
    m = torchvision.models.resnet18(weights=None)
    m.conv1 = torch.nn.Conv2d(2, 64, kernel_size=7, stride=2, padding=3, bias=False)
    m.fc = torch.nn.Linear(512, n_out)
    return m


@pytest.mark.parametrize("cpo", [False, True])
def test_patched_update_matches_reference_shaped_class(cpo):
    """A 50-step rollout written in place into (T + 1, B, .) rollout slots, as ppo_trainer.py:332-336 does: the
    patched class against the unpatched one with the same torchvision ResNets (23-column location head, 21-column
    classifier).  The patched update launches one kernel after the networks and never synchronises with the host."""
    pytest.importorskip("torchvision")
    from soundspaces_b200.belief import patch_belief_predictor
    T, B, shape = 50, 8, SHAPES[0]
    torch.manual_seed(7)
    predictor, classifier = _resnet(23).cuda().eval(), _resnet(21).cuda().eval()
    Ref, Patched = make_reference_class(), make_reference_class()
    patch_belief_predictor(Patched)
    ref = Ref(B, w=0.5, current_pred_only=cpo, predictor=predictor, classifier=classifier)
    pat = Patched(B, w=0.5, current_pred_only=cpo, predictor=predictor, classifier=classifier)
    seq = bo.make_sequence(21 + cpo, T, B, p_done=0.08)
    dims = {"spectrogram": shape, "pose": (4,), "location_belief": (2,), "category_belief": (21,)}
    storage = {}
    for side in ("ref", "pat"):
        storage[side] = {k: torch.zeros((T + 1, B) + d, device="cuda") for k, d in dims.items()}
        s = storage[side]
        for t in range(T):
            s["spectrogram"][t + 1] = torch.from_numpy(bo.make_spectrograms(seq["silent"][t], shape, t)).cuda() * 4.0
            s["pose"][t + 1] = torch.from_numpy(seq["pose"][t]).cuda()
    prev = (torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark)
    torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = True, False
    ops = _ops()
    try:
        for t in range(T):
            dones = [bool(d) for d in seq["dones"][t]]
            ref.update({k: v[t + 1] for k, v in storage["ref"].items()}, dones)
            obs = {k: v[t + 1] for k, v in storage["pat"].items()}
            before = ops.ctx.launch_count
            torch.cuda.synchronize()
            torch.cuda.set_sync_debug_mode("error")
            try:
                pat.update(obs, dones)
            finally:
                torch.cuda.set_sync_debug_mode(0)
            assert ops.ctx.launch_count == before + 1
        # the sync debug mode does not see every synchronising call: queue ~0.1 s of device work ahead of one more
        # update and check that the update returned while that work was still running
        obs = {k: v[T] for k, v in storage["pat"].items()}
        loc_before, cat_before = obs["location_belief"].clone(), obs["category_belief"].clone()
        torch.cuda.synchronize()
        torch.cuda._sleep(200_000_000)
        busy = torch.cuda.Event()
        busy.record()
        pat.update(obs, [False] * B)
        assert not busy.query()
        torch.cuda.synchronize()
        obs["location_belief"].copy_(loc_before)
        obs["category_belief"].copy_(cat_before)
    finally:
        torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = prev
    r, p = storage["ref"], storage["pat"]
    assert torch.equal(p["category_belief"], r["category_belief"])
    assert torch.equal(p["location_belief"] == 10, r["location_belief"] == 10)
    scale = max(r["location_belief"].abs().max().item(), r["pose"][..., :2].abs().max().item())
    err = (p["location_belief"] - r["location_belief"]).abs().max().item()
    assert err <= bo.location_bound(scale), err
    assert (r["category_belief"][1:] == np.float32(1 / 21)).all(-1).any()      # silent first steps were exercised
    assert all(x is None for x in pat.last_pointgoal) and any(x is not None for x in ref.last_pointgoal)
