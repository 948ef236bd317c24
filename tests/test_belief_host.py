"""Host side of SAVi's belief update: the float32 model in ``belief_oracle`` against the recording of the real
``BeliefPredictor.update`` (tests/golden/belief_golden.npz), the dispatch of ``patch_belief_predictor`` on a stand-in
shaped like the reference class, and the argument handling of ``WaveformOps.belief_update``.  No GPU: the device call
is replaced by a recorder."""
import ctypes as C
import os
from types import SimpleNamespace

import numpy as np
import pytest

torch = pytest.importorskip("torch")
nn = torch.nn

import belief_oracle as bo  # noqa: E402
from soundspaces_b200 import belief  # noqa: E402

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "belief_golden.npz")
CONFIGS = ("both", "current_pred_only", "location_only", "label_only")


def load_golden(name):
    with np.load(GOLDEN) as z:
        return {k.split("/", 1)[1]: z[k] for k in z.files if k.startswith(name + "/")}


def golden_scale(g):
    return max(np.abs(g["pose"][..., :2]).max(), np.abs(g["loc_out"]).max(), np.abs(g["last_pg"]).max())


# ---------------------------------------------------------------------------
# a stand-in with the reference class's attributes and update (belief_predictor.py:55-202)
# ---------------------------------------------------------------------------
class Head(nn.Module):
    """Spectrogram (B, 2, H, W) -> (B, n): mean over H, W, then Linear.  Cheap stand-in for the ResNets."""

    def __init__(self, n):
        super().__init__()
        self.fc = nn.Linear(2, n)

    def forward(self, x):
        return self.fc(x.float().mean(dim=(2, 3)) * 50.0)


class Fixed(nn.Module):
    """A network whose output is set from outside (``.out``): seeded predictions in place of the ResNets."""

    def forward(self, x):
        return self.out


def make_reference_class():
    """A fresh class (patch_belief_predictor patches in place) shaped like ``BeliefPredictor``: the same attributes,
    ``cnn_forward``, and an ``update`` that does what the reference's does, per env on the host."""

    class BeliefPredictor(nn.Module):
        def __init__(self, num_env, loc=True, label=True, w=0.5, current_pred_only=False, predictor=None,
                     classifier=None):
            super().__init__()
            self.config = SimpleNamespace(weighting_factor=w, current_pred_only=current_pred_only)
            self.predict_location, self.predict_label = loc, label
            self.predictor = predictor if predictor is not None else Head(2)
            self.classifier = classifier if classifier is not None else Head(21)
            self.last_pointgoal = [None] * num_env
            self.last_label = [None] * num_env

        def cnn_forward(self, observations):
            return self.predictor(observations["spectrogram"].permute(0, 3, 1, 2))

        def update(self, observations, dones):
            spec = observations["spectrogram"]
            B = spec.size(0)
            w = self.config.weighting_factor
            if self.predict_location:
                with torch.no_grad():
                    pg = self.cnn_forward(observations).cpu().numpy()
                for i in range(B):
                    pose = observations["pose"][i].cpu().numpy()
                    if dones is not None and dones[i]:
                        self.last_pointgoal[i] = None
                    if spec[i].sum().item() != 0:
                        base = np.array([-pg[i][1], pg[i][0]])
                        if self.last_pointgoal[i] is None or self.config.current_pred_only:
                            avg = base
                        else:
                            avg = (1 - w) * base + w * bo.odom_to_base(self.last_pointgoal[i], pose)
                        self.last_pointgoal[i] = bo.base_to_odom(avg, pose)
                    else:
                        avg = (np.array([10, 10]) if self.last_pointgoal[i] is None
                               else bo.odom_to_base(self.last_pointgoal[i], pose))
                    observations["location_belief"][i].copy_(torch.from_numpy(avg))
            if self.predict_label:
                with torch.no_grad():
                    labels = self.classifier(spec.permute(0, 3, 1, 2))[:, :21].cpu().numpy()
                for i in range(B):
                    if dones is not None and dones[i]:
                        self.last_label[i] = None
                    if spec[i].sum().item() != 0:
                        if self.last_label[i] is None or self.config.current_pred_only:
                            avg = labels[i]
                        else:
                            avg = (1 - w) * labels[i] + w * self.last_label[i]
                        self.last_label[i] = avg
                    else:
                        avg = np.ones(21) / 21 if self.last_label[i] is None else self.last_label[i]
                    observations["category_belief"][i].copy_(torch.from_numpy(avg))

    return BeliefPredictor


class FakeCuda(torch.Tensor):
    """A CPU tensor that reports ``is_cuda``: lets the CPU suite reach the device branch of the dispatch."""

    @property
    def is_cuda(self):
        return True


@pytest.fixture
def device_calls(monkeypatch):
    """Replace the device path with a recorder."""
    from soundspaces_b200.renderer import WaveformOps
    calls = []

    class Recorder:
        def belief_update(self, spec, dones, w, current_pred_only, **kw):
            calls.append(dict(spec=spec, dones=dones, w=w, current_pred_only=current_pred_only, **kw))

    monkeypatch.setattr(WaveformOps, "get", classmethod(lambda cls, device="cuda:0": Recorder()))
    return calls


def make_obs(B, seed=0, silent=(), fake_cuda=False):
    g = torch.Generator().manual_seed(seed)
    spec = torch.rand((B, 65, 26, 2), generator=g)
    spec[list(silent)] = 0
    obs = {"spectrogram": spec, "pose": torch.randn((B, 4), generator=g), "location_belief": torch.zeros(B, 2),
           "category_belief": torch.zeros(B, 21)}
    if fake_cuda:
        obs = {k: v.as_subclass(FakeCuda) for k, v in obs.items()}
    return obs


# ---------------------------------------------------------------------------
# the model against the recording of the real class
# ---------------------------------------------------------------------------
@pytest.mark.parametrize("name", CONFIGS)
def test_oracle_matches_reference_recording(name):
    """Label belief, label state and every branch decision exactly; location belief and state within
    ``belief_oracle.location_bound`` (the two sides share numpy here, so in practice they are equal too)."""
    g = load_golden(name)
    T, B = g["silent"].shape
    assert T == 60 and B == 8
    assert g["silent"][0].all() and g["dones"].any() and (g["silent"][1:] & g["dones"][:-1]).any()
    bound = bo.location_bound(golden_scale(g))
    st = bo.new_state(B)
    for t in range(T):
        valid_before = (st["loc_valid"] | st["label_valid"]).copy()
        lo, co, dec = bo.step(st, g["silent"][t], g["pose"][t], g["loc_pred"][t] if g["loc"] else None,
                              g["label_pred"][t] if g["label"] else None, g["dones"][t], float(g["w"]), bool(g["cpo"]))
        assert np.array_equal(st["loc_valid"], g["loc_valid"][t]) and np.array_equal(st["label_valid"], g["label_valid"][t])
        # decisions: silent is the reference's sum() == 0; the state exists after a sounding step only
        assert np.array_equal(dec[:, 0], g["silent"][t]) and np.array_equal(dec[:, 1], g["dones"][t])
        ref_valid = g["loc_valid"][t] if g["loc"] else g["label_valid"][t]
        assert np.array_equal(ref_valid, ~g["silent"][t] | (valid_before & ~g["dones"][t]))
        assert np.array_equal(dec[:, 2], ~g["silent"][t] & (g["dones"][t] | ~valid_before))
        assert np.array_equal(co, g["cat_out"][t])
        assert np.array_equal(st["last_label"][st["label_valid"]], g["last_label"][t][g["label_valid"][t]])
        assert np.abs(lo - g["loc_out"][t]).max() <= bound
        v = st["loc_valid"]
        assert np.abs(st["last_pg"][v] - g["last_pg"][t][v]).max(initial=0.0) <= bound
    if g["loc"]:
        assert (g["loc_out"] == 10).all(axis=2).any()                      # silent without a state: (10, 10)
    if g["label"]:
        assert (g["cat_out"] == np.float32(1 / 21)).all(axis=2).any()     # silent without a state: 1/21


def test_stand_in_matches_reference_recording():
    """The stand-in's host ``update`` (what the GPU test compares the patched class against) reproduces the
    recording of the real class."""
    Ref = make_reference_class()
    for name in CONFIGS:
        g = load_golden(name)
        T, B = g["silent"].shape
        model = Ref(B, loc=bool(g["loc"]), label=bool(g["label"]), w=float(g["w"]), current_pred_only=bool(g["cpo"]),
                    predictor=Fixed(), classifier=Fixed())
        for t in range(T):
            model.predictor.out = torch.from_numpy(g["loc_pred"][t].copy())
            model.classifier.out = torch.from_numpy(g["label_pred"][t].copy())
            obs = {"spectrogram": torch.from_numpy(bo.make_spectrograms(g["silent"][t], (65, 26, 2), t)),
                   "pose": torch.from_numpy(g["pose"][t].copy()), "location_belief": torch.zeros(B, 2),
                   "category_belief": torch.zeros(B, 21)}
            model.update(obs, list(g["dones"][t]))
            assert np.array_equal(obs["category_belief"].numpy(), g["cat_out"][t])
            assert np.array_equal(obs["location_belief"].numpy(), g["loc_out"][t])


def test_silence_sum_and_any_agree_on_spectrograms():
    x = bo.make_spectrograms(np.array([True, False, False, True]), (65, 69, 2), seed=3)
    x[2] = 0
    x[2, 64, 68, 1] = np.float32(1e-30)          # one tiny value: still sounding
    for row in x:
        assert (row.sum() != 0) == bool((row != 0).any())


# ---------------------------------------------------------------------------
# dispatch of the patched update
# ---------------------------------------------------------------------------
def test_patch_replaces_only_update():
    Ref = make_reference_class()
    before = dict(vars(Ref))
    assert belief.patch_belief_predictor(Ref) is Ref
    after = dict(vars(Ref))
    assert set(before) == set(after)
    assert [k for k in before if before[k] is not after[k]] == ["update"]
    assert Ref.update._ssb_original is before["update"]
    belief.patch_belief_predictor(Ref)                     # patching twice keeps the same original
    assert Ref.update._ssb_original is before["update"]


def test_device_path_calls_networks_once_in_order(device_calls):
    Ref = make_reference_class()
    belief.patch_belief_predictor(Ref)
    model = Ref(8, w=0.3, current_pred_only=True)
    order = []
    model.predictor.register_forward_hook(lambda m, i, o: order.append(("predictor", torch.is_grad_enabled())))
    model.classifier.register_forward_hook(lambda m, i, o: order.append(("classifier", torch.is_grad_enabled())))
    obs = make_obs(6, fake_cuda=True)
    dones = [False, True, 0, 1, None, np.bool_(True)]
    model.update(obs, dones)
    assert order == [("predictor", False), ("classifier", False)]
    (c,) = device_calls
    assert c["spec"] is obs["spectrogram"] and c["pose"] is obs["pose"] and c["dones"] is dones
    assert c["loc_out"] is obs["location_belief"] and c["cat_out"] is obs["category_belief"]
    assert c["w"] == 0.3 and c["current_pred_only"] is True
    assert c["loc_pred"].shape == (6, 2) and c["label_pred"].shape == (6, 21)
    assert c["last_pg"].shape == (8, 2) and c["last_label"].shape == (8, 21)
    assert c["loc_valid"].dtype == torch.uint8 and c["label_valid"].shape == (8,)
    assert not obs["location_belief"].any() and not obs["category_belief"].any()    # nothing written on the host
    assert model.last_pointgoal == [None] * 8 and model.last_label == [None] * 8     # the lists are left alone


@pytest.mark.parametrize("loc,label", [(True, False), (False, True)])
def test_one_belief(loc, label, device_calls):
    Ref = make_reference_class()
    belief.patch_belief_predictor(Ref)
    model = Ref(4, loc=loc, label=label)
    obs = make_obs(4, fake_cuda=True)
    if not loc:
        obs["pose"] = obs["pose"].double()             # not read without the location belief
        del obs["location_belief"]
    if not label:
        del obs["category_belief"]
    model.update(obs, None)
    (c,) = device_calls
    assert (c["loc_pred"] is not None) == loc and (c["label_pred"] is not None) == label
    assert (c["pose"] is not None) == loc and (c["cat_out"] is not None) == label


def _fallback_cases():
    def cpu(o):
        return {k: v.as_subclass(torch.Tensor) for k, v in o.items()}

    def f64(o):
        o["spectrogram"] = o["spectrogram"].double().as_subclass(FakeCuda)
        return o

    def pose_f64(o):
        o["pose"] = o["pose"].double().as_subclass(FakeCuda)
        return o

    def row_gaps(o):                                  # a (B, 2) view of a (B, 4) tensor
        o["location_belief"] = torch.zeros(o["pose"].shape[0], 4)[:, :2].as_subclass(FakeCuda)
        return o

    def cat_gaps(o):
        o["category_belief"] = torch.zeros(o["pose"].shape[0], 42)[:, ::2].as_subclass(FakeCuda)
        return o

    def spec_nchw(o):                                 # not the (B, H, W, 2) layout
        o["spectrogram"] = o["spectrogram"].permute(0, 3, 1, 2).contiguous()
        return o
    return dict(cpu=cpu, float64=f64, pose_float64=pose_f64, row_gaps=row_gaps, cat_gaps=cat_gaps, spec_nchw=spec_nchw)


@pytest.mark.parametrize("case", sorted(_fallback_cases()))
def test_fallback_runs_the_original(case, device_calls):
    Ref = make_reference_class()
    torch.manual_seed(0)
    ref_model = Ref(5)
    model = Ref(5)
    model.load_state_dict(ref_model.state_dict())
    belief.patch_belief_predictor(Ref)
    obs = _fallback_cases()[case](make_obs(5, seed=1, silent=(2,), fake_cuda=True))
    ref_obs = {k: v.clone() for k, v in obs.items()}
    if case == "spec_nchw":                            # the original cannot run this layout either
        with pytest.raises(Exception):
            Ref.update._ssb_original(ref_model, ref_obs, None)
        with pytest.raises(Exception):
            model.update(obs, None)
    else:
        Ref.update._ssb_original(ref_model, ref_obs, [False, True, False, False, False])
        model.update(obs, [False, True, False, False, False])
        for k in ("location_belief", "category_belief"):
            assert torch.equal(obs[k].as_subclass(torch.Tensor), ref_obs[k].as_subclass(torch.Tensor))
        assert model.last_pointgoal[0] is not None and model.last_pointgoal[2] is None
    assert not device_calls


def test_prediction_dtype_falls_back(device_calls):
    """Network outputs that are not float32: the original update runs (and evaluates the networks again)."""
    Ref = make_reference_class()
    belief.patch_belief_predictor(Ref)
    model = Ref(3)
    model.classifier.forward = lambda x, f=model.classifier.forward: f(x).double()
    calls = []
    model.predictor.register_forward_hook(lambda *a: calls.append(1))
    model.update(make_obs(3, fake_cuda=True), None)
    assert not device_calls and len(calls) == 2 and model.last_label[0] is not None


def test_batch_larger_than_num_env(device_calls):
    Ref = make_reference_class()
    belief.patch_belief_predictor(Ref)
    with pytest.raises(ValueError, match="last_pointgoal"):
        Ref(4).update(make_obs(5, fake_cuda=True), None)
    with pytest.raises(ValueError, match="last_label"):
        Ref(4, loc=False).update(make_obs(5, fake_cuda=True), None)
    model = Ref(4)
    model.last_label = [None] * 3
    with pytest.raises(ValueError, match="last_label"):
        model.update(make_obs(4, fake_cuda=True), None)
    assert not device_calls
    with pytest.raises(IndexError):                   # the reference itself
        Ref.update._ssb_original(Ref(4), make_obs(5), None)


def test_more_envs_than_the_device_update_takes_run_the_original(device_calls):
    """ssb_belief_update_batch takes at most belief.MAX_ENVS envs: a larger batch runs the original update, even when
    the lists hold that many envs."""
    Ref = make_reference_class()
    n = belief.MAX_ENVS + 1
    torch.manual_seed(0)
    ref_model = Ref(n)
    model = Ref(n)
    model.load_state_dict(ref_model.state_dict())
    belief.patch_belief_predictor(Ref)
    obs = make_obs(n, seed=3, silent=(4,), fake_cuda=True)
    ref_obs = {k: v.clone() for k, v in obs.items()}
    Ref.update._ssb_original(ref_model, ref_obs, None)
    model.update(obs, None)
    for k in ("location_belief", "category_belief"):
        assert torch.equal(obs[k].as_subclass(torch.Tensor), ref_obs[k].as_subclass(torch.Tensor))
    assert model.last_pointgoal[n - 1] is not None and model.last_pointgoal[4] is None
    assert not device_calls
    belief.patch_belief_predictor(Ref)
    model.update(make_obs(belief.MAX_ENVS, fake_cuda=True), None)      # at the limit: the device path
    assert len(device_calls) == 1


def test_subclass_inherits_the_patch(device_calls):
    Ref = make_reference_class()

    class Mixin:
        def init_distributed(self):
            pass

    class BeliefPredictorDDP(Ref, Mixin):
        pass

    belief.patch_belief_predictor(Ref)
    assert BeliefPredictorDDP.update is Ref.update
    BeliefPredictorDDP(4).update(make_obs(4, fake_cuda=True), None)
    assert len(device_calls) == 1


def test_state_starts_over_when_the_lists_are_replaced(device_calls):
    Ref = make_reference_class()
    belief.patch_belief_predictor(Ref)
    model = Ref(6)
    model.update(make_obs(4, fake_cuda=True), None)
    model.update(make_obs(4, fake_cuda=True), None)
    a, b = device_calls
    for k in ("last_pg", "loc_valid", "last_label", "label_valid"):
        assert a[k] is b[k]                           # kept across calls
    a["loc_valid"].fill_(1)
    a["label_valid"].fill_(1)
    model.last_pointgoal[0] = "mutated in place"      # not a replacement
    model.update(make_obs(4, fake_cuda=True), None)
    assert device_calls[2]["last_pg"] is a["last_pg"]
    model.last_pointgoal = [None] * 9                 # replaced: fresh, zeroed state of the new length
    model.update(make_obs(4, fake_cuda=True), None)
    c = device_calls[3]
    assert c["last_pg"] is not a["last_pg"] and c["last_pg"].shape == (9, 2) and not c["loc_valid"].any()
    assert c["last_label"].shape == (6, 21) and not c["label_valid"].any()
    model.last_label = list(model.last_label)         # an equal but new list also starts over
    model.update(make_obs(4, fake_cuda=True), None)
    assert device_calls[4]["last_label"] is not c["last_label"]


# ---------------------------------------------------------------------------
# WaveformOps.belief_update: argument checks and the dones bytes, with the ABI replaced by a recorder
# ---------------------------------------------------------------------------
class FakeLib:
    def __init__(self):
        self.calls = []

    def ssb_belief_update_batch(self, *args):
        self.calls.append(args)
        return 0


def _cpu_ops():
    from soundspaces_b200.renderer import WaveformOps
    ops = object.__new__(WaveformOps)
    ops.device = torch.device("cpu")
    ops.lib = FakeLib()
    ops.ctx = SimpleNamespace(handle=None, check=lambda rc, what: None)
    ops._stream = lambda: None
    return ops


def _args(B=5, N=8, loc=True, label=True):
    a = dict(spec=torch.rand(B, 65, 69, 2))
    if loc:
        a.update(pose=torch.randn(B, 4), loc_pred=torch.randn(B, 23), last_pg=torch.zeros(N, 2),
                 loc_valid=torch.zeros(N, dtype=torch.uint8), loc_out=torch.zeros(B, 2))
    if label:
        a.update(label_pred=torch.randn(B, 21), last_label=torch.zeros(N, 21),
                 label_valid=torch.zeros(N, dtype=torch.uint8), cat_out=torch.zeros(B, 21))
    return a


def test_dones_are_passed_as_bytes():
    ops = _cpu_ops()
    a = _args(B=5)
    spec = a.pop("spec")
    ops.belief_update(spec, [True, False, 1, 0, np.bool_(True), True], 0.5, False, **a)   # extra dones are ignored
    args = ops.lib.calls[-1]
    assert args[1:6] == (5, 8, spec.data_ptr(), 65, 69)
    assert args[7] == 4 and args[9] == 23 and args[11] == 21    # row strides
    assert bytes(args[12]) == bytes([1, 0, 1, 0, 1])
    assert args[13] == 0.5 and args[14] == 0
    ops.belief_update(spec, None, 0.25, True, **a)
    assert ops.lib.calls[-1][12] is None and ops.lib.calls[-1][14] == 1


def test_one_belief_passes_null_pointers():
    ops = _cpu_ops()
    a = _args(loc=False)
    ops.belief_update(a.pop("spec"), None, 0.5, False, pose=torch.randn(5, 2), **a)   # pose unused: not checked
    args = ops.lib.calls[-1]
    assert args[6] is None and args[8] is None and args[15] is None and args[16] is None and args[19] is None
    assert args[10] is not None and args[20] is not None


def _bad(name):
    a = _args()
    if name == "few_dones":
        return a, dict(dones=[False] * 4)
    if name == "no_prediction":
        for k in ("loc_pred", "label_pred"):
            a[k] = None
    elif name == "b_over_num_env":
        a["last_pg"], a["loc_valid"] = torch.zeros(4, 2), torch.zeros(4, dtype=torch.uint8)
    elif name == "spec_not_2_ears":
        a["spec"] = torch.rand(5, 65, 69, 3)
    elif name == "spec_f64":
        a["spec"] = a["spec"].double()
    elif name == "pose_2_cols":
        a["pose"] = torch.randn(5, 2)
    elif name == "loc_pred_col_stride":
        a["loc_pred"] = torch.randn(2, 5).t()
    elif name == "label_pred_20":
        a["label_pred"] = torch.randn(5, 20)
    elif name == "loc_out_rows":
        a["loc_out"] = torch.zeros(4, 2)
    elif name == "cat_out_gaps":
        a["cat_out"] = torch.zeros(5, 42)[:, ::2]
    elif name == "valid_dtype":
        a["label_valid"] = torch.zeros(8, dtype=torch.bool)
    elif name == "valid_rows":
        a["loc_valid"] = torch.zeros(7, dtype=torch.uint8)
    elif name == "state_missing":
        a["last_label"] = None
    return a, {}


@pytest.mark.parametrize("name", ["few_dones", "no_prediction", "b_over_num_env", "spec_not_2_ears", "spec_f64",
                                  "pose_2_cols", "loc_pred_col_stride", "label_pred_20", "loc_out_rows", "cat_out_gaps",
                                  "valid_dtype", "valid_rows", "state_missing"])
def test_belief_update_refuses(name):
    ops = _cpu_ops()
    a, extra = _bad(name)
    with pytest.raises(ValueError):
        ops.belief_update(a.pop("spec"), extra.get("dones"), 0.5, False, **a)
    assert not ops.lib.calls


def test_abi_prototype():
    from soundspaces_b200 import _lib
    restype, argtypes = _lib.EXPORTS["ssb_belief_update_batch"]
    assert restype is C.c_int and len(argtypes) == 22 and argtypes[13] is C.c_double
