"""Host side of the SMT location predictor's online training (``patch_belief_predictor(..., training=True)``): the
patch leaves ``cnn_forward`` alone without the flag, keeps the original reachable, patches once, and calls that do not
qualify (here: CPU tensors) run the original."""
import pytest

torch = pytest.importorskip("torch")

from belief_nets_models import smt_net  # noqa: E402


class _Predictor(torch.nn.Module):
    def __init__(self, n_labels=0):
        super().__init__()
        self.has_distractor_sound = bool(n_labels)
        self.predictor = smt_net(2 + n_labels, (65, 26))

    def cnn_forward(self, observations):
        s = observations["spectrogram"].permute(0, 3, 1, 2)
        if self.has_distractor_sound:
            labels = observations["category"]
            s = torch.cat([s, labels.reshape(labels.shape + (1, 1)).expand(labels.shape + s.shape[-2:])], dim=1)
        return self.predictor(s)

    def update(self, observations, dones):
        raise NotImplementedError


def _fresh():
    class P(_Predictor):
        pass
    return P


def test_flag_off_keeps_cnn_forward():
    from soundspaces_b200.belief import patch_belief_predictor
    P = _fresh()
    before = P.cnn_forward
    patch_belief_predictor(P, networks=True)
    assert P.cnn_forward is before


def test_patch_keeps_the_original_and_patches_once():
    from soundspaces_b200.belief import patch_belief_predictor
    P = _fresh()
    original = P.cnn_forward
    patch_belief_predictor(P, networks=True, training=True)
    assert P.cnn_forward is not original and P.cnn_forward._ssb_original is original
    patch_belief_predictor(P, networks=True, training=True)
    assert P.cnn_forward._ssb_original is original


@pytest.mark.parametrize("n_labels", [0, 21])
def test_cpu_calls_run_the_original(n_labels):
    from soundspaces_b200.belief import patch_belief_predictor
    from soundspaces_b200.belief_nets import smt_resnet18_train_error
    P = _fresh()
    patch_belief_predictor(P, training=True)
    m = P(n_labels)
    obs = {"spectrogram": torch.rand(3, 65, 26, 2)}
    if n_labels:
        obs["category"] = torch.eye(n_labels)[:3]
    assert smt_resnet18_train_error(m, obs) == "the spectrogram is not a CUDA tensor"
    got = m.cnn_forward(obs)
    want = _Predictor.cnn_forward(m, obs)
    assert torch.equal(got, want) and got.grad_fn is not None


def test_fallback_reasons_without_a_device():
    from soundspaces_b200.belief_nets import smt_resnet18_train_error
    m = _Predictor()
    assert smt_resnet18_train_error(m, {}) == "the spectrogram is not a CUDA tensor"
    assert smt_resnet18_train_error(m, {"spectrogram": [1.0]}) == "the spectrogram is not a CUDA tensor"


@pytest.fixture(scope="module")
def golden():
    import os
    import numpy as np
    path = os.path.join(os.path.dirname(__file__), "golden", "smt_resnet_train_golden.npz")
    return dict(np.load(path))


def _case(name):
    from belief_nets_models import SmtResNet
    from smt_resnet_train_models import CASES, case_inputs, set_params
    net = set_params(SmtResNet(2 + CASES[name])).double()
    return net, case_inputs(name)


@pytest.mark.parametrize("name", ["smt2", "smt23"])
def test_stand_in_reproduces_the_golden(golden, name):
    """The float64 stand-in against the unmodified reference custom_resnet18's forward and masked-MSE gradients."""
    import numpy as np
    from smt_resnet_train_models import check_grad, torch_grads
    net, (x, labels, gts) = _case(name)
    pred, grads = torch_grads(net, x, labels, gts)
    assert np.abs(pred.numpy() - golden[f"{name}/pred"]).max() <= 1e-12 * np.abs(golden[f"{name}/pred"]).max()
    for j, g in enumerate(grads):
        check_grad(name, j, g.numpy(), golden, 1e-10)


@pytest.mark.parametrize("name", ["smt2", "smt23"])
def test_numpy_model_of_the_kernels_reproduces_the_golden(golden, name):
    """The kernels' equations (live-row compaction, threshold_backward on the saved output, GroupNorm backward from
    the saved statistics, residual split, padded stride-2 gather dX, label-tap sums) in float64 against the golden."""
    import numpy as np
    from soundspaces_b200.belief_nets import conv_norm_pairs, smt_resnet18_params
    from smt_resnet_train_models import check_grad, numpy_model
    net, (x, labels, gts) = _case(name)
    params = [p.detach().numpy() for p in smt_resnet18_params(net)]
    eps = [n.eps for _, n in conv_norm_pairs(net)]
    pred, grads = numpy_model(params, eps, x.numpy(), None if labels is None else labels.numpy(), gts.numpy())
    assert np.abs(pred - golden[f"{name}/pred"]).max() <= 1e-10 * np.abs(golden[f"{name}/pred"]).max()
    for j, g in enumerate(grads):
        check_grad(name, j, g, golden, 1e-9)
