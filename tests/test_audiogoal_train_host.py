"""Host side of SAVi's audio-goal predictor training (``patch_audiogoal_predictor``, ``belief_nets.ResNetFunction``):
a float64 stand-in and a numpy model of the kernels' equations against the golden of the unmodified reference, the
layout check in both BatchNorm modes, the fallback reasons a CPU call meets, torch's ValueError for one value per
channel, and the patch keeping the original, patching once and leaving numpy and CPU calls to it."""
import logging

import numpy as np
import pytest

torch = pytest.importorskip("torch")

from audiogoal_train_models import CASES, case_inputs, check, set_params, torch_step, tv_net  # noqa: E402


@pytest.fixture(scope="module")
def golden():
    import os
    path = os.path.join(os.path.dirname(__file__), "golden", "audiogoal_train_golden.npz")
    return dict(np.load(path))


def _net(name):
    H, W, n_out, B, mode, steps = CASES[name]
    return set_params(tv_net(n_out)).double().train(mode == "train"), steps


@pytest.mark.parametrize("name", list(CASES))
def test_stand_in_reproduces_the_golden(golden, name):
    """torchvision's resnet18 in float64 against the unmodified reference AudioGoalPredictor: logits, the gradients
    of the pretraining loss and the running statistics after each step."""
    from soundspaces_b200.belief_nets import resnet18_buffers
    net, steps = _net(name)
    for step in range(steps):
        x, gts = case_inputs(name, step)
        pred, grads = torch_step(net, x, gts)
        ref = golden[f"{name}/{step}/pred"]
        assert np.abs(pred.numpy() - ref).max() <= 1e-12 * np.abs(ref).max()
        check(f"{name}/{step}/g", [g.numpy() for g in grads], golden, 1e-10)
        check(f"{name}/{step}/s", [t.numpy() for t in resnet18_buffers(net)[:40]], golden, 1e-12)


@pytest.mark.parametrize("name", list(CASES))
def test_numpy_model_of_the_kernels_reproduces_the_golden(golden, name):
    """The kernels' equations (batch statistics and their backward over every row, the running update, the first-
    maximum maxpool rule in gather form, AdaptiveAvgPool2d's spread, padded strided conv gradients) in float64."""
    from soundspaces_b200.belief_nets import conv_norm_pairs, resnet18_buffers, resnet18_params
    from audiogoal_train_models import MOMENTUM, numpy_model
    net, steps = _net(name)
    training = CASES[name][4] == "train"
    params = [p.detach().numpy() for p in resnet18_params(net)]
    stats = [t.numpy().copy() for t in resnet18_buffers(net)[:40]]
    eps = [n.eps for _, n in conv_norm_pairs(net)]
    for step in range(steps):
        x, gts = case_inputs(name, step)
        pred, grads, stats = numpy_model(params, stats, eps, MOMENTUM, training, x.numpy(), gts.numpy())
        ref = golden[f"{name}/{step}/pred"]
        assert np.abs(pred - ref).max() <= 1e-10 * np.abs(ref).max()
        check(f"{name}/{step}/g", grads, golden, 1e-9)
        check(f"{name}/{step}/s", stats, golden, 1e-12)


def test_maxpool_ties_go_to_the_first_maximum():
    """A window of equal values routes its gradient to its first valid element, as torch's max_pool2d does: the
    silent row of the golden cases normalises to one value per channel, so its windows are whole ties."""
    from audiogoal_train_models import _maxpool
    y = np.zeros((1, 1, 5, 5))
    y[0, 0, 2, 2] = 1.0
    out, arg = _maxpool(y)
    assert out.shape == (1, 1, 3, 3)
    assert arg[0, 0, 0, 0] == 4          # rows and columns -1..1: the first valid element is (0, 0), index 3 + 1
    assert arg[0, 0, 1, 1] == 4          # the maximum at (2, 2)
    assert arg[0, 0, 2, 2] == 0          # rows and columns 3..5: all 0, the first is (3, 3)


def test_layout_in_both_modes():
    from soundspaces_b200.belief_nets import resnet18_layout_error
    net = tv_net(23)
    assert resnet18_layout_error(net.eval()) == ""
    assert "training mode" in resnet18_layout_error(net.train())
    assert resnet18_layout_error(net.train(), training=True) == ""
    assert resnet18_layout_error(net.eval(), training=True) == ""
    net.layer3[1].bn2 = torch.nn.GroupNorm(16, 256)
    assert "expected BatchNorm2d" in resnet18_layout_error(net, training=True)


class AudioGoalPredictor(torch.nn.Module):
    """The reference class's interface (audiogoal_predictor.py:18-38) on the CPU: the one-time shape log, the numpy
    branch (without the move to cuda:0), the permute and the predictor."""

    def __init__(self, n_out=23):
        super().__init__()
        self.input_shape_printed = False
        self.predictor = tv_net(n_out)

    def forward(self, audio_feature):
        if not self.input_shape_printed:
            logging.info('Audiogoal predictor input audio feature shape: {}'.format(audio_feature["spectrogram"].shape))
            self.input_shape_printed = True
        x = audio_feature["spectrogram"]
        if not torch.is_tensor(x):
            x = torch.from_numpy(x).unsqueeze(0)
        return self.predictor(x.permute(0, 3, 1, 2))


def _fresh():
    class P(AudioGoalPredictor):
        pass
    return P


def test_patch_keeps_the_original_and_patches_once():
    from soundspaces_b200.pretraining import patch_audiogoal_predictor
    P = _fresh()
    original = P.forward
    assert patch_audiogoal_predictor(P) is P
    assert P.forward is not original and P.forward._ssb_original is original
    patch_audiogoal_predictor(P)
    assert P.forward._ssb_original is original
    patch_audiogoal_predictor(P, training=False)
    assert P.forward._ssb_original is original


@pytest.mark.parametrize("mode", ["train", "eval"])
def test_cpu_and_numpy_calls_run_the_original(mode, caplog):
    from soundspaces_b200.pretraining import patch_audiogoal_predictor
    P = _fresh()
    patch_audiogoal_predictor(P)
    torch.manual_seed(0)
    m = P()
    ref = AudioGoalPredictor()
    ref.load_state_dict(m.state_dict())
    m.train(mode == "train")
    ref.train(mode == "train")
    x = torch.rand(3, 65, 26, 2)
    with caplog.at_level(logging.INFO):
        got = m({"spectrogram": x})
        m({"spectrogram": x})
    assert [r.getMessage() for r in caplog.records] == [
        "Audiogoal predictor input audio feature shape: torch.Size([3, 65, 26, 2])"]
    want = ref({"spectrogram": x})
    assert torch.equal(got, want) and got.grad_fn is not None
    one = m({"spectrogram": x[0].numpy()})
    assert one.shape == (1, 23)
    assert int(m.predictor.bn1.num_batches_tracked) == (3 if mode == "train" else 0)


def test_fallback_reasons_without_a_device():
    from soundspaces_b200.belief_nets import resnet18_train_error
    m = AudioGoalPredictor()
    assert resnet18_train_error(m, {}) == "the spectrogram is not a CUDA tensor"
    assert resnet18_train_error(m, {"spectrogram": [1.0]}) == "the spectrogram is not a CUDA tensor"
    assert resnet18_train_error(m, {"spectrogram": torch.rand(2, 65, 26, 2)}) == "the spectrogram is not a CUDA tensor"


@pytest.mark.parametrize("B,H,W", [(1, 17, 17), (1, 3, 3), (1, 1, 1)])
def test_one_value_per_channel_raises_torchs_value_error(B, H, W):
    """check_batch_norm_values raises what BatchNorm2d raises in training mode, at the same norm."""
    from soundspaces_b200.belief_nets import check_batch_norm_values
    net = tv_net(23).train()
    with pytest.raises(ValueError) as want:
        net(torch.rand(B, 2, H, W))
    with pytest.raises(ValueError) as got:
        check_batch_norm_values(B, H, W)
    assert str(got.value) == str(want.value)
    check_batch_norm_values(2, H, W)
    check_batch_norm_values(1, 65, 26)
