"""Host side of the fused audio encoder: the layout check behind ``WaveformOps.audio_encoder`` and the dispatch of
``patch_audio_cnn`` on stand-ins shaped like the reference's three ``AudioCNN`` classes
(ss_baselines/{av_nav,av_wan,savi}/models/audio_cnn.py).  No GPU: the fused path is replaced by a recorder."""
import copy

import numpy as np
import pytest

torch = pytest.importorskip("torch")
nn = torch.nn

from soundspaces_b200 import encoder  # noqa: E402


class Flatten(nn.Module):
    """ss_baselines.common.utils.Flatten."""

    def forward(self, x):
        return x.reshape(x.size(0), -1)


Flatten.__module__ = "ss_baselines.common.utils"


def make_cnn(spec_shape, c3=64, hidden=512, in_ch=2, flatten=Flatten):
    """audio_cnn.py's Sequential for an (H, W, in_ch) observation: 8x8/4, 4x4/2, 3x3/1, or 5/3/3 under 30 pixels."""
    h, w = spec_shape[:2]
    if h < 30 or w < 30:
        ks, st = [(5, 5), (3, 3), (3, 3)], [(2, 2), (2, 2), (1, 1)]
    else:
        ks, st = [(8, 8), (4, 4), (3, 3)], [(4, 4), (2, 2), (1, 1)]
    dims = [h, w]
    for k, s in zip(ks, st):
        dims = [int(np.floor((d - (kk - 1) - 1) / ss + 1)) for d, kk, ss in zip(dims, k, s)]
    return nn.Sequential(
        nn.Conv2d(in_ch, 32, ks[0], st[0]), nn.ReLU(True), nn.Conv2d(32, 64, ks[1], st[1]), nn.ReLU(True),
        nn.Conv2d(64, c3, ks[2], st[2]), flatten(), nn.Linear(c3 * dims[0] * dims[1], hidden), nn.ReLU(True))


def reference_classes():
    """Fresh stand-ins for the three reference AudioCNN classes (patch_audio_cnn patches a class in place)."""

    class AvNavAudioCNN(nn.Module):
        def __init__(self, spec_shape, hidden=512, audiogoal_sensor="spectrogram"):
            super().__init__()
            self._audiogoal_sensor = audiogoal_sensor
            self.cnn = make_cnn(spec_shape, 64, hidden)

        def forward(self, observations):
            x = observations[self._audiogoal_sensor].permute(0, 3, 1, 2)
            return self.cnn(torch.cat([x], dim=1))

    class AvWanAudioCNN(nn.Module):
        def __init__(self, spec_shape, hidden=512):
            super().__init__()
            self.cnn = make_cnn(spec_shape, 32, hidden)

        def forward(self, observations):
            x = observations["spectrogram"].permute(0, 3, 1, 2)
            return self.cnn(torch.cat([x], dim=1))

    class SaviAudioCNN(nn.Module):
        def __init__(self, spec_shape, hidden=512, audiogoal_sensor="audiogoal", has_distractor_sound=False):
            super().__init__()
            self._audiogoal_sensor = audiogoal_sensor
            self._has_distractor_sound = has_distractor_sound
            self._n_input_category = 21 if has_distractor_sound else 0
            self.cnn = make_cnn(spec_shape, 64, hidden, in_ch=2 + self._n_input_category)

        def forward(self, observations):
            x = observations[self._audiogoal_sensor].permute(0, 3, 1, 2)
            inputs = [x]
            if self._has_distractor_sound:
                labels = observations["category"]
                inputs.append(labels.reshape(labels.shape + (1, 1)).expand(labels.shape + x.shape[-2:]))
            return self.cnn(torch.cat(inputs, dim=1))

    return AvNavAudioCNN, AvWanAudioCNN, SaviAudioCNN


class FakeCuda(torch.Tensor):
    """A CPU tensor that reports ``is_cuda``: lets the CPU suite reach the fused branch of the dispatch."""

    @property
    def is_cuda(self):
        return True


@pytest.fixture
def fused_calls(monkeypatch):
    """Replace the fused path with a recorder that returns zeros of the right shape."""
    from soundspaces_b200.renderer import WaveformOps
    calls = []

    class Recorder:
        def audio_encoder(self, x, cnn):
            calls.append((tuple(x.shape), cnn))
            return torch.zeros(x.shape[0], cnn[6].out_features)

    monkeypatch.setattr(WaveformOps, "get", classmethod(lambda cls, device="cuda:0": Recorder()))
    return calls


SHAPES = [(65, 26, 2), (65, 69, 2)]


def _obs(model, x):
    return {getattr(model, "_audiogoal_sensor", "spectrogram"): x, "category": torch.zeros(x.shape[0], 21)}


def test_patch_replaces_only_forward():
    for cls in reference_classes():
        before = dict(vars(cls))
        assert encoder.patch_audio_cnn(cls) is cls
        after = dict(vars(cls))
        assert set(before) == set(after)
        assert [k for k in before if before[k] is not after[k]] == ["forward"]
        assert cls.forward._ssb_original is before["forward"]
        encoder.patch_audio_cnn(cls)                     # patching twice keeps the same original
        assert cls.forward._ssb_original is before["forward"]


@pytest.mark.parametrize("shape", SHAPES)
def test_dispatch(shape, fused_calls):
    torch.manual_seed(0)
    for cls in reference_classes():
        model = cls(shape, hidden=40)
        x = torch.rand((3,) + shape)
        ref = model(_obs(model, x))
        encoder.patch_audio_cnn(cls)
        assert torch.equal(model(_obs(model, x)), ref)                       # grad enabled: original forward
        with torch.no_grad():
            assert torch.equal(model(_obs(model, x)), ref)                   # CPU tensor: original forward
            assert not fused_calls
            got = model(_obs(model, x.as_subclass(FakeCuda)))                # CUDA float32 (N, H, W, 2): fused
            assert fused_calls and fused_calls[-1] == ((3,) + shape, model.cnn) and got.shape == (3, 40)
            n = len(fused_calls)
            model64 = copy.deepcopy(model).double()
            model64(_obs(model64, x.double().as_subclass(FakeCuda)))        # float64: original
            model(_obs(model, x.as_subclass(FakeCuda).permute(0, 2, 1, 3).contiguous().permute(0, 2, 1, 3)))
            assert len(fused_calls) == n                                     # not contiguous: original
        fused_calls.clear()


def test_dispatch_savi_with_category_channels(fused_calls):
    _, _, Savi = reference_classes()
    encoder.patch_audio_cnn(Savi)
    model = Savi((65, 26, 2), hidden=40, has_distractor_sound=True)
    assert model.cnn[0].in_channels == 23
    x = torch.rand(2, 65, 26, 2)
    with torch.no_grad():
        out = model(_obs(model, x.as_subclass(FakeCuda)))
    assert not fused_calls and out.shape == (2, 40)


def _bad_layouts():
    base = lambda: make_cnn((65, 26, 2))           # noqa: E731
    cases = {}
    m = base(); m[0] = nn.Conv2d(2, 32, 5, 2, padding=1); cases["padding"] = m
    m = base(); m[2] = nn.Conv2d(32, 64, 3, 2, dilation=2); cases["dilation"] = m
    m = base(); m[4] = nn.Conv2d(64, 64, 3, 1, groups=2); cases["groups"] = m
    m = base(); m[0] = nn.Conv2d(3, 32, 5, 2); cases["in_channels"] = m
    cases["savi_category"] = make_cnn((65, 26, 2), in_ch=23)
    m = base(); cases["missing_relu"] = nn.Sequential(*[m[i] for i in (0, 2, 3, 4, 5, 6, 7)])
    m = base(); cases["missing_final_relu"] = nn.Sequential(*[m[i] for i in range(7)])
    m = base(); cases["reordered"] = nn.Sequential(*[m[i] for i in (0, 1, 2, 3, 4, 6, 5, 7)])
    m = base(); cases["relu_after_conv3"] = nn.Sequential(*[m[i] for i in (0, 1, 2, 3, 4, 1, 5, 6)])
    m = base(); m[1] = nn.Tanh(); cases["tanh"] = m
    m = base(); m[5] = nn.Flatten(0); cases["flatten_dim0"] = m
    m = base(); m[2] = nn.Conv2d(16, 64, 3, 2); cases["channel_chain"] = m
    cases["not_sequential"] = list(base())
    return cases


@pytest.mark.parametrize("name", sorted(_bad_layouts()))
def test_layout_refused(name):
    cnn = _bad_layouts()[name]
    assert encoder.encoder_layout_error(cnn)
    with pytest.raises(ValueError):
        encoder.check_encoder_layout(cnn)


@pytest.mark.parametrize("flatten", [Flatten, nn.Flatten])
def test_layout_accepted(flatten):
    for c3 in (64, 32):
        for shape in SHAPES:
            cnn = make_cnn(shape, c3, flatten=flatten)
            assert encoder.encoder_layout_error(cnn) == ""
            encoder.check_encoder_layout(cnn)


def test_flatten_from_elsewhere_is_refused():
    class Flatten(nn.Module):                    # same name, not the reference's module
        def forward(self, x):
            return x.reshape(x.size(0), -1)
    assert encoder.encoder_layout_error(make_cnn((65, 26, 2), flatten=Flatten))
