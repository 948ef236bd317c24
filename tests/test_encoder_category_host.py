"""Host side of the fused encoder for SAVi with a distractor sound: the identity that lets the kernel fold the category
channels into a per-env conv1 bias, the layout check with category channels, and the dispatch of
``patch_audio_cnn(cls, category=True)`` on the stand-ins of ``test_encoder_host``.  No GPU: the fused path is replaced
by a recorder."""
import copy

import pytest

torch = pytest.importorskip("torch")
nn = torch.nn

from soundspaces_b200 import encoder  # noqa: E402
from test_encoder_host import FakeCuda, make_cnn, reference_classes  # noqa: E402

SHAPES = [(65, 26, 2), (65, 69, 2)]          # 16 kHz (conv1 5x5 / 2) and 44.1 kHz (8x8 / 4)


def _labels(kind, n, gen):
    if kind == "one_hot":
        return nn.functional.one_hot(torch.randint(0, 21, (n,), generator=gen), 21).double()
    if kind == "zero":
        return torch.zeros(n, 21, dtype=torch.float64)
    return torch.rand(n, 21, generator=gen, dtype=torch.float64) * 2.0 - 1.0      # signed soft values


@pytest.mark.parametrize("kind", ["one_hot", "zero", "soft"])
@pytest.mark.parametrize("shape", SHAPES)
def test_fold_identity(shape, kind):
    """conv1(cat(x, expand(l))) == conv1_ears(x) + b + sum_c l[c] sum_k W[:, 2 + c, k], in float64."""
    gen = torch.Generator().manual_seed(shape[1])
    conv = make_cnn(shape, in_ch=23)[0].double()
    with torch.no_grad():
        conv.bias.uniform_(-0.5, 0.5, generator=gen)
        x = torch.rand((4, 2) + shape[:2], generator=gen, dtype=torch.float64)
        lab = _labels(kind, 4, gen)
        ref = conv(torch.cat([x, lab[:, :, None, None].expand(4, 21, *shape[:2])], dim=1))
        W = conv.weight
        ears = nn.functional.conv2d(x, W[:, :2], None, conv.stride)
        fold = conv.bias[None] + lab @ W[:, 2:].sum(dim=(2, 3)).T              # (n, C1)
        got = ears + fold[:, :, None, None]
    assert (got - ref).abs().max().item() <= 1e-12 * max(1.0, ref.abs().max().item())


@pytest.fixture
def fused_calls(monkeypatch):
    """Replace the fused path with a recorder that returns zeros of the right shape."""
    from soundspaces_b200.renderer import WaveformOps
    calls = []

    class Recorder:
        def audio_encoder(self, x, cnn, features=None, category=None):
            calls.append((tuple(x.shape), cnn, category))
            return torch.zeros(x.shape[0], cnn[6].out_features)

    monkeypatch.setattr(WaveformOps, "get", classmethod(lambda cls, device="cuda:0": Recorder()))
    return calls


def _savi(shape, distractor=True):
    _, _, Savi = reference_classes()
    torch.manual_seed(3)
    return Savi, Savi(shape, hidden=40, has_distractor_sound=distractor)


@pytest.mark.parametrize("shape", SHAPES)
def test_dispatch_category(shape, fused_calls):
    Savi, model = _savi(shape)
    x = torch.rand((3,) + shape)
    lab = torch.rand(3, 21)
    ref = model({"audiogoal": x, "category": lab})
    encoder.patch_audio_cnn(Savi, category=True)
    assert torch.equal(model({"audiogoal": x, "category": lab}), ref)                  # grad enabled: original
    assert not fused_calls
    with torch.no_grad():
        fx, flab = x.as_subclass(FakeCuda), lab.as_subclass(FakeCuda)
        got = model({"audiogoal": fx, "category": flab})
        assert len(fused_calls) == 1 and got.shape == (3, 40)
        assert fused_calls[0][0] == (3,) + shape and fused_calls[0][1] is model.cnn and fused_calls[0][2] is flab
        wide = torch.full((3, 30), float("nan")).as_subclass(FakeCuda)
        wide[:, 4:25] = flab
        model({"audiogoal": fx, "category": wide[:, 4:25]})                          # row stride 30: fused
        assert len(fused_calls) == 2 and fused_calls[-1][2].stride() == (30, 1)

        assert torch.equal(model({"audiogoal": x, "category": lab}), ref)             # CPU observation and labels
        assert torch.equal(model({"audiogoal": fx, "category": lab}), ref)            # CPU labels
        model64 = copy.deepcopy(model).double()
        model64({"audiogoal": fx.double(), "category": flab.double()})                # float64 observation
        with pytest.raises(RuntimeError):                                            # float64 labels: the original,
            model({"audiogoal": fx, "category": lab.double().as_subclass(FakeCuda)})  # whose cat promotes to float64
        cols = torch.rand(21, 3).as_subclass(FakeCuda).T                              # column stride 3
        assert torch.allclose(model({"audiogoal": fx, "category": cols}),
                              model({"audiogoal": x, "category": cols.contiguous().as_subclass(torch.Tensor)}))
        with pytest.raises(RuntimeError):                                            # 20 columns: the original's cat
            model({"audiogoal": fx, "category": torch.rand(3, 20).as_subclass(FakeCuda)})   # makes 22 channels
        with pytest.raises(RuntimeError):                                            # 2 rows for 3 envs
            model({"audiogoal": fx, "category": flab[:2]})
        with pytest.raises(KeyError):                                                # no category: the original
            model({"audiogoal": fx})
        assert len(fused_calls) == 2


def test_dispatch_category_is_opt_in(fused_calls):
    """Without category=True a SAVi model with a distractor sound keeps the original forward."""
    Savi, model = _savi((65, 26, 2))
    encoder.patch_audio_cnn(Savi)
    with torch.no_grad():
        x = torch.rand(2, 65, 26, 2).as_subclass(FakeCuda)
        out = model({"audiogoal": x, "category": torch.rand(2, 21).as_subclass(FakeCuda)})
    assert not fused_calls and out.shape == (2, 40)


@pytest.mark.parametrize("shape", SHAPES)
def test_dispatch_without_distractor_is_unchanged(shape, fused_calls):
    """av_nav, av_wan and SAVi without a distractor sound dispatch as with the default: no category is passed."""
    for cls in reference_classes():
        encoder.patch_audio_cnn(cls, category=True)
        torch.manual_seed(0)
        model = cls(shape, hidden=40)
        key = getattr(model, "_audiogoal_sensor", "spectrogram")
        x = torch.rand((3,) + shape)
        obs = {key: x, "category": torch.zeros(3, 21)}
        ref = model(obs)
        with torch.no_grad():
            assert torch.equal(model(obs), ref)                                      # CPU: original
            assert not fused_calls
            obs[key] = x.as_subclass(FakeCuda)
            obs["category"] = obs["category"].as_subclass(FakeCuda)
            model(obs)
        assert len(fused_calls) == 1 and fused_calls[0][2] is None and fused_calls[0][1] is model.cnn
        fused_calls.clear()


@pytest.mark.parametrize("shape", SHAPES)
def test_layout_with_category(shape):
    cnn = make_cnn(shape, in_ch=23)
    assert encoder.encoder_layout_error(cnn, n_category=21) == ""
    encoder.check_encoder_layout(cnn, n_category=21)
    assert encoder.encoder_layout_error(cnn)                                         # the default refuses 23 channels
    for in_ch in (2, 22, 24):
        other = make_cnn(shape, in_ch=in_ch)
        assert "in_channels" in encoder.encoder_layout_error(other, n_category=21)
        with pytest.raises(ValueError, match=r"Conv2d\(23 -> C1\)"):
            encoder.check_encoder_layout(other, n_category=21)
    bad = make_cnn(shape, in_ch=23)
    bad[0] = nn.Conv2d(23, 32, 5, 2, padding=1)
    assert encoder.encoder_layout_error(bad, n_category=21)
