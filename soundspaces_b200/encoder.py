"""The policy's audio encoder at rollout time: ``AudioCNN.cnn`` of the reference's audio-goal baselines
(ss_baselines/av_nav/models/audio_cnn.py:50-75, av_wan/models/audio_cnn.py:51-76, savi/models/audio_cnn.py:61-92)
run by ``ssb_audio_encoder_batch`` (two launches) instead of seven PyTorch / cuDNN layers.

    from soundspaces_b200.encoder import patch_audio_cnn
    patch_audio_cnn(AudioCNN)       # the class of ss_baselines.av_nav / av_wan / savi models.audio_cnn
    patch_audio_cnn(AudioCNN, category=True)     # savi: also SAVi with a distractor sound

The patched ``forward`` takes the fused path only for inference on a contiguous CUDA float32 ``(N, H, W, 2)``
observation through a ``cnn`` of exactly the reference layout (:func:`check_encoder_layout`); the PPO update (grad
enabled) and CPU tensors run the original ``forward``.  SAVi with a distractor sound (``_has_distractor_sound``)
concatenates the ``(N, 21)`` category observation, broadcast over every pixel, after the two ears, so its conv1 has
23 input channels.  By default it runs the original ``forward``; with ``category=True`` it takes the fused path too
(``ssb_audio_encoder_category_batch``, the label channels folded into a per-env conv1 bias) when ``category`` is a
CUDA float32 ``(N, 21)`` tensor on the observation's device with unit column stride.
"""
from __future__ import annotations

import torch
import torch.nn as nn


def _is_flatten(m: nn.Module) -> bool:
    if isinstance(m, nn.Flatten):
        return m.start_dim == 1 and m.end_dim == -1
    # ss_baselines.common.utils.Flatten: x.reshape(x.size(0), -1), no parameters
    return (type(m).__name__ == "Flatten" and type(m).__module__ == "ss_baselines.common.utils"
            and not any(True for _ in m.parameters()))


def encoder_layout_error(cnn, n_category: int = 0) -> str:
    """Why ``cnn`` is not ``Conv2d(2 + n_category -> C1) ReLU Conv2d ReLU Conv2d Flatten Linear ReLU`` with unpadded,
    undilated, ungrouped convolutions chained channel to channel; ``""`` when it is."""
    if not isinstance(cnn, nn.Sequential) or len(cnn) != 8:
        return "expected an nn.Sequential of 8 modules"
    kinds = (nn.Conv2d, nn.ReLU, nn.Conv2d, nn.ReLU, nn.Conv2d, None, nn.Linear, nn.ReLU)
    for i, (m, kind) in enumerate(zip(cnn, kinds)):
        ok = _is_flatten(m) if kind is None else type(m) is kind
        if not ok:
            want = "Flatten" if kind is None else kind.__name__
            return f"module {i} is {type(m).__name__}, expected {want}"
    in_ch = 2 + n_category
    for i in (0, 2, 4):
        c = cnn[i]
        if c.in_channels != in_ch:
            return f"module {i}: in_channels {c.in_channels}, expected {in_ch}"
        if (tuple(c.padding) != (0, 0) or tuple(c.dilation) != (1, 1) or c.groups != 1
                or c.padding_mode != "zeros"):
            return f"module {i}: only unpadded, undilated, ungrouped convolutions are fused"
        in_ch = c.out_channels
    return ""


def check_encoder_layout(cnn, n_category: int = 0):
    """Raise ``ValueError`` unless ``cnn`` has the layout :func:`encoder_layout_error` accepts."""
    err = encoder_layout_error(cnn, n_category)
    if err:
        raise ValueError(f"audio_encoder fuses AudioCNN.cnn = Conv2d({2 + n_category} -> C1) ReLU Conv2d ReLU Conv2d "
                         "Flatten Linear ReLU: " + err)


def _fusable(x) -> bool:
    return (isinstance(x, torch.Tensor) and x.is_cuda and x.dtype == torch.float32 and x.ndim == 4
            and x.shape[3] == 2 and x.is_contiguous())


def _fusable_category(labels, x, cnn) -> bool:
    """SAVi's ``(N, 21)`` category observation as the fused path reads it: on ``x``'s device, float32, one row per
    env, unit column stride, as many columns as ``cnn``'s conv1 has label channels."""
    return (isinstance(labels, torch.Tensor) and labels.is_cuda and labels.device == x.device
            and labels.dtype == torch.float32 and labels.ndim == 2 and labels.shape[0] == x.shape[0]
            and labels.stride(1) == 1 and (labels.shape[0] <= 1 or labels.stride(0) >= labels.shape[1])
            and isinstance(cnn, nn.Sequential) and len(cnn) == 8 and isinstance(cnn[0], nn.Conv2d)
            and labels.shape[1] == cnn[0].in_channels - 2 and not encoder_layout_error(cnn, labels.shape[1]))


def patch_audio_cnn(cls, category: bool = False):
    """Replace ``cls.forward`` of an ``AudioCNN`` class (av_nav, av_wan or savi) in place, nothing else.  The
    observation is ``observations[self._audiogoal_sensor]`` (av_nav, savi) or ``observations["spectrogram"]``
    (av_wan, which has no ``_audiogoal_sensor``).  ``category=True`` also fuses SAVi models built with
    ``has_distractor_sound=True``, reading ``observations["category"]``; without it they run the original."""
    original = getattr(cls.forward, "_ssb_original", cls.forward)

    def forward(self, observations):
        x = observations[getattr(self, "_audiogoal_sensor", "spectrogram")]
        if category and getattr(self, "_has_distractor_sound", False):
            if torch.is_grad_enabled() or not _fusable(x) or "category" not in observations:
                return original(self, observations)
            labels = observations["category"]
            if not _fusable_category(labels, x, self.cnn):
                return original(self, observations)
            from .renderer import WaveformOps
            return WaveformOps.get(x.device).audio_encoder(x, self.cnn, category=labels)
        if torch.is_grad_enabled() or not _fusable(x) or encoder_layout_error(self.cnn):
            return original(self, observations)
        from .renderer import WaveformOps
        return WaveformOps.get(x.device).audio_encoder(x, self.cnn)

    forward._ssb_original = original
    forward.__doc__ = original.__doc__
    cls.forward = forward
    return cls
