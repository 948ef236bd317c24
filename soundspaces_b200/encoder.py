"""The policy's audio encoder at rollout time: ``AudioCNN.cnn`` of the reference's audio-goal baselines
(ss_baselines/av_nav/models/audio_cnn.py:50-75, av_wan/models/audio_cnn.py:51-76, savi/models/audio_cnn.py:61-92)
run by ``ssb_audio_encoder_batch`` (two launches) instead of seven PyTorch / cuDNN layers.

    from soundspaces_b200.encoder import patch_audio_cnn
    patch_audio_cnn(AudioCNN)       # the class of ss_baselines.av_nav / av_wan / savi models.audio_cnn

The patched ``forward`` takes the fused path only for inference on a contiguous CUDA float32 ``(N, H, W, 2)``
observation through a ``cnn`` of exactly the reference layout (:func:`check_encoder_layout`); the PPO update (grad
enabled), CPU tensors and SAVi with category channels (``in_channels != 2``) run the original ``forward``.
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


def encoder_layout_error(cnn) -> str:
    """Why ``cnn`` is not ``Conv2d(2 -> C1) ReLU Conv2d ReLU Conv2d Flatten Linear ReLU`` with unpadded, undilated,
    ungrouped convolutions chained channel to channel; ``""`` when it is."""
    if not isinstance(cnn, nn.Sequential) or len(cnn) != 8:
        return "expected an nn.Sequential of 8 modules"
    kinds = (nn.Conv2d, nn.ReLU, nn.Conv2d, nn.ReLU, nn.Conv2d, None, nn.Linear, nn.ReLU)
    for i, (m, kind) in enumerate(zip(cnn, kinds)):
        ok = _is_flatten(m) if kind is None else type(m) is kind
        if not ok:
            want = "Flatten" if kind is None else kind.__name__
            return f"module {i} is {type(m).__name__}, expected {want}"
    in_ch = 2
    for i in (0, 2, 4):
        c = cnn[i]
        if c.in_channels != in_ch:
            return f"module {i}: in_channels {c.in_channels}, expected {in_ch}"
        if (tuple(c.padding) != (0, 0) or tuple(c.dilation) != (1, 1) or c.groups != 1
                or c.padding_mode != "zeros"):
            return f"module {i}: only unpadded, undilated, ungrouped convolutions are fused"
        in_ch = c.out_channels
    return ""


def check_encoder_layout(cnn):
    """Raise ``ValueError`` unless ``cnn`` has the layout :func:`encoder_layout_error` accepts."""
    err = encoder_layout_error(cnn)
    if err:
        raise ValueError("audio_encoder fuses AudioCNN.cnn = Conv2d(2 -> C1) ReLU Conv2d ReLU Conv2d Flatten Linear "
                         "ReLU: " + err)


def _fusable(x) -> bool:
    return (isinstance(x, torch.Tensor) and x.is_cuda and x.dtype == torch.float32 and x.ndim == 4
            and x.shape[3] == 2 and x.is_contiguous())


def patch_audio_cnn(cls):
    """Replace ``cls.forward`` of an ``AudioCNN`` class (av_nav, av_wan or savi) in place, nothing else.  The
    observation is ``observations[self._audiogoal_sensor]`` (av_nav, savi) or ``observations["spectrogram"]``
    (av_wan, which has no ``_audiogoal_sensor``)."""
    original = getattr(cls.forward, "_ssb_original", cls.forward)

    def forward(self, observations):
        x = observations[getattr(self, "_audiogoal_sensor", "spectrogram")]
        if torch.is_grad_enabled() or not _fusable(x) or encoder_layout_error(self.cnn):
            return original(self, observations)
        from .renderer import WaveformOps
        return WaveformOps.get(x.device).audio_encoder(x, self.cnn)

    forward._ssb_original = original
    forward.__doc__ = original.__doc__
    cls.forward = forward
    return cls
