"""The policy's state encoder at rollout time: ``RNNStateEncoder.single_forward`` of the reference's baselines
(ss_baselines/av_nav/models/rnn_state_encoder.py:80-90; av_wan and SAVi's ``AudioNavBaselineNet`` import the same
class) run by ``ssb_gru_step_batch`` (one launch) instead of the mask multiply and a cuDNN GRU step.

    from soundspaces_b200.rnn import patch_rnn_state_encoder
    patch_rnn_state_encoder(RNNStateEncoder)     # ss_baselines.av_nav.models.rnn_state_encoder.RNNStateEncoder

Only ``single_forward`` is replaced.  The reference's ``forward`` already routes rollout steps there
(``x.size(0) == hidden_states.size(1)``); ``seq_forward``, which the PPO update runs, is untouched.  The fused path
takes a one-layer, unidirectional ``nn.GRU`` with bias (:func:`gru_layout_error`) under no-grad on contiguous CUDA
float32 tensors; an LSTM (SAVi's DD-PPO ``resnet_policy.py`` default), a multi-layer GRU and everything else run the
original.
"""
from __future__ import annotations

import torch
import torch.nn as nn


def gru_layout_error(rnn) -> str:
    """Why ``rnn`` is not an ``nn.GRU`` with one layer, bias, one direction, ``batch_first=False`` and no projection;
    ``""`` when it is."""
    if type(rnn) is not nn.GRU:
        return f"{type(rnn).__name__} is not nn.GRU"
    if rnn.num_layers != 1:
        return f"num_layers is {rnn.num_layers}, expected 1"
    if not rnn.bias:
        return "bias=False"
    if rnn.bidirectional:
        return "bidirectional"
    if rnn.batch_first:
        return "batch_first=True"
    if getattr(rnn, "proj_size", 0) != 0:
        return f"proj_size is {rnn.proj_size}"
    return ""


def _dense(t, device) -> bool:
    return isinstance(t, torch.Tensor) and t.is_cuda and t.device == device and t.dtype == torch.float32 and t.is_contiguous()


def fused_single_forward(module, x, hidden_states, masks):
    """``module.single_forward(x, hidden_states, masks)`` through the library -> ``(out (N, Hd), h (1, N, Hd))``, or
    None (the caller runs the original) when grad is enabled, ``module.rnn`` does not qualify
    (:func:`gru_layout_error`), a tensor or parameter is not a contiguous CUDA float32 tensor on ``x``'s device, or
    the shapes are not x (N, I), hidden_states (1, N, Hd) and masks (N, 1), or N > 65535."""
    if torch.is_grad_enabled() or not isinstance(x, torch.Tensor):
        return None
    rnn = getattr(module, "rnn", None)
    if gru_layout_error(rnn):
        return None
    dev = x.device
    if not all(_dense(t, dev) for t in (x, hidden_states, masks)):
        return None
    if not all(_dense(p, dev) for p in (rnn.weight_ih_l0, rnn.weight_hh_l0, rnn.bias_ih_l0, rnn.bias_hh_l0)):
        return None
    if x.ndim != 2:
        return None
    N = x.shape[0]
    if (N > 65535 or x.shape[1] != rnn.input_size or tuple(hidden_states.shape) != (1, N, rnn.hidden_size)
            or tuple(masks.shape) != (N, 1)):
        return None
    from .renderer import WaveformOps
    out, h = WaveformOps.get(dev).gru_step(x, hidden_states[0], masks, rnn)
    return out, h.unsqueeze(0)


def patch_rnn_state_encoder(cls):
    """Replace ``cls.single_forward`` of ``RNNStateEncoder`` in place, nothing else; the original stays reachable as
    ``cls.single_forward._ssb_original`` and patching twice changes nothing.  Qualifying calls
    (:func:`fused_single_forward`) run in the library, anything else runs the original."""
    original = getattr(cls.single_forward, "_ssb_original", cls.single_forward)

    def single_forward(self, x, hidden_states, masks):
        out = fused_single_forward(self, x, hidden_states, masks)
        return original(self, x, hidden_states, masks) if out is None else out

    single_forward._ssb_original = original
    single_forward.__doc__ = original.__doc__
    cls.single_forward = single_forward
    return cls
