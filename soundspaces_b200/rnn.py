"""The policy's state encoder: ``RNNStateEncoder.single_forward`` at rollout time and, on request, ``seq_forward`` and
its backward in PPO's update, of the reference's baselines (ss_baselines/av_nav/models/rnn_state_encoder.py:80-143;
av_wan and SAVi's ``AudioNavBaselineNet`` import the same class).

    from soundspaces_b200.rnn import patch_rnn_state_encoder
    patch_rnn_state_encoder(RNNStateEncoder)                  # single_forward only
    patch_rnn_state_encoder(RNNStateEncoder, sequence=True)   # single_forward and seq_forward

``single_forward`` runs ``ssb_gru_step_batch`` (one launch) instead of the mask multiply and a cuDNN GRU step, under
no-grad.  With ``sequence=True``, ``seq_forward`` runs ``ssb_gru_seq_forward_batch`` (two launches) with or without
grad, and its backward ``ssb_gru_seq_backward_batch`` (at most four launches), instead of the host-synchronising split
at done steps, one cuDNN call per segment and their backward.  The mask multiplies the carried state only at a
segment start (t = 0, or a step at which some env's mask is 0.0), as the reference's split does; the library finds
those steps on the device.  Both take a one-layer, unidirectional ``nn.GRU`` with bias (:func:`gru_layout_error`) on
contiguous CUDA float32 tensors (:func:`gru_seq_error` for the sequence); an LSTM (SAVi's DD-PPO ``resnet_policy.py``
default), a multi-layer GRU and everything else run the original.
"""
from __future__ import annotations

import torch
import torch.nn as nn
from torch.autograd.function import once_differentiable

MAX_STEPS = 4096        # ssb_gru_seq_*'s limits (include/ssb200.h)
MAX_ENVS = 256
MAX_HIDDEN = 1024


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


def _params(rnn):
    return rnn.weight_ih_l0, rnn.weight_hh_l0, rnn.bias_ih_l0, rnn.bias_hh_l0


def gru_seq_error(module, x, hidden_states, masks) -> str:
    """Why ``module.seq_forward(x, hidden_states, masks)`` does not run in the library; ``""`` when it does: a
    qualifying ``module.rnn`` (:func:`gru_layout_error`), x, hidden_states, masks and the GRU's parameters contiguous
    CUDA float32 tensors on x's device, x (T N, input_size) and hidden_states (1, N, hidden_size) with T >= 2, masks of
    T N values that do not require grad, T, N and hidden_size within the library's limits, autocast off."""
    rnn = getattr(module, "rnn", None)
    err = gru_layout_error(rnn)
    if err:
        return err
    if not isinstance(x, torch.Tensor):
        return "x is not a tensor"
    dev = x.device
    named = [("x", x), ("hidden_states", hidden_states), ("masks", masks)]
    named += list(zip(("weight_ih_l0", "weight_hh_l0", "bias_ih_l0", "bias_hh_l0"), _params(rnn)))
    for name, t in named:
        if not _dense(t, dev):
            return f"{name} is not a contiguous CUDA float32 tensor on {dev}"
    I, Hd = rnn.input_size, rnn.hidden_size
    if x.ndim != 2 or x.shape[1] != I:
        return f"x has shape {tuple(x.shape)}, expected (T * N, {I})"
    if hidden_states.ndim != 3 or hidden_states.shape[0] != 1 or hidden_states.shape[2] != Hd:
        return f"hidden_states has shape {tuple(hidden_states.shape)}, expected (1, N, {Hd})"
    N = hidden_states.shape[1]
    if N < 1 or x.shape[0] % N or x.shape[0] // N < 2:
        return f"x has {x.shape[0]} rows, not T * N for N={N} and some T >= 2"
    T = x.shape[0] // N
    if masks.numel() != T * N:
        return f"masks hold {masks.numel()} values, expected T * N = {T * N}"
    if T > MAX_STEPS or N > MAX_ENVS or Hd > MAX_HIDDEN:
        return (f"T={T}, N={N}, hidden_size={Hd}: the library takes T <= {MAX_STEPS}, N <= {MAX_ENVS} and "
                f"hidden_size <= {MAX_HIDDEN}")
    if masks.requires_grad:
        return "masks require grad"
    if torch.is_autocast_enabled("cuda"):
        return "autocast is on"
    return ""


class GruSeqFunction(torch.autograd.Function):
    """``(out, h_last) = seq_forward`` through the library, differentiable in x, h0 and the four GRU parameters (not
    in the masks); the backward computes only the gradients autograd asks for and is not itself differentiable.
    ``grad``: whether grad mode was on at the call (``needs_input_grad`` reflects only ``requires_grad``); without it
    nothing is saved for a backward."""

    @staticmethod
    def forward(ctx, grad, x, h0, masks, w_ih, w_hh, b_ih, b_hh):
        from .renderer import WaveformOps
        ops = WaveformOps.get(x.device)
        save = grad and any(ctx.needs_input_grad[1:])
        out, h_last, saved = ops.gru_seq_forward(x, h0, masks, (w_ih, w_hh, b_ih, b_hh), save=save)
        if save:
            ctx.save_for_backward(x, masks, w_ih, w_hh, saved)
            ctx.n_envs = h0.shape[1]
            ctx.set_materialize_grads(False)
        return out, h_last

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_out, grad_h_last):
        from .renderer import WaveformOps
        x, masks, w_ih, w_hh, saved = ctx.saved_tensors
        need = ctx.needs_input_grad
        grads = WaveformOps.get(x.device).gru_seq_backward(
            x, ctx.n_envs, masks, w_ih, w_hh, saved,
            None if grad_out is None else grad_out.contiguous(),
            None if grad_h_last is None else grad_h_last.contiguous(),
            need=(need[1], need[2], need[4], need[5], need[6], need[7]))
        dx, dh0, dw_ih, dw_hh, db_ih, db_hh = grads
        return None, dx, dh0, None, dw_ih, dw_hh, db_ih, db_hh


def fused_seq_forward(module, x, hidden_states, masks):
    """``module.seq_forward(x, hidden_states, masks)`` through the library -> ``(out (T N, Hd), h_last (1, N, Hd))``,
    or None (the caller runs the original) when :func:`gru_seq_error` gives a reason."""
    if gru_seq_error(module, x, hidden_states, masks):
        return None
    return GruSeqFunction.apply(torch.is_grad_enabled(), x, hidden_states, masks, *_params(module.rnn))


def patch_rnn_state_encoder(cls, sequence=False):
    """Replace ``cls.single_forward`` of ``RNNStateEncoder`` in place, and with ``sequence=True`` also
    ``cls.seq_forward``; nothing else.  The originals stay reachable as ``._ssb_original`` and patching again changes
    nothing (a ``sequence=True`` patch after a plain one adds ``seq_forward``).  Qualifying calls
    (:func:`fused_single_forward`, :func:`gru_seq_error`) run in the library, anything else runs the original."""
    original = getattr(cls.single_forward, "_ssb_original", cls.single_forward)

    def single_forward(self, x, hidden_states, masks):
        out = fused_single_forward(self, x, hidden_states, masks)
        return original(self, x, hidden_states, masks) if out is None else out

    single_forward._ssb_original = original
    single_forward.__doc__ = original.__doc__
    cls.single_forward = single_forward
    if sequence:
        seq_original = getattr(cls.seq_forward, "_ssb_original", cls.seq_forward)

        def seq_forward(self, x, hidden_states, masks):
            out = fused_seq_forward(self, x, hidden_states, masks)
            return seq_original(self, x, hidden_states, masks) if out is None else out

        seq_forward._ssb_original = seq_original
        seq_forward.__doc__ = seq_original.__doc__
        cls.seq_forward = seq_forward
    return cls
