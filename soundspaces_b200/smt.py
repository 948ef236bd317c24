"""SAVi's scene memory transformer at rollout time: ``SMTStateEncoder.single_forward``
(ss_baselines/savi/models/smt_state_encoder.py:92-157), called by ``AudioNavSMTNet.forward`` (savi/ppo/policy.py:380-403)
on every rollout step, in ``get_value`` and in eval, run by ``ssb_smt_state_encoder_batch`` (six launches) instead of
dozens of eager PyTorch ops over every allocated memory slot.

    from soundspaces_b200.smt import patch_smt_state_encoder
    patch_smt_state_encoder(SMTStateEncoder)     # ss_baselines.savi.models.smt_state_encoder

    patch_smt_state_encoder(SMTStateEncoder, training=True)   # PPO's update too (:class:`SmtFunction`)

The module is recognised by structure (:func:`smt_layout_error`), never by class name.  Anything that does not qualify
(grad enabled without ``training=True``, CPU or non-float32 tensors, other topologies, shapes past the library's
limits) runs the original ``single_forward``.  The library computes on valid tokens only and never reads a masked slot's memory row; the
reference multiplies a masked slot's zero attention weight by its values, so a NaN or Inf there reaches its output but
not the library's.
"""
from __future__ import annotations

import torch
import torch.nn as nn
import torch.nn.functional as F

from torch.autograd.function import once_differentiable

from . import _lib

MAX_ENVS = 1024        # SMT_MAX_ENVS of ssb200.cu
MAX_TOKENS = 1024      # M + 1
MAX_D_MODEL = 512
MAX_HEAD_DIM = 128
MAX_D_IN = 1024
MAX_TRAIN_ENVS = 65535  # SMT_MAX_TRAIN_ENVS: rows per ssb_smt_state_encoder_train_* call


def _linear_error(m, i, o, where):
    if not isinstance(m, nn.Linear):
        return f"{where} is {type(m).__name__}, expected Linear"
    if (m.in_features, m.out_features) != (i, o) or m.bias is None:
        return f"{where} is Linear({m.in_features}, {m.out_features}, bias={m.bias is not None}), expected Linear({i}, {o})"
    return ""


def _norm_error(m, d, where):
    if type(m) is not nn.LayerNorm:
        return f"{where} is {type(m).__name__}, expected LayerNorm"
    if tuple(m.normalized_shape) != (d,) or not m.elementwise_affine or m.weight is None or m.bias is None:
        return f"{where}: expected an affine LayerNorm({d}) with a bias"
    if not m.eps > 0:
        return f"{where}: eps must be positive"
    return ""


def _mha_error(m, d, nhead, where):
    if type(m) is not nn.MultiheadAttention:
        return f"{where} is {type(m).__name__}, expected MultiheadAttention"
    if m.embed_dim != d or m.num_heads != nhead or not m._qkv_same_embed_dim or m.in_proj_weight is None:
        return f"{where}: expected MultiheadAttention({d}, {nhead}) with one in_proj"
    if m.in_proj_bias is None or m.out_proj.bias is None:
        return f"{where}: expected biased projections"
    if m.bias_k is not None or m.bias_v is not None or m.add_zero_attn:
        return f"{where}: add_bias_kv / add_zero_attn are not supported"
    if m.batch_first:
        return f"{where}: batch_first is not supported"
    return _linear_error(m.out_proj, d, d, f"{where}.out_proj")


def _is_relu(act):
    return act is F.relu or type(act) is nn.ReLU


def _layer_error(layer, d, nhead, decoder, where):
    if getattr(layer, "norm_first", None) is not False:
        return f"{where}: expected post-norm (norm_first=False)"
    if not _is_relu(getattr(layer, "activation", None)):
        return f"{where}: expected a ReLU activation"
    err = _mha_error(layer.self_attn, d, nhead, f"{where}.self_attn")
    if not err and decoder:
        err = _mha_error(layer.multihead_attn, d, nhead, f"{where}.multihead_attn")
    err = err or _linear_error(layer.linear1, d, d, f"{where}.linear1") or _linear_error(layer.linear2, d, d, f"{where}.linear2")
    for n in ("norm1", "norm2") + (("norm3",) if decoder else ()):
        err = err or _norm_error(getattr(layer, n, None), d, f"{where}.{n}")
    return err


def _dropouts(module):
    ps = [m.p for m in module.modules() if isinstance(m, nn.Dropout)]
    return ps + [m.dropout for m in module.modules() if isinstance(m, nn.MultiheadAttention)]


def smt_parameters(module):
    """The tensors the library reads, in ``ssb_smt_params`` order (pose_encoder's first when it has one)."""
    tr = module.transformer
    enc, dec = tr.encoder.layers[0], tr.decoder.layers[0]
    lins = [module.fusion_encoder[0], module.fusion_encoder[2], enc.linear1, enc.linear2, enc.self_attn.out_proj,
            dec.self_attn.out_proj, dec.multihead_attn.out_proj, dec.linear1, dec.linear2]
    if getattr(module, "_use_pose_encoding", False):
        lins.insert(0, module.pose_encoder)
    norms = [enc.norm1, enc.norm2, tr.encoder.norm, dec.norm1, dec.norm2, dec.norm3, tr.decoder.norm]
    ts = [t for m in lins for t in (m.weight, m.bias)] + [t for m in norms for t in (m.weight, m.bias)]
    for mha in (enc.self_attn, dec.self_attn, dec.multihead_attn):
        ts += [mha.in_proj_weight, mha.in_proj_bias]
    return ts


def smt_layout_error(module, device=None) -> str:
    """Why ``module`` is not an ``SMTStateEncoder`` with one encoder and one decoder layer the library runs, with
    contiguous float32 parameters on ``device`` (not checked when None); ``""`` when it is.  Dropout must be 0 unless
    the module is in eval mode."""
    if not isinstance(module, nn.Module):
        return "not a module"
    tr = getattr(module, "transformer", None)
    fusion = getattr(module, "fusion_encoder", None)
    if type(tr) is not nn.Transformer:
        return "transformer is not an nn.Transformer"
    if getattr(tr, "batch_first", False):
        return "transformer: batch_first is not supported"
    enc, dec = tr.encoder, tr.decoder
    if len(enc.layers) != 1 or len(dec.layers) != 1:
        return f"expected 1 encoder and 1 decoder layer, got {len(enc.layers)} and {len(dec.layers)}"
    d = tr.d_model
    nhead = tr.nhead
    if d % nhead:
        return f"d_model {d} is not a multiple of nhead {nhead}"
    err = (_layer_error(enc.layers[0], d, nhead, False, "transformer.encoder.layers.0")
           or _layer_error(dec.layers[0], d, nhead, True, "transformer.decoder.layers.0")
           or _norm_error(enc.norm, d, "transformer.encoder.norm") or _norm_error(dec.norm, d, "transformer.decoder.norm"))
    if err:
        return err
    if type(fusion) is not nn.Sequential or len(fusion) != 3 or type(fusion[1]) is not nn.ReLU:
        return "fusion_encoder must be Sequential(Linear, ReLU, Linear)"
    use_pose = bool(getattr(module, "_use_pose_encoding", False))
    if use_pose:
        idx = getattr(module, "_pose_indices", None)
        if not idx or not isinstance(idx[0], int) or idx[0] < 0:
            return "_pose_indices must start at a non-negative int"
        err = _linear_error(getattr(module, "pose_encoder", None), 5, 16, "pose_encoder")
        width = idx[0] + 16
    else:
        width = fusion[0].in_features if isinstance(fusion[0], nn.Linear) else -1
    err = err or _linear_error(fusion[0], width, d, "fusion_encoder.0") or _linear_error(fusion[2], d, d, "fusion_encoder.2")
    if err:
        return err
    if not isinstance(getattr(module, "_pretraining", False), bool):
        return "_pretraining must be a bool"
    if module.training and any(p != 0 for p in _dropouts(module)):
        return "dropout > 0 in training mode"
    if device is not None:
        for t in smt_parameters(module):
            if t.device != device or t.dtype != torch.float32 or not t.is_contiguous():
                return f"parameters must be contiguous float32 tensors on {device}"
    return ""


def smt_params(module, d_in: int):
    """The ``ssb_smt_params`` of ``module`` for tokens of width ``d_in`` (pointers of the live parameters)."""
    tr = module.transformer
    enc, dec = tr.encoder.layers[0], tr.decoder.layers[0]

    def lin(m):
        return _lib.Linear(m.weight.data_ptr(), m.bias.data_ptr())

    def qkv(m):
        return _lib.Linear(m.in_proj_weight.data_ptr(), m.in_proj_bias.data_ptr())

    def ln(m):
        return _lib.LayerNorm(m.weight.data_ptr(), m.bias.data_ptr(), float(m.eps), 0)

    use_pose = bool(getattr(module, "_use_pose_encoding", False))
    return _lib.SmtParams(
        d_in, module._pose_indices[0] if use_pose else -1, tr.d_model, tr.nhead, int(bool(module._pretraining)),
        lin(module.pose_encoder) if use_pose else _lib.Linear(), lin(module.fusion_encoder[0]),
        lin(module.fusion_encoder[2]), qkv(enc.self_attn), lin(enc.self_attn.out_proj), lin(enc.linear1),
        lin(enc.linear2), ln(enc.norm1), ln(enc.norm2), ln(tr.encoder.norm), qkv(dec.self_attn),
        lin(dec.self_attn.out_proj), qkv(dec.multihead_attn), lin(dec.multihead_attn.out_proj), lin(dec.linear1),
        lin(dec.linear2), ln(dec.norm1), ln(dec.norm2), ln(dec.norm3), ln(tr.decoder.norm))


def _dense(t, device) -> bool:
    return isinstance(t, torch.Tensor) and t.is_cuda and t.device == device and t.dtype == torch.float32 and t.is_contiguous()


def fused_single_forward(module, x, memory, memory_masks, goal=None):
    """``module.single_forward(x, memory, memory_masks, goal)`` through the library -> (N, d_model), or None (the
    caller runs the original) when grad is enabled, a tensor is not a contiguous CUDA float32 tensor on ``x``'s
    device, the shapes disagree (x (N, D), memory (M, N, D), memory_masks (N, M), goal (N, d_model)), a limit is
    exceeded (N <= 1024, M + 1 <= 1024, d_model <= 512, head dim <= 128, D <= 1024, pose index + 4 <= D with pose
    encoding; without it D is fusion_encoder[0]'s input width) or the module
    does not qualify (:func:`smt_layout_error`)."""
    if torch.is_grad_enabled() or not isinstance(x, torch.Tensor):
        return None
    dev = x.device
    if not all(_dense(t, dev) for t in (x, memory, memory_masks)) or (goal is not None and not _dense(goal, dev)):
        return None
    if x.ndim != 2 or memory.ndim != 3 or memory_masks.ndim != 2:
        return None
    N, D = x.shape
    M = memory.shape[0]
    if tuple(memory.shape[1:]) != (N, D) or tuple(memory_masks.shape) != (N, M):
        return None
    tr = getattr(module, "transformer", None)
    d = getattr(tr, "d_model", None)
    if goal is not None and (goal.ndim != 2 or tuple(goal.shape) != (N, d)):
        return None
    if not isinstance(d, int) or N > MAX_ENVS or M + 1 > MAX_TOKENS or D > MAX_D_IN or d > MAX_D_MODEL:
        return None
    if smt_layout_error(module, dev) or d // tr.nhead > MAX_HEAD_DIM:
        return None
    if getattr(module, "_use_pose_encoding", False) and module._pose_indices[0] + 4 > D:
        return None
    if not getattr(module, "_use_pose_encoding", False) and module.fusion_encoder[0].in_features != D:
        return None
    from .renderer import WaveformOps
    return WaveformOps.get(dev).smt_state_encoder(module, x, memory, memory_masks, goal)


def smt_train_parameters(module):
    """The parameters :class:`SmtFunction` takes, in ``ssb_smt_params`` order: pose_encoder's weight and bias first
    when it has one, then fusion_encoder, the encoder layer's in_proj, out_proj, linear1, linear2, its norms and
    encoder.norm, the decoder layer's self-attention and cross-attention in_proj / out_proj, linear1, linear2, its
    norms and decoder.norm (40 tensors with pose encoding, 38 without)."""
    tr = module.transformer
    enc, dec = tr.encoder.layers[0], tr.decoder.layers[0]
    mods = [module.fusion_encoder[0], module.fusion_encoder[2]]
    if getattr(module, "_use_pose_encoding", False):
        mods.insert(0, module.pose_encoder)
    ts = [t for m in mods for t in (m.weight, m.bias)]
    ts += [enc.self_attn.in_proj_weight, enc.self_attn.in_proj_bias]
    for m in (enc.self_attn.out_proj, enc.linear1, enc.linear2, enc.norm1, enc.norm2, tr.encoder.norm):
        ts += [m.weight, m.bias]
    for mha in (dec.self_attn, dec.multihead_attn):
        ts += [mha.in_proj_weight, mha.in_proj_bias, mha.out_proj.weight, mha.out_proj.bias]
    for m in (dec.linear1, dec.linear2, dec.norm1, dec.norm2, dec.norm3, tr.decoder.norm):
        ts += [m.weight, m.bias]
    return ts


def smt_train_error(module, x, memory, masks, goal) -> str:
    """Why ``module.single_forward(x, memory, masks, goal)`` under grad mode does not run through
    :class:`SmtFunction`; ``""`` when it does.  It does when autocast is off; the module qualifies
    (:func:`smt_layout_error`, parameters contiguous float32 on x's device); x (N, D), memory (M, N, D), masks (N, M)
    and goal (N, d_model) or None are contiguous CUDA float32 tensors on one device; memory and masks do not require
    grad; and 1 <= N <= 65535, M + 1 <= 1024, d_model <= 512, head dim <= 128, D <= 1024, with pose encoding pose
    index + 4 <= D and without it D = fusion_encoder[0]'s input width."""
    if torch.is_autocast_enabled("cuda"):
        return "autocast is on"
    err = smt_layout_error(module)
    if err:
        return err
    for name, t in (("x", x), ("memory", memory), ("masks", masks), ("goal", goal)):
        if t is None and name == "goal":
            continue
        if not (isinstance(t, torch.Tensor) and t.is_cuda):
            return f"{name} is not a CUDA tensor"
        if t.dtype != torch.float32 or not t.is_contiguous():
            return f"{name} is not a contiguous float32 tensor"
        if t.device != x.device:
            return f"{name} is not on {x.device}"
    if memory.requires_grad or masks.requires_grad:
        return "memory or masks require grad"
    tr = module.transformer
    d = tr.d_model
    if x.ndim != 2 or memory.ndim != 3 or masks.ndim != 2:
        return "x, memory and masks must be 2-d, 3-d and 2-d"
    N, D = x.shape
    M = memory.shape[0]
    if tuple(memory.shape[1:]) != (N, D) or tuple(masks.shape) != (N, M) or (
            goal is not None and tuple(goal.shape) != (N, d)):
        return (f"shapes x {tuple(x.shape)}, memory {tuple(memory.shape)}, masks {tuple(masks.shape)}, goal "
                f"{None if goal is None else tuple(goal.shape)} disagree")
    if not 1 <= N <= MAX_TRAIN_ENVS:
        return f"{N} rows, outside 1..{MAX_TRAIN_ENVS}"
    if M + 1 > MAX_TOKENS or D > MAX_D_IN or d > MAX_D_MODEL or d // tr.nhead > MAX_HEAD_DIM:
        return (f"M + 1 = {M + 1}, D = {D}, d_model = {d} or head dim {d // tr.nhead} past the limits "
                f"({MAX_TOKENS}, {MAX_D_IN}, {MAX_D_MODEL}, {MAX_HEAD_DIM})")
    if getattr(module, "_use_pose_encoding", False):
        if module._pose_indices[0] + 4 > D:
            return f"pose index {module._pose_indices[0]} + 4 > D = {D}"
    elif module.fusion_encoder[0].in_features != D:
        return f"x has {D} columns, fusion_encoder.0 takes {module.fusion_encoder[0].in_features}"
    if smt_layout_error(module, x.device):
        return f"the parameters are not contiguous float32 tensors on {x.device}"
    return ""


class SmtFunction(torch.autograd.Function):
    """``module.single_forward(x, memory, masks, goal)`` through the library, differentiable in x, goal and every
    parameter (:func:`smt_train_parameters`), each an input of the function so that autograd (and DDP's
    unused-parameter search) sees them; not in memory or masks.  The backward computes only the gradients autograd
    asks for and is not itself differentiable.  ``grad``: whether grad mode was on at the call; without it, or when no
    input requires grad, nothing is saved for a backward."""

    @staticmethod
    def forward(ctx, grad, module, x, memory, masks, goal, *params):
        from .renderer import WaveformOps
        ops = WaveformOps.get(x.device)
        out, ws = ops.smt_train_forward(module, x, memory, masks, goal)
        needs = ctx.needs_input_grad
        if grad and (needs[2] or needs[5] or any(needs[6:])):
            ctx.save_for_backward(x, memory, masks, goal, ws, *params)
            ctx.module = module
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_out):
        from .renderer import WaveformOps
        x, memory, masks, goal, ws = ctx.saved_tensors[:5]
        needs = ctx.needs_input_grad
        ops = WaveformOps.get(ws.device)
        *grads, dx, dgoal = ops.smt_train_backward(ctx.module, x, memory, masks, goal, ws, grad_out,
                                                   need=tuple(needs[6:]) + (needs[2], needs[5]))
        return (None, None, dx, None, None, dgoal) + tuple(grads)


def patch_smt_state_encoder(cls, training: bool = False):
    """Replace ``cls.single_forward`` of SAVi's ``SMTStateEncoder`` in place, nothing else; the original stays
    reachable as ``cls.single_forward._ssb_original`` and patching twice changes nothing.  Qualifying calls
    (:func:`fused_single_forward`) run in the library, anything else runs the original.  ``training=True`` also runs
    grad-mode calls (PPO's ``evaluate_actions``) in the library through :class:`SmtFunction` when
    :func:`smt_train_error` allows; without it they run the original."""
    original = getattr(cls.single_forward, "_ssb_original", cls.single_forward)

    def single_forward(self, x, memory, memory_masks, goal=None):
        if training and torch.is_grad_enabled():
            if smt_train_error(self, x, memory, memory_masks, goal):
                return original(self, x, memory, memory_masks, goal)
            return SmtFunction.apply(True, self, x, memory, memory_masks, goal, *smt_train_parameters(self))
        out = fused_single_forward(self, x, memory, memory_masks, goal)
        return original(self, x, memory, memory_masks, goal) if out is None else out

    single_forward._ssb_original = original
    single_forward.__doc__ = original.__doc__
    cls.single_forward = single_forward
    return cls
