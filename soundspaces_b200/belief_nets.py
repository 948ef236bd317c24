"""The two ResNet-18 topologies of SAVi's ``BeliefPredictor`` (ss_baselines/savi/models/belief_predictor.py:65-80),
recognised by structure and packed into the parameter table of ``ssb_resnet18_batch`` / ``ssb_smt_resnet18_batch``.

- torchvision ``resnet18`` with ``conv1 = Conv2d(2, 64, 7, 2, 3, bias=False)`` and any ``fc = Linear(512, n)``:
  the label classifier and the location predictor without online training.  BatchNorm in eval mode.
- ``custom_resnet18`` (savi/models/smt_resnet.py) with ``fc = Linear(128 H4 W4, n)``: the location predictor with
  online training.  7x7 stride-1 stem to 16 channels, stages of widths 16/32/64/128, every norm ``GroupNorm(16, C)``,
  no pooling.

The checks look at module types, attribute names, convolution geometry and widths only, never at class names (the
reference's ``CustomResNet`` need not be importable).  Parameters must be contiguous float32 tensors on the
observation's device.
"""
from __future__ import annotations

import ctypes as C

import torch
import torch.nn as nn
from torch.autograd.function import once_differentiable

from . import _lib

TV_WIDTHS = (64, 128, 256, 512)
SMT_WIDTHS = (16, 32, 64, 128)
N_CONVS = 20          # stem + 8 blocks x 2 + 3 downsample convs
SMT_GROUPS = 16
MAX_ENVS = 1024       # RN_MAX_ENVS of ssb200.cu: both entries refuse larger batches
MAX_HW = 256          # RN_MAX_HW: and observations taller or wider than this


def _names_error(m, names, where):
    got = [n for n, _ in m.named_children()]
    return "" if got == list(names) else f"{where} has modules {got}, expected {list(names)}"


def _conv_error(c, ic, oc, k, s, p, where):
    if type(c) is not nn.Conv2d:
        return f"{where} is {type(c).__name__}, expected Conv2d"
    if (c.in_channels, c.out_channels) != (ic, oc):
        return f"{where} is Conv2d({c.in_channels}, {c.out_channels}), expected Conv2d({ic}, {oc})"
    if (tuple(c.kernel_size) != (k, k) or tuple(c.stride) != (s, s) or not isinstance(c.padding, tuple)
            or tuple(c.padding) != (p, p) or tuple(c.dilation) != (1, 1) or c.groups != 1 or c.padding_mode != "zeros"
            or c.bias is not None):
        return f"{where}: expected kernel {k}, stride {s}, padding {p}, no dilation, groups or bias"
    return ""


def _norm_error(m, ch, bn, where, training=False):
    if bn:
        if type(m) is not nn.BatchNorm2d:
            return f"{where} is {type(m).__name__}, expected BatchNorm2d"
        if m.num_features != ch or not m.affine or not m.track_running_stats or m.running_mean is None:
            return f"{where}: expected an affine BatchNorm2d({ch}) with running statistics"
        if m.training and not training:
            return f"{where} is in training mode"
    else:
        if type(m) is not nn.GroupNorm:
            return f"{where} is {type(m).__name__}, expected GroupNorm"
        if m.num_groups != SMT_GROUPS or m.num_channels != ch or not m.affine:
            return f"{where}: expected an affine GroupNorm({SMT_GROUPS}, {ch})"
    if not m.eps > 0:
        return f"{where}: eps must be positive"
    return ""


def _layers_error(net, widths, bn, training=False):
    """layer1..layer4: two blocks each, conv1 norm1 relu conv2 norm2 [downsample = Sequential(1x1 conv, norm)]."""
    ic = widths[0]
    for s, oc in enumerate(widths):
        layer = getattr(net, f"layer{s + 1}")
        where = f"layer{s + 1}"
        if type(layer) is not nn.Sequential or len(layer) != 2:
            return f"{where} must be a Sequential of 2 blocks"
        for j, blk in enumerate(layer):
            w = f"{where}.{j}"
            stride = 2 if s > 0 and j == 0 else 1
            ds = stride == 2
            err = _names_error(blk, ("conv1", "bn1", "relu", "conv2", "bn2") + (("downsample",) if ds else ()), w)
            err = err or ("" if type(blk.relu) is nn.ReLU else f"{w}.relu is {type(blk.relu).__name__}")
            err = (err or _conv_error(blk.conv1, ic, oc, 3, stride, 1, f"{w}.conv1")
                   or _norm_error(blk.bn1, oc, bn, f"{w}.bn1", training)
                   or _conv_error(blk.conv2, oc, oc, 3, 1, 1, f"{w}.conv2")
                   or _norm_error(blk.bn2, oc, bn, f"{w}.bn2", training))
            if not err and ds:
                d = blk.downsample
                err = ("" if type(d) is nn.Sequential and len(d) == 2 else f"{w}.downsample must be Sequential(conv, norm)")
                err = (err or _conv_error(d[0], ic, oc, 1, 2, 0, f"{w}.downsample.0")
                       or _norm_error(d[1], oc, bn, f"{w}.downsample.1", training))
            if err:
                return err
            ic = oc
    return ""


def _linear_error(fc, in_features):
    if type(fc) is not nn.Linear:
        return f"fc is {type(fc).__name__}, expected Linear"
    if fc.in_features != in_features:
        return f"fc takes {fc.in_features} features, expected {in_features}"
    return ""


def conv_norm_pairs(net):
    """The 20 (conv, norm) pairs in the documented order: conv1/bn1, then per block conv1/bn1, conv2/bn2 and, in the
    first block of layer2..layer4, downsample.0/downsample.1."""
    pairs = [(net.conv1, net.bn1)]
    for s in range(4):
        for blk in getattr(net, f"layer{s + 1}"):
            pairs += [(blk.conv1, blk.bn1), (blk.conv2, blk.bn2)]
            if "downsample" in blk._modules and blk.downsample is not None:
                pairs.append((blk.downsample[0], blk.downsample[1]))
    return pairs


def _tensor_error(net, device, bn):
    tensors = [net.fc.weight] + ([net.fc.bias] if net.fc.bias is not None else [])
    for conv, norm in conv_norm_pairs(net):
        tensors += [conv.weight, norm.weight, norm.bias] + ([norm.running_mean, norm.running_var] if bn else [])
    for t in tensors:
        if t.device != device or t.dtype != torch.float32 or not t.is_contiguous():
            return f"parameters must be contiguous float32 tensors on {device}"
    return ""


def resnet18_layout_error(net, device=None, training=False) -> str:
    """Why ``net`` is not torchvision's resnet18 with a 2-channel ``Conv2d(2, 64, 7, 2, 3, bias=False)`` stem, eval-mode
    BatchNorm (either mode with ``training``) and ``fc = Linear(512, n)`` whose parameters live on ``device`` (not
    checked when None); ``""`` when it is."""
    if not isinstance(net, nn.Module):
        return "not a module"
    err = _names_error(net, ("conv1", "bn1", "relu", "maxpool", "layer1", "layer2", "layer3", "layer4", "avgpool", "fc"),
                       "the network")
    if err:
        return err
    mp, ap = net.maxpool, net.avgpool
    if type(net.relu) is not nn.ReLU:
        return f"relu is {type(net.relu).__name__}"
    if (type(mp) is not nn.MaxPool2d or mp.kernel_size not in (3, (3, 3)) or mp.stride not in (2, (2, 2))
            or mp.padding not in (1, (1, 1)) or mp.dilation not in (1, (1, 1)) or mp.ceil_mode):
        return "maxpool must be MaxPool2d(3, 2, 1)"
    if type(ap) is not nn.AdaptiveAvgPool2d or ap.output_size not in (1, (1, 1)):
        return "avgpool must be AdaptiveAvgPool2d((1, 1))"
    err = (_conv_error(net.conv1, 2, 64, 7, 2, 3, "conv1") or _norm_error(net.bn1, 64, True, "bn1", training)
           or _layers_error(net, TV_WIDTHS, True, training) or _linear_error(net.fc, TV_WIDTHS[-1]))
    if err or device is None:
        return err
    return _tensor_error(net, device, True)


def smt_out_hw(H: int, W: int):
    """Spatial size after the SMT network's three stride-2 stages: (9, 4) for the 65 x 26 observation."""
    for _ in range(3):
        H, W = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    return H, W


def smt_resnet18_layout_error(net, in_channels: int, hw=None, device=None) -> str:
    """Why ``net`` is not the SMT ``custom_resnet18`` with ``in_channels`` input channels (2, or 23 with the category
    channels), GroupNorm(16, C) everywhere and an ``fc`` that takes the flattened ``(128, H4, W4)`` activation of an
    ``hw = (H, W)`` observation (not checked when None), whose parameters live on ``device``; ``""`` when it is."""
    if not isinstance(net, nn.Module):
        return "not a module"
    err = _names_error(net, ("conv1", "bn1", "relu", "layer1", "layer2", "layer3", "layer4", "fc"), "the network")
    if err:
        return err
    if type(net.relu) is not nn.ReLU:
        return f"relu is {type(net.relu).__name__}"
    err = (_conv_error(net.conv1, in_channels, 16, 7, 1, 3, "conv1") or _norm_error(net.bn1, 16, False, "bn1")
           or _layers_error(net, SMT_WIDTHS, False))
    if not err and type(net.fc) is not nn.Linear:
        err = f"fc is {type(net.fc).__name__}, expected Linear"
    if not err and hw is not None:
        h4, w4 = smt_out_hw(*hw)
        err = _linear_error(net.fc, SMT_WIDTHS[-1] * h4 * w4)
    if err or device is None:
        return err
    return _tensor_error(net, device, False)


def conv_table(net, bn: bool):
    """The host array of 20 ``ssb_resnet_conv`` for ``net`` (pointers of the live parameters, read at call time)."""
    table = (_lib.ResnetConv * N_CONVS)()
    for i, (conv, norm) in enumerate(conv_norm_pairs(net)):
        table[i] = _lib.ResnetConv(conv.weight.data_ptr(), norm.weight.data_ptr(), norm.bias.data_ptr(),
                                   norm.running_mean.data_ptr() if bn else None,
                                   norm.running_var.data_ptr() if bn else None, float(norm.eps), 0)
    return table


def fusable_observation(x) -> bool:
    return (isinstance(x, torch.Tensor) and x.is_cuda and x.dtype == torch.float32 and x.ndim == 4
            and x.shape[3] == 2 and x.is_contiguous())


def fusable_labels(labels, x, n: int) -> bool:
    """SAVi's ``(B, n)`` category observation as the SMT kernels read it: float32 on ``x``'s device, unit column
    stride, row stride >= n."""
    return (isinstance(labels, torch.Tensor) and labels.device == x.device and labels.dtype == torch.float32
            and labels.ndim == 2 and labels.shape == (x.shape[0], n) and labels.stride(1) == 1
            and (labels.shape[0] <= 1 or labels.stride(0) >= n))


def fused_forward(net, x, labels=None):
    """``net(input)`` through the library for a qualifying network, or None: ``input`` is ``x.permute(0, 3, 1, 2)``,
    with ``labels`` broadcast over the pixels and concatenated after the two ears when given.  None (the caller runs
    the module) when grad is enabled, ``x`` is not a contiguous CUDA float32 ``(B, H, W, 2)`` observation, B exceeds
    ``MAX_ENVS``, H or W exceeds ``MAX_HW``, or ``net`` / its parameters / ``labels`` do not qualify."""
    if torch.is_grad_enabled() or not fusable_observation(x):
        return None
    if x.shape[0] > MAX_ENVS or max(x.shape[1], x.shape[2]) > MAX_HW:
        return None
    from .renderer import WaveformOps
    if labels is None and not resnet18_layout_error(net, x.device):
        return WaveformOps.get(x.device).resnet18(x, net)
    n = 0 if labels is None else (labels.shape[1] if isinstance(labels, torch.Tensor) and labels.ndim == 2 else -1)
    if n < 0 or (n and not fusable_labels(labels, x, n)):
        return None
    if smt_resnet18_layout_error(net, 2 + n, tuple(x.shape[1:3]), x.device):
        return None
    return WaveformOps.get(x.device).smt_resnet18(x, net, labels)


# ---------------------------------------------------------------------------
# Online training of the SMT location predictor (ppo_trainer.py:342-400, train_belief_predictor): cnn_forward through
# ssb_smt_resnet18_train_forward_batch, differentiable in every predictor parameter.
# ---------------------------------------------------------------------------
TRAIN_MAX_ENVS = 65535    # SRN_MAX_ENVS of ssb200.cu


def smt_resnet18_params(net):
    """The 62 parameters the train entries take, in their order: the 20 conv weights, the 20 GroupNorm weights
    (gamma), the 20 GroupNorm biases (beta), fc.weight and fc.bias (None without a bias)."""
    pairs = conv_norm_pairs(net)
    return ([c.weight for c, _ in pairs] + [n.weight for _, n in pairs] + [n.bias for _, n in pairs]
            + [net.fc.weight, net.fc.bias])


def _train_labels(model, observations):
    """SAVi's category observation when the model reads it (``has_distractor_sound``), else None."""
    return observations.get("category") if getattr(model, "has_distractor_sound", False) else None


def _train_spectrogram_error(x) -> str:
    """Why ``x`` is not a spectrogram the train entries take (autocast off, a contiguous CUDA float32 (B, H, W, 2)
    tensor that does not require grad, 1 <= B <= 65535, H, W <= 256); ``""`` when it is."""
    if torch.is_autocast_enabled("cuda"):
        return "autocast is on"
    if not isinstance(x, torch.Tensor) or not x.is_cuda:
        return "the spectrogram is not a CUDA tensor"
    if x.dtype != torch.float32:
        return "the spectrogram is not float32"
    if x.ndim != 4 or x.shape[3] != 2:
        return "the spectrogram is not a (B, H, W, 2) tensor"
    if not x.is_contiguous():
        return "the spectrogram is not contiguous"
    if x.requires_grad:
        return "the spectrogram requires grad"
    if not 1 <= x.shape[0] <= TRAIN_MAX_ENVS:
        return f"{x.shape[0]} rows, outside 1..{TRAIN_MAX_ENVS}"
    if max(x.shape[1], x.shape[2]) > MAX_HW:
        return f"a {x.shape[1]}x{x.shape[2]} spectrogram exceeds {MAX_HW}x{MAX_HW}"
    return ""


def smt_resnet18_train_error(model, observations) -> str:
    """Why ``model.cnn_forward(observations)`` (SAVi's BeliefPredictor) does not run through
    :class:`SmtResNetFunction`; ``""`` when it does.  It does when autocast is off; ``model.predictor`` is the SMT
    ``custom_resnet18`` (:func:`smt_resnet18_layout_error`; not the torchvision predictor of a model without online
    training) for 2 input channels, or 2 + L with ``has_distractor_sound``; ``observations["spectrogram"]`` is a
    contiguous CUDA float32 (B, H, W, 2) tensor with 1 <= B <= 65535 and H, W <= 256; with ``has_distractor_sound``,
    ``observations["category"]`` is a CUDA float32 (B, L) tensor with unit column stride on that device; neither
    requires grad; and every predictor parameter is a contiguous CUDA float32 tensor on that device."""
    obs = observations if isinstance(observations, dict) else {}
    x = obs.get("spectrogram")
    err = _train_spectrogram_error(x)
    if err:
        return err
    labels = _train_labels(model, obs)
    n = 0
    if getattr(model, "has_distractor_sound", False):
        if not isinstance(labels, torch.Tensor) or labels.ndim != 2:
            return "has_distractor_sound without a (B, L) category tensor"
        if labels.requires_grad:
            return "the category requires grad"
        if not fusable_labels(labels, x, labels.shape[1]):
            return f"the category is not a float32 ({x.shape[0]}, L) tensor on {x.device} with unit column stride"
        n = labels.shape[1]
    net = getattr(model, "predictor", None)
    err = smt_resnet18_layout_error(net, 2 + n, tuple(x.shape[1:3]))
    if err:
        return "the predictor is not the SMT custom_resnet18: " + err
    if _tensor_error(net, x.device, False):
        return f"the predictor's parameters are not contiguous float32 tensors on {x.device}"
    return ""


class SmtResNetFunction(torch.autograd.Function):
    """The SMT location predictor on ``x.permute(0, 3, 1, 2)`` (with ``labels`` broadcast over the pixels and
    concatenated after the two ears when given) through the library, differentiable in all 62 predictor parameters,
    each an input of the function so that autograd (and DDP's unused-parameter search) sees them; not in ``x`` or
    ``labels``.  The backward computes only the gradients autograd asks for and is not itself differentiable.
    ``grad``: whether grad mode was on at the call; without it, or when no parameter requires grad (a frozen
    predictor), nothing is saved for a backward."""

    @staticmethod
    def forward(ctx, grad, eps, x, labels, *params):
        from .renderer import WaveformOps
        ops = WaveformOps.get(x.device)
        out, ws = ops.smt_resnet18_train_forward(x, labels, params, eps)
        if grad and any(ctx.needs_input_grad[4:]):
            ctx.save_for_backward(x, labels, ws, *params)
            ctx.eps = eps
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_out):
        from .renderer import WaveformOps
        x, labels, ws, *params = ctx.saved_tensors
        ops = WaveformOps.get(x.device)
        grads = ops.smt_resnet18_train_backward(x, labels, params, ctx.eps, ws, grad_out.contiguous(),
                                                need=ctx.needs_input_grad[4:])
        return (None,) * 4 + tuple(grads)


def smt_resnet18_train_forward(model, observations):
    """``model.cnn_forward(observations)`` through :class:`SmtResNetFunction`; the caller has checked
    :func:`smt_resnet18_train_error`."""
    net = model.predictor
    eps = tuple(float(n.eps) for _, n in conv_norm_pairs(net))
    return SmtResNetFunction.apply(torch.is_grad_enabled(), eps, observations["spectrogram"],
                                   _train_labels(model, observations), *smt_resnet18_params(net))


# ---------------------------------------------------------------------------
# Training of SAVi's audio-goal predictor (pretraining/audiogoal_trainer.py:69-124): torchvision's resnet18 through
# ssb_resnet18_train_forward_batch, BatchNorm in training or eval mode, differentiable in every parameter.
# ---------------------------------------------------------------------------
def resnet18_params(net):
    """The 62 parameters ``ssb_resnet18_train_*`` take, in :func:`smt_resnet18_params`' order: the 20 conv weights,
    the 20 BatchNorm weights (gamma), the 20 BatchNorm biases (beta), fc.weight and fc.bias (None without a bias)."""
    return smt_resnet18_params(net)


def resnet18_buffers(net):
    """The 20 running means, the 20 running variances and the 20 ``num_batches_tracked`` counters, in
    :func:`conv_norm_pairs` order."""
    norms = [n for _, n in conv_norm_pairs(net)]
    return ([n.running_mean for n in norms] + [n.running_var for n in norms]
            + [n.num_batches_tracked for n in norms])


def tv_norm_shapes(B: int, H: int, W: int):
    """The input size of each of the 20 BatchNorms of the torchvision ResNet-18 on a (B, 2, H, W) input, in
    :func:`conv_norm_pairs` order."""
    h, w = (H - 1) // 2 + 1, (W - 1) // 2 + 1                     # conv1, stride 2
    shapes = [(B, TV_WIDTHS[0], h, w)]
    h, w = (h - 1) // 2 + 1, (w - 1) // 2 + 1                     # MaxPool2d(3, 2, 1)
    for s, c in enumerate(TV_WIDTHS):
        if s:
            h, w = (h - 1) // 2 + 1, (w - 1) // 2 + 1
        shapes += [(B, c, h, w)] * (5 if s else 4)               # conv1, conv2 [, downsample] of two blocks
    return shapes


def check_batch_norm_values(B: int, H: int, W: int):
    """Raise torch's ``ValueError`` when a BatchNorm in training mode would see one value per channel
    (``F.batch_norm``'s ``_verify_batch_size``); the library refuses that shape too."""
    for shape in tv_norm_shapes(B, H, W):
        if shape[0] * shape[2] * shape[3] == 1:
            raise ValueError(f"Expected more than 1 value per channel when training, got input size "
                             f"{torch.Size(shape)}")


def resnet18_train_error(model, observations) -> str:
    """Why ``model(observations)`` (SAVi's AudioGoalPredictor) does not run through :class:`ResNetFunction`; ``""``
    when it does.  It does when autocast is off; ``observations["spectrogram"]`` is a contiguous CUDA float32
    (B, H, W, 2) tensor that does not require grad, with 1 <= B <= 65535 and H, W <= 256; ``model.predictor`` is
    torchvision's resnet18 of :func:`resnet18_layout_error` with every BatchNorm in the same mode and with the same
    float momentum (not None, torch's cumulative average); and its parameters and running statistics are contiguous
    float32 tensors, and its ``num_batches_tracked`` int64 tensors, on that device."""
    obs = observations if isinstance(observations, dict) else {}
    x = obs.get("spectrogram")
    err = _train_spectrogram_error(x)
    if err:
        return err
    net = getattr(model, "predictor", None)
    err = resnet18_layout_error(net, training=True)
    if err:
        return "the predictor is not torchvision's resnet18: " + err
    norms = [n for _, n in conv_norm_pairs(net)]
    if len({n.training for n in norms}) != 1:
        return "the BatchNorms are not all in the same mode"
    if any(n.momentum is None for n in norms):
        return "a BatchNorm has momentum=None (cumulative average)"
    if len({float(n.momentum) for n in norms}) != 1:
        return "the BatchNorms' momenta differ"
    if _tensor_error(net, x.device, True) or any(
            n.num_batches_tracked is None or n.num_batches_tracked.device != x.device
            or n.num_batches_tracked.dtype != torch.int64 for n in norms):
        return f"the predictor's parameters or buffers are not contiguous float32 tensors on {x.device}"
    return ""


class ResNetFunction(torch.autograd.Function):
    """torchvision's ResNet-18 on ``x.permute(0, 3, 1, 2)`` through the library, BatchNorm with batch statistics
    (``training``: the running statistics and ``num_batches_tracked`` in ``stats`` updated in place) or with the
    running ones, differentiable in all 62 parameters, each an input of the function so that autograd sees them; not
    in ``x``.  The backward computes only the gradients autograd asks for and is not itself differentiable.
    ``grad``: whether grad mode was on at the call; without it, or when no parameter requires grad (a frozen
    network), nothing is saved for a backward."""

    @staticmethod
    def forward(ctx, grad, eps, training, momentum, x, stats, *params):
        from .renderer import WaveformOps
        ops = WaveformOps.get(x.device)
        out, ws = ops.resnet18_train_forward(x, params, stats, eps, training, momentum)
        if grad and any(ctx.needs_input_grad[6:]):
            ctx.save_for_backward(x, ws, *params)
            ctx.eps, ctx.training, ctx.stats = eps, training, stats
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_out):
        from .renderer import WaveformOps
        x, ws, *params = ctx.saved_tensors
        ops = WaveformOps.get(x.device)
        grads = ops.resnet18_train_backward(x, params, ctx.stats, ctx.eps, ctx.training, ws, grad_out.contiguous(),
                                            need=ctx.needs_input_grad[6:])
        return (None,) * 6 + tuple(grads)


def resnet18_train_forward(model, observations):
    """``model.predictor(observations["spectrogram"].permute(0, 3, 1, 2))`` through :class:`ResNetFunction`, in the
    BatchNorms' mode; the caller has checked :func:`resnet18_train_error`.  ``ValueError`` as torch's in training mode
    when a BatchNorm would see one value per channel."""
    net = model.predictor
    norms = [n for _, n in conv_norm_pairs(net)]
    x = observations["spectrogram"]
    training = norms[0].training
    if training:
        check_batch_norm_values(*x.shape[:3])
    eps = tuple(float(n.eps) for n in norms)
    return ResNetFunction.apply(torch.is_grad_enabled(), eps, training, float(norms[0].momentum), x,
                                tuple(resnet18_buffers(net)), *resnet18_params(net))
