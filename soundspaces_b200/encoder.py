"""The policy's audio encoder at rollout time: ``AudioCNN.cnn`` of the reference's audio-goal baselines
(ss_baselines/av_nav/models/audio_cnn.py:50-75, av_wan/models/audio_cnn.py:51-76, savi/models/audio_cnn.py:61-92)
run by ``ssb_audio_encoder_batch`` (two launches) instead of seven PyTorch / cuDNN layers.

    from soundspaces_b200.encoder import patch_audio_cnn
    patch_audio_cnn(AudioCNN)       # the class of ss_baselines.av_nav / av_wan / savi models.audio_cnn
    patch_audio_cnn(AudioCNN, category=True)     # savi: also SAVi with a distractor sound

The patched ``forward`` takes the fused path only for inference on a contiguous CUDA float32 ``(N, H, W, 2)``
observation through a ``cnn`` of exactly the reference layout (:func:`check_encoder_layout`) that the library takes
(at most 65535 envs, a Linear that matches conv3 and a shape within the shared-memory limit,
:func:`audio_encoder_smem_bytes`); the PPO update (grad enabled), CPU tensors and anything else run the original
``forward``.  SAVi with a distractor sound (``_has_distractor_sound``) concatenates the ``(N, 21)`` category
observation, broadcast over every pixel, after the two ears, so its conv1 has 23 input channels.  By default it runs the original ``forward``; with ``category=True`` it takes the fused path too
(``ssb_audio_encoder_category_batch``, the label channels folded into a per-env conv1 bias) when ``category`` is a
CUDA float32 ``(N, 21)`` tensor on the observation's device with unit column stride.

The policy's visual encoder, ``VisualCNN`` (ss_baselines/av_nav/models/visual_cnn.py:53-161, av_wan :17-118,
savi :17-188), has the same ``cnn`` layout with RGB and depth channels in conv1; :func:`patch_visual_cnn` runs it by
``ssb_visual_encoder_batch`` (two launches) from the raw ``observations["rgb"]`` / ``["depth"]``:

    from soundspaces_b200.encoder import patch_visual_cnn
    patch_visual_cnn(VisualCNN)     # the class of ss_baselines.av_nav / av_wan / savi models.visual_cnn

AV-WaN's map encoders, ``MapCNN`` (ss_baselines/av_wan/models/map_cnn.py:17-104) on the geometric map ``gm`` and the
acoustic map ``am``, have the same layout too; :func:`patch_map_cnn` runs them by ``ssb_map_encoder_batch`` (two
launches), whose cluster kernel spreads conv1's activations over the cluster so that the 200 x 200 and 400 x 400
geometric maps fit:

    from soundspaces_b200.encoder import patch_map_cnn
    patch_map_cnn(MapCNN)           # the class of ss_baselines.av_wan.models.map_cnn

With ``training=True`` each of the three patches also runs grad-mode calls (PPO's ``evaluate_actions``) through
:class:`ConvStackFunction`: ``ssb_conv_stack_train_forward_batch``, whose features and output are bit-identical to
the rollout-time entries, and ``ssb_conv_stack_train_backward_batch`` for the ``cnn``'s parameter gradients.
:func:`conv_stack_train_error` says why a call runs the original instead.
"""
from __future__ import annotations

import torch
import torch.nn as nn
from torch.autograd.function import once_differentiable


def _is_flatten(m: nn.Module) -> bool:
    if isinstance(m, nn.Flatten):
        return m.start_dim == 1 and m.end_dim == -1
    # ss_baselines.common.utils.Flatten: x.reshape(x.size(0), -1), no parameters
    return (type(m).__name__ == "Flatten" and type(m).__module__ == "ss_baselines.common.utils"
            and not any(True for _ in m.parameters()))


def encoder_layout_error(cnn, n_category: int = 0) -> str:
    """Why ``cnn`` is not ``Conv2d(2 + n_category -> C1) ReLU Conv2d ReLU Conv2d Flatten Linear ReLU`` with unpadded,
    undilated, ungrouped convolutions chained channel to channel; ``""`` when it is."""
    return conv_stack_layout_error(cnn, 2 + n_category)


def conv_stack_layout_error(cnn, in_channels: int) -> str:
    """Why ``cnn`` is not ``Conv2d(in_channels -> C1) ReLU Conv2d ReLU Conv2d Flatten Linear ReLU`` with unpadded,
    undilated, ungrouped convolutions chained channel to channel; ``""`` when it is.  The layout of both
    ``AudioCNN.cnn`` and ``VisualCNN.cnn``."""
    if not isinstance(cnn, nn.Sequential) or len(cnn) != 8:
        return "expected an nn.Sequential of 8 modules"
    kinds = (nn.Conv2d, nn.ReLU, nn.Conv2d, nn.ReLU, nn.Conv2d, None, nn.Linear, nn.ReLU)
    for i, (m, kind) in enumerate(zip(cnn, kinds)):
        ok = _is_flatten(m) if kind is None else type(m) is kind
        if not ok:
            want = "Flatten" if kind is None else kind.__name__
            return f"module {i} is {type(m).__name__}, expected {want}"
    in_ch = in_channels
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


AUDIO_SMEM_LIMIT = 232448          # bytes of shared memory ssb_audio_encoder_batch may use per CTA
AUDIO_MAX_ENVS = 65535


def _conv_shapes(cnn, H, W):
    """[(C, ho, wo, kh, kw)] of the three convs of ``cnn`` on an H x W input, or None when a layer's output is empty."""
    shapes, h, w = [], H, W
    for conv in (cnn[0], cnn[2], cnn[4]):
        (kh, kw), (sh, sw) = conv.kernel_size, conv.stride
        if kh > h or kw > w:
            return None
        h, w = (h - kh) // sh + 1, (w - kw) // sw + 1
        shapes.append((conv.out_channels, h, w, kh, kw))
    return shapes


def audio_encoder_smem_bytes(cnn, n_labels: int, H: int, W: int):
    """Shared memory ``ssb_audio_encoder_batch`` (``ssb_audio_encoder_category_batch`` with ``n_labels`` label
    channels) needs per CTA for ``cnn`` (a layout :func:`encoder_layout_error` accepts) on an (H, W, 2) observation,
    and the number of conv3 features: ``(bytes, F)``, or ``None`` when a layer's output is empty.  Mirrors the entries'
    limit (include/ssb200.h)."""
    shapes = _conv_shapes(cnn, H, W)
    if shapes is None:
        return None
    (c1, h1, w1, kh1, kw1), (c2, h2, w2, kh2, kw2), (c3, h3, w3, kh3, kw3) = shapes
    wslice = max(-(-c1 // 8) * (2 + n_labels) * kh1 * kw1, -(-c2 // 8) * c1 * kh2 * kw2, -(-c3 // 8) * c2 * kh3 * kw3)
    return 4 * (H * W * 2 + c1 * h1 * w1 + c2 * h2 * w2 + wslice), c3 * h3 * w3


def _audio_fits(cnn, n_labels, x) -> bool:
    """Whether the entries take ``cnn`` (a checked layout) on the observation ``x``: at most 65535 envs, every layer's
    output non-empty, Linear.in_features equal to conv3's size and the shared-memory footprint within the limit."""
    N, H, W = x.shape[:3]
    sizes = audio_encoder_smem_bytes(cnn, n_labels, H, W)
    return (N <= AUDIO_MAX_ENVS and sizes is not None and sizes[0] <= AUDIO_SMEM_LIMIT
            and cnn[6].in_features == sizes[1])


def _conv_stack_kind(module) -> str:
    if hasattr(module, "_map_type"):
        return "map"
    if hasattr(module, "_n_input_rgb") or hasattr(module, "_n_input_depth"):
        return "visual"
    return "audio"


def _train_inputs(module, observations):
    """(kind, x, depth, labels) the conv-stack entries read for ``module`` (AudioCNN, VisualCNN or MapCNN), or a
    ``str`` saying why they cannot."""
    from ._lib import CONV_INPUT_MAP, CONV_INPUT_SPECTROGRAM, CONV_INPUT_VISUAL
    kind = _conv_stack_kind(module)
    if kind == "audio":
        x = observations.get(getattr(module, "_audiogoal_sensor", "spectrogram"))
        labels = observations.get("category") if getattr(module, "_has_distractor_sound", False) else None
        if labels is None and getattr(module, "_has_distractor_sound", False):
            return "no category observation"
        return CONV_INPUT_SPECTROGRAM, x, None, labels
    if kind == "map":
        return CONV_INPUT_MAP, observations.get(module._map_type), None, None
    if getattr(module, "_n_input_semantic", 0) > 0:
        return "semantic channels are not fused"
    n_rgb, n_depth = getattr(module, "_n_input_rgb", 0), getattr(module, "_n_input_depth", 0)
    if n_rgb + n_depth == 0:
        return "a blind encoder"
    return (CONV_INPUT_VISUAL, observations.get("rgb") if n_rgb else None,
            observations.get("depth") if n_depth else None, None)


def _params(cnn):
    return (cnn[0].weight, cnn[0].bias, cnn[2].weight, cnn[2].bias, cnn[4].weight, cnn[4].bias, cnn[6].weight,
            cnn[6].bias)


def conv_stack_train_error(module, observations) -> str:
    """Why ``module(observations)`` (an AudioCNN, VisualCNN or MapCNN) does not run through :class:`ConvStackFunction`;
    ``""`` when it does.  It does when autocast is off; the ``cnn`` has the reference layout
    (:func:`conv_stack_layout_error`); its observations (and SAVi's ``(B, 21)`` category) are contiguous CUDA float32
    tensors on one device that do not require grad, with the channel counts the module expects; the parameters are
    contiguous CUDA float32 tensors there; and the library takes the shape
    (``ssb_conv_stack_train_workspace_bytes``: B <= 65535, non-empty layers, a Linear that matches conv3, the per-layer
    limits of include/ssb200.h)."""
    if torch.is_autocast_enabled("cuda"):
        return "autocast is on"
    got = _train_inputs(module, observations)
    if isinstance(got, str):
        return got
    kind, x, depth, labels = got
    cnn = getattr(module, "cnn", None)
    first = x if x is not None else depth
    if not isinstance(first, torch.Tensor) or not first.is_cuda:
        return "the observation is not a CUDA tensor"
    dev = first.device
    named = [("observation", x), ("depth", depth), ("category", labels)]
    for name, t in named:
        if t is None:
            continue
        if not (isinstance(t, torch.Tensor) and t.is_cuda and t.device == dev and t.dtype == torch.float32
                and t.is_contiguous()):
            return f"{name} is not a contiguous CUDA float32 tensor on {dev}"
        if t.requires_grad:
            return f"{name} requires grad"
    if first.ndim != 4 or (depth is not None and x is not None and (depth.ndim != 4 or depth.shape[:3] != x.shape[:3])):
        return "the observations are not (B, H, W, C) tensors of equal B, H and W"
    B = first.shape[0]
    if labels is not None and (labels.ndim != 2 or labels.shape[0] != B):
        return f"category has shape {tuple(labels.shape)}, expected ({B}, L)"
    if kind == 0 and first.shape[3] != 2:
        return "the spectrogram does not have 2 channels"
    if kind == 1:
        want = ((x, getattr(module, "_n_input_rgb", 0)), (depth, getattr(module, "_n_input_depth", 0)))
        if any(t is not None and t.shape[3] != c for t, c in want):
            return "the RGB / depth channels do not match _n_input_rgb / _n_input_depth"
    if kind == 2 and first.shape[3] != module._n_input_gm:
        return "the map does not have _n_input_gm channels"
    in_ch = sum(t.shape[3] for t in (x, depth) if t is not None) + (labels.shape[1] if labels is not None else 0)
    err = conv_stack_layout_error(cnn, in_ch)
    if err:
        return err
    for p in _params(cnn):
        if p is not None and not (p.is_cuda and p.device == dev and p.dtype == torch.float32 and p.is_contiguous()):
            return f"the parameters are not contiguous CUDA float32 tensors on {dev}"
    if B == 0:
        return "no envs"
    import ctypes
    from ._lib import Conv2dLayer, ConvStackInput, load_library
    # the shape check reads no memory: any non-NULL pointer stands for a present input
    n_labels = labels.shape[1] if labels is not None else 0
    inp = ConvStackInput(d_x=16 if x is not None else None, d_depth=16 if depth is not None else None,
                         d_labels=16 if n_labels else None, label_stride=n_labels, kind=kind, H=first.shape[1],
                         W=first.shape[2], channels=x.shape[3] if x is not None else 0,
                         n_depth=depth.shape[3] if depth is not None else 0, n_labels=n_labels)
    layers = (Conv2dLayer * 3)()
    for i, conv in enumerate((cnn[0], cnn[2], cnn[4])):
        layers[i] = Conv2dLayer(16, None, conv.out_channels, *conv.kernel_size, *conv.stride, int(i < 2))
    if load_library().ssb_conv_stack_train_workspace_bytes(B, ctypes.byref(inp), layers, cnn[6].in_features,
                                                           cnn[6].out_features, 1) < 0:
        return "the library refuses this shape (include/ssb200.h, ssb_conv_stack_train_*)"
    return ""


class ConvStackFunction(torch.autograd.Function):
    """``cnn(input)`` of an AudioCNN, VisualCNN or MapCNN through the library, differentiable in the eight parameters
    of the ``cnn`` (not in the observations or labels); the backward computes only the gradients autograd asks for
    and is not itself differentiable.  ``grad``: whether grad mode was on at the call; without it, or when no
    parameter requires grad (a frozen encoder), nothing is saved for a backward."""

    @staticmethod
    def forward(ctx, grad, kind, strides, x, depth, labels, *params):
        from .renderer import WaveformOps
        first = x if x is not None else depth
        ops = WaveformOps.get(first.device)
        out, features, saved = ops.conv_stack_train_forward(kind, x, depth, labels, params, strides)
        if grad and any(ctx.needs_input_grad[6:]):
            ctx.save_for_backward(x, depth, labels, features, out, saved, *params)
            ctx.kind, ctx.strides = kind, strides
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_out):
        from .renderer import WaveformOps
        x, depth, labels, features, out, saved, *params = ctx.saved_tensors
        ops = WaveformOps.get(out.device)
        grads = ops.conv_stack_train_backward(ctx.kind, x, depth, labels, params, ctx.strides, features, out, saved,
                                              grad_out.contiguous(), need=ctx.needs_input_grad[6:])
        return (None,) * 6 + tuple(grads)


def conv_stack_train_forward(module, observations):
    """``module(observations)`` through :class:`ConvStackFunction`; the caller has checked
    :func:`conv_stack_train_error`."""
    kind, x, depth, labels = _train_inputs(module, observations)
    cnn = module.cnn
    strides = tuple(tuple(c.stride) for c in (cnn[0], cnn[2], cnn[4]))
    return ConvStackFunction.apply(torch.is_grad_enabled(), kind, strides, x, depth, labels, *_params(cnn))


def _train_forward(self, observations, original):
    """The grad-mode call of a ``training=True`` patch: the library when :func:`conv_stack_train_error` allows."""
    if conv_stack_train_error(self, observations):
        return original(self, observations)
    return conv_stack_train_forward(self, observations)


def patch_audio_cnn(cls, category: bool = False, training: bool = False):
    """Replace ``cls.forward`` of an ``AudioCNN`` class (av_nav, av_wan or savi) in place, nothing else.  The
    observation is ``observations[self._audiogoal_sensor]`` (av_nav, savi) or ``observations["spectrogram"]``
    (av_wan, which has no ``_audiogoal_sensor``).  ``category=True`` also fuses SAVi models built with
    ``has_distractor_sound=True``, reading ``observations["category"]``; without it they run the original.  Calls the
    library cannot take run the original too: more than 65535 envs, a layer whose output is empty, a Linear whose
    in_features is not conv3's size, or a shape past the shared-memory limit (:func:`audio_encoder_smem_bytes`).
    ``training=True`` also runs grad-mode calls (PPO's ``evaluate_actions``) through :class:`ConvStackFunction` when
    :func:`conv_stack_train_error` allows; without it they run the original."""
    original = getattr(cls.forward, "_ssb_original", cls.forward)

    def forward(self, observations):
        if training and torch.is_grad_enabled():
            if getattr(self, "_has_distractor_sound", False) and not category:
                return original(self, observations)
            return _train_forward(self, observations, original)
        x = observations[getattr(self, "_audiogoal_sensor", "spectrogram")]
        if category and getattr(self, "_has_distractor_sound", False):
            if torch.is_grad_enabled() or not _fusable(x) or "category" not in observations:
                return original(self, observations)
            labels = observations["category"]
            if not _fusable_category(labels, x, self.cnn) or not _audio_fits(self.cnn, labels.shape[1], x):
                return original(self, observations)
            from .renderer import WaveformOps
            return WaveformOps.get(x.device).audio_encoder(x, self.cnn, category=labels)
        if (torch.is_grad_enabled() or not _fusable(x) or encoder_layout_error(self.cnn)
                or not _audio_fits(self.cnn, 0, x)):
            return original(self, observations)
        from .renderer import WaveformOps
        return WaveformOps.get(x.device).audio_encoder(x, self.cnn)

    forward._ssb_original = original
    forward.__doc__ = original.__doc__
    cls.forward = forward
    return cls


VISUAL_SMEM_LIMIT = 232448          # bytes of shared memory ssb_visual_encoder_batch may use per CTA
VISUAL_MAX_ENVS = 65535
ENCODER_MAX_FEATURES = 2 ** 31 - 1  # conv3 features the visual and map entries take (the Linear's F is an int)


def visual_encoder_smem_bytes(cnn, in_channels: int, H: int, W: int):
    """Shared memory ``ssb_visual_encoder_batch`` needs per CTA for ``cnn`` (a layout
    :func:`conv_stack_layout_error` accepts) on an H x W input, and the number of conv3 features:
    ``(bytes, F)``, or ``None`` when a layer's output is empty.  Mirrors the entry's limit (include/ssb200.h)."""
    shapes = _conv_shapes(cnn, H, W)
    if shapes is None:
        return None
    (c1, h1, w1, kh1, kw1), (c2, h2, w2, kh2, kw2), (c3, h3, w3, kh3, kw3) = shapes
    region2 = max(c2 * h2 * w2, c1 * in_channels * kh1 * kw1 + in_channels * kh1 * W)
    wslice = max(-(-c2 // 8) * c1 * kh2 * kw2, -(-c3 // 8) * c2 * kh3 * kw3)
    return 4 * (c1 * h1 * w1 + region2 + wslice), c3 * h3 * w3


def _visual_obs(t, channels, like=None) -> bool:
    return (isinstance(t, torch.Tensor) and t.is_cuda and t.dtype == torch.float32 and t.ndim == 4
            and t.shape[3] == channels and t.is_contiguous()
            and (like is None or (t.device == like.device and t.shape[:3] == like.shape[:3])))


def fused_visual_forward(module, observations):
    """``module.forward(observations)`` of a ``VisualCNN`` (av_nav, av_wan or savi) through the library -> (N, hidden),
    or None (the caller runs the original) for: grad enabled, SAVi semantic channels, a blind encoder, an observation
    that is not a contiguous CUDA float32 (N, H, W, C) tensor with C = ``_n_input_rgb`` / ``_n_input_depth`` (RGB and
    depth on one device with equal N, H, W), a ``cnn`` :func:`conv_stack_layout_error` refuses, a Linear whose
    in_features is not conv3's output size, more than 65535 envs, a shape past the entry's shared-memory limit, or more
    than 2^31 - 1 conv3 features."""
    if torch.is_grad_enabled() or getattr(module, "_n_input_semantic", 0) > 0:
        return None
    n_rgb, n_depth = getattr(module, "_n_input_rgb", 0), getattr(module, "_n_input_depth", 0)
    if n_rgb + n_depth == 0:
        return None
    rgb = observations.get("rgb") if n_rgb > 0 else None
    depth = observations.get("depth") if n_depth > 0 else None
    if (n_rgb > 0 and not _visual_obs(rgb, n_rgb)) or (n_depth > 0 and not _visual_obs(depth, n_depth, rgb)):
        return None
    first = rgb if rgb is not None else depth
    N, H, W = first.shape[:3]
    cnn = module.cnn
    if N > VISUAL_MAX_ENVS or conv_stack_layout_error(cnn, n_rgb + n_depth):
        return None
    sizes = visual_encoder_smem_bytes(cnn, n_rgb + n_depth, H, W)
    if (sizes is None or sizes[0] > VISUAL_SMEM_LIMIT or cnn[6].in_features != sizes[1]
            or sizes[1] > ENCODER_MAX_FEATURES):
        return None
    from .renderer import WaveformOps
    return WaveformOps.get(first.device).visual_encoder(rgb, depth, cnn)


def patch_visual_cnn(cls, training: bool = False):
    """Replace ``cls.forward`` of a ``VisualCNN`` class (ss_baselines.av_nav / av_wan / savi models.visual_cnn) in
    place, nothing else; the original stays reachable as ``cls.forward._ssb_original`` and patching twice changes
    nothing.  Qualifying calls (:func:`fused_visual_forward`) run in the library, anything else runs the original.
    ``training=True`` also runs grad-mode calls through :class:`ConvStackFunction` when
    :func:`conv_stack_train_error` allows."""
    original = getattr(cls.forward, "_ssb_original", cls.forward)

    def forward(self, observations):
        if training and torch.is_grad_enabled():
            return _train_forward(self, observations, original)
        out = fused_visual_forward(self, observations)
        return original(self, observations) if out is None else out

    forward._ssb_original = original
    forward.__doc__ = original.__doc__
    cls.forward = forward
    return cls


MAP_SMEM_LIMIT = 232448             # bytes of shared memory ssb_map_encoder_batch may use per CTA
MAP_MAX_ENVS = 65535


def map_encoder_smem_bytes(cnn, C: int, H: int, W: int):
    """Shared memory ``ssb_map_encoder_batch`` needs per CTA for ``cnn`` (a layout :func:`conv_stack_layout_error`
    accepts) on an (H, W, C) map, and the number of conv3 features: ``(bytes, F)``, or ``None`` when a layer's output
    is empty.  Mirrors the entry's formula (include/ssb200.h)."""
    shapes = _conv_shapes(cnn, H, W)
    if shapes is None:
        return None
    (c1, h1, w1, kh1, kw1), (c2, h2, w2, kh2, kw2), (c3, h3, w3, kh3, kw3) = shapes
    rows1 = c1 * -(-h1 // 8) * w1
    conv1 = c1 * C * kh1 * kw1 + C * kh1 * W
    conv2 = c1 * kh2 * w1 + -(-c2 // 8) * c1 * kh2 * kw2
    conv3 = c2 * h2 * w2 + -(-c3 // 8) * c2 * kh3 * kw3
    return 4 * (max(rows1 + max(conv1, conv2), conv3) + -(-c2 // 8) * h2 * w2), c3 * h3 * w3


def fused_map_forward(module, observations):
    """``module.forward(observations)`` of AV-WaN's ``MapCNN`` through the library -> (N, hidden), or None (the caller
    runs the original) for: grad enabled, an ``observations[module._map_type]`` that is not a contiguous CUDA float32
    (N, H, W, C) tensor with C = ``module._n_input_gm``, a ``cnn`` :func:`conv_stack_layout_error` refuses, a Linear
    whose in_features is not conv3's output size, more than 65535 envs, a shape past the entry's shared-memory
    limit (:func:`map_encoder_smem_bytes`), or more than 2^31 - 1 conv3 features."""
    if torch.is_grad_enabled():
        return None
    x, C = observations.get(module._map_type), module._n_input_gm
    if not (isinstance(x, torch.Tensor) and x.is_cuda and x.dtype == torch.float32 and x.ndim == 4
            and x.shape[3] == C and x.is_contiguous()):
        return None
    N, H, W = x.shape[:3]
    cnn = module.cnn
    if N > MAP_MAX_ENVS or conv_stack_layout_error(cnn, C):
        return None
    sizes = map_encoder_smem_bytes(cnn, C, H, W)
    if sizes is None or sizes[0] > MAP_SMEM_LIMIT or cnn[6].in_features != sizes[1] or sizes[1] > ENCODER_MAX_FEATURES:
        return None
    from .renderer import WaveformOps
    return WaveformOps.get(x.device).map_encoder(x, cnn)


def patch_map_cnn(cls, training: bool = False):
    """Replace ``cls.forward`` of AV-WaN's ``MapCNN`` class (ss_baselines.av_wan.models.map_cnn), which encodes both
    the geometric and the acoustic map, in place, nothing else; the original stays reachable as
    ``cls.forward._ssb_original`` and patching twice changes nothing.  Qualifying calls (:func:`fused_map_forward`)
    run in the library in two launches, anything else runs the original.  ``training=True`` also runs grad-mode
    calls through :class:`ConvStackFunction` when :func:`conv_stack_train_error` allows."""
    original = getattr(cls.forward, "_ssb_original", cls.forward)

    def forward(self, observations):
        if training and torch.is_grad_enabled():
            return _train_forward(self, observations, original)
        out = fused_map_forward(self, observations)
        return original(self, observations) if out is None else out

    forward._ssb_original = original
    forward.__doc__ = original.__doc__
    cls.forward = forward
    return cls


SMT_CNN_CROP = 64                  # ResizeCenterCropper(size=(64, 64)) of SMTCNN's default obs_transform
SMT_CNN_MAX_HW = 1024               # ssb_smt_cnn_batch refuses taller or wider observations
SMT_CNN_MAX_ENVS = 1024


def resize_center_crop_geometry(H: int, W: int, size: int = SMT_CNN_CROP):
    """``(h', w', crop_y, crop_x)`` of ``ResizeCenterCropper(size=(size, size))`` on an H x W image, with the
    reference's own expressions (ss_baselines/common/utils.py: ``image_resize_shortest_edge`` and ``center_crop``)."""
    scale = size / min(H, W)
    h, w = int(H * scale), int(W * scale)
    return h, w, h // 2 - size // 2, w // 2 - size // 2


def crop_inside(h: int, w: int, cy: int, cx: int, size: int = SMT_CNN_CROP) -> bool:
    """Whether the size x size crop at (cy, cx) lies inside the h x w resized image.  It does not when rounding makes
    the short edge ``size - 1`` (short edges 49, 98, 103, ...): the reference's slice then degenerates and its ``fc``
    raises."""
    return 0 <= cy <= h - size and 0 <= cx <= w - size


def _is_resize_center_cropper(m) -> bool:
    """ss_baselines.common.utils.ResizeCenterCropper(size=(64, 64)) on channels-first input, no parameters."""
    if type(m).__name__ != "ResizeCenterCropper" or type(m).__module__ != "ss_baselines.common.utils":
        return False
    size = getattr(m, "_size", None)
    return (isinstance(size, (tuple, list)) and tuple(size) == (SMT_CNN_CROP, SMT_CNN_CROP)
            and getattr(m, "channels_last", None) is False and not any(True for _ in m.parameters()))


def smt_cnn_layout_error(module) -> str:
    """Why ``module`` is not an ``SMTCNN`` (ss_baselines/savi/models/smt_cnn.py:17-113) the library runs: RGB and / or
    depth only, each encoder the SMT ``custom_resnet18`` with the modality's channels and an fc on the 64 x 64 crop
    (:func:`soundspaces_b200.belief_nets.smt_resnet18_layout_error`), and an ``obs_transform`` that is None or
    ``ResizeCenterCropper(size=(64, 64))`` on channels-first input; ``""`` when it is.  Parameters are not checked
    here."""
    from .belief_nets import smt_resnet18_layout_error
    mods = getattr(module, "input_modalities", None)
    if not isinstance(mods, list) or not mods or any(m not in ("rgb", "depth") for m in mods) or len(set(mods)) != len(mods):
        return f"input_modalities {mods!r}: only 'rgb' and / or 'depth' are fused"
    t = getattr(module, "obs_transform", None)
    if t is not None and not _is_resize_center_cropper(t):
        return f"obs_transform is {type(t).__name__}, expected None or ResizeCenterCropper(size=(64, 64))"
    for m in mods:
        net = getattr(module, f"{m}_encoder", None)
        conv1 = getattr(net, "conv1", None)
        if not isinstance(conv1, nn.Conv2d):
            return f"{m}_encoder has no Conv2d conv1"
        err = smt_resnet18_layout_error(net, conv1.in_channels, (SMT_CNN_CROP, SMT_CNN_CROP))
        if err:
            return f"{m}_encoder: {err}"
    return ""


def fused_smt_cnn_forward(module, observations):
    """``module.forward(observations)`` of an ``SMTCNN`` through ``ssb_smt_cnn_batch`` -> (B, 64 n_modalities), or None
    (the caller runs the original) for: grad enabled, a layout :func:`smt_cnn_layout_error` refuses (a semantic
    modality among them), an observation that is not a contiguous CUDA float32 (B, H, W, C) tensor with the encoder's C
    (both on one device with equal B), B = 0 or B > 1024, H or W past 1024, an input that is not 64 x 64 without a
    transform, a resize whose short edge rounds to 63 (:func:`crop_inside`), or parameters that are not contiguous
    float32 on the observation's device."""
    if torch.is_grad_enabled() or smt_cnn_layout_error(module):
        return None
    from .belief_nets import smt_resnet18_layout_error
    resize = module.obs_transform is not None
    first = None
    for m in module.input_modalities:
        x, net = observations.get(m), getattr(module, f"{m}_encoder")
        if not (isinstance(x, torch.Tensor) and x.is_cuda and x.dtype == torch.float32 and x.ndim == 4
                and x.shape[3] == net.conv1.in_channels and x.is_contiguous()
                and (first is None or (x.device == first.device and x.shape[0] == first.shape[0]))):
            return None
        first = first if first is not None else x
        H, W = x.shape[1:3]
        if max(H, W) > SMT_CNN_MAX_HW:
            return None
        if resize:
            if not crop_inside(*resize_center_crop_geometry(H, W)):
                return None
        elif (H, W) != (SMT_CNN_CROP, SMT_CNN_CROP):
            return None
        if smt_resnet18_layout_error(net, x.shape[3], (SMT_CNN_CROP, SMT_CNN_CROP), x.device):
            return None
    if not 0 < first.shape[0] <= SMT_CNN_MAX_ENVS:
        return None
    from .renderer import WaveformOps
    rgb = observations["rgb"] if "rgb" in module.input_modalities else None
    depth = observations["depth"] if "depth" in module.input_modalities else None
    return WaveformOps.get(first.device).smt_cnn(rgb, depth, getattr(module, "rgb_encoder", None),
                                                 getattr(module, "depth_encoder", None), resize=resize)


SMT_CNN_TRAIN_MAX_ENVS = 65535      # SRN_MAX_ENVS of ssb200.cu: rows per ssb_smt_cnn_train_* call


def smt_cnn_params(module):
    """The parameters :class:`SmtCnnFunction` takes: 62 per present encoder, RGB first, each in the order of
    :func:`soundspaces_b200.belief_nets.smt_resnet18_params`."""
    from .belief_nets import smt_resnet18_params
    return [p for m in ("rgb", "depth") if m in module.input_modalities
            for p in smt_resnet18_params(getattr(module, f"{m}_encoder"))]


def _smt_cnn_observations(module):
    """The present modalities in the order their features appear: RGB first."""
    return [m for m in ("rgb", "depth") if m in module.input_modalities]


def smt_cnn_train_error(module, observations) -> str:
    """Why ``module(observations)`` (SAVi's ``SMTCNN``) does not run through :class:`SmtCnnFunction` or, with every
    parameter frozen, through ``ssb_smt_cnn_batch`` in chunks; ``""`` when it does.  It does when autocast is off; the
    layout is one :func:`smt_cnn_layout_error` accepts (no semantic modality); each observation is a contiguous CUDA
    float32 (B, H, W, C) tensor with the encoder's C that does not require grad, all on one device with equal B, 1 <= B
    <= 65535, H, W <= 1024, 64 x 64 without a transform and otherwise a resize whose crop lies inside it
    (:func:`crop_inside`); and every encoder parameter is a contiguous float32 tensor on that device."""
    if torch.is_autocast_enabled("cuda"):
        return "autocast is on"
    err = smt_cnn_layout_error(module)
    if err:
        return err
    from .belief_nets import smt_resnet18_layout_error
    obs = observations if isinstance(observations, dict) else {}
    first = None
    for m in _smt_cnn_observations(module):
        x, net = obs.get(m), getattr(module, f"{m}_encoder")
        if not (isinstance(x, torch.Tensor) and x.is_cuda):
            return f"{m} is not a CUDA tensor"
        if x.dtype != torch.float32 or not x.is_contiguous():
            return f"{m} is not a contiguous float32 tensor"
        if x.requires_grad:
            return f"{m} requires grad"
        if x.ndim != 4 or x.shape[3] != net.conv1.in_channels:
            return f"{m} is not a (B, H, W, {net.conv1.in_channels}) tensor"
        if first is not None and (x.device != first.device or x.shape[0] != first.shape[0]):
            return "the observations are not on one device with equal B"
        first = first if first is not None else x
        H, W = x.shape[1:3]
        if max(H, W) > SMT_CNN_MAX_HW:
            return f"a {H}x{W} {m} exceeds {SMT_CNN_MAX_HW}x{SMT_CNN_MAX_HW}"
        if module.obs_transform is not None:
            if not crop_inside(*resize_center_crop_geometry(H, W)):
                return f"the {SMT_CNN_CROP}x{SMT_CNN_CROP} crop does not lie inside the resized {H}x{W} {m}"
        elif (H, W) != (SMT_CNN_CROP, SMT_CNN_CROP):
            return f"without a transform, {m} must be {SMT_CNN_CROP}x{SMT_CNN_CROP}, not {H}x{W}"
        if smt_resnet18_layout_error(net, x.shape[3], (SMT_CNN_CROP, SMT_CNN_CROP), x.device):
            return f"the {m}_encoder parameters are not contiguous float32 tensors on {x.device}"
    if not 1 <= first.shape[0] <= SMT_CNN_TRAIN_MAX_ENVS:
        return f"{first.shape[0]} rows, outside 1..{SMT_CNN_TRAIN_MAX_ENVS}"
    return ""


class SmtCnnFunction(torch.autograd.Function):
    """``SMTCNN.forward`` on RGB and / or depth through the library, differentiable in all 62 parameters of each
    present encoder, each an input of the function so that autograd (and DDP's unused-parameter search) sees them; not
    in the observations.  The backward computes only the gradients autograd asks for and is not itself
    differentiable.  ``grad``: whether grad mode was on at the call; without it, or when no parameter requires grad,
    nothing is saved for a backward."""

    @staticmethod
    def forward(ctx, grad, eps, resize, rgb, depth, *params):
        from .renderer import WaveformOps
        ops = WaveformOps.get((rgb if rgb is not None else depth).device)
        out, ws = ops.smt_cnn_train_forward(rgb, depth, params, eps, resize)
        if grad and any(ctx.needs_input_grad[5:]):
            ctx.save_for_backward(rgb, depth, ws, *params)
            ctx.eps, ctx.resize = eps, resize
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_out):
        from .renderer import WaveformOps
        rgb, depth, ws, *params = ctx.saved_tensors
        ops = WaveformOps.get(ws.device)
        grads = ops.smt_cnn_train_backward(rgb, depth, params, ctx.eps, ctx.resize, ws, grad_out.contiguous(),
                                           need=ctx.needs_input_grad[5:])
        return (None,) * 5 + tuple(grads)


def smt_cnn_train_forward(module, observations):
    """``module(observations)`` of an ``SMTCNN`` under grad mode; the caller has checked :func:`smt_cnn_train_error`.
    With some parameter requiring grad, through :class:`SmtCnnFunction`.  With every parameter frozen (SAVi's second
    stage, ``freeze_encoders``), through ``ssb_smt_cnn_batch`` in chunks of at most 1024 rows: the rollout's bits, no
    workspace and no autograd node."""
    from .belief_nets import conv_norm_pairs
    mods = _smt_cnn_observations(module)
    params = smt_cnn_params(module)
    if not any(p.requires_grad for p in params if p is not None):
        B = observations[mods[0]].shape[0]
        with torch.no_grad():
            outs = [fused_smt_cnn_forward(module, {m: observations[m][i:i + SMT_CNN_MAX_ENVS] for m in mods})
                    for i in range(0, B, SMT_CNN_MAX_ENVS)]
        return outs[0] if len(outs) == 1 else torch.cat(outs)
    eps = tuple(float(n.eps) for m in mods for _, n in conv_norm_pairs(getattr(module, f"{m}_encoder")))
    return SmtCnnFunction.apply(torch.is_grad_enabled(), eps, module.obs_transform is not None,
                                observations["rgb"] if "rgb" in mods else None,
                                observations["depth"] if "depth" in mods else None, *params)


def patch_smt_cnn(cls, training: bool = False):
    """Replace ``cls.forward`` of SAVi's ``SMTCNN`` class (ss_baselines/savi/models/smt_cnn.py) in place, nothing
    else; the original stays reachable as ``cls.forward._ssb_original`` and patching twice changes nothing.
    Qualifying calls (:func:`fused_smt_cnn_forward`) run in the library in 39 launches, anything else runs the
    original.  ``training=True`` also runs grad-mode calls (PPO's ``evaluate_actions``) in the library when
    :func:`smt_cnn_train_error` allows (:func:`smt_cnn_train_forward`); without it they run the original."""
    original = getattr(cls.forward, "_ssb_original", cls.forward)

    def forward(self, observations):
        if training and torch.is_grad_enabled():
            if smt_cnn_train_error(self, observations):
                return original(self, observations)
            return smt_cnn_train_forward(self, observations)
        out = fused_smt_cnn_forward(self, observations)
        return original(self, observations) if out is None else out

    forward._ssb_original = original
    forward.__doc__ = original.__doc__
    cls.forward = forward
    return cls
