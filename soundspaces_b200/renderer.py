"""Batched device-side audio renderer: the host half of the H100 audio path.

Owns the device-resident RIR bank (SURVEY.md N1), the source clips with their
cached overlap-save window spectra (the per-sound cache of
``soundspaces/simulator.py:595-600`` moved to the device), and the scratch the
kernels need.  One ``render()`` call replaces, for a whole batch of envs, one
cache-missing ``get_current_spectrogram_observation`` each
(``soundspaces/simulator.py:690-701`` -> ``_compute_audiogoal`` ``:608-666`` ->
``SpectrogramSensor.compute_spectrogram`` ``soundspaces/tasks/nav.py:86-100``).

PyTorch is used for device memory and streams only; all arithmetic runs in
``libssb200.so`` (hand-written sm_90a CUDA) through the C ABI.
"""
from __future__ import annotations

import contextlib
import ctypes as C
import os
from dataclasses import dataclass
from typing import Optional, Sequence

import numpy as np
import torch

from . import _lib, belief_nets
from .encoder import check_encoder_layout, conv_stack_layout_error
from .planning import window_layout
from ._lib import PAD_MODES, REQ_DTYPE, SSB_FLAG_SILENT

N_FFT, HOP, WIN, POOL, SPEC_ROWS = 512, 160, 400, 4, 65
SH_CHANNELS = (1, 4, 9, 16)     # ambisonic orders 0 to 3


def sh_hrtf_bank(n_channels: int = 16) -> np.ndarray:
    """The ambisonic decoder's (K, 2, 256) float32 HRTF bank: the first K rows of the AmbisonicBinauralizer's one
    nested 16-row bank.  Rows 0-8 are ``data/sh_hrtf_bank.npy``; the third-order rows 9-15 are stored as text in
    ``data/sh_hrtf_bank_order3.txt`` (one line per (row, ear), 10 significant digits: exact for float32)."""
    if n_channels not in SH_CHANNELS:
        raise ValueError(f"{n_channels} channels: 1, 4, 9 or 16")
    data = os.path.join(os.path.dirname(os.path.abspath(__file__)), "data")
    bank = np.load(os.path.join(data, "sh_hrtf_bank.npy"))
    if n_channels > 9:
        order3 = np.loadtxt(os.path.join(data, "sh_hrtf_bank_order3.txt"), dtype=np.float64)
        bank = np.concatenate([bank, order3.astype(np.float32).reshape(7, 2, 256)])
    return np.ascontiguousarray(bank[:n_channels])


def spectrogram_shape(sr: int):
    """(65, ceil((1 + sr//160)/4), 2): (65, 26, 2) @16 kHz, (65, 69, 2) @44.1 kHz."""
    frames = 1 + sr // HOP
    return (SPEC_ROWS, -(-frames // POOL), 2)


@dataclass
class AudioRequest:
    """One env-step.  ``out[m] = sum_k rir[k] * src[offset + m - k]`` for m < out_samples.

    offset: 0 for 1-s clips (simulator.py:629-632); ``index * sr`` for multi-second clips
    (simulator.py:634-647, both the early and the ``valid`` branch); the running
    ``_current_sample_index`` for the continuous simulator (continuous_simulator.py:428-456).
    """
    rir: int                       # id in the RIR bank; -1 => unreadable/empty file => zero RIR (simulator.py:617-624)
    source: int                    # id of the source clip
    offset: int = 0
    out_samples: Optional[int] = None      # default sr; int(sr*STEP_TIME) for the continuous simulator
    wrap: bool = False             # continuous_simulator.py:443-445 wrap-around of the clip
    silent: bool = False           # simulator.py:610-612
    distractor_rir: Optional[int] = None   # simulator.py:649-664
    distractor_source: Optional[int] = None
    # transient RIR supplied inline ((L, 2) array; overrides ``rir``): the RIR habitat-sim renders every step
    # (simulator.py:626, continuous_simulator.py:419).  Uploaded for the one call and dropped afterwards.
    rir_array: Optional[object] = None


class _PoolReset(Exception):
    """The window-spectra pool was recycled while a batch was being prepared."""


@dataclass
class PreparedBatch:
    n: int
    reqs_host: np.ndarray
    reqs_dev: torch.Tensor
    plan: object = None            # the ssb_plan the requests were resolved for (partitioned or single-block)


def _dev_index(device):
    device = torch.device(device)
    if device.type != "cuda":
        raise RuntimeError("BatchedAudioRenderer needs a CUDA device; there is no CPU fallback")
    return torch.cuda.current_device() if device.index is None else device.index


class WaveformOps:
    """Kernels that only need a context -- the STFT front end and the AV-WaN intensity reduction on waveforms the
    caller already holds -- without a convolution plan, RIR bank or window-spectra pool.  One per device; this is
    what ``SpectrogramSensor.compute_spectrogram`` (a static method other modules import and call on host arrays of
    any length, savi/ppo/ppo_trainer.py:52,374, belief_predictor.py:15,124) runs on."""

    _instances: dict = {}

    def __init__(self, device="cuda:0"):
        self.device = torch.device("cuda", _dev_index(device))
        self.ctx = _lib.Context(self.device.index)
        self.lib = self.ctx.lib
        self._smt_scratch = {}        # (N, M, d_model) -> device scratch of ssb_smt_state_encoder_batch

    @classmethod
    def get(cls, device="cuda:0") -> "WaveformOps":
        key = _dev_index(device)
        if key not in cls._instances:
            cls._instances[key] = cls(torch.device("cuda", key))
        return cls._instances[key]

    def _stream(self):
        return C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    def spectrogram(self, wave: torch.Tensor, pad_mode: str = "reflect", out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """(n, 2, S) CUDA float32 -> (n, 65, T', 2) for any S >= 512 (nav.py:86-100)."""
        if wave.ndim == 2:
            wave = wave[None]
        wave = wave.to(self.device, torch.float32).contiguous()
        n, _, S = wave.shape
        spec = out if out is not None else torch.empty((n,) + spectrogram_shape(S), dtype=torch.float32, device=self.device)
        self.ctx.check(self.lib.ssb_spectrogram_batch(self.ctx.handle, n, wave.data_ptr(), S, S, PAD_MODES[pad_mode],
                                                      spec.data_ptr(), self._stream()), "ssb_spectrogram_batch")
        return spec

    def frame_gather(self, n: int, sensors) -> None:
        """``ssb_frame_gather_batch``: ``n`` rows of every sensor in ONE launch.  ``sensors``: up to
        ``_lib.FRAME_MAX_SENSORS`` tuples ``(bank, stage, dst, index, fill)`` -- ``bank`` a (rows, row_elems) uint8 or
        float32 CUDA tensor on this device, ``stage`` the (len(fill), row_elems) rows uploaded for this call (same
        dtype) or None, ``dst`` a float32 tensor whose n rows are ``dst.stride(0)`` floats apart and contiguous
        within, ``index`` / ``fill`` int32 sequences as the entry takes them (include/ssb200.h)."""
        table = (_lib.FrameSensor * max(1, len(sensors)))()
        keep = []
        for q, (bank, stage, dst, index, fill) in enumerate(sensors):
            index = np.ascontiguousarray(index, dtype=np.int32)
            fill = np.ascontiguousarray(fill, dtype=np.int32)
            keep += [index, fill]
            table[q] = _lib.FrameSensor(
                bank.data_ptr(), stage.data_ptr() if stage is not None and len(fill) else None,
                dst.data_ptr() if n else None, index.ctypes.data if n else None, fill.ctypes.data if len(fill) else None,
                bank.shape[1], bank.shape[0], dst.stride(0) if n else bank.shape[1], len(fill),
                _lib.FRAME_DTYPES[np.dtype(str(bank.dtype).replace("torch.", ""))])
        self.ctx.check(self.lib.ssb_frame_gather_batch(self.ctx.handle, len(sensors), table, n, self._stream()),
                       "ssb_frame_gather_batch")

    def intensity(self, wave: torch.Tensor, num_frame: int = 150) -> torch.Tensor:
        """AV-WaN ``Intensity`` (avwan_sensors.py:91-100) for a (n, 2, S) CUDA batch -> (n,) mean squares."""
        if wave.ndim == 2:
            wave = wave[None]
        wave = wave.to(self.device, torch.float32).contiguous()
        out = torch.empty(wave.shape[0], dtype=torch.float32, device=self.device)
        self.ctx.check(self.lib.ssb_intensity_batch(self.ctx.handle, wave.shape[0], wave.data_ptr(), wave.shape[2],
                                                    wave.shape[2], int(num_frame), out.data_ptr(), self._stream()),
                       "ssb_intensity_batch")
        return out

    @torch.no_grad()
    def audio_conv1(self, spec: torch.Tensor, conv: "torch.nn.Conv2d", relu: bool = True) -> torch.Tensor:
        """SURVEY.md N2: ``relu(conv(spec.permute(0, 3, 1, 2)))`` for the first layer of ``AudioCNN``
        (audio_cnn.py:51-58,86) straight from the (n, 65, T', 2) observation: no permuted copy, one launch.
        Inference only (rollout collection); ``conv`` must be an unpadded, undilated 2-input-channel ``Conv2d``."""
        if not (spec.is_cuda and spec.dtype == torch.float32 and spec.ndim == 4 and spec.shape[3] == 2 and spec.is_contiguous()):
            raise ValueError("expected a contiguous CUDA float32 (n, H, W, 2) observation")
        if (conv.in_channels != 2 or tuple(conv.padding) != (0, 0) or tuple(conv.dilation) != (1, 1) or conv.groups != 1
                or conv.padding_mode != "zeros"):
            raise ValueError("audio_conv1 fuses Conv2d(2 -> OC, k, stride) without padding / dilation / groups")
        n, H, W, _ = spec.shape
        (kh, kw), (sh, sw) = conv.kernel_size, conv.stride
        out = torch.empty((n, conv.out_channels, (H - kh) // sh + 1, (W - kw) // sw + 1), dtype=torch.float32, device=self.device)
        w = conv.weight.detach().to(self.device, torch.float32).contiguous()
        b = conv.bias.detach().to(self.device, torch.float32).contiguous() if conv.bias is not None else None
        self.ctx.check(self.lib.ssb_audio_conv1_batch(
            self.ctx.handle, n, spec.data_ptr(), H, W, w.data_ptr(), b.data_ptr() if b is not None else None,
            conv.out_channels, kh, kw, sh, sw, int(bool(relu)), out.data_ptr(), self._stream()), "ssb_audio_conv1_batch")
        return out

    @torch.no_grad()
    def audio_encoder(self, spec: torch.Tensor, cnn: "torch.nn.Sequential",
                      features: Optional[torch.Tensor] = None, category: Optional[torch.Tensor] = None) -> torch.Tensor:
        """``cnn(spec.permute(0, 3, 1, 2))`` for ``AudioCNN.cnn`` (audio_cnn.py: Conv2d(2 -> C1) ReLU Conv2d ReLU Conv2d
        Flatten Linear ReLU) straight from the (n, H, W, 2) observation in two launches -> (n, hidden).  Inference
        only.  ``features``: optional (n, F) float32 CUDA tensor that receives the flattened conv3 output.
        ``category``: SAVi with a distractor sound (savi/models/audio_cnn.py:135-150), an (n, L) float32 tensor on
        this device with unit column stride; ``cnn`` then takes ``cat(permute(spec), expand(category))``, i.e. conv1
        has 2 + L input channels (``ssb_audio_encoder_category_batch``).
        ``ValueError`` for any other layout (see :func:`soundspaces_b200.encoder.check_encoder_layout`)."""
        if not (spec.is_cuda and spec.dtype == torch.float32 and spec.ndim == 4 and spec.shape[3] == 2 and spec.is_contiguous()):
            raise ValueError("expected a contiguous CUDA float32 (n, H, W, 2) observation")
        n, H, W, _ = spec.shape
        if category is not None:
            if not (isinstance(category, torch.Tensor) and category.device == self.device
                    and category.dtype == torch.float32 and category.ndim == 2 and category.shape[0] == n
                    and category.stride(1) == 1 and (n <= 1 or category.stride(0) >= category.shape[1])):
                raise ValueError(f"category must be a float32 ({n}, L) tensor on {self.device} with unit column stride "
                                 "and row stride >= L")
            check_encoder_layout(cnn, n_category=category.shape[1])
        else:
            check_encoder_layout(cnn)
        keep, layers, lw, lb, features, out = self._conv_stack_args(cnn, n, H, W, features)
        if n == 0:                    # empty tensors have NULL data pointers, which the library refuses
            return out
        lin = cnn[6]
        if category is None:
            self.ctx.check(self.lib.ssb_audio_encoder_batch(
                self.ctx.handle, n, spec.data_ptr(), H, W, layers, lw.data_ptr(), lb.data_ptr() if lb is not None else None,
                lin.out_features, 1, features.data_ptr(), out.data_ptr(), self._stream()), "ssb_audio_encoder_batch")
        else:
            L = category.shape[1]         # a one-row tensor may report any row stride; only row 0 is read
            self.ctx.check(self.lib.ssb_audio_encoder_category_batch(
                self.ctx.handle, n, spec.data_ptr(), H, W, layers, category.data_ptr() if L else None, L,
                max(category.stride(0), L), lw.data_ptr(), lb.data_ptr() if lb is not None else None, lin.out_features,
                1, features.data_ptr(), out.data_ptr(), self._stream()), "ssb_audio_encoder_category_batch")
        return out

    def _conv_stack_args(self, cnn, n, H, W, features):
        """The ``ssb_conv2d_layer`` array of a checked ``Conv2d ReLU Conv2d ReLU Conv2d Flatten Linear ReLU`` for an
        H x W input, with the tensors it points into, the Linear's weight and bias, the (n, F) features and the
        (n, hidden) output buffer."""
        h, w = H, W
        keep, layers = [], (_lib.Conv2dLayer * 3)()
        for i, (conv, relu) in enumerate(((cnn[0], 1), (cnn[2], 1), (cnn[4], 0))):
            (kh, kw), (sh, sw) = conv.kernel_size, conv.stride
            h, w = (h - kh) // sh + 1, (w - kw) // sw + 1
            if h < 1 or w < 1:
                raise ValueError(f"layer {i + 1} output is empty for a {H}x{W} observation")
            wt = conv.weight.detach().to(self.device, torch.float32).contiguous()
            b = conv.bias.detach().to(self.device, torch.float32).contiguous() if conv.bias is not None else None
            keep += [wt, b]
            layers[i] = _lib.Conv2dLayer(wt.data_ptr(), b.data_ptr() if b is not None else None, conv.out_channels,
                                         kh, kw, sh, sw, relu)
        lin = cnn[6]
        F = cnn[4].out_channels * h * w
        if lin.in_features != F:
            raise ValueError(f"Linear.in_features is {lin.in_features}; conv3 yields {F} features for a {H}x{W} input")
        lw = lin.weight.detach().to(self.device, torch.float32).contiguous()
        lb = lin.bias.detach().to(self.device, torch.float32).contiguous() if lin.bias is not None else None
        if features is None:
            features = torch.empty((n, F), dtype=torch.float32, device=self.device)
        elif not (features.is_cuda and features.dtype == torch.float32 and features.is_contiguous()
                  and tuple(features.shape) == (n, F)):
            raise ValueError(f"features must be a contiguous CUDA float32 ({n}, {F}) tensor")
        out = torch.empty((n, lin.out_features), dtype=torch.float32, device=self.device)
        return keep, layers, lw, lb, features, out

    @torch.no_grad()
    def visual_encoder(self, rgb: Optional[torch.Tensor], depth: Optional[torch.Tensor], cnn: "torch.nn.Sequential",
                       features: Optional[torch.Tensor] = None) -> torch.Tensor:
        """``VisualCNN.cnn(cat(rgb.permute(0, 3, 1, 2) / 255.0, depth.permute(0, 3, 1, 2)))`` (visual_cnn.py: Conv2d
        ReLU Conv2d ReLU Conv2d Flatten Linear ReLU) straight from the (n, H, W, C_rgb) and (n, H, W, C_depth)
        observations in two launches -> (n, hidden).  Either input may be None (not both).  Inference only.
        ``features``: optional (n, F) float32 CUDA tensor that receives the flattened conv3 output.  ``ValueError``
        for other tensors or layouts (:func:`soundspaces_b200.encoder.conv_stack_layout_error` with
        C_rgb + C_depth input channels); ``RuntimeError`` when the library refuses the shape
        (``ssb_visual_encoder_batch``)."""
        present = [t for t in (rgb, depth) if t is not None]
        if not present:
            raise ValueError("visual_encoder needs rgb, depth or both")
        n, H, W = present[0].shape[:3] if present[0].ndim == 4 else (0, 0, 0)
        for t in present:
            if not (isinstance(t, torch.Tensor) and t.device == self.device and t.dtype == torch.float32 and t.ndim == 4
                    and tuple(t.shape[:3]) == (n, H, W) and t.shape[3] >= 1 and t.is_contiguous()):
                raise ValueError(f"expected contiguous float32 (n, H, W, C) observations on {self.device} with the "
                                 "same n, H and W")
        n_rgb = rgb.shape[3] if rgb is not None else 0
        n_depth = depth.shape[3] if depth is not None else 0
        err = conv_stack_layout_error(cnn, n_rgb + n_depth)
        if err:
            raise ValueError(f"visual_encoder fuses VisualCNN.cnn = Conv2d({n_rgb + n_depth} -> C1) ReLU Conv2d ReLU "
                             "Conv2d Flatten Linear ReLU: " + err)
        keep, layers, lw, lb, features, out = self._conv_stack_args(cnn, n, H, W, features)
        if n == 0:                    # empty tensors have NULL data pointers, which the library refuses
            return out
        self.ctx.check(self.lib.ssb_visual_encoder_batch(
            self.ctx.handle, n, rgb.data_ptr() if rgb is not None else None, n_rgb,
            depth.data_ptr() if depth is not None else None, n_depth, H, W, layers, lw.data_ptr(),
            lb.data_ptr() if lb is not None else None, cnn[6].out_features, 1, features.data_ptr(), out.data_ptr(),
            self._stream()), "ssb_visual_encoder_batch")
        return out

    @torch.no_grad()
    def map_encoder(self, x: torch.Tensor, cnn: "torch.nn.Sequential",
                    features: Optional[torch.Tensor] = None) -> torch.Tensor:
        """``MapCNN.cnn(x.permute(0, 3, 1, 2))`` (av_wan/models/map_cnn.py: Conv2d ReLU Conv2d ReLU Conv2d Flatten
        Linear ReLU) straight from the (n, H, W, C) geometric or acoustic map in two launches -> (n, hidden).
        Inference only.  ``features``: optional (n, F) float32 CUDA tensor that receives the flattened conv3 output.
        ``ValueError`` for other tensors or layouts (:func:`soundspaces_b200.encoder.conv_stack_layout_error` with C
        input channels); ``RuntimeError`` when the library refuses the shape (``ssb_map_encoder_batch``)."""
        if not (isinstance(x, torch.Tensor) and x.device == self.device and x.dtype == torch.float32 and x.ndim == 4
                and x.shape[3] >= 1 and x.is_contiguous()):
            raise ValueError(f"expected a contiguous float32 (n, H, W, C) map on {self.device}")
        n, H, W, C = x.shape
        err = conv_stack_layout_error(cnn, C)
        if err:
            raise ValueError(f"map_encoder fuses MapCNN.cnn = Conv2d({C} -> C1) ReLU Conv2d ReLU Conv2d Flatten Linear "
                             "ReLU: " + err)
        keep, layers, lw, lb, features, out = self._conv_stack_args(cnn, n, H, W, features)
        if n == 0:                    # empty tensors have NULL data pointers, which the library refuses
            return out
        self.ctx.check(self.lib.ssb_map_encoder_batch(
            self.ctx.handle, n, x.data_ptr(), C, H, W, layers, lw.data_ptr(), lb.data_ptr() if lb is not None else None,
            cnn[6].out_features, 1, features.data_ptr(), out.data_ptr(), self._stream()), "ssb_map_encoder_batch")
        return out

    def _conv_stack_train_args(self, kind, x, depth, labels, params, strides):
        """The ``ssb_conv_stack_input`` and ``ssb_conv2d_layer`` array of a conv-stack call, with B and the Linear's
        sizes.  ``params``: (w1, b1, w2, b2, w3, b3, w_lin, b_lin), biases optional; ``strides``: conv1-3's (sh, sw)."""
        first = x if x is not None else depth
        B, H, W = first.shape[:3]
        inp = _lib.ConvStackInput()
        inp.kind, inp.H, inp.W = kind, H, W
        inp.d_x = x.data_ptr() if x is not None and B else None
        inp.channels = x.shape[3] if x is not None else 0
        if depth is not None:
            inp.d_depth, inp.n_depth = depth.data_ptr() if B else None, depth.shape[3]
        if labels is not None:
            inp.d_labels, inp.n_labels = labels.data_ptr() if B else None, labels.shape[1]
            inp.label_stride = max(labels.stride(0), labels.shape[1])
        layers = (_lib.Conv2dLayer * 3)()
        for i in range(3):
            w, b = params[2 * i], params[2 * i + 1]
            layers[i] = _lib.Conv2dLayer(w.data_ptr(), b.data_ptr() if b is not None else None, w.shape[0],
                                         w.shape[2], w.shape[3], strides[i][0], strides[i][1], int(i < 2))
        hidden, F = params[6].shape
        return B, inp, layers, F, hidden

    def _conv_stack_workspace(self, B, inp, layers, F, hidden, backward):
        nbytes = int(self.lib.ssb_conv_stack_train_workspace_bytes(B, C.byref(inp), layers, F, hidden, int(backward)))
        if nbytes < 0:
            raise RuntimeError("conv_stack_train: the library refuses this shape "
                               "(ssb_conv_stack_train_workspace_bytes, include/ssb200.h)")
        return torch.empty(max(nbytes, 16), dtype=torch.uint8, device=self.device)

    @torch.no_grad()
    def conv_stack_train_forward(self, kind: int, x: Optional[torch.Tensor], depth: Optional[torch.Tensor],
                                 labels: Optional[torch.Tensor], params, strides):
        """``Conv2d ReLU Conv2d ReLU Conv2d Flatten Linear ReLU`` of an encoder's ``cnn`` on the current stream
        (``ssb_conv_stack_train_forward_batch``, 4 launches, 5 with labels).  ``kind``: ``_lib.CONV_INPUT_*``; x the
        (B, H, W, C) spectrogram, RGB or map, ``depth`` VisualCNN's depth, ``labels`` SAVi's (B, L) category, each
        contiguous float32 on this device (x or depth may be None for a visual input).  -> (out (B, hidden),
        features (B, F), saved): ``saved`` is the workspace holding conv1's and conv2's outputs, which
        :meth:`conv_stack_train_backward` reads.  ``RuntimeError`` when the library refuses the call."""
        B, inp, layers, F, hidden = self._conv_stack_train_args(kind, x, depth, labels, params, strides)
        features = torch.empty((B, F), dtype=torch.float32, device=self.device)
        out = torch.empty((B, hidden), dtype=torch.float32, device=self.device)
        saved = self._conv_stack_workspace(B, inp, layers, F, hidden, False)
        lb = params[7]
        self.ctx.check(self.lib.ssb_conv_stack_train_forward_batch(
            self.ctx.handle, B, C.byref(inp), layers, params[6].data_ptr(), lb.data_ptr() if lb is not None else None,
            F, hidden, 1, features.data_ptr(), out.data_ptr(), saved.data_ptr(), self._stream()),
            "ssb_conv_stack_train_forward_batch")
        return out, features, saved

    @torch.no_grad()
    def conv_stack_train_backward(self, kind: int, x, depth, labels, params, strides, features: torch.Tensor,
                                  out: torch.Tensor, saved: torch.Tensor, grad_out: torch.Tensor, need=(True,) * 8):
        """The backward of :meth:`conv_stack_train_forward` (``ssb_conv_stack_train_backward_batch``) from its
        features, out and saved workspace and the (B, hidden) gradient of out.  ``need``: which of the eight parameter
        gradients (w1, b1, w2, b2, w3, b3, w_lin, b_lin) to compute.  -> those eight, None where not needed."""
        B, inp, layers, F, hidden = self._conv_stack_train_args(kind, x, depth, labels, params, strides)
        grads = [torch.empty_like(p) if n and p is not None else None for p, n in zip(params, need)]
        if B == 0 or not any(g is not None for g in grads):
            return tuple(grads)
        ws = self._conv_stack_workspace(B, inp, layers, F, hidden, True)
        ptr = lambda t: None if t is None else t.data_ptr()                   # noqa: E731
        dw = (C.c_void_p * 4)(*[ptr(g) for g in grads[0::2]])
        db = (C.c_void_p * 4)(*[ptr(g) for g in grads[1::2]])
        self.ctx.check(self.lib.ssb_conv_stack_train_backward_batch(
            self.ctx.handle, B, C.byref(inp), layers, params[6].data_ptr(), F, hidden, 1, features.data_ptr(),
            out.data_ptr(), saved.data_ptr(), grad_out.data_ptr(), ws.data_ptr(), dw, db, self._stream()),
            "ssb_conv_stack_train_backward_batch")
        return tuple(grads)

    def map_update(self, geometry: "_lib.MapGeometry", gmap: torch.Tensor, amap: torch.Tensor, records: np.ndarray,
                   ego: np.ndarray) -> None:
        """Replay AV-WaN map-update records (``soundspaces_b200.maps.RECORD_DTYPE``, host) into the device maps
        ``gmap`` (uint8 (n_slots, pitch)) and ``amap`` (float64 (n_slots, M, M)) in one launch; ``ego``: host uint8
        bytes the records' ``ego_offset`` point into.  ``RuntimeError`` when the library refuses a record
        (``ssb_map_update_batch``)."""
        records = np.ascontiguousarray(records)
        ego = np.ascontiguousarray(ego, dtype=np.uint8)
        self.ctx.check(self.lib.ssb_map_update_batch(
            self.ctx.handle, C.byref(geometry), gmap.data_ptr(), amap.data_ptr(), len(records),
            records.ctypes.data if len(records) else None, ego.ctypes.data if ego.size else None, ego.size,
            self._stream()), "ssb_map_update_batch")

    def map_update_device_intensity(self, geometry: "_lib.MapGeometry", gmap: torch.Tensor, amap: torch.Tensor,
                                    records: np.ndarray, ego: np.ndarray, intensity: torch.Tensor) -> None:
        """:meth:`map_update` with the acoustic values on the device: with an acoustic map, an update record's value is
        ``intensity[record.reserved]`` (``intensity``: contiguous float32 on this device), applied in float64 with
        half = 0.5 * value (``ssb_map_update_device_intensity_batch``)."""
        if not (intensity.device == self.device and intensity.dtype == torch.float32 and intensity.ndim == 1
                and intensity.is_contiguous()):
            raise ValueError(f"intensity must be a contiguous float32 1-d tensor on {self.device}")
        records = np.ascontiguousarray(records)
        ego = np.ascontiguousarray(ego, dtype=np.uint8)
        self.ctx.check(self.lib.ssb_map_update_device_intensity_batch(
            self.ctx.handle, C.byref(geometry), gmap.data_ptr(), amap.data_ptr(), len(records),
            records.ctypes.data if len(records) else None, ego.ctypes.data if ego.size else None, ego.size,
            intensity.data_ptr() if intensity.numel() else None, intensity.numel(), self._stream()),
            "ssb_map_update_device_intensity_batch")

    def map_observe(self, geometry: "_lib.MapGeometry", gmap: torch.Tensor, amap: torch.Tensor, poses: np.ndarray,
                    tables: np.ndarray, gm: Optional[torch.Tensor] = None, am: Optional[torch.Tensor] = None,
                    action: Optional[torch.Tensor] = None) -> None:
        """Write the egocentric ``gm`` / ``am`` / ``action`` maps (each optional, float32 on this device with
        contiguous rows) of the envs at ``poses`` (host int32 (B, 4): slot, x, y, orientation) in one launch;
        ``tables``: host int32 (4, 2, L) navigable xs / ys (``ssb_map_observe_batch``)."""
        poses = np.ascontiguousarray(poses, dtype=np.int32)
        tables = np.ascontiguousarray(tables, dtype=np.int32)
        B = poses.shape[0]

        def arg(t):
            if t is None or B == 0:
                return None, 0
            return t.data_ptr(), t.stride(0) if B > 1 else t[0].numel()
        (g_p, g_s), (a_p, a_s), (x_p, x_s) = arg(gm), arg(am), arg(action)
        self.ctx.check(self.lib.ssb_map_observe_batch(
            self.ctx.handle, C.byref(geometry), gmap.data_ptr(), amap.data_ptr(), B, poses.ctypes.data if B else None,
            tables.ctypes.data, tables.shape[2], g_p, g_s, a_p, a_s, x_p, x_s, self._stream()),
            "ssb_map_observe_batch")

    @torch.no_grad()
    def gru_step(self, x: torch.Tensor, h: torch.Tensor, masks: torch.Tensor, rnn: "torch.nn.GRU"):
        """One step of ``rnn`` (a one-layer, unidirectional ``nn.GRU`` with bias) on ``masks * h``: x (n, I), h (n, Hd),
        masks n values (``(n, 1)`` as RNNStateEncoder passes them) -> (out, h_out), two distinct (n, Hd) tensors with
        equal values (``ssb_gru_step_batch``, one launch).  Inference only.  ``ValueError`` for any other tensor or
        module (:func:`soundspaces_b200.rnn.gru_layout_error`)."""
        from .rnn import gru_layout_error
        err = gru_layout_error(rnn)
        if err:
            raise ValueError("gru_step fuses a one-layer unidirectional nn.GRU with bias: " + err)
        n, Hd, I = x.shape[0] if x.ndim == 2 else -1, rnn.hidden_size, rnn.input_size
        want = {"x": (x, (n, I)), "h": (h, (n, Hd)), "masks": (masks, None)}
        for name, (t, shape) in want.items():
            if not (isinstance(t, torch.Tensor) and t.device == self.device and t.dtype == torch.float32
                    and t.is_contiguous() and (shape is None or tuple(t.shape) == shape)):
                raise ValueError(f"{name} must be a contiguous float32 tensor on {self.device}"
                                 + (f" of shape {shape}" if shape else ""))
        if masks.numel() != n:
            raise ValueError(f"masks must hold {n} values")
        params = [rnn.weight_ih_l0, rnn.weight_hh_l0, rnn.bias_ih_l0, rnn.bias_hh_l0]
        for p in params:
            if not (p.device == self.device and p.dtype == torch.float32 and p.is_contiguous()):
                raise ValueError(f"the GRU's parameters must be contiguous float32 tensors on {self.device}")
        out = torch.empty((n, Hd), dtype=torch.float32, device=self.device)
        h_out = torch.empty((n, Hd), dtype=torch.float32, device=self.device)
        if n == 0:                    # empty tensors have NULL data pointers, which the library refuses
            return out, h_out
        self.ctx.check(self.lib.ssb_gru_step_batch(
            self.ctx.handle, n, I, Hd, x.data_ptr(), h.data_ptr(), masks.data_ptr(),
            *[p.data_ptr() for p in params], out.data_ptr(), h_out.data_ptr(), self._stream()), "ssb_gru_step_batch")
        return out, h_out

    def _gru_seq_check(self, what, tensors, sizes):
        """Every tensor a contiguous float32 tensor on this device holding ``sizes[name]`` values."""
        for name, t in tensors.items():
            if not (isinstance(t, torch.Tensor) and t.device == self.device and t.dtype == torch.float32
                    and t.is_contiguous()):
                raise ValueError(f"{what}: {name} must be a contiguous float32 tensor on {self.device}")
            if t.numel() != sizes[name]:
                raise ValueError(f"{what}: {name} has shape {tuple(t.shape)}, expected {sizes[name]} values")

    def _gru_seq_workspace(self, T, N, I, Hd):
        nbytes = int(self.lib.ssb_gru_seq_workspace_bytes(T, N, I, Hd))
        if nbytes < 0:
            raise RuntimeError(f"gru_seq: T={T} N={N} I={I} Hd={Hd} is outside the library's limits")
        return torch.empty(nbytes, dtype=torch.uint8, device=self.device)

    @staticmethod
    def _gru_seq_dims(x, N, w_ih, w_hh, what):
        Hd, I = (w_hh.shape[1], w_ih.shape[1]) if w_hh.ndim == 2 and w_ih.ndim == 2 else (0, 0)
        if x.ndim != 2 or N < 1 or x.shape[0] % N or x.shape[1] != I or w_hh.shape[0] != 3 * Hd:
            raise ValueError(f"{what}: x {tuple(x.shape)}, N={N}, weight_ih {tuple(w_ih.shape)} and weight_hh "
                             f"{tuple(w_hh.shape)} disagree")
        return x.shape[0] // N, I, Hd

    @torch.no_grad()
    def gru_seq_forward(self, x: torch.Tensor, h0: torch.Tensor, masks: torch.Tensor, params, save: bool = False):
        """``RNNStateEncoder.seq_forward``'s arithmetic on the current stream (``ssb_gru_seq_forward_batch``, two
        launches): x (T N, I), h0 (1, N, Hd), masks T N values, ``params`` the GRU's (weight_ih_l0, weight_hh_l0,
        bias_ih_l0, bias_hh_l0), all contiguous float32 on this device.  -> (out (T N, Hd), h_last (1, N, Hd), saved),
        saved the (5, T N, Hd) state :meth:`gru_seq_backward` takes when ``save``, else None.  ``ValueError`` for other
        tensors; ``RuntimeError`` when the library refuses the shape."""
        w_ih, w_hh, b_ih, b_hh = params
        N = h0.shape[1] if h0.ndim == 3 else 0
        T, I, Hd = self._gru_seq_dims(x, N, w_ih, w_hh, "gru_seq_forward")
        self._gru_seq_check("gru_seq_forward", dict(x=x, h0=h0, masks=masks, w_ih=w_ih, w_hh=w_hh, b_ih=b_ih, b_hh=b_hh),
                            dict(x=T * N * I, h0=N * Hd, masks=T * N, w_ih=3 * Hd * I, w_hh=3 * Hd * Hd, b_ih=3 * Hd,
                                 b_hh=3 * Hd))
        ws = self._gru_seq_workspace(T, N, I, Hd)
        out = torch.empty((T * N, Hd), dtype=torch.float32, device=self.device)
        h_last = torch.empty((1, N, Hd), dtype=torch.float32, device=self.device)
        saved = torch.empty((5, T * N, Hd), dtype=torch.float32, device=self.device) if save else None
        self.ctx.check(self.lib.ssb_gru_seq_forward_batch(
            self.ctx.handle, T, N, I, Hd, x.data_ptr(), h0.data_ptr(), masks.data_ptr(),
            *[p.data_ptr() for p in params], out.data_ptr(), h_last.data_ptr(),
            saved.data_ptr() if save else None, ws.data_ptr(), self._stream()), "ssb_gru_seq_forward_batch")
        return out, h_last, saved

    @torch.no_grad()
    def gru_seq_backward(self, x: torch.Tensor, N: int, masks: torch.Tensor, w_ih: torch.Tensor, w_hh: torch.Tensor,
                         saved: torch.Tensor, grad_out: Optional[torch.Tensor], grad_h_last: Optional[torch.Tensor],
                         need=(True,) * 6):
        """The backward of :meth:`gru_seq_forward` for N envs on the current stream (``ssb_gru_seq_backward_batch``)
        from its ``saved`` state and the gradients of out (T N, Hd) and h_last (1, N, Hd), either None for zero;
        contiguous float32 on this device.  ``need``: which of (dx, dh0, dw_ih, dw_hh, db_ih, db_hh) to compute.
        -> those six, each None when not needed, dh0 (1, N, Hd)."""
        T, I, Hd = self._gru_seq_dims(x, N, w_ih, w_hh, "gru_seq_backward")
        tensors = dict(x=x, masks=masks, w_ih=w_ih, w_hh=w_hh, saved=saved)
        sizes = dict(x=T * N * I, masks=T * N, w_ih=3 * Hd * I, w_hh=3 * Hd * Hd, saved=5 * T * N * Hd,
                     grad_out=T * N * Hd, grad_h_last=N * Hd)
        for name, g in (("grad_out", grad_out), ("grad_h_last", grad_h_last)):
            if g is not None:
                tensors[name] = g
        self._gru_seq_check("gru_seq_backward", tensors, sizes)
        shapes = ((T * N, I), (1, N, Hd), (3 * Hd, I), (3 * Hd, Hd), (3 * Hd,), (3 * Hd,))
        grads = [torch.empty(s, dtype=torch.float32, device=self.device) if n else None for s, n in zip(shapes, need)]
        if not any(need):
            return tuple(grads)
        ws = self._gru_seq_workspace(T, N, I, Hd)
        ptr = lambda t: None if t is None else t.data_ptr()                  # noqa: E731
        self.ctx.check(self.lib.ssb_gru_seq_backward_batch(
            self.ctx.handle, T, N, I, Hd, x.data_ptr(), masks.data_ptr(), w_ih.data_ptr(), w_hh.data_ptr(),
            saved.data_ptr(), ptr(grad_out), ptr(grad_h_last), ws.data_ptr(), *[ptr(g) for g in grads],
            self._stream()), "ssb_gru_seq_backward_batch")
        return tuple(grads)

    @torch.no_grad()
    def policy_head(self, features: torch.Tensor, actor: "torch.nn.Linear", critic: "torch.nn.Linear",
                    masked: bool = False, mask: Optional[torch.Tensor] = None, q: Optional[torch.Tensor] = None,
                    want_probs: bool = False):
        """A policy's action and value heads on ``features`` (n, H) in one launch (``ssb_policy_head_batch``):
        ``actor`` the ``nn.Linear(H, A)`` of CategoricalNet (``masked`` False) or CategoricalNetWithMask (``masked``
        True, ``mask`` (n, A) or None when masking is off), ``critic`` CriticHead's ``nn.Linear(H, 1)``; ``q`` (n, A)
        the Exp(1) draws of ``torch.multinomial``'s single-sample path, None for the mode.  All contiguous float32 on
        this device.  -> (value (n, 1), action (n, 1) int64, log_prob (n, 1), probs (n, A) or None, status (1,) int32
        on the device: the number of rows the reference would refuse, whose action is -1).  Nothing is read back.
        ``ValueError`` for other tensors or modules; ``RuntimeError`` when the library refuses the shape."""
        if not (isinstance(features, torch.Tensor) and features.device == self.device
                and features.dtype == torch.float32 and features.ndim == 2 and features.is_contiguous()):
            raise ValueError(f"features must be a contiguous float32 (n, H) tensor on {self.device}")
        (n, H), A = features.shape, actor.out_features
        for name, lin, rows in (("actor", actor, A), ("critic", critic, 1)):
            if not (isinstance(lin, torch.nn.Linear) and lin.bias is not None and lin.in_features == H
                    and lin.out_features == rows):
                raise ValueError(f"{name} must be an nn.Linear({H}, {rows}) with bias")
            for p in (lin.weight, lin.bias):
                if not (p.device == self.device and p.dtype == torch.float32 and p.is_contiguous()):
                    raise ValueError(f"the {name}'s parameters must be contiguous float32 tensors on {self.device}")
        for name, t in (("mask", mask), ("q", q)):
            if t is not None and not (isinstance(t, torch.Tensor) and t.device == self.device
                                      and t.dtype == torch.float32 and tuple(t.shape) == (n, A) and t.is_contiguous()):
                raise ValueError(f"{name} must be a contiguous float32 ({n}, {A}) tensor on {self.device}")
        if mask is not None and not masked:
            raise ValueError("a mask needs the masked head")
        value = torch.empty((n, 1), dtype=torch.float32, device=self.device)
        action = torch.empty((n, 1), dtype=torch.int64, device=self.device)
        log_prob = torch.empty((n, 1), dtype=torch.float32, device=self.device)
        probs = torch.empty((n, A), dtype=torch.float32, device=self.device) if want_probs else None
        status = torch.empty(1, dtype=torch.int32, device=self.device)
        if n == 0:                    # empty tensors have NULL data pointers, which the library refuses
            status.zero_()
            return value, action, log_prob, probs, status
        self.ctx.check(self.lib.ssb_policy_head_batch(
            self.ctx.handle, n, H, A, features.data_ptr(), actor.weight.data_ptr(), actor.bias.data_ptr(),
            critic.weight.data_ptr(), critic.bias.data_ptr(), int(bool(masked)),
            mask.data_ptr() if mask is not None else None, q.data_ptr() if q is not None else None,
            value.data_ptr(), action.data_ptr(), log_prob.data_ptr(), probs.data_ptr() if probs is not None else None,
            status.data_ptr(), self._stream()), "ssb_policy_head_batch")
        return value, action, log_prob, probs, status

    @torch.no_grad()
    def policy_head_train_forward(self, features: torch.Tensor, actor: "torch.nn.Linear", critic: "torch.nn.Linear",
                                  masked: bool, mask: Optional[torch.Tensor], action: torch.Tensor):
        """The heads of ``evaluate_actions`` on ``features`` (n, H) for the given ``action`` (n, 1) int64 in one launch
        (``ssb_policy_head_train_forward_batch``); modules and ``mask`` as :meth:`policy_head`, all contiguous on this
        device, checked by the caller (:func:`soundspaces_b200.policy._evaluate_inputs`).  -> (value (n, 1),
        log_prob (n, 1), entropy (n,), saved (n, A) for the backward, status (1,) int32 on the device: the number of
        refused rows, whose outputs are NaN).  Nothing is read back."""
        (n, H), A = features.shape, actor.out_features
        new = lambda *s: torch.empty(s, dtype=torch.float32, device=self.device)   # noqa: E731
        value, log_prob, entropy, saved = new(n, 1), new(n, 1), new(n), new(n, A)
        status = torch.empty(1, dtype=torch.int32, device=self.device)
        if n == 0:
            return value, log_prob, entropy, saved, status.zero_()
        self.ctx.check(self.lib.ssb_policy_head_train_forward_batch(
            self.ctx.handle, n, H, A, features.data_ptr(), actor.weight.data_ptr(), actor.bias.data_ptr(),
            critic.weight.data_ptr(), critic.bias.data_ptr(), int(bool(masked)),
            mask.data_ptr() if mask is not None else None, action.data_ptr(), value.data_ptr(), log_prob.data_ptr(),
            entropy.data_ptr(), saved.data_ptr(), status.data_ptr(), self._stream()),
            "ssb_policy_head_train_forward_batch")
        return value, log_prob, entropy, saved, status

    @torch.no_grad()
    def policy_head_train_backward(self, features: torch.Tensor, actor_weight: torch.Tensor,
                                   critic_weight: torch.Tensor, masked: bool, mask: Optional[torch.Tensor],
                                   action: torch.Tensor,
                                   saved: torch.Tensor, grad_value: torch.Tensor, grad_log_prob: torch.Tensor,
                                   grad_entropy: torch.Tensor, need=(True,) * 5):
        """The backward of :meth:`policy_head_train_forward` (``ssb_policy_head_train_backward_batch``, at most two
        launches) from its ``saved`` rows, the heads' weights and the gradients of value, log_prob and entropy
        (n values each).  ``need``:
        which of (features, actor weight, actor bias, critic weight, critic bias) to compute -> those gradients, None
        where not needed."""
        (n, H), A = features.shape, actor_weight.shape[0]
        shapes = ((n, H), (A, H), (A,), (1, H), (1,))
        grads = [torch.empty(s, dtype=torch.float32, device=self.device) if w else None for s, w in zip(shapes, need)]
        if n == 0 or not any(need):
            return tuple(g.zero_() if g is not None else None for g in grads)
        ws = self._train_workspace(self.lib.ssb_policy_head_train_workspace_bytes(n, H, A))
        gv, glp, gh = (g.reshape(n).float().contiguous() for g in (grad_value, grad_log_prob, grad_entropy))
        ptr = lambda t: None if t is None else t.data_ptr()                  # noqa: E731
        self.ctx.check(self.lib.ssb_policy_head_train_backward_batch(
            self.ctx.handle, n, H, A, features.data_ptr(), actor_weight.data_ptr(), critic_weight.data_ptr(),
            int(bool(masked)), ptr(mask), action.data_ptr(), saved.data_ptr(), gv.data_ptr(), glp.data_ptr(),
            gh.data_ptr(), ws.data_ptr(), *[ptr(g) for g in grads], self._stream()),
            "ssb_policy_head_train_backward_batch")
        return tuple(grads)

    @staticmethod
    def _rollout_fields(fields):
        """ctypes array of ``ssb_rollout_field`` from (src_ptr, dst_ptr, row_bytes, src_t_stride, src_outer_stride,
        T, outer[, on_host]) tuples (pointers and strides in bytes)."""
        return (_lib.RolloutField * max(1, len(fields)))(*[_lib.RolloutField(*f) for f in fields])

    def rollout_insert(self, n: int, fields, memory: Optional[dict] = None) -> None:
        """One ``RolloutStorage.insert`` of ``n`` envs in one launch (``ssb_rollout_insert_batch``): ``fields`` as in
        :meth:`_rollout_fields`, copied on this device; a field with ``on_host`` reads host memory, which the library
        stages through its pinned ring.  ``memory``: SAVi's external-memory update, a dict of ``masks`` (n, total),
        ``not_done`` (n float32 values on this device or the CPU), ``em_masks_out`` ((n, total) or None), ``status``
        ((1 + n,) int32), ``capacity``, ``idx`` and ``step``.  Nothing is read back; the pointers are the caller's to
        keep valid until the call returns (host sources) or the launch has run (device ones)."""
        em = None
        if memory is not None:
            nd, out = memory["not_done"], memory["em_masks_out"]
            em = _lib.RolloutMemory(memory["masks"].data_ptr(), nd.data_ptr(),
                                    out.data_ptr() if out is not None else None, memory["status"].data_ptr(),
                                    memory["masks"].shape[1], memory["capacity"], memory["idx"], memory["step"],
                                    int(nd.device.type == "cpu"), 0)
        self.ctx.check(self.lib.ssb_rollout_insert_batch(
            self.ctx.handle, n, self._rollout_fields(fields), len(fields), C.byref(em) if em is not None else None,
            self._stream()), "ssb_rollout_insert_batch")

    def rollout_returns(self, rewards, value_preds, returns, masks, next_value, T: int, use_gae: bool, gamma: float,
                        tau: float, adv: Optional[torch.Tensor] = None, normalize: bool = True,
                        scan: bool = True) -> None:
        """``compute_returns`` over steps ``[0, T)`` of (S + 1, n, 1) float32 storage (``ssb_rollout_returns_batch``),
        then with ``adv`` (S, n, 1) the advantages ``returns[:S] - value_preds[:S]``, normalised when asked.  With
        ``scan`` False only the advantages.  gamma and gamma * tau are rounded to float32 here, as torch rounds a
        Python scalar it multiplies a float32 tensor by."""
        S, n = value_preds.shape[0] - 1, value_preds.shape[1]
        ptr = lambda t: t.data_ptr() if t is not None else None  # noqa: E731
        self.ctx.check(self.lib.ssb_rollout_returns_batch(
            self.ctx.handle, n, S, int(T), int(bool(scan)), int(bool(use_gae)), float(gamma), float(gamma * tau),
            ptr(rewards), value_preds.data_ptr(), returns.data_ptr(), ptr(masks), ptr(next_value), ptr(adv),
            int(bool(normalize)), self._stream()), "ssb_rollout_returns_batch")

    def rollout_gather(self, fields, n_cols: int, cols: Optional[Sequence[int]] = None, max_col: int = 0) -> None:
        """One minibatch of ``recurrent_generator`` (``cols`` the env columns, each below ``max_col``) or
        ``after_update``'s copies (``cols`` None: columns 0 .. n_cols-1) in one launch (``ssb_rollout_gather_batch``)."""
        h_cols = (C.c_int64 * len(cols))(*cols) if cols is not None else None
        self.ctx.check(self.lib.ssb_rollout_gather_batch(
            self.ctx.handle, self._rollout_fields(fields), len(fields), int(n_cols), h_cols, int(max_col),
            self._stream()), "ssb_rollout_gather_batch")

    def _resnet_input(self, x, what):
        if not (isinstance(x, torch.Tensor) and x.device == self.device and x.dtype == torch.float32 and x.ndim == 4
                and x.shape[3] == 2 and x.is_contiguous()):
            raise ValueError(f"{what}: expected a contiguous float32 (B, H, W, 2) observation on {self.device}")
        return x.shape[:3]

    @torch.no_grad()
    def resnet18(self, x: torch.Tensor, net: "torch.nn.Module") -> torch.Tensor:
        """``net(x.permute(0, 3, 1, 2))`` for SAVi's torchvision ResNet-18s (belief_predictor.py:73-80: the label
        classifier, and the location predictor without online training) in eval mode, straight from the (B, H, W, 2)
        observation, on the current stream -> (B, fc.out_features).  ``ssb_resnet18_batch``, 39 launches.
        ``ValueError`` for any other layout (:func:`soundspaces_b200.belief_nets.resnet18_layout_error`)."""
        B, H, W = self._resnet_input(x, "resnet18")
        err = belief_nets.resnet18_layout_error(net, self.device)
        if err:
            raise ValueError("resnet18: " + err)
        fc = net.fc
        out = torch.empty((B, fc.out_features), dtype=torch.float32, device=self.device)
        self.ctx.check(self.lib.ssb_resnet18_batch(
            self.ctx.handle, B, x.data_ptr(), H, W, belief_nets.conv_table(net, True), fc.weight.data_ptr(),
            fc.bias.data_ptr() if fc.bias is not None else None, fc.in_features, fc.out_features, out.data_ptr(),
            self._stream()), "ssb_resnet18_batch")
        return out

    @torch.no_grad()
    def smt_resnet18(self, x: torch.Tensor, net: "torch.nn.Module", labels: Optional[torch.Tensor] = None) -> torch.Tensor:
        """SAVi's online-trained location predictor (smt_resnet.py ``custom_resnet18``, belief_predictor.py:66-71) on
        ``x.permute(0, 3, 1, 2)``, with ``labels`` (B, L) broadcast over the pixels and concatenated after the two ears
        when given (``cnn_forward``, :123-134), on the current stream -> (B, fc.out_features).
        ``ssb_smt_resnet18_batch``, 38 launches.  ``labels``: float32 on this device with unit column stride.
        ``ValueError`` for any other layout (:func:`soundspaces_b200.belief_nets.smt_resnet18_layout_error`)."""
        B, H, W = self._resnet_input(x, "smt_resnet18")
        L = 0
        if labels is not None:
            L = labels.shape[1] if isinstance(labels, torch.Tensor) and labels.ndim == 2 else -1
            if L < 0 or not belief_nets.fusable_labels(labels, x, L):
                raise ValueError(f"smt_resnet18: labels must be a float32 ({B}, L) tensor on {self.device} with unit "
                                 "column stride and row stride >= L")
        err = belief_nets.smt_resnet18_layout_error(net, 2 + L, (H, W), self.device)
        if err:
            raise ValueError("smt_resnet18: " + err)
        fc = net.fc
        out = torch.empty((B, fc.out_features), dtype=torch.float32, device=self.device)
        self.ctx.check(self.lib.ssb_smt_resnet18_batch(
            self.ctx.handle, B, x.data_ptr(), H, W, labels.data_ptr() if L else None, L,
            max(labels.stride(0), L) if L else 0, belief_nets.conv_table(net, False), fc.weight.data_ptr(),
            fc.bias.data_ptr() if fc.bias is not None else None, fc.in_features, fc.out_features, out.data_ptr(),
            self._stream()), "ssb_smt_resnet18_batch")
        return out

    def _smt_train_args(self, x, labels, params, eps):
        """(B, H, W, L, label pointer, label stride, the 20-entry conv table) of a train call; ``params`` as
        :func:`soundspaces_b200.belief_nets.smt_resnet18_params` orders them, ``eps`` the 20 GroupNorm eps."""
        B, H, W = x.shape[:3]
        L = labels.shape[1] if labels is not None else 0
        table = (_lib.ResnetConv * belief_nets.N_CONVS)()
        for i in range(belief_nets.N_CONVS):
            w, g, b = params[i], params[20 + i], params[40 + i]
            table[i] = _lib.ResnetConv(w.data_ptr(), g.data_ptr(), b.data_ptr(), None, None, float(eps[i]), 0)
        lp = labels.data_ptr() if L and B else None
        return B, H, W, L, lp, (max(labels.stride(0), L) if L else 0), table

    def smt_resnet18_train_workspace(self, B: int, H: int, W: int, n_labels: int, n_out: int) -> torch.Tensor:
        return self._train_workspace(self.lib.ssb_smt_resnet18_train_workspace_bytes(B, H, W, n_labels, n_out))

    def resnet18_train_workspace(self, B: int, H: int, W: int, n_out: int) -> torch.Tensor:
        return self._train_workspace(self.lib.ssb_resnet18_train_workspace_bytes(B, H, W, n_out))

    def _train_workspace(self, nbytes: int) -> torch.Tensor:
        """The workspace of a ResNet-18 train forward and its backward, ``nbytes`` as a ``*_train_workspace_bytes``
        ABI function returned it."""
        if nbytes < 0:
            raise RuntimeError("the library refuses this shape (*_train_workspace_bytes, include/ssb200.h)")
        return torch.empty(max(int(nbytes), 16), dtype=torch.uint8, device=self.device)

    @staticmethod
    def _train_grads(B: int, params, need, n_params: int = 62):
        """The gradient buffers of a ResNet-18 train backward (None where not needed), and whether the entry has any
        work: at B = 0 the needed gradients are zeros."""
        need = need if need is not None else (True,) * n_params
        grads = [torch.empty_like(p) if n and p is not None else None for p, n in zip(params[:n_params], need)]
        if B == 0:
            for g in grads:
                if g is not None:
                    g.zero_()
        return grads, B > 0 and any(g is not None for g in grads)

    @torch.no_grad()
    def smt_resnet18_train_forward(self, x: torch.Tensor, labels: Optional[torch.Tensor], params, eps):
        """The forward of :meth:`smt_resnet18` for training (``ssb_smt_resnet18_train_forward_batch``, 38 launches):
        bit-identical output, B up to 65535, and the workspace the backward reads.  ``params``: the 20 conv weights,
        20 GroupNorm gammas, 20 betas, fc weight and fc bias (or None); ``eps`` the 20 GroupNorm eps -> (out (B, n_out),
        workspace)."""
        B, H, W, L, lp, ls, table = self._smt_train_args(x, labels, params, eps)
        fw, fb = params[60], params[61]
        n_out, fc_in = fw.shape
        out = torch.empty((B, n_out), dtype=torch.float32, device=self.device)
        ws = self.smt_resnet18_train_workspace(B, H, W, L, n_out)
        if B == 0:
            return out, ws
        self.ctx.check(self.lib.ssb_smt_resnet18_train_forward_batch(
            self.ctx.handle, B, x.data_ptr(), H, W, lp, L, ls, table, fw.data_ptr(),
            fb.data_ptr() if fb is not None else None, fc_in, n_out, out.data_ptr(), ws.data_ptr(), self._stream()),
            "ssb_smt_resnet18_train_forward_batch")
        return out, ws

    @torch.no_grad()
    def smt_resnet18_train_backward(self, x: torch.Tensor, labels: Optional[torch.Tensor], params, eps,
                                    workspace: torch.Tensor, grad_out: torch.Tensor, need=None):
        """The backward of :meth:`smt_resnet18_train_forward` (``ssb_smt_resnet18_train_backward_batch``) from its
        workspace and the (B, n_out) gradient of its output.  ``need``: which of the 62 parameter gradients (weights,
        gammas, betas, fc weight, fc bias) to compute, all when None.  -> those 62, None where not needed."""
        B, H, W, L, lp, ls, table = self._smt_train_args(x, labels, params, eps)
        grads, work = self._train_grads(B, params, need)
        if not work:
            return tuple(grads)
        ptr = lambda t: None if t is None else t.data_ptr()                   # noqa: E731
        arr = lambda ts: (C.c_void_p * 20)(*[ptr(t) for t in ts])              # noqa: E731
        fw = params[60]
        n_out, fc_in = fw.shape
        self.ctx.check(self.lib.ssb_smt_resnet18_train_backward_batch(
            self.ctx.handle, B, x.data_ptr(), H, W, lp, L, ls, table, fw.data_ptr(), fc_in, n_out,
            grad_out.data_ptr(), workspace.data_ptr(), arr(grads[0:20]), arr(grads[20:40]), arr(grads[40:60]),
            ptr(grads[60]), ptr(grads[61]), self._stream()), "ssb_smt_resnet18_train_backward_batch")
        return tuple(grads)

    @staticmethod
    def _resnet_train_table(params, stats, eps):
        """The 20-entry conv table of a torchvision train call: ``params`` as
        :func:`soundspaces_b200.belief_nets.resnet18_params` orders them, ``stats`` as
        :func:`soundspaces_b200.belief_nets.resnet18_buffers`, ``eps`` the 20 BatchNorm eps."""
        table = (_lib.ResnetConv * belief_nets.N_CONVS)()
        for i in range(belief_nets.N_CONVS):
            table[i] = _lib.ResnetConv(params[i].data_ptr(), params[20 + i].data_ptr(), params[40 + i].data_ptr(),
                                       stats[i].data_ptr(), stats[20 + i].data_ptr(), float(eps[i]), 0)
        return table

    @torch.no_grad()
    def resnet18_train_forward(self, x: torch.Tensor, params, stats, eps, training: bool, momentum: float):
        """The torchvision ResNet-18 of :meth:`resnet18` for training (``ssb_resnet18_train_forward_batch``): BatchNorm
        with batch statistics, updating the running statistics and counters in place (``training``, 79 launches), or
        with the running ones and output bit-identical to :meth:`resnet18` (59 launches); B up to 65535.  ``params``:
        the 20 conv weights, 20 BatchNorm gammas, 20 betas, fc weight and fc bias (or None); ``stats``: the 20
        running means, 20 running variances and 20 ``num_batches_tracked``; ``eps`` the 20 BatchNorm eps ->
        (out (B, n_out), workspace)."""
        B, H, W = x.shape[:3]
        fw, fb = params[60], params[61]
        n_out, fc_in = fw.shape
        out = torch.empty((B, n_out), dtype=torch.float32, device=self.device)
        ws = self.resnet18_train_workspace(B, H, W, n_out)
        if B == 0:
            return out, ws
        nbt = (C.c_void_p * 20)(*[t.data_ptr() for t in stats[40:60]])
        self.ctx.check(self.lib.ssb_resnet18_train_forward_batch(
            self.ctx.handle, B, x.data_ptr(), H, W, self._resnet_train_table(params, stats, eps), fw.data_ptr(),
            fb.data_ptr() if fb is not None else None, fc_in, n_out, int(training), float(momentum), nbt,
            out.data_ptr(), ws.data_ptr(), self._stream()), "ssb_resnet18_train_forward_batch")
        return out, ws

    @torch.no_grad()
    def resnet18_train_backward(self, x: torch.Tensor, params, stats, eps, training: bool, workspace: torch.Tensor,
                                grad_out: torch.Tensor, need=None):
        """The backward of :meth:`resnet18_train_forward` (``ssb_resnet18_train_backward_batch``, 115 launches) from its
        workspace and the (B, n_out) gradient of its output.  ``need``: which of the 62 parameter gradients (weights,
        gammas, betas, fc weight, fc bias) to compute, all when None.  -> those 62, None where not needed."""
        B, H, W = x.shape[:3]
        grads, work = self._train_grads(B, params, need)
        if not work:
            return tuple(grads)
        ptr = lambda t: None if t is None else t.data_ptr()                   # noqa: E731
        arr = lambda ts: (C.c_void_p * 20)(*[ptr(t) for t in ts])              # noqa: E731
        fw = params[60]
        n_out, fc_in = fw.shape
        self.ctx.check(self.lib.ssb_resnet18_train_backward_batch(
            self.ctx.handle, B, x.data_ptr(), H, W, self._resnet_train_table(params, stats, eps), fw.data_ptr(), fc_in,
            n_out, int(training), grad_out.data_ptr(), workspace.data_ptr(), arr(grads[0:20]), arr(grads[20:40]),
            arr(grads[40:60]), ptr(grads[60]), ptr(grads[61]), self._stream()), "ssb_resnet18_train_backward_batch")
        return tuple(grads)

    @torch.no_grad()
    def smt_cnn(self, rgb: Optional[torch.Tensor], depth: Optional[torch.Tensor],
                rgb_encoder: Optional["torch.nn.Module"], depth_encoder: Optional["torch.nn.Module"],
                resize: bool = True) -> torch.Tensor:
        """SAVi's visual encoder ``SMTCNN.forward`` (savi/models/smt_cnn.py:76-113) for RGB and / or depth on the current
        stream -> (B, n_out_rgb + n_out_depth), the features side by side in that order: ``rgb_encoder(T(rgb.permute(0,
        3, 1, 2) / 255.0))`` and ``depth_encoder(T(depth.permute(0, 3, 1, 2)))``, where T is ResizeCenterCropper(size=
        (64, 64)) when ``resize`` and the identity otherwise.  ``ssb_smt_cnn_batch``, 39 launches.  ``rgb`` / ``depth``:
        contiguous float32 (B, H, W, C) on this device with equal B (H, W may differ); either may be None, not both.
        ``ValueError`` for other tensors, a missing encoder, an encoder
        :func:`soundspaces_b200.belief_nets.smt_resnet18_layout_error` refuses for C channels on a 64 x 64 input, or an
        observation that is not 64 x 64 without ``resize``; ``RuntimeError`` when the library refuses the shape (B >
        1024, H or W past 1024, a resize whose crop does not lie inside it)."""
        from .encoder import SMT_CNN_CROP, resize_center_crop_geometry
        inputs = [(x, net, name, scale) for x, net, name, scale in ((rgb, rgb_encoder, "rgb", 1),
                                                                     (depth, depth_encoder, "depth", 0)) if x is not None]
        if not inputs:
            raise ValueError("smt_cnn needs rgb, depth or both")
        B = inputs[0][0].shape[0] if isinstance(inputs[0][0], torch.Tensor) else -1
        table = (_lib.SmtCnnInput * len(inputs))()
        n_out = 0
        for k, (x, net, name, scale) in enumerate(inputs):
            if not (isinstance(x, torch.Tensor) and x.device == self.device and x.dtype == torch.float32 and x.ndim == 4
                    and x.shape[0] == B and x.shape[3] >= 1 and x.is_contiguous()):
                raise ValueError(f"smt_cnn: {name} must be a contiguous float32 (B, H, W, C) observation on "
                                 f"{self.device}, B equal for both")
            _, H, W, Cin = x.shape
            err = belief_nets.smt_resnet18_layout_error(net, Cin, (SMT_CNN_CROP, SMT_CNN_CROP), self.device)
            if err:
                raise ValueError(f"smt_cnn: {name}_encoder: " + err)
            if resize:
                rh, rw, cy, cx = resize_center_crop_geometry(H, W)
            elif (H, W) == (SMT_CNN_CROP, SMT_CNN_CROP):
                rh, rw, cy, cx = SMT_CNN_CROP, SMT_CNN_CROP, 0, 0
            else:
                raise ValueError(f"smt_cnn: without resize, {name} must be {SMT_CNN_CROP} x {SMT_CNN_CROP}, not {H} x {W}")
            fc = net.fc
            table[k] = _lib.SmtCnnInput(x.data_ptr(), Cin, H, W, scale, rh, rw, cy, cx,
                                        belief_nets.conv_table(net, False), fc.weight.data_ptr(),
                                        fc.bias.data_ptr() if fc.bias is not None else None, fc.in_features,
                                        fc.out_features)
            n_out += fc.out_features
        out = torch.empty((B, n_out), dtype=torch.float32, device=self.device)
        if B == 0:                    # empty tensors have NULL data pointers, which the library refuses
            return out
        self.ctx.check(self.lib.ssb_smt_cnn_batch(self.ctx.handle, B, len(inputs), table, out.data_ptr(),
                                                  self._stream()), "ssb_smt_cnn_batch")
        return out

    @staticmethod
    def _smt_cnn_train_table(rgb, depth, params, eps, resize: bool):
        """(B, the ssb_smt_cnn_input table, n_inputs, sum of n_out) of a train call: ``params`` 62 per present input
        (RGB first) as :func:`soundspaces_b200.belief_nets.smt_resnet18_params` orders them, ``eps`` 20 per input."""
        from .encoder import SMT_CNN_CROP, resize_center_crop_geometry
        inputs = [(x, scale) for x, scale in ((rgb, 1), (depth, 0)) if x is not None]
        table = (_lib.SmtCnnInput * len(inputs))()
        ld = 0
        for k, (x, scale) in enumerate(inputs):
            _, H, W, Cin = x.shape
            geo = resize_center_crop_geometry(H, W) if resize else (SMT_CNN_CROP, SMT_CNN_CROP, 0, 0)
            p, e = params[62 * k:62 * k + 62], eps[20 * k:20 * k + 20]
            convs = (_lib.ResnetConv * belief_nets.N_CONVS)()
            for i in range(belief_nets.N_CONVS):
                convs[i] = _lib.ResnetConv(p[i].data_ptr(), p[20 + i].data_ptr(), p[40 + i].data_ptr(), None, None,
                                           float(e[i]), 0)
            fw, fb = p[60], p[61]
            table[k] = _lib.SmtCnnInput(x.data_ptr(), Cin, H, W, scale, *geo, convs, fw.data_ptr(),
                                        fb.data_ptr() if fb is not None else None, fw.shape[1], fw.shape[0])
            ld += fw.shape[0]
        return inputs[0][0].shape[0], table, len(inputs), ld

    def smt_cnn_train_workspace(self, B: int, table, n_inputs: int) -> torch.Tensor:
        return self._train_workspace(self.lib.ssb_smt_cnn_train_workspace_bytes(B, n_inputs, table))

    @torch.no_grad()
    def smt_cnn_train_forward(self, rgb: Optional[torch.Tensor], depth: Optional[torch.Tensor], params, eps,
                              resize: bool = True):
        """The forward of :meth:`smt_cnn` for training (``ssb_smt_cnn_train_forward_batch``, 1 + 38 n_inputs launches):
        bit-identical output, B up to 65535, and the workspace the backward reads.  ``params``: 62 per present input,
        RGB first (:func:`soundspaces_b200.encoder.smt_cnn_params`); ``eps``: 20 GroupNorm eps per input -> (out
        (B, sum n_out), workspace)."""
        B, table, n, ld = self._smt_cnn_train_table(rgb, depth, params, eps, resize)
        out = torch.empty((B, ld), dtype=torch.float32, device=self.device)
        ws = self.smt_cnn_train_workspace(B, table, n)
        if B == 0:
            return out, ws
        self.ctx.check(self.lib.ssb_smt_cnn_train_forward_batch(self.ctx.handle, B, n, table, out.data_ptr(),
                                                                ws.data_ptr(), self._stream()),
                       "ssb_smt_cnn_train_forward_batch")
        return out, ws

    @torch.no_grad()
    def smt_cnn_train_backward(self, rgb: Optional[torch.Tensor], depth: Optional[torch.Tensor], params, eps,
                               resize: bool, workspace: torch.Tensor, grad_out: torch.Tensor, need=None):
        """The backward of :meth:`smt_cnn_train_forward` (``ssb_smt_cnn_train_backward_batch``, 80 launches per input)
        from its workspace and the contiguous (B, sum n_out) gradient of its output.  ``need``: which of the 62 n
        parameter gradients to compute, all when None.  -> those 62 n, None where not needed."""
        B, table, n, _ = self._smt_cnn_train_table(rgb, depth, params, eps, resize)
        grads, work = self._train_grads(B, params, need, 62 * n)
        if not work:
            return tuple(grads)
        ptrs = (C.c_void_p * (62 * n))(*[None if g is None else g.data_ptr() for g in grads])
        self.ctx.check(self.lib.ssb_smt_cnn_train_backward_batch(
            self.ctx.handle, B, n, table, grad_out.data_ptr(), workspace.data_ptr(), ptrs, self._stream()),
            "ssb_smt_cnn_train_backward_batch")
        return tuple(grads)

    @torch.no_grad()
    def smt_state_encoder(self, module: "torch.nn.Module", x: torch.Tensor, memory: torch.Tensor,
                          masks: torch.Tensor, goal: Optional[torch.Tensor] = None) -> torch.Tensor:
        """``SMTStateEncoder.single_forward(x, memory, masks, goal)`` (savi/models/smt_state_encoder.py:92-157) on the
        current stream -> (N, d_model), in six launches whatever N, M and the masks (``ssb_smt_state_encoder_batch``).
        ``x`` (N, D), ``memory`` (M, N, D), ``masks`` (N, M) and ``goal`` (N, d_model) or None: contiguous float32 on
        this device.  Only valid tokens are computed; masked memory rows are never read.  ``ValueError`` for a module
        :func:`soundspaces_b200.smt.smt_layout_error` refuses or malformed inputs; ``RuntimeError`` past the library's
        limits."""
        from . import smt
        for name, t, ndim in (("x", x, 2), ("memory", memory, 3), ("masks", masks, 2), ("goal", goal, 2)):
            if t is None and name == "goal":
                continue
            if not (isinstance(t, torch.Tensor) and t.device == self.device and t.dtype == torch.float32
                    and t.ndim == ndim and t.is_contiguous()):
                raise ValueError(f"smt_state_encoder: {name} must be a contiguous float32 {ndim}-d tensor on {self.device}")
        N, D = x.shape
        M = memory.shape[0]
        d = getattr(getattr(module, "transformer", None), "d_model", 0)
        if tuple(memory.shape[1:]) != (N, D) or tuple(masks.shape) != (N, M) or (goal is not None and tuple(goal.shape) != (N, d)):
            raise ValueError(f"smt_state_encoder: shapes x {tuple(x.shape)}, memory {tuple(memory.shape)}, masks "
                             f"{tuple(masks.shape)}, goal {None if goal is None else tuple(goal.shape)} disagree")
        err = smt.smt_layout_error(module, self.device)
        if err:
            raise ValueError("smt_state_encoder: " + err)
        # without pose encoding the kernels read fusion_encoder[0].weight with row stride D
        if not getattr(module, "_use_pose_encoding", False) and D != module.fusion_encoder[0].in_features:
            raise ValueError(f"smt_state_encoder: x has {D} columns, fusion_encoder.0 takes "
                             f"{module.fusion_encoder[0].in_features}")
        out = torch.empty((N, d), dtype=torch.float32, device=self.device)
        if N == 0:
            return out
        params = smt.smt_params(module, D)
        key = (N, M, d)
        scratch = self._smt_scratch.get(key)
        if scratch is None:
            nbytes = int(self.lib.ssb_smt_scratch_bytes(N, M, C.byref(params)))
            if nbytes < 0:
                raise ValueError(f"smt_state_encoder: no scratch size for N={N} M={M} d_model={d}")
            scratch = torch.empty(max(nbytes, 16), dtype=torch.uint8, device=self.device)
            self._smt_scratch[key] = scratch
        self.ctx.check(self.lib.ssb_smt_state_encoder_batch(
            self.ctx.handle, N, M, x.data_ptr(), memory.data_ptr() if M else None, masks.data_ptr() if M else None,
            goal.data_ptr() if goal is not None else None, C.byref(params), scratch.data_ptr(), out.data_ptr(),
            self._stream()), "ssb_smt_state_encoder_batch")
        return out

    def smt_train_workspace(self, N: int, M: int, params) -> torch.Tensor:
        """The workspace of :meth:`smt_train_forward` and :meth:`smt_train_backward` for ``params`` (an
        ``ssb_smt_params`` from :func:`soundspaces_b200.smt.smt_params`)."""
        return self._train_workspace(self.lib.ssb_smt_train_workspace_bytes(N, M, C.byref(params)))

    @torch.no_grad()
    def smt_train_forward(self, module: "torch.nn.Module", x: torch.Tensor, memory: torch.Tensor, masks: torch.Tensor,
                          goal: Optional[torch.Tensor] = None):
        """The forward of :meth:`smt_state_encoder` for training (``ssb_smt_state_encoder_train_forward_batch``, the
        same six launches): bit-identical output, N up to 65535, and the workspace the backward reads.  The caller
        has checked the inputs (:func:`soundspaces_b200.smt.smt_train_error`) -> (out (N, d_model), workspace)."""
        from . import smt
        N, D = x.shape
        M = memory.shape[0]
        params = smt.smt_params(module, D)
        out = torch.empty((N, module.transformer.d_model), dtype=torch.float32, device=self.device)
        ws = self.smt_train_workspace(N, M, params)
        if N == 0:
            return out, ws
        self.ctx.check(self.lib.ssb_smt_state_encoder_train_forward_batch(
            self.ctx.handle, N, M, x.data_ptr(), memory.data_ptr() if M else None, masks.data_ptr() if M else None,
            goal.data_ptr() if goal is not None else None, C.byref(params), ws.data_ptr(), out.data_ptr(),
            self._stream()), "ssb_smt_state_encoder_train_forward_batch")
        return out, ws

    @torch.no_grad()
    def smt_train_backward(self, module: "torch.nn.Module", x: torch.Tensor, memory: torch.Tensor,
                           masks: torch.Tensor, goal: Optional[torch.Tensor], workspace: torch.Tensor,
                           grad_out: torch.Tensor, need=None):
        """The backward of :meth:`smt_train_forward` (``ssb_smt_state_encoder_train_backward_batch``, 10 launches)
        from its workspace and the (N, d_model) gradient of its output (unit column stride).  ``need``: which of (the
        parameters of :func:`soundspaces_b200.smt.smt_train_parameters`..., x, goal) to compute, all when None ->
        those gradients, None where not needed."""
        from . import smt
        N, D = x.shape
        M = memory.shape[0]
        params = smt.smt_train_parameters(module)
        n = len(params)
        need = tuple(need) if need is not None else (True,) * (n + 2)
        grads, _ = self._train_grads(N, params, need[:n], n)
        dx = torch.empty_like(x) if need[n] else None
        dgoal = torch.empty_like(goal) if goal is not None and need[n + 1] else None
        if N == 0 or not any(g is not None for g in grads + [dx, dgoal]):
            for g in (dx, dgoal):
                if g is not None:
                    g.zero_()
            return tuple(grads) + (dx, dgoal)
        if grad_out.stride(1) != 1:
            grad_out = grad_out.contiguous()
        ptrs = (C.c_void_p * n)(*[None if g is None else g.data_ptr() for g in grads])
        self.ctx.check(self.lib.ssb_smt_state_encoder_train_backward_batch(
            self.ctx.handle, N, M, x.data_ptr(), memory.data_ptr() if M else None, masks.data_ptr() if M else None,
            goal.data_ptr() if goal is not None else None, C.byref(smt.smt_params(module, D)), grad_out.data_ptr(),
            grad_out.stride(0), workspace.data_ptr(), ptrs, dx.data_ptr() if dx is not None else None,
            dgoal.data_ptr() if dgoal is not None else None, self._stream()),
            "ssb_smt_state_encoder_train_backward_batch")
        return tuple(grads) + (dx, dgoal)

    def belief_update(self, spec: torch.Tensor, dones, w: float, current_pred_only: bool, *,
                      pose: Optional[torch.Tensor] = None, loc_pred: Optional[torch.Tensor] = None,
                      last_pg: Optional[torch.Tensor] = None, loc_valid: Optional[torch.Tensor] = None,
                      loc_out: Optional[torch.Tensor] = None, label_pred: Optional[torch.Tensor] = None,
                      last_label: Optional[torch.Tensor] = None, label_valid: Optional[torch.Tensor] = None,
                      cat_out: Optional[torch.Tensor] = None) -> None:
        """The per-env part of SAVi's ``BeliefPredictor.update`` (belief_predictor.py:150-202) in one launch, on the
        current stream, with no host synchronisation (``ssb_belief_update_batch``).  ``spec``: the (B, H, W, 2)
        observation; ``dones``: None or B truthy values (host).  Location belief when ``loc_pred`` is given:
        ``pose`` (B, >= 3) and ``loc_pred`` (B, >= 2) with unit column stride, state ``last_pg`` (N, 2) float32 and
        ``loc_valid`` (N,) uint8, output ``loc_out`` (B, 2).  Label belief when ``label_pred`` (B, >= 21) is given:
        state ``last_label`` (N, 21) and ``label_valid`` (N,) uint8, output ``cat_out`` (B, 21).  State rows >= B are
        not touched.  ``ValueError`` for anything else."""
        def need(name, t, ndim, dtype=torch.float32, rows=None, min_cols=None, cols=None, dense=True):
            ok = (isinstance(t, torch.Tensor) and t.device == self.device and t.dtype == dtype and t.ndim == ndim
                  and (rows is None or t.shape[0] == rows) and (min_cols is None or t.shape[1] >= min_cols)
                  and (cols is None or t.shape[1] == cols)
                  and (t.is_contiguous() if dense else (t.shape[0] <= 1 or t.stride(0) >= t.shape[1]) and t.stride(1) == 1))
            if not ok:
                raise ValueError(f"belief_update: {name} must be a {'contiguous ' if dense else ''}{dtype} tensor on "
                                 f"{self.device} with {ndim} dims" + (f", {rows} rows" if rows is not None else "")
                                 + (f", >= {min_cols} columns of unit stride" if min_cols is not None else "")
                                 + (f", {cols} columns" if cols is not None else ""))

        need("spec", spec, 4)
        if spec.shape[3] != 2:
            raise ValueError("belief_update: spec must be (B, H, W, 2)")
        B, H, W, _ = spec.shape
        if loc_pred is None and label_pred is None:
            raise ValueError("belief_update: give loc_pred, label_pred or both")
        num_env = None
        if loc_pred is not None:
            need("pose", pose, 2, rows=B, min_cols=3, dense=False)
            need("loc_pred", loc_pred, 2, rows=B, min_cols=2, dense=False)
            need("last_pg", last_pg, 2, cols=2)
            need("loc_valid", loc_valid, 1, dtype=torch.uint8, rows=last_pg.shape[0])
            need("loc_out", loc_out, 2, rows=B, cols=2)
            num_env = last_pg.shape[0]
        if label_pred is not None:
            need("label_pred", label_pred, 2, rows=B, min_cols=21, dense=False)
            need("last_label", last_label, 2, cols=21)
            need("label_valid", label_valid, 1, dtype=torch.uint8, rows=last_label.shape[0])
            need("cat_out", cat_out, 2, rows=B, cols=21)
            num_env = last_label.shape[0] if num_env is None else min(num_env, last_label.shape[0])
        if B > num_env:
            raise ValueError(f"belief_update: batch of {B} envs, but the state has {num_env} rows")
        if dones is not None and len(dones) < B:
            raise ValueError(f"belief_update: {len(dones)} dones for {B} envs")
        h_dones = None if dones is None else (C.c_uint8 * max(B, 1))(*[1 if dones[i] else 0 for i in range(B)])

        def ptr(t):
            return t.data_ptr() if t is not None else None

        def stride(t):                    # a one-row tensor may report any row stride; only row 0 is read
            return max(t.stride(0), t.shape[1]) if t is not None else 0

        if loc_pred is None:
            pose = None
        self.ctx.check(self.lib.ssb_belief_update_batch(
            self.ctx.handle, B, num_env, spec.data_ptr(), H, W, ptr(pose), stride(pose), ptr(loc_pred), stride(loc_pred),
            ptr(label_pred), stride(label_pred), h_dones, float(w), int(bool(current_pred_only)), ptr(last_pg), ptr(loc_valid), ptr(last_label), ptr(label_valid), ptr(loc_out),
            ptr(cat_out), self._stream()), "ssb_belief_update_batch")


class BatchedAudioRenderer:
    def __init__(self, sr: int, max_taps: int, device="cuda:0", n_terms: int = 1, log2n: int = 0,
                 pad_mode: str = "reflect", xpool_bytes: int = 512 << 20, prefer_block64: Optional[bool] = None):
        self.sr = int(sr)
        self.device = torch.device("cuda", _dev_index(device))
        self.pad_mode = PAD_MODES[pad_mode]
        # No global side effect: the caller's current CUDA device is left alone.  Every C-ABI entry selects the
        # context's device itself (and restores the caller's); tensors are allocated with an explicit device and
        # streams are taken from torch's current stream OF THAT device.
        self.ctx = _lib.Context(self.device.index)
        self.lib = self.ctx.lib
        self.max_taps = int(max_taps)
        # Two plans (include/ssb200.h).  The partitioned overlap-save plan handles every request; the single-block plan
        # (one fused 65536-point cluster kernel per env, no H / Y intermediates in DRAM) serves batches whose requests
        # all have one term and at most 65536 - sr + 1 effective taps.
        # prefer_block64=True (or SSB200_BLOCK64=1) takes it whenever a batch is eligible -- chosen per batch in
        # _prepare_columns; log2n = 16 forces it (requests that do not fit raise).  DESIGN.md section 4 has the numbers.
        self.plan64 = None
        self.block64_taps = 65536 - self.sr + 1
        if prefer_block64 is None:
            prefer_block64 = os.environ.get("SSB200_BLOCK64", "0") == "1"
        if (log2n == 16 or (log2n == 0 and prefer_block64)) and self.sr <= 65536 - 4096:
            self.plan64 = self.ctx.make_plan(self.sr, min(self.max_taps, self.block64_taps), 1, 16)
        self.force_block64 = log2n == 16
        if self.force_block64 and (self.plan64 is None or self.max_taps > self.block64_taps or n_terms != 1):
            raise ValueError(f"log2n=16 (single-block plan) needs n_terms=1 and max_taps <= {self.block64_taps} at sr={self.sr}")
        self.plan = self.ctx.make_plan(self.sr, self.max_taps, n_terms, 0 if log2n == 16 else log2n)
        self.N = 1 << self.plan.log2n
        self.P = self.plan.block
        self.spec_shape = spectrogram_shape(self.sr)
        assert self.spec_shape[1] == self.lib.ssb_spec_cols(self.sr)
        # RIR bank: (total_taps, 2) float32, interleaved ears == one complex signal
        self._bank = torch.zeros((1, 2), dtype=torch.float32, device=self.device)
        self._bank_used = 0
        self._rir_off: list[int] = []
        self._rir_len: list[int] = []
        self._bank_index = None               # numpy copies of the two lists, rebuilt when the bank changes
        # sources + window-spectra pool
        self._sources: list[torch.Tensor] = []
        # window-spectra pool: allocated on first use (a renderer that only runs the STFT / intensity kernels on
        # waveforms it is handed -- SpectrogramSensor.compute_spectrogram on a host array -- never needs it)
        self._xpool_elems = max(xpool_bytes // 8, 64 * self.N, 8 * 65536 if self.plan64 is not None else 0)   # float2 elements
        self._xpool_t = None
        self._xpool_used = 0                  # float2 elements
        self._xcache: dict = {}
        self._hscratch = None
        self._wave = None
        self._prev_wave = None
        self._hbanks = {}             # channel count -> (K, 2, 256) device HRTF bank

    @property
    def _xpool(self) -> torch.Tensor:
        if self._xpool_t is None:
            self._xpool_t = torch.empty(self._xpool_elems * 2, dtype=torch.float32, device=self.device)
        return self._xpool_t

    def set_conv_mode(self, mode: int):
        """0 = per-bin partition sums then inverse FFTs (default); 1 = fused into the inverse-FFT kernel."""
        self.ctx.check(self.lib.ssb_set_conv_mode(self.ctx.handle, int(mode)), "ssb_set_conv_mode")

    def set_streams(self, n: int):
        """Run render() as n sub-batches on n internal streams (overlaps kernel tails)."""
        self.ctx.check(self.lib.ssb_set_streams(self.ctx.handle, int(n)), "ssb_set_streams")

    def set_chunks(self, n: int):
        """Each internal stream works through n sub-batches in turn (smaller L2 footprint per sub-batch)."""
        self.ctx.check(self.lib.ssb_set_chunks(self.ctx.handle, int(n)), "ssb_set_chunks")

    # ------------------------------------------------------------------ banks
    def add_rirs(self, rirs: Sequence) -> list:
        """Append RIRs ((L, 2) float32 arrays / tensors; None or empty => zero-RIR fallback).
        All-or-nothing: every entry is validated and converted BEFORE the index lists or the bank are touched,
        so a bad entry in the middle of the list leaves the bank exactly as it was."""
        offs, lens, chunks, total = [], [], [], 0
        for r in rirs:
            if r is None or len(r) == 0:
                offs.append(0)
                lens.append(0)
                continue
            t = torch.as_tensor(r, dtype=torch.float32)
            if t.ndim != 2 or t.shape[1] != 2:
                raise ValueError(f"RIR must be (L, 2), got {tuple(t.shape)}")
            offs.append(self._bank_used + total)
            lens.append(t.shape[0])
            chunks.append(t)
            total += t.shape[0]
        if total:
            need = self._bank_used + total
            if need > self._bank.shape[0]:
                grown = torch.empty((max(need, 2 * self._bank.shape[0]), 2), dtype=torch.float32, device=self.device)
                grown[: self._bank_used] = self._bank[: self._bank_used]
                self._bank = grown
            if all(c.is_cuda for c in chunks):
                host = torch.cat(chunks)
            else:
                host = torch.cat([c.cpu() if c.is_cuda else c for c in chunks])
            self._bank[self._bank_used: need].copy_(host, non_blocking=True)
            self._bank_used = need
        first = len(self._rir_off)
        self._rir_off.extend(offs)
        self._rir_len.extend(lens)
        self._bank_index = None
        return list(range(first, first + len(offs)))

    def compact_bank(self, keep_ids: Sequence[int]) -> list:
        """Keep only the given RIRs (one device-side gather into a fresh arena) and return their new ids, in the
        order given; every other id becomes invalid.  The file-backed service calls this when the resident bank
        outgrows its budget, keeping the recently used part of the working set instead of re-reading it."""
        keep_ids = [int(i) for i in keep_ids]
        lens = [self._rir_len[i] for i in keep_ids]
        total = sum(lens)
        arena = torch.empty((max(total, 1), 2), dtype=torch.float32, device=self.device)
        offs, pos = [], 0
        for i, n in zip(keep_ids, lens):
            offs.append(pos if n else 0)
            if n:
                arena[pos: pos + n].copy_(self._bank[self._rir_off[i]: self._rir_off[i] + n])
                pos += n
        self._bank, self._bank_used = arena, total
        self._rir_off, self._rir_len = offs, lens
        self._bank_index = None
        return list(range(len(keep_ids)))

    def reset_bank(self):
        """Forget every RIR (ids become invalid).  Used by the file-backed service when the resident
        bank outgrows its budget: the working set of a scene is reloaded on demand."""
        self._bank_used = 0
        self._bank_index = None
        self._rir_off.clear()
        self._rir_len.clear()

    @property
    def bank_bytes(self) -> int:
        return self._bank_used * 8

    def bank_mark(self):
        """Stack mark for transient RIRs (the continuous simulator renders a new RIR every step)."""
        return (self._bank_used, len(self._rir_off))

    def bank_release(self, mark):
        """Drop every RIR added since ``mark``.  Safe while kernels are in flight: later uploads
        are ordered after them on the same stream."""
        self._bank_used, n = mark
        self._bank_index = None
        del self._rir_off[n:]
        del self._rir_len[n:]

    def set_dense_rir_bank(self, rirs: torch.Tensor) -> list:
        """Adopt an already device-resident (n, L, 2) float32 tensor as the bank (no copy)."""
        if not (rirs.is_cuda and rirs.dtype == torch.float32 and rirs.is_contiguous() and rirs.ndim == 3
                and rirs.shape[2] == 2):
            raise ValueError("expected a contiguous CUDA float32 (n, L, 2) tensor")
        n, L, _ = rirs.shape
        self._bank = rirs.view(n * L, 2)
        self._bank_used = n * L
        self._rir_off = [i * L for i in range(n)]
        self._rir_len = [L] * n
        self._bank_index = None
        return list(range(n))

    def add_source(self, samples) -> int:
        """Register a mono clip already at ``sr`` (float32).  Returns its id."""
        t = torch.as_tensor(samples, dtype=torch.float32).reshape(-1).to(self.device).contiguous()
        if t.numel() == 0:
            raise ValueError("empty source clip")
        self._sources.append(t)
        return len(self._sources) - 1

    def add_source_pcm16(self, pcm) -> int:
        """Register an int16 clip; decoded on the device as float32(x)/32768 (bit-exact
        with the soundfile decode behind ``librosa.load``, simulator.py:597)."""
        p = torch.as_tensor(np.ascontiguousarray(pcm, dtype=np.int16)).to(self.device)
        out = torch.empty(p.numel(), dtype=torch.float32, device=self.device)
        self.ctx.check(self.lib.ssb_pcm16_decode(self.ctx.handle, p.data_ptr(), p.numel(), out.data_ptr(),
                                                 self._stream()), "ssb_pcm16_decode")
        self._sources.append(out)
        return len(self._sources) - 1

    def encode_pcm16(self, wave: torch.Tensor, mode: str = "round") -> torch.Tensor:
        w = wave.contiguous()
        out = torch.empty(w.shape, dtype=torch.int16, device=self.device)
        self.ctx.check(self.lib.ssb_pcm16_encode(self.ctx.handle, w.data_ptr(), w.numel(),
                                                 {"round": 0, "demo": 1}[mode], out.data_ptr(), self._stream()),
                       "ssb_pcm16_encode")
        return out

    def intensity(self, wave: torch.Tensor, num_frame: int = 150) -> torch.Tensor:
        """AV-WaN ``Intensity`` (avwan_sensors.py:91-100) for a (n, 2, sr) CUDA batch -> (n,) mean squares."""
        if wave.ndim == 2:
            wave = wave[None]
        wave = wave.to(self.device, torch.float32).contiguous()
        out = torch.empty(wave.shape[0], dtype=torch.float32, device=self.device)
        self.ctx.check(self.lib.ssb_intensity_batch(self.ctx.handle, wave.shape[0], wave.data_ptr(), wave.shape[2],
                                                    wave.shape[2], int(num_frame), out.data_ptr(), self._stream()),
                       "ssb_intensity_batch")
        return out

    # ------------------------------------------------------------ SH decode
    def _sh_inputs(self, amb, hbank):
        """(n, L, K) float32 contiguous device tensor and the (K, 2, 256) bank: by default the first K rows of
        :func:`sh_hrtf_bank`, uploaded once per K.  A bank given by the caller serves that call only and leaves the
        default in place, so a decode without ``hbank`` never depends on an earlier call."""
        amb = torch.as_tensor(amb, dtype=torch.float32).to(self.device).contiguous()
        if amb.ndim != 3 or amb.shape[2] not in SH_CHANNELS:
            raise ValueError(f"ambisonic RIRs must be (n, L, K) with K in {SH_CHANNELS}, got {tuple(amb.shape)}")
        K = amb.shape[2]
        if hbank is not None:
            hb = torch.as_tensor(np.ascontiguousarray(hbank, dtype=np.float32))
            if tuple(hb.shape) != (K, 2, 256):
                raise ValueError(f"HRTF bank must be ({K}, 2, 256)")
            return amb, hb.to(self.device)
        if K not in self._hbanks:
            self._hbanks[K] = torch.from_numpy(sh_hrtf_bank(K)).to(self.device)
        return amb, self._hbanks[K]

    def _sh_azimuths(self, azimuth_deg):
        """Azimuths in degrees as a flat float32 device tensor.  Any finite value is accepted (the kernel reduces it
        exactly, so ``az`` and ``az + 360`` decode alike).  Values given on the host are refused when NaN or infinite;
        a tensor already on the device is not read back, and a non-finite value in it gives NaN rows."""
        az = torch.as_tensor(azimuth_deg, dtype=torch.float32).reshape(-1)
        if not az.is_cuda and not bool(torch.isfinite(az).all()):
            raise ValueError(f"azimuths must be finite, got {az.tolist()}")
        return az.to(self.device)

    def sh_decode(self, amb: torch.Tensor, azimuth_deg, hbank=None) -> torch.Tensor:
        """Ambisonic (n, L, K) -> binaural (n, L, 2) RIRs on the device, K in {1, 4, 9, 16} (orders 0 to 3, ACN):
        SH rotation about the vertical axis + the K x 2 x 256-tap HRTF bank (scripts/ambisonic_to_binaural.py:14-19),
        one azimuth per RIR.  The result can be handed to :meth:`set_dense_rir_bank` / :meth:`add_rirs`."""
        amb, hb = self._sh_inputs(amb, hbank)
        n, L, K = amb.shape
        az = self._sh_azimuths(azimuth_deg)
        if az.numel() != n:
            raise ValueError("one azimuth per RIR")
        out = torch.empty((n, L, 2), dtype=torch.float32, device=self.device)
        if K == 9:
            filt = torch.empty((n, 9, 256, 2), dtype=torch.float32, device=self.device)
            self.ctx.check(self.lib.ssb_sh_decode_batch(self.ctx.handle, n, amb.data_ptr(), L, az.data_ptr(),
                                                        hb.data_ptr(), filt.data_ptr(), out.data_ptr(),
                                                        self._stream()), "ssb_sh_decode_batch")
            return out
        # the multi-azimuth entry decodes every input at every azimuth: one call per RIR here
        filt = torch.empty((K, 256, 2), dtype=torch.float32, device=self.device)
        for i in range(n):
            self._sh_decode_multi(amb[i:i + 1], az[i:i + 1], hb, filt, out[i:i + 1])
        return out

    def sh_decode_angles(self, amb: torch.Tensor, angles, hbank=None) -> torch.Tensor:
        """Ambisonic (n, L, K) -> binaural (n, A, L, 2): every input decoded at each of the A azimuths (degrees), K in
        {1, 4, 9, 16}.  Each input is read once for all azimuths; row [i, a] is bit-identical to decoding input i
        alone at angles[a]."""
        amb, hb = self._sh_inputs(amb, hbank)
        n, L, K = amb.shape
        az = self._sh_azimuths(angles)
        if az.numel() < 1:
            raise ValueError("at least one angle")
        out = torch.empty((n, az.numel(), L, 2), dtype=torch.float32, device=self.device)
        filt = torch.empty((az.numel(), K, 256, 2), dtype=torch.float32, device=self.device)
        self._sh_decode_multi(amb, az, hb, filt, out)
        return out

    def _sh_decode_multi(self, amb, az, hb, filt, out):
        n, L, K = amb.shape
        self.ctx.check(self.lib.ssb_sh_decode_multi_batch(self.ctx.handle, n, K, L, amb.data_ptr(), az.numel(),
                                                          az.data_ptr(), hb.data_ptr(), filt.data_ptr(),
                                                          out.data_ptr(), self._stream()), "ssb_sh_decode_multi_batch")

    # ---------------------------------------------------------------- helpers
    def _stream(self):
        return C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    def _windows(self, source: int, offset: int, wrap: bool, out_samples: int, block64: bool = False):
        """Cached source spectra of (clip, offset): the overlap-save window set of the partitioned plan, or the one
        65536-point spectrum of the single-block plan.  Returns (x_offset, nw, wofs)."""
        if block64:
            nblk, wofs, nw = 1, 0, 1
            key = (source, offset, bool(wrap), "block64")
            plan, need = self.plan64, 65536
        else:
            nblk, wofs, nw = window_layout(self.P, self.plan.max_parts, offset, out_samples)
            key = (source, offset, bool(wrap), nblk, wofs)
            plan, need = self.plan, nw * self.N
        hit = self._xcache.get(key)
        if hit is not None:
            return hit
        if self._xpool_used + need > self._xpool.numel() // 2:
            if need > self._xpool.numel() // 2:
                raise RuntimeError("window-spectra pool too small for one clip; raise xpool_bytes")
            # simplest policy: drop every cached set (they are recomputed on demand).  Offsets handed out
            # earlier in the current prepare() are stale now: signal it to restart.
            torch.cuda.current_stream(self.device).synchronize()
            self._xcache.clear()
            self._xpool_used = 0
            raise _PoolReset()
        x_off = self._xpool_used
        src = self._sources[source]
        self.ctx.check(self.lib.ssb_source_windows(
            self.ctx.handle, C.byref(plan), src.data_ptr(), src.numel(), int(offset), int(bool(wrap)),
            nw, wofs, self._xpool.data_ptr() + 8 * x_off, self._stream()), "ssb_source_windows")
        self._xpool_used += need
        self._xcache[key] = (x_off, nw, wofs)
        return self._xcache[key]

    def _fill_terms(self, terms, rows, rir_ids, sources, offsets, wraps, out_samples, block64=False):
        """Vectorised fill of one convolution term for the requests ``rows`` (indices into the batch):
        bank offsets and effective tap counts by array indexing, one window-set lookup per distinct
        ``(source, offset, wrap, out_samples)`` instead of one per request."""
        if rows.size == 0:
            return
        n_bank = len(self._rir_len)
        if rir_ids.size and int(rir_ids.max()) >= n_bank:
            raise ValueError(f"unknown RIR id {int(rir_ids.max())}")
        if self._bank_index is None:
            self._bank_index = (np.asarray(self._rir_off, dtype=np.int64), np.asarray(self._rir_len, dtype=np.int64))
        off_arr, len_arr = self._bank_index
        valid = rir_ids >= 0
        lens = np.where(valid, len_arr[np.where(valid, rir_ids, 0)] if n_bank else 0, 0)
        has = lens > 0                                          # None / -1 / empty file => zero RIR: rir_taps stays 0
        if not has.any():
            return
        rows, rir_ids, lens = rows[has], rir_ids[has], lens[has]
        sources, offsets, wraps, out_samples = sources[has], offsets[has], wraps[has], out_samples[has]
        taps = np.minimum(lens, offsets + out_samples)          # planning.effective_taps
        too_long = taps > (self.block64_taps if block64 else self.plan.max_parts * self.P)
        if too_long.any():
            k = int(np.argmax(too_long))
            raise ValueError(f"RIR {int(rir_ids[k])} needs {int(taps[k])} taps > max_taps={self.max_taps} the renderer was sized for")
        keys = np.stack([sources, offsets, wraps.astype(np.int64), out_samples], axis=1)
        if (keys == keys[0]).all():                             # the usual step: every env plays the same clip window
            xs = np.asarray([self._windows(int(keys[0, 0]), int(keys[0, 1]), bool(keys[0, 2]), int(keys[0, 3]), block64)], dtype=np.int64)
            inverse = np.zeros(rows.size, dtype=np.int64)
        else:
            uniq, first, inverse = np.unique(keys, axis=0, return_index=True, return_inverse=True)
            inverse = inverse.reshape(-1)
            xs = np.empty((uniq.shape[0], 3), dtype=np.int64)
            for u in np.argsort(first):                         # allocate window sets in request order
                src, off, wrap, outs = (int(v) for v in uniq[u])
                xs[u] = self._windows(src, off, bool(wrap), outs, block64)
        terms["rir_offset"][rows] = off_arr[rir_ids]
        terms["x_offset"][rows] = xs[inverse, 0]
        terms["rir_taps"][rows] = taps
        terms["x_nw"][rows] = xs[inverse, 1]
        terms["x_wofs"][rows] = xs[inverse, 2]

    # ----------------------------------------------------------------- render
    def prepare(self, requests: Sequence[AudioRequest]) -> PreparedBatch:
        """Resolve requests into the device request array.  A PreparedBatch stays valid until the
        window-spectra pool is recycled (only when it overflows) or the RIR bank is reset."""
        try:
            return self._prepare(requests)
        except _PoolReset:
            try:
                return self._prepare(requests)            # pool is empty now: the whole batch must fit
            except _PoolReset:
                raise RuntimeError("window-spectra pool too small for this batch; raise xpool_bytes") from None

    def _prepare(self, requests: Sequence[AudioRequest]) -> PreparedBatch:
        """Host cost matters here: a step of 128 envs takes about 0.2 ms on an H100, so the request array is filled
        with array operations (one pass over the request objects, then :meth:`_prepare_columns`)."""
        n = len(requests)
        if n == 0:
            return self._prepare_columns(np.zeros((0, 8), dtype=np.int64))
        sr = self.sr
        f = np.array([(-1 if r.rir is None else r.rir, r.source, r.offset, r.wrap, r.silent,
                       sr if r.out_samples is None else r.out_samples,
                       -1 if r.distractor_rir is None else r.distractor_rir,
                       -1 if r.distractor_source is None else r.distractor_source) for r in requests], dtype=np.int64)
        return self._prepare_columns(f)

    def prepare_arrays(self, rir, source, offset=0, out_samples=None, wrap=False, silent=False,
                       distractor_rir=-1, distractor_source=-1) -> PreparedBatch:
        """:meth:`prepare` for callers that already hold their requests as arrays (one entry per env, scalars
        broadcast; -1 = no RIR / no distractor): skips the per-request Python objects altogether."""
        rir = np.atleast_1d(np.asarray(rir, dtype=np.int64))
        f = np.empty((rir.shape[0], 8), dtype=np.int64)
        cols = (rir, source, offset, wrap, silent, self.sr if out_samples is None else out_samples,
                distractor_rir, distractor_source)
        for k, c in enumerate(cols):
            f[:, k] = np.asarray(c, dtype=np.int64)
        try:
            return self._prepare_columns(f)
        except _PoolReset:
            try:
                return self._prepare_columns(f)
            except _PoolReset:
                raise RuntimeError("window-spectra pool too small for this batch; raise xpool_bytes") from None

    def _prepare_columns(self, f: np.ndarray) -> PreparedBatch:
        """f: (n, 8) int64 columns rir, source, offset, wrap, silent, out_samples, distractor_rir, distractor_source."""
        n = f.shape[0]
        reqs = np.zeros(n, dtype=REQ_DTYPE)
        if n:
            out_samples = f[:, 5]
            if out_samples.min() <= 0 or out_samples.max() > self.sr:
                raise ValueError("out_samples must be in (0, sr]")
            silent = f[:, 4] != 0
            reqs["out_samples"] = out_samples
            reqs["flags"][silent] = SSB_FLAG_SILENT
            rows = np.flatnonzero(~silent)
            g = f[rows]
            terms = reqs["term"]
            sel = g[:, 7] >= 0
            block64 = self._block64_eligible(g, sel)
            self._fill_terms(terms[:, 0], rows, g[:, 0], g[:, 1], g[:, 2], g[:, 3] != 0, g[:, 5], block64)
            if sel.any():
                if self.plan.n_terms < 2:
                    raise ValueError("renderer was created with n_terms=1; distractors need n_terms=2")
                # the whole distractor clip is convolved in full mode and cut to [:sr] (simulator.py:661-664)
                d = g[sel]
                k = d.shape[0]
                self._fill_terms(terms[:, 1], rows[sel], d[:, 6], d[:, 7], np.zeros(k, np.int64), np.zeros(k, bool), d[:, 5])
        else:
            block64 = self.plan64 is not None
        dev = self._upload_requests(reqs)
        return PreparedBatch(n, reqs, dev, self.plan64 if block64 else self.plan)

    def _upload_requests(self, reqs: np.ndarray) -> torch.Tensor:
        """Request array -> device.  A plain (synchronous, pageable) copy of the 9 KB array: staging it through a ring of
        pinned buffers with completion events costs more bookkeeping than the copy."""
        return torch.from_numpy(reqs.view(np.uint8).reshape(-1)).to(self.device, non_blocking=False)

    def _block64_eligible(self, g: np.ndarray, has_distractor: np.ndarray) -> bool:
        """Single-block plan for this batch?  Every non-silent request must have one term and at most
        65536 - sr + 1 EFFECTIVE taps (min(file taps, offset + out_samples), planning.effective_taps)."""
        if self.plan64 is None:
            return False
        ok = not has_distractor.any()
        if ok and g.shape[0]:
            if self._bank_index is None:
                self._bank_index = (np.asarray(self._rir_off, dtype=np.int64), np.asarray(self._rir_len, dtype=np.int64))
            len_arr = self._bank_index[1]
            ids = g[:, 0]
            if ids.size and int(ids.max()) >= len(len_arr):
                raise ValueError(f"unknown RIR id {int(ids.max())}")
            lens = np.where(ids >= 0, len_arr[np.where(ids >= 0, ids, 0)] if len(len_arr) else 0, 0)
            ok = bool((np.minimum(lens, g[:, 2] + g[:, 5]) <= self.block64_taps).all())
        if self.force_block64 and not ok:
            raise ValueError(f"log2n=16: a request has a distractor or more than {self.block64_taps} effective taps")
        return ok

    def _scratch(self, n, plan=None):
        h_elems = n * (self.plan if plan is None else plan).h_elems_per_env
        if self._hscratch is None or self._hscratch.numel() < 2 * h_elems:
            self._hscratch = torch.empty(max(2 * h_elems, 2), dtype=torch.float32, device=self.device)
        if self._wave is None or self._wave.shape[0] < n:
            self._wave = torch.empty((n, 2, self.sr), dtype=torch.float32, device=self.device)
        return self._hscratch, self._wave[:n]

    def execute(self, batch: PreparedBatch, want_wave: bool = False, out: Optional[torch.Tensor] = None,
                channels_first: bool = False):
        """Run convolution + spectrogram for a prepared batch on the current stream.
        Returns spec (n, 65, T', 2) [, wave (n, 2, sr)] as CUDA tensors.  The waveform buffer is
        owned by the renderer and overwritten by the next call (clone to keep).

        ``out`` may be any contiguous CUDA tensor of the right shape, e.g. the rollout-storage slot
        ``rollouts.observations["spectrogram"][step + 1]`` (ss_baselines/common/rollout_storage.py:88-91):
        the observation is then written in place and ``insert`` has nothing to copy.
        ``channels_first=True`` emits (n, 2, 65, T') -- the layout ``AudioCNN.forward`` asks for with
        ``permute(0, 3, 1, 2)`` (ss_baselines/av_nav/models/audio_cnn.py:86); ``spec.permute(0, 2, 3, 1)`` is
        then the reference-shaped view and the CNN's permute of it is contiguous for free."""
        n = batch.n
        shape = (n, 2, self.spec_shape[0], self.spec_shape[1]) if channels_first else (n,) + self.spec_shape
        spec = out if out is not None else torch.empty(shape, dtype=torch.float32, device=self.device)
        if n == 0:
            return (spec, self._scratch(0)[1]) if want_wave else spec
        if not (spec.is_cuda and spec.is_contiguous() and tuple(spec.shape) == shape and spec.dtype == torch.float32):
            raise ValueError("bad output tensor")
        hs, wave = self._scratch(n, batch.plan)
        self.ctx.check(self.lib.ssb_render_batch(
            self.ctx.handle, C.byref(batch.plan), n, batch.reqs_dev.data_ptr(), self._bank.data_ptr(),
            self._xpool.data_ptr(), hs.data_ptr(), wave.data_ptr(), self.sr,
            self.pad_mode | (0x100 if channels_first else 0), spec.data_ptr(), self._stream()), "ssb_render_batch")
        return (spec, wave) if want_wave else spec

    @contextlib.contextmanager
    def transient_windows(self):
        """Window-spectra sets created inside the block are dropped at its end (stack discipline, like
        :meth:`bank_mark` / :meth:`bank_release` for RIRs).  The continuous simulator asks for a new
        ``(clip, sample offset)`` every step; without this each step would leave a dead set behind until the pool
        overflowed and was reset wholesale with a stream synchronise.  Safe while kernels are in flight: the next
        ``ssb_source_windows`` into the reclaimed space is ordered after them on the same stream."""
        used, keys = self._xpool_used, set(self._xcache)
        try:
            yield
        finally:
            if self._xpool_used >= used:                  # not recycled meanwhile
                for k in [k for k in self._xcache if k not in keys]:
                    del self._xcache[k]
                self._xpool_used = used

    @contextlib.contextmanager
    def _inline_rirs(self, *request_lists):
        """Upload the inline (transient) RIRs of one call behind a bank mark and drop them afterwards."""
        inline, seen = [], set()
        for reqs in request_lists:
            for r in reqs:
                if r is not None and r.rir_array is not None and not getattr(r, "_inline_live", False) \
                        and id(r) not in seen:
                    inline.append(r)
                    seen.add(id(r))
        if not inline:
            yield
            return
        mark = self.bank_mark()
        saved = [r.rir for r in inline]
        try:
            ids = self.add_rirs([np.asarray(r.rir_array, dtype=np.float32) for r in inline])
            for r, i in zip(inline, ids):
                r.rir = i
                r._inline_live = True                     # nested calls (render_crossfade -> convolve) reuse the upload
            yield
        finally:
            for r, old in zip(inline, saved):
                r.rir = old
                r._inline_live = False
            self.bank_release(mark)                       # later uploads are stream-ordered after the kernels

    def render(self, requests: Sequence[AudioRequest], want_wave: bool = False):
        with self._inline_rirs(requests):
            return self.execute(self.prepare(requests), want_wave=want_wave)

    def convolve_prepared(self, batch: PreparedBatch) -> torch.Tensor:
        """Waveforms (n, 2, sr) of a prepared batch (renderer-owned buffer, overwritten by the next call)."""
        hs, wave = self._scratch(batch.n, batch.plan)
        if batch.n:
            self.ctx.check(self.lib.ssb_convolve_batch(
                self.ctx.handle, C.byref(batch.plan), batch.n, batch.reqs_dev.data_ptr(), self._bank.data_ptr(),
                self._xpool.data_ptr(), hs.data_ptr(), wave.data_ptr(), self.sr, self._stream()),
                "ssb_convolve_batch")
        return wave

    def convolve(self, requests: Sequence[AudioRequest]) -> torch.Tensor:
        """Waveforms only: (n, 2, sr) -- ``get_current_audiogoal_observation`` for a batch."""
        with self._inline_rirs(requests):
            return self.convolve_prepared(self.prepare(requests))

    def render_crossfade(self, cur: Sequence[AudioRequest], prev: Sequence[Optional[AudioRequest]],
                         want_wave: bool = False):
        """Continuous simulator with CROSSFADE (continuous_simulator.py:422-424): render with the
        previous RIR and with the current one, blend the first int(0.05*sr)+1 samples."""
        n = len(cur)
        enable = torch.tensor([p is not None for p in prev], dtype=torch.uint8, device=self.device)
        prev_reqs = [p if p is not None else c for p, c in zip(prev, cur)]
        with self._inline_rirs(cur, prev):
            return self._render_crossfade(cur, prev_reqs, enable, n, want_wave)

    def _render_crossfade(self, cur, prev_reqs, enable, n, want_wave):
        w_prev = self.convolve(prev_reqs)
        if self._prev_wave is None or self._prev_wave.shape[0] < n:
            self._prev_wave = torch.empty((n, 2, self.sr), dtype=torch.float32, device=self.device)
        pw = self._prev_wave[:n]
        pw.copy_(w_prev)
        wave = self.convolve(cur)
        self.ctx.check(self.lib.ssb_crossfade_batch(self.ctx.handle, n, pw.data_ptr(), wave.data_ptr(), self.sr,
                                                    self.sr, enable.data_ptr(), self._stream()), "ssb_crossfade_batch")
        spec = self.spectrogram(wave)
        return (spec, wave) if want_wave else spec

    def spectrogram(self, wave: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """``SpectrogramSensor.compute_spectrogram`` (nav.py:86-100) for a (n, 2, sr) CUDA batch."""
        if wave.ndim == 2:
            wave = wave[None]
        if not (wave.is_cuda and wave.dtype == torch.float32 and wave.shape[1] == 2 and wave.shape[2] == self.sr):
            raise ValueError(f"expected CUDA float32 (n, 2, {self.sr})")
        wave = wave.contiguous()
        n = wave.shape[0]
        spec = out if out is not None else torch.empty((n,) + self.spec_shape, dtype=torch.float32, device=self.device)
        self.ctx.check(self.lib.ssb_spectrogram_batch(self.ctx.handle, n, wave.data_ptr(), self.sr, self.sr,
                                                      self.pad_mode, spec.data_ptr(), self._stream()),
                       "ssb_spectrogram_batch")
        return spec

    # ------------------------------------------------------------- log-mel (extension)
    def logmel_shape(self, n_mels: int = 64):
        """(n_mels, 1 + sr//160, 2)."""
        return (int(n_mels), self.lib.ssb_logmel_frames(self.sr), 2)

    def logmel(self, wave: torch.Tensor, n_mels: int = 64, power: int = 2, out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """EXTENSION (the reference has no mel front end; BASELINE.json configs[2] names one): per ear
        ``log1p(librosa.feature.melspectrogram(y, sr, n_fft=512, hop_length=160, win_length=400, n_mels, power))``
        on the reference's STFT geometry (nav.py:89-92) for a (n, 2, sr) CUDA batch -> (n, n_mels, 1 + sr//160, 2)."""
        if wave.ndim == 2:
            wave = wave[None]
        if not (wave.is_cuda and wave.dtype == torch.float32 and wave.shape[1] == 2 and wave.shape[2] == self.sr):
            raise ValueError(f"expected CUDA float32 (n, 2, {self.sr})")
        wave = wave.contiguous()
        n = wave.shape[0]
        shape = (n,) + self.logmel_shape(n_mels)
        res = out if out is not None else torch.empty(shape, dtype=torch.float32, device=self.device)
        if not (res.is_cuda and res.is_contiguous() and tuple(res.shape) == shape and res.dtype == torch.float32):
            raise ValueError("bad output tensor")
        self.ctx.check(self.lib.ssb_logmel_batch(self.ctx.handle, n, wave.data_ptr(), self.sr, self.sr, int(n_mels),
                                                 int(power), self.pad_mode, res.data_ptr(), self._stream()),
                       "ssb_logmel_batch")
        return res

    def render_logmel(self, requests: Sequence[AudioRequest], n_mels: int = 64, power: int = 2,
                      out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Convolution (every reference branch, as :meth:`convolve`) followed by :meth:`logmel`."""
        return self.logmel(self.convolve(requests), n_mels=n_mels, power=power, out=out)

    # --------------------------------------------------------- host-buffer path
    def make_host_session(self, n: int, taps: int, want_wave: bool = False, n_chunks: int = 4):
        """Pinned host buffers + device staging for the host-buffer entry (the e2e path)."""
        return HostSession(self, n, taps, want_wave, n_chunks)


class HostSession:
    """End-to-end entry with HOST buffers: per step the (n, taps, 2) RIRs are copied from pinned
    host memory, rendered, and the spectrograms (optionally waveforms) are copied back --
    what the reference's per-env numpy API hands over and gets back."""

    def __init__(self, r: BatchedAudioRenderer, n: int, taps: int, want_wave: bool, n_chunks: int = 4):
        self.r, self.n, self.taps, self.n_chunks = r, n, taps, n_chunks
        self.h_rir = torch.empty((n, taps, 2), dtype=torch.float32).pin_memory()
        self.h_spec = torch.empty((n,) + r.spec_shape, dtype=torch.float32).pin_memory()
        self.h_wave = torch.empty((n, 2, r.sr), dtype=torch.float32).pin_memory() if want_wave else None
        self.h_reqs = torch.empty(n * REQ_DTYPE.itemsize, dtype=torch.uint8).pin_memory()
        # two device staging sets, alternated per step: the copy of step k+1 overlaps the kernels of step k
        self.d_rir = [torch.empty((n, taps, 2), dtype=torch.float32, device=r.device) for _ in range(2)]
        self.d_reqs = [torch.empty(n * REQ_DTYPE.itemsize, dtype=torch.uint8, device=r.device) for _ in range(2)]
        self._step = 0
        self.d_spec = torch.empty((n,) + r.spec_shape, dtype=torch.float32, device=r.device)
        self.h2d_bytes = self.h_rir.numel() * 4 + self.h_reqs.numel()
        self.d2h_bytes = self.h_spec.numel() * 4 + (self.h_wave.numel() * 4 if want_wave else 0)

    def set_requests(self, source: int, silent=None, taps=None):
        """All envs play ``source`` through their own RIR row (the 1-s clip branch)."""
        r = self.r
        reqs = np.zeros(self.n, dtype=REQ_DTYPE)
        eff = np.minimum(self.taps if taps is None else np.asarray(taps), r.sr)
        self.block64 = r.plan64 is not None and int(np.max(eff)) <= r.block64_taps
        self.plan = r.plan64 if self.block64 else r.plan
        for i in range(self.n):
            reqs[i]["out_samples"] = r.sr
            if silent is not None and silent[i]:
                reqs[i]["flags"] = SSB_FLAG_SILENT
                continue
            L = self.taps if taps is None else int(taps[i])
            if L == 0:
                continue
            x_off, nw, wofs = r._windows(source, 0, False, r.sr, self.block64)
            t = reqs[i]["term"][0]
            t["rir_offset"], t["x_offset"] = i * self.taps, x_off
            t["rir_taps"] = min(L, r.sr, r.block64_taps if self.block64 else r.plan.max_parts * r.P)
            t["x_nw"], t["x_wofs"] = nw, wofs
        self.h_reqs.numpy()[:] = reqs.view(np.uint8).reshape(-1)

    def run(self):
        """Enqueue H2D + kernels + D2H (asynchronous; the current stream completes when the results
        have landed in ``h_spec`` / ``h_wave``).  ``h_rir`` must not be refilled before that."""
        r = self.r
        hs, wave = r._scratch(self.n, self.plan)
        d_rir, d_reqs = self.d_rir[self._step & 1], self.d_reqs[self._step & 1]
        self._step += 1
        r.ctx.check(r.lib.ssb_render_batch_host(
            r.ctx.handle, C.byref(self.plan), self.n, self.h_reqs.data_ptr(), self.h_rir.data_ptr(),
            self.h_rir.numel() * 4, d_rir.data_ptr(), d_reqs.data_ptr(), r._xpool.data_ptr(),
            hs.data_ptr(), wave.data_ptr(), r.sr, r.pad_mode, self.d_spec.data_ptr(), self.h_spec.data_ptr(),
            self.h_wave.data_ptr() if self.h_wave is not None else None, self.n_chunks, r._stream()),
            "ssb_render_batch_host")
        h2d, d2h = C.c_int64(), C.c_int64()
        r.lib.ssb_host_copy_bytes(r.ctx.handle, C.byref(h2d), C.byref(d2h))
        self.h2d_bytes, self.d2h_bytes = h2d.value, d2h.value      # what this step really moved (silent envs need no RIR)
        return self.h_spec
