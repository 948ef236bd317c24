"""Stand-ins for SAVi's visual encoder, written from its description (ss_baselines/savi/models/smt_cnn.py and
ss_baselines/common/utils.py:341-466): ``ResizeCenterCropper(size=(64, 64))`` resizes the shortest edge to 64 with
area averaging (bins ``[floor(i h / h'), ceil((i + 1) h / h'))``) and centre-crops 64 x 64 at ``(h' // 2 - 32,
w' // 2 - 32)``; ``SMTCNN`` runs one SMT ``custom_resnet18`` per modality on ``rgb.permute(0, 3, 1, 2) / 255`` and
``depth.permute(0, 3, 1, 2)`` and concatenates the features.  The area resize here is an explicit float64 sum, not
``F.interpolate``.  Parameters come from a seed keyed by module name, so the reference and the stand-in get equal
weights without storing them."""
import zlib

import numpy as np
import torch
import torch.nn as nn

from belief_nets_models import SmtResNet

CROP = 64


def geometry(H, W, size=CROP):
    """(h', w', crop_y, crop_x): image_resize_shortest_edge's and center_crop's expressions."""
    scale = size / min(H, W)
    h, w = int(H * scale), int(W * scale)
    return h, w, h // 2 - size // 2, w // 2 - size // 2


def area_matrix(n_in, n_out, dtype=torch.float64):
    """(n_out, n_in): row i averages inputs [floor(i n_in / n_out), ceil((i + 1) n_in / n_out))."""
    m = torch.zeros(n_out, n_in, dtype=dtype)
    for i in range(n_out):
        a, b = (i * n_in) // n_out, -((-(i + 1) * n_in) // n_out)
        m[i, a:b] = 1.0 / (b - a)
    return m


def bins(n_in, n_out, start, count=CROP):
    """(lo, hi) int64 arrays: the input range [floor(i n_in / n_out), ceil((i + 1) n_in / n_out)) of resized indices
    i = start .. start + count - 1 (adaptive_avg_pool2d's start_index / end_index)."""
    i = np.arange(start, start + count, dtype=np.int64)
    return i * n_in // n_out, -(-(i + 1) * n_in // n_out)


def crop_area_rows(n_in, n_out, start, count=CROP, dtype=torch.float64):
    """Rows start .. start + count - 1 of ``area_matrix(n_in, n_out)``, without building the others (a 65536-long
    resize of 1024 inputs would take 512 MB in float64)."""
    lo, hi = bins(n_in, n_out, start, count)
    m = torch.zeros(count, n_in, dtype=dtype)
    for r, (a, b) in enumerate(zip(lo.tolist(), hi.tolist())):
        m[r, a:b] = 1.0 / (b - a)
    return m


def resize_crop64(x, rh, rw, cy, cx):
    """The 64 x 64 crop at (cy, cx) of x's (..., H, W) area resize to rh x rw, as float64 matrix products."""
    H, W = x.shape[-2:]
    return crop_area_rows(H, rh, cy).to(x.device) @ x.double() @ crop_area_rows(W, rw, cx).to(x.device).T


def prep_image_f32(obs, mul, rh, rw, cy, cx):
    """The [B][C][64][64] float32 image ``ssb_smt_cnn_batch`` documents for the (B, H, W, C) observation ``obs``
    (include/ssb200.h): crop pixel (y, x) is resized pixel (y + cy, x + cx); every value of its bin is multiplied by
    ``mul`` and rounded to float32, the products are summed in float32 row by row, each row left to right, and the sum
    is divided by the bin's height and then by its width.  Vectorised over envs, channels and pixels by looping over
    the offsets inside the largest bin: an offset past a smaller bin adds 0, which leaves the sum unchanged, and reads
    a pixel inside the bin, so values outside every bin (NaN, Inf) never reach the sum."""
    x = np.asarray(obs, dtype=np.float32)
    B, H, W, C = x.shape
    mul = np.float32(mul)
    h0, h1 = bins(H, rh, cy)
    w0, w1 = bins(W, rw, cx)
    s = np.zeros((B, CROP, CROP, C), dtype=np.float32)
    for dy in range(int((h1 - h0).max())):
        rows = np.minimum(h0 + dy, h1 - 1)
        for dx in range(int((w1 - w0).max())):
            cols = np.minimum(w0 + dx, w1 - 1)
            v = x[:, rows[:, None], cols[None, :], :] * mul
            ok = ((h0 + dy < h1)[:, None] & (w0 + dx < w1)[None, :])[None, :, :, None]
            s = s + np.where(ok, v, np.float32(0))
    kh = (h1 - h0).astype(np.float32)[None, :, None, None]
    kw = (w1 - w0).astype(np.float32)[None, None, :, None]
    return np.ascontiguousarray((s / kh / kw).transpose(0, 3, 1, 2))


class ResizeCenterCropper(nn.Module):
    def __init__(self, size=(CROP, CROP), channels_last=False):
        super().__init__()
        self._size = tuple(size)
        self.channels_last = channels_last

    def forward(self, x):
        H, W = x.shape[-2:]
        h, w, cy, cx = geometry(H, W, max(self._size))
        dt = x.dtype if x.dtype == torch.float64 else torch.float32
        y = area_matrix(H, h, dt).to(x.device) @ x.to(dt) @ area_matrix(W, w, dt).to(x.device).T
        return y[..., cy:cy + self._size[0], cx:cx + self._size[1]].to(x.dtype)


ResizeCenterCropper.__module__ = "ss_baselines.common.utils"


class SMTCNN(nn.Module):
    """``channels``: {"rgb": C, "depth": C} (either may be absent); ``n_out``: the fc widths, 64 unless given per
    modality; ``no_bias``: the modalities whose fc has no bias."""

    def __init__(self, channels, obs_transform="default", n_out=None, no_bias=()):
        super().__init__()
        self.obs_transform = ResizeCenterCropper() if obs_transform == "default" else obs_transform
        self.input_modalities = []
        for m in ("rgb", "depth"):
            if m in channels:
                self.input_modalities.append(m)
                net = SmtResNet(channels[m], (n_out or {}).get(m, 64), 128 * 8 * 8)
                if m in no_bias:
                    net.fc = nn.Linear(128 * 8 * 8, net.fc.out_features, bias=False)
                setattr(self, f"{m}_encoder", net)

    def forward(self, observations):
        feats = []
        for m in self.input_modalities:
            x = observations[m].permute(0, 3, 1, 2)
            if m == "rgb":
                x = x / 255.0
            if self.obs_transform:
                x = self.obs_transform(x)
            feats.append(getattr(self, f"{m}_encoder")(x))
        return torch.cat(feats, dim=1)


def set_params(module, seed):
    """Every Conv2d / Linear / GroupNorm of ``module`` from a generator seeded by (seed, module name): convs at He
    scale, Linear at 1 / sqrt(fan_in) with a 0.1 bias, GroupNorm affines around (1, 0)."""
    with torch.no_grad():
        for name, m in module.named_modules():
            if not isinstance(m, (nn.Conv2d, nn.Linear, nn.GroupNorm)):
                continue
            g = torch.Generator().manual_seed(seed * 1000003 + zlib.crc32(name.encode()))
            if isinstance(m, nn.Conv2d):
                fan_in = m.in_channels * m.kernel_size[0] * m.kernel_size[1]
                m.weight.copy_(torch.randn(m.weight.shape, generator=g, dtype=torch.float64) * (2.0 / fan_in) ** 0.5)
            elif isinstance(m, nn.Linear):
                m.weight.copy_(torch.randn(m.weight.shape, generator=g, dtype=torch.float64) / m.in_features ** 0.5)
                if m.bias is not None:
                    m.bias.copy_(0.1 * torch.randn(m.bias.shape, generator=g, dtype=torch.float64))
            else:
                m.weight.copy_(1.0 + 0.3 * torch.randn(m.weight.shape, generator=g, dtype=torch.float64))
                m.bias.copy_(0.2 * torch.randn(m.bias.shape, generator=g, dtype=torch.float64))
    return module


def observations(B, H, W, seed, rgb=3, depth=1):
    """Seeded float32 observations: integer-valued RGB in [0, 255] and depth in multiples of 1 / 1000 in [0, 1],
    with a smooth gradient so resized images are not pure noise.  Returns {"rgb", "depth"} as (B, H, W, C)."""
    rng = np.random.default_rng(seed)
    yy, xx = np.meshgrid(np.linspace(0, 1, H), np.linspace(0, 1, W), indexing="ij")
    out = {}
    if rgb:
        base = 120 * (yy + xx)[None, :, :, None]
        out["rgb"] = torch.from_numpy(np.clip(base + rng.integers(0, 60, (B, H, W, rgb)), 0, 255).astype(np.float32))
    if depth:
        k = np.clip(500 * yy[None, :, :, None] + rng.integers(0, 500, (B, H, W, depth)), 0, 1000).astype(np.uint16)
        out["depth"] = torch.from_numpy(k.astype(np.float32) / np.float32(1000))
    return out
