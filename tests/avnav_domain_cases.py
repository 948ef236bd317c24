"""The cases of tests/test_gpu_avnav_policy_domain.py as plain data, shared with tests/test_avnav_domain_host.py, which
checks through a restatement of the kernels' tiling that they reach every tile edge, dispatch instance and limit.

A visual case is a dict made by :func:`conv_stack`: conv1 takes ``IC = n_rgb + n_depth`` channels (RGB first), and
layer i has ``C[i]`` output channels, kernel ``K[i] = (kh, kw)`` and stride ``S[i] = (sh, sw)`` on an H x W input,
followed by a Linear to ``hidden``.  A GRU case is a tuple ``(I, Hd, B, masks, scales)``: ``masks`` is ``"mixed"``
(0 / 1) or a tuple of values given to env b in turn, ``scales`` is ``(weights, x, biases)``.
"""
import torch
import torch.nn as nn

REF_K = ((8, 8), (4, 4), (3, 3))
AV_NAV_S = ((4, 4), (2, 2), (2, 2))
AV_NAV_C = (32, 64, 64)


def conv_stack(IC, C, K, S, H, W, hidden, bias=True, n_rgb=None, name=""):
    """One visual layout.  ``n_rgb`` defaults to 3 when IC > 3 (RGB-D), else 0 (depth only)."""
    if n_rgb is None:
        n_rgb = 3 if IC > 3 else 0
    return dict(name=name, IC=IC, n_rgb=n_rgb, n_depth=IC - n_rgb, C=tuple(C), K=tuple(K), S=tuple(S), H=H, W=W,
                hidden=hidden, bias=bias)


def layer_shapes(c):
    """[(C, ho, wo, kh, kw, sh, sw)] of the three convs, or None when a layer's output is empty."""
    out, h, w = [], c["H"], c["W"]
    for oc, (kh, kw), (sh, sw) in zip(c["C"], c["K"], c["S"]):
        if kh > h or kw > w:
            return None
        h, w = (h - kh) // sh + 1, (w - kw) // sw + 1
        out.append((oc, h, w, kh, kw, sh, sw))
    return out


def features(c):
    oc, h, w = layer_shapes(c)[2][:3]
    return oc * h * w


def make_cnn(c, seed=0):
    """``VisualCNN.cnn`` of a case on the CPU in float32, with biases in [-0.1, 0.1] so that every ReLU clips."""
    torch.manual_seed(seed)
    convs, ic = [], c["IC"]
    for oc, k, s in zip(c["C"], c["K"], c["S"]):
        convs.append(nn.Conv2d(ic, oc, k, s, bias=c["bias"]))
        ic = oc
    cnn = nn.Sequential(convs[0], nn.ReLU(True), convs[1], nn.ReLU(True), convs[2], nn.Flatten(),
                        nn.Linear(features(c), c["hidden"], bias=c["bias"]), nn.ReLU(True))
    with torch.no_grad():
        for m in cnn:
            if getattr(m, "bias", None) is not None:
                m.bias.uniform_(-0.1, 0.1)
    return cnn.eval()


VISUAL = [
    # every kernel and stride non-square; conv2 (3 x 4) and conv3 (2 x 3) take the generic instance
    conv_stack(4, (16, 32, 32), ((8, 5), (3, 4), (2, 3)), ((4, 3), (1, 2), (2, 1)), 96, 128, 100, name="nonsquare"),
    # the reference 8 / 4 / 3 kernels at non-square strides: the 4 x 4 and 3 x 3 instances at sh != sw
    conv_stack(4, AV_NAV_C, REF_K, ((4, 2), (2, 1), (1, 2)), 64, 40, 64, name="ref_kernels_nonsquare_strides"),
    # one input channel, 1 / 3 / 1 output channels: most ranks idle in every layer, H1 = 7
    conv_stack(1, (1, 3, 1), REF_K, ((4, 4), (1, 1), (1, 1)), 32, 37, 5, name="tiny_channels"),
    # odd channel counts (17: a 3-channel slice per rank), strides larger than the kernels, RGB only
    conv_stack(3, (7, 9, 17), ((3, 2), (2, 2), (1, 1)), ((5, 6), (3, 3), (1, 2)), 64, 80, 513, n_rgb=3,
               name="odd_channels"),
    # conv1's kernel is the whole input: H1 = W1 = 1, C1 = 33; F = 3
    conv_stack(4, (33, 8, 3), ((12, 20), (1, 1), (1, 1)), ((1, 1), (1, 1), (1, 1)), 12, 20, 3, name="kernel_is_input"),
    # H1 = 7 with W1 = 10 (a tail of 2 pixels); 3 x 3 conv2 / conv3 at unit stride
    conv_stack(4, AV_NAV_C, ((8, 8), (3, 3), (3, 3)), ((4, 4), (1, 1), (1, 1)), 32, 44, 64, name="short_rows_tail2"),
    # RGB + 2 depth channels, W1 = 17 (a tail of 1), hidden = 130
    conv_stack(5, (32, 64, 32), REF_K, AV_NAV_S, 64, 72, 130, name="rgb_2depth"),
    # 12 input channels, W1 = 19 (a tail of 3); a 4 x 5 conv2 takes the generic instance
    conv_stack(12, (16, 16, 8), ((4, 4), (4, 5), (3, 3)), ((2, 2), (2, 2), (1, 1)), 40, 40, 64, n_rgb=9,
               name="ic12"),
    # bias=False on every layer
    conv_stack(1, AV_NAV_C, REF_K, AV_NAV_S, 64, 64, 16, bias=False, name="no_bias"),
    # F = 1 and hidden = 1; W1 = 8
    conv_stack(1, (4, 4, 1), REF_K, AV_NAV_S, 36, 36, 1, name="one_feature"),
    # F = 257, just past the 256-wide feature stride
    conv_stack(1, (8, 8, 257), REF_K, AV_NAV_S, 36, 36, 8, name="f257"),
]

# av_nav's layout at the shared-memory limit, through each branch of max(C2 H2 W2, C1 IC KH KW + IC KH W): RGB-D
# 48 x 382 (conv1 weights and input rows) and depth 44 x 484 (conv2 activations) need exactly 232448 bytes; the nearest
# wider shapes, 48 x 383 and 44 x 488, are over it
LIMIT = [conv_stack(4, AV_NAV_C, REF_K, AV_NAV_S, 48, 382, 8, name="limit_rgbd"),
         conv_stack(1, AV_NAV_C, REF_K, AV_NAV_S, 44, 484, 8, name="limit_depth")]
OVER_LIMIT = [conv_stack(4, AV_NAV_C, REF_K, AV_NAV_S, 48, 383, 8, name="over_rgbd"),
              conv_stack(1, AV_NAV_C, REF_K, AV_NAV_S, 44, 488, 8, name="over_depth")]
SMEM_LIMIT = 232448

# the layout for the input-domain cases (NaN, Inf, scales) and the largest batch
INPUT_LAYOUT = conv_stack(4, AV_NAV_C, REF_K, AV_NAV_S, 48, 64, 64, name="inputs_rgbd")
BIG_B_LAYOUT = conv_stack(1, AV_NAV_C, REF_K, AV_NAV_S, 36, 36, 32, name="big_b_depth")
MAX_ENVS = 65535
SCALES = (1e-6, 1e3)

GRU_WIDTHS = (1, 31, 255, 256, 257, 513, 4096)
GRU_BATCHES = (1, 15, 16, 17, 129)
MASK_VALUES = (0.5, 2.0, -1.0, float("inf"), float("-inf"), float("nan"), 0.0, 1.0)
GRU = [
    (1, 1, 17, "mixed", (1, 1, 1)),
    (31, 257, 129, "mixed", (1, 1, 1)),
    (255, 31, 16, "mixed", (1, 1, 1)),
    (256, 513, 15, "mixed", (1, 1, 1)),
    (257, 256, 1, "mixed", (1, 1, 1)),
    (513, 255, 17, "mixed", (1, 1, 1)),
    (4096, 1, 16, "mixed", (1, 1, 1)),
    (1, 4096, 15, "mixed", (1, 1, 1)),
    # every mask value, at I = Hd = 1 and off the tiles
    (1, 1, 16, MASK_VALUES, (1, 1, 1)),
    (257, 31, 17, MASK_VALUES, (1, 1, 1)),
    # saturated gates, badly scaled x, zero biases.  x * 1e3 at I = 1: with I = 255 the gate sums reach ~1e4, and
    # float32 rounding alone (torch's CPU forward) is 1.8e-4 of the output where a tanh argument crosses 0
    (255, 257, 17, "mixed", (30, 1, 1)),
    (1, 257, 17, "mixed", (1, 1e3, 1)),
    (255, 257, 17, "mixed", (1, 1e-6, 1)),
    (255, 257, 17, "mixed", (1, 1, 0)),
]
GRU_BIG_B = (31, 31)
