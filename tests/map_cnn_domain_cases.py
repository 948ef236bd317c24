"""The cases of tests/test_gpu_map_cnn_domain.py as plain data, shared with tests/test_map_cnn_domain_host.py, which
checks through a restatement of ``ssb_map_encoder_batch``'s tiling that they reach every tile edge, kernel instance and
limit.

A case is a dict made by :func:`conv_stack`: conv1 takes the map's ``C`` channels, and layer i has ``Cs[i]`` output
channels, kernel ``K[i] = (kh, kw)``, stride ``S[i] = (sh, sw)`` and a bias when ``bias[i]`` (``bias[3]``: the
Linear's) on an H x W map, followed by a Linear to ``hidden``.
"""
import torch
import torch.nn as nn

REF_C = (32, 64, 32)
GM200 = (((8, 8), (4, 4), (3, 3)), ((4, 4), (2, 2), (1, 1)))      # MapCNN's kernels and strides at MAP_SIZE 200
GM400 = (((8, 8), (4, 4), (3, 3)), ((5, 5), (4, 4), (2, 2)))      # MAP_SIZE 400
AM = (((5, 5), (3, 3), (3, 3)), ((2, 2), (1, 1), (1, 1)))         # the acoustic map


def conv_stack(C, Cs, K, S, H, W, hidden, bias=True, name=""):
    """One layout.  ``bias``: one flag for every layer, or four (conv1, conv2, conv3, Linear)."""
    bias = (bias,) * 4 if isinstance(bias, bool) else tuple(bias)
    assert len(bias) == 4
    return dict(name=name, C=C, Cs=tuple(Cs), K=tuple(K), S=tuple(S), H=H, W=W, hidden=hidden, bias=bias)


def layer_shapes(c):
    """[(C, ho, wo, kh, kw, sh, sw)] of the three convs, or None when a layer's output is empty."""
    out, h, w = [], c["H"], c["W"]
    for oc, (kh, kw), (sh, sw) in zip(c["Cs"], c["K"], c["S"]):
        if kh > h or kw > w:
            return None
        h, w = (h - kh) // sh + 1, (w - kw) // sw + 1
        out.append((oc, h, w, kh, kw, sh, sw))
    return out


def features(c):
    oc, h, w = layer_shapes(c)[2][:3]
    return oc * h * w


def make_cnn(c, seed=0):
    """``MapCNN.cnn`` of a case on the CPU in float32, with biases in [-0.1, 0.1] so that every ReLU clips."""
    torch.manual_seed(seed)
    convs, ic = [], c["C"]
    for oc, k, s, b in zip(c["Cs"], c["K"], c["S"], c["bias"]):
        convs.append(nn.Conv2d(ic, oc, k, s, bias=b))
        ic = oc
    cnn = nn.Sequential(convs[0], nn.ReLU(True), convs[1], nn.ReLU(True), convs[2], nn.Flatten(),
                        nn.Linear(features(c), c["hidden"], bias=c["bias"][3]), nn.ReLU(True))
    with torch.no_grad():
        for m in cnn:
            if getattr(m, "bias", None) is not None:
                m.bias.uniform_(-0.1, 0.1)
    return cnn.eval()


LAYOUTS = [
    # the <8, 4> instance with KH1 = 6 and sh != sw in conv1 and conv2; overlapping conv1 windows; H1 = 17 (rank 0
    # holds three rows, the others two), W1 = 24; conv3 3 x 3 at sh != sw
    conv_stack(2, REF_C, ((6, 8), (4, 4), (3, 3)), ((3, 4), (2, 1), (1, 2)), 54, 100, 130, name="inst84_kh6"),
    # the <5, 3> instance with KH1 = 4; C1 = 7, C2 = 9, C3 = 17 (three-channel conv3 slices, an odd ENC_OCT tail);
    # H1 = 9, W1 = 9; conv3 4 x 4 at sh != sw; biases on conv2 and the Linear only
    conv_stack(1, (7, 9, 17), ((4, 5), (3, 3), (4, 4)), ((1, 2), (1, 1), (2, 1)), 12, 21, 3,
               bias=(False, True, False, True), name="inst53_kh4"),
    # conv1 kw = 8 before a 3 x 4 conv2: the generic instance; H1 = 9, W1 = 11, columns 48 and 49 never read; C2 = 5
    # (ranks 5 - 7 hold no conv2 channel); conv3 2 x 3 at sh != sw
    conv_stack(3, (16, 5, 24), ((8, 8), (3, 4), (2, 3)), ((4, 4), (2, 3), (3, 2)), 40, 50, 1, name="kw8_conv2_3x4"),
    # conv1 kw = 8 before a 4 x 3 conv2: the generic instance; five map channels, H1 = 8; C2 = 3; a 3 x 5 conv3 at
    # sh != sw; no bias on conv3 and the Linear
    conv_stack(5, (12, 3, 8), ((3, 8), (4, 3), (3, 5)), ((2, 1), (1, 2), (2, 1)), 17, 18, 130,
               bias=(True, True, False, False), name="kw8_conv2_4x3"),
    # a 4 x 4 conv2 after a conv1 with kw = 7: the generic instance; eight map channels; C1 = 9; H1 = 12 with rows 38
    # and 39 never read, W1 = 18; C3 = 1; a 4 x 2 conv3 at sh != sw
    conv_stack(8, (9, 16, 1), ((5, 7), (4, 4), (4, 2)), ((3, 2), (1, 3), (1, 2)), 40, 41, 130, name="conv2_4x4_kw7"),
    # conv1 strides that skip input (1 x 2 kernel at stride 2 x 3, row 9 and column 8 never read): H1 = 5 (ranks 5 - 7
    # idle in conv1), W1 = 3; a conv2 stride larger than its kernel; C3 = 3
    conv_stack(2, (4, 10, 3), ((1, 2), (2, 1), (1, 1)), ((2, 3), (3, 2), (1, 1)), 10, 9, 3, name="skip_idle_ranks"),
    # conv1's kernel is as tall as the map: H1 = 1 (ranks 1 - 7 hold no conv1 row), W1 = 10
    conv_stack(1, (3, 2, 1), ((6, 4), (1, 3), (1, 1)), ((1, 1), (1, 1), (1, 1)), 6, 13, 1, name="h1_one"),
    # conv2 as tall as conv1's output: H1 = 5, KH2 = 5, H2 = 1; a 1 x 4 conv3 at sh != sw
    conv_stack(3, (8, 8, 16), ((3, 3), (5, 2), (1, 4)), ((1, 2), (1, 1), (1, 3)), 7, 21, 130, name="conv2_full_height"),
    # F = 257: C3 = 257 on a 1 x 1 conv3 output (33-channel slices: an odd ENC_OCT tail); the <5, 3> instance
    conv_stack(1, (8, 8, 257), ((5, 5), (3, 3), (1, 1)), ((2, 2), (1, 1), (1, 1)), 9, 9, 3, name="f257"),
    # F = 256 (16 x 4 x 4); H1 = W1 = 8; a 4 x 4 conv2 after a 4 x 4 conv1: the generic instance
    conv_stack(2, (16, 24, 16), ((4, 4), (3, 3), (3, 3)), ((1, 1), (1, 1), (1, 1)), 11, 11, 130, name="f256"),
    # F = 255 (15 x 1 x 17); W1 = 19
    conv_stack(3, (5, 6, 15), ((2, 2), (2, 2), (2, 2)), ((2, 2), (1, 1), (1, 1)), 6, 38, 130, name="f255"),
    # F = 1, hidden = 1, no bias anywhere
    conv_stack(1, (2, 1, 1), ((3, 3), (2, 2), (1, 1)), ((3, 3), (1, 1), (1, 1)), 6, 6, 1, bias=False, name="f1_no_bias"),
]

# the shared-memory limit through each branch of max(rows1 + max(conv1 phase, conv2 phase), conv3 phase): MapCNN at
# MAP_SIZE 200 on 52 x 945 x 4 (conv1 phase: weights and staged input rows) and at MAP_SIZE 400 on 323 x 653 x 1
# (conv2 phase: gathered rows and weight slice) need exactly 232448 bytes, as does the acoustic geometry with channels
# 32 / 12 / 32 on 47 x 420 x 1 (conv3 phase: the gathered conv2 output).  The nearest wider shapes past the limit are
# 946, 658 and 421 columns wide (654 - 657 still need exactly 232448 bytes at MAP_SIZE 400).
SMEM_LIMIT = 232448
LIMIT = [conv_stack(4, REF_C, *GM200, 52, 945, 8, name="limit_conv1_phase"),
         conv_stack(1, REF_C, *GM400, 323, 653, 8, name="limit_conv2_phase"),
         conv_stack(1, (32, 12, 32), *AM, 47, 420, 8, name="limit_conv3_phase")]
OVER_LIMIT = [conv_stack(4, REF_C, *GM200, 52, 946, 8, name="over_conv1_phase"),
              conv_stack(1, REF_C, *GM400, 323, 658, 8, name="over_conv2_phase"),
              conv_stack(1, (32, 12, 32), *AM, 47, 421, 8, name="over_conv3_phase")]

# the layout of the input-value cases: MapCNN at MAP_SIZE 200 on a 64 x 66 x 2 map.  Input row r (4 <= r < 60) is read
# by conv1 rows r // 4 - 1 and r // 4, which two ranks own; columns 64 and 65 are never read
INPUT_LAYOUT = conv_stack(2, REF_C, *GM200, 64, 66, 64, name="inputs_gm")
UNREAD_PIXEL = (17, 65)
SHARED_ROW_PIXEL = (21, 30)
# the largest batch: MapCNN's acoustic geometry on a 20 x 20 x 1 map
BIG_B_LAYOUT = conv_stack(1, REF_C, *AM, 20, 20, 32, name="big_b_am")
MAX_ENVS = 65535
SCALES = (1e-6, 1e3)
# batch-size and permutation identity: the generic instance with idle ranks in conv1 and conv3
IDENTITY_LAYOUT = LAYOUTS[5]
IDENTITY_BATCHES = (1, 16, 17, 129)
# the per-layer relu flags through the entry
RELU_LAYOUT = LAYOUTS[1]

# F past INT32_MAX within the shared-memory limit: a 120 x 120 x 1 input through three 1 x 1 stride-1 convs with
# C1 = C2 = 1 and C3 = 149131 (189768 bytes of shared memory in the map and visual entries)
HUGE_F = conv_stack(1, (1, 1, 149131), ((1, 1),) * 3, ((1, 1),) * 3, 120, 120, 1, name="huge_f")
HUGE_F_FEATURES = 2147486400
HUGE_F_SMEM = 189768
