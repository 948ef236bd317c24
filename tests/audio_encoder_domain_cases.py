"""The cases of tests/test_gpu_audio_encoder_domain.py as plain data, shared with tests/test_audio_encoder_domain_host.py,
which checks through a restatement of the kernels' tiling that they reach every tile edge, dispatch instance and limit.

A case is a dict made by :func:`audio_stack`: the observation is (H, W, 2) (the two ears, as ssb_spectrogram_batch
writes it), conv1 takes ``2 + NL`` channels (``NL`` category labels after the ears, read with a row stride of
``label_stride`` floats), layer i has ``C[i]`` output channels, kernel ``K[i] = (kh, kw)`` and stride ``S[i] = (sh, sw)``,
followed by a Linear to ``hidden``.  ``bias`` says which of conv1, conv2, conv3 and the Linear have a bias.  ``B`` is the
batch the case runs at.
"""
import torch
import torch.nn as nn

SMEM_LIMIT = 232448
MAX_ENVS = 65535

# the reference's two conv stacks (ss_baselines/*/models/audio_cnn.py): under 30 pixels, and from 30 up
SMALL_K, SMALL_S = ((5, 5), (3, 3), (3, 3)), ((2, 2), (2, 2), (1, 1))
REF_K, REF_S = ((8, 8), (4, 4), (3, 3)), ((4, 4), (2, 2), (1, 1))
UNIT = ((1, 1), (1, 1), (1, 1))


def audio_stack(name, H, W, C, K, S, hidden, NL=0, label_stride=None, bias=True, B=3):
    if isinstance(bias, bool):
        bias = (bias,) * 4
    return dict(name=name, H=H, W=W, C=tuple(C), K=tuple(K), S=tuple(S), hidden=hidden, NL=NL,
                label_stride=NL if label_stride is None else label_stride, bias=tuple(bias), B=B)


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
    """``AudioCNN.cnn`` of a case on the CPU in float32, with biases in [-0.2, 0.2] so that every ReLU clips."""
    torch.manual_seed(seed)
    convs, ic = [], 2 + c["NL"]
    for oc, k, s, b in zip(c["C"], c["K"], c["S"], c["bias"]):
        convs.append(nn.Conv2d(ic, oc, k, s, bias=b))
        ic = oc
    cnn = nn.Sequential(convs[0], nn.ReLU(True), convs[1], nn.ReLU(True), convs[2], nn.Flatten(),
                        nn.Linear(features(c), c["hidden"], bias=c["bias"][3]), nn.ReLU(True))
    with torch.no_grad():
        for m in cnn:
            if getattr(m, "bias", None) is not None:
                m.bias.uniform_(-0.2, 0.2)
    return cnn.eval()


def make_inputs(c, B, seed=1, kind=("soft", 1.0), device="cpu"):
    """(observation, labels) of a case on ``device``, drawn on the CPU: the observation uniform in [0, 3) (a
    log-magnitude spectrogram) with env 2 all zero when B > 2; labels None when NL = 0, else a (B, NL) view with row stride ``label_stride`` of a
    buffer whose other columns are NaN (never read), of the given (kind, scale)."""
    g = torch.Generator().manual_seed(seed)
    x = torch.rand((B, c["H"], c["W"], 2), generator=g) * 3.0
    if B > 2:
        x[2] = 0.0
    if not c["NL"]:
        return x.to(device), None
    name, scale = kind
    NL = c["NL"]
    if name == "one_hot":
        lab = nn.functional.one_hot(torch.randint(0, NL, (B,), generator=g), NL).float()
    elif name == "zero":
        lab = torch.zeros(B, NL)
    elif name == "negative":
        lab = -torch.rand((B, NL), generator=g)
    else:
        lab = torch.rand((B, NL), generator=g) * 2.0 - 1.0
    buf = torch.full((B, c["label_stride"]), float("nan"))
    buf[:, :NL] = lab * scale
    return x.to(device), buf.to(device)[:, :NL]


AUDIO = [
    # one conv1 channel: 7 idle ranks in conv1, 5 in conv2 (C2 = 3), 3 in conv3 (C3 = 5)
    audio_stack("c1_1_idle_ranks", 65, 26, (1, 3, 5), SMALL_K, SMALL_S, 3, B=17),
    # non-square conv1 kernel and stride; conv2 3 x 5 (generic) and conv3 4 x 4 at sh != sw; hidden off LIN_ROWS
    audio_stack("c1_3_nonsquare", 65, 40, (3, 12, 7), ((7, 3), (3, 5), (4, 4)), ((3, 1), (1, 2), (1, 2)), 130, B=16),
    # conv1 strides larger than its kernel; conv2 3 x 3 at sh != sw; conv3 4 x 6 (generic), C3 = 17: chunks of 3
    audio_stack("c1_9_stride_over_kernel", 65, 69, (9, 16, 17), ((2, 3), (3, 3), (4, 6)), ((4, 5), (2, 1), (2, 1)), 1,
                B=15),
    # conv1's kernel is the whole input: H1 = W1 = 1; C1 = 17 (a partial last chunk), C2 = 9, C3 = 33 (chunks of 5)
    audio_stack("c1_17_kernel_is_input", 16, 12, (17, 9, 33), ((16, 12), (1, 1), (1, 1)), UNIT, 3, B=129),
    # W = 1, what ssb_spectrogram_batch gives at sr = 512: k x 1 kernels, conv2 4 x 1 and conv3 3 x 1 (generic)
    audio_stack("c1_33_w1", 65, 1, (33, 10, 7), ((8, 1), (4, 1), (3, 1)), ((4, 1), (2, 1), (1, 1)), 130, B=1),
    # F = 1 and hidden = 1: conv3 2 x 2 (generic) over a 2 x 2 map
    audio_stack("f1", 16, 16, (4, 4, 1), ((5, 5), (3, 3), (2, 2)), SMALL_S, 1, B=16),
    # F = 255: C3 = 15 over a 1 x 17 map
    audio_stack("f255", 8, 40, (8, 16, 15), ((8, 4), (1, 2), (1, 2)), ((1, 2), (1, 1), (1, 1)), 3, B=17),
    # F = 256 and F = 257 (C3 = 257: a chunk of 33) over the reference kernels on a 36 x 36 input
    audio_stack("f256", 36, 36, (32, 64, 256), REF_K, REF_S, 130, B=129),
    audio_stack("f257", 36, 36, (32, 64, 257), REF_K, REF_S, 3, B=17),
    # bias=False on every layer, the reference's 16 kHz network
    audio_stack("no_bias", 65, 26, (32, 64, 64), SMALL_K, SMALL_S, 130, bias=False, B=17),
]

# SAVi with a distractor sound: the category entry.  Each case runs with every kind of label in LABEL_KINDS
LABELS = [
    # one label, conv1 1 x 1 (KK1 = 1) at a non-square stride, labels in every third float
    audio_stack("lab1_kk1", 65, 26, (9, 8, 3), ((1, 1), (3, 3), (3, 3)), ((2, 3), (2, 2), (1, 2)), 3, NL=1,
                label_stride=3, B=17),
    # SAVi's 21 labels, conv1 16 x 12 (KK1 = 192) without a bias: the fold starts from 0
    audio_stack("lab21_kk192_no_conv1_bias", 65, 26, (32, 64, 64), ((16, 12), (4, 4), (3, 3)),
                ((4, 2), (1, 1), (1, 1)), 130, NL=21, bias=(False, True, True, True), B=16),
    # 222 labels in rows of 230 floats; conv2 4 x 4 at sh != sw
    audio_stack("lab222", 16, 20, (17, 8, 4), ((5, 4), (4, 4), (2, 3)), ((2, 3), (2, 1), (1, 1)), 1, NL=222,
                label_stride=230, B=15),
]
# (kind, scale): one-hot, zero, signed soft in [-1, 1), all negative in [-1, 0), and soft labels scaled
LABEL_KINDS = (("one_hot", 1.0), ("zero", 1.0), ("soft", 1.0), ("negative", 1.0), ("soft", 1e-3), ("soft", 1e3))

# the shared-memory limit, exactly 232448 bytes, through each branch of the weight-slice max; the first two are the
# shapes of test_gpu_encoder.py::test_shared_memory_limit (conv2's slice) and test_gpu_encoder_category.py::
# test_shared_memory_limit_with_conv1_slice_largest (conv1's slice, 222 labels).  The last has the observation staged
# as 98 % of the footprint.  OVER_LIMIT: the same networks on the nearest wider observation.
LIMIT = [
    audio_stack("limit_conv1_slice_labels", 16, 16, (8, 248, 4), ((16, 16), (1, 1), (1, 1)), UNIT, 33, NL=222),
    audio_stack("limit_conv2_slice", 32, 8, (96, 123, 4), UNIT, UNIT, 33),
    audio_stack("limit_conv3_slice", 16, 16, (33, 128, 5), ((1, 1), (1, 1), (16, 8)), ((1, 1), (1, 1), (1, 4)), 33),
    audio_stack("limit_observation", 65, 439, (2, 5, 3), ((65, 3), (1, 4), (1, 3)), ((1, 3), (1, 2), (1, 2)), 33),
]
OVER_LIMIT = [dict(c, name=c["name"].replace("limit", "over"), W=c["W"] + 1) for c in LIMIT]

# the reference's own AudioCNN at H = 65: the widest observation that fits and the next one, for av_nav / savi
# (C3 = 64), av_wan (C3 = 32) and SAVi with a distractor sound (21 labels)
REF_FITS = [audio_stack("ref_avnav_w183", 65, 183, (32, 64, 64), REF_K, REF_S, 512),
            audio_stack("ref_avwan_w187", 65, 187, (32, 64, 32), REF_K, REF_S, 512),
            audio_stack("ref_savi_labels_w179", 65, 179, (32, 64, 64), REF_K, REF_S, 128, NL=21)]
REF_OVER = [dict(c, name=c["name"][:-3] + str(c["W"] + 1), W=c["W"] + 1) for c in REF_FITS]

# the layouts for the input-domain cases (NaN, Inf, all-zero env, ReLU flags) and the largest batch
INPUT_LAYOUT = audio_stack("inputs", 65, 26, (32, 64, 64), SMALL_K, SMALL_S, 130, B=5)
INPUT_LABELS = dict(INPUT_LAYOUT, name="inputs_labels", NL=21, label_stride=21)
BIG_B_LAYOUT = audio_stack("big_b", 16, 8, (8, 16, 8), ((4, 3), (3, 3), (3, 2)), ((2, 1), (2, 1), (1, 1)), 32)
BIG_B_LABELS = dict(BIG_B_LAYOUT, name="big_b_labels", NL=3, label_stride=3)
