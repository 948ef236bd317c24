"""The cases of tests/test_gpu_conv_stack_train_domain.py as plain data, shared with
tests/test_conv_stack_train_domain_host.py, which checks through a restatement of ``cs_plan`` and ``cs_launch_gemm``
(soundspaces_b200/csrc/ssb200.cu) that they reach every tile edge, residue class and limit of the training kernels.

A case is a dict made by :func:`case`, the call as ``ssb_conv_stack_train_*_batch`` sees it: ``kind`` "audio" (a
(B, H, W, 2) spectrogram with ``NL`` labels in rows of ``label_stride`` floats), "visual" (``nA`` RGB channels, times
1 / 255, then ``nB`` depth channels) or "map" (``nA`` channels); layer i has ``C[i]`` output channels, kernel
``K[i] = (kh, kw)``, stride ``S[i] = (sh, sw)`` and ReLU flag ``relu[i]``; then a Linear to ``hidden`` with ReLU flag
``lin_relu``.  ``bias`` says which of conv1, conv2, conv3 and the Linear have a bias.  ``B`` is the batch the case runs
at and ``family`` the group whose error bar the host calibrates.

The inference entries accept the reused layouts (the rollout domain cases), so the training forward's bits are
compared with them there; the rest are the training kernels' own edges, checked against float64.
"""
import torch

import audio_encoder_domain_cases as ac
import avnav_domain_cases as vc
import map_cnn_domain_cases as mc

MAX_B, MAX_K, MAX_LABELS = 65535, 2048, 256
MAX_STRIDE_AREA, MAX_HIDDEN = 65535, 4194240            # the two grid limits of the backward
INT32_MAX = 2 ** 31 - 1
BM, BN, BK, RCHUNK = 128, 32, 16, 2048                 # cs_gemm_kernel's tile and the weight gradients' chunk
GG_BM, GG_BN = 64, 64                                  # the Linear's GEMM tile (gru_gemm_kernel)
UNIT = ((1, 1), (1, 1), (1, 1))


def case(name, kind, nA, H, W, C, K, S, hidden, nB=0, NL=0, label_stride=None, bias=True, relu=(1, 1, 0),
         lin_relu=1, B=3, family="edges"):
    bias = (bias,) * 4 if isinstance(bias, bool) else tuple(bias)
    return dict(name=name, kind=kind, nA=nA, nB=nB, H=H, W=W, NL=NL, label_stride=NL if label_stride is None else
                label_stride, C=tuple(C), K=tuple(K), S=tuple(S), bias=bias, hidden=hidden, relu=tuple(relu),
                lin_relu=lin_relu, B=B, family=family)


def from_audio(c, family="reused"):
    return case(c["name"], "audio", 2, c["H"], c["W"], c["C"], c["K"], c["S"], c["hidden"], NL=c["NL"],
                label_stride=c["label_stride"], bias=c["bias"], B=c["B"], family=family)


def from_visual(c, family="reused"):
    return case("visual_" + c["name"], "visual", c["n_rgb"], c["H"], c["W"], c["C"], c["K"], c["S"], c["hidden"],
                nB=c["n_depth"], bias=c["bias"], B=3, family=family)


def from_map(c, family="reused"):
    return case("map_" + c["name"], "map", c["C"], c["H"], c["W"], c["Cs"], c["K"], c["S"], c["hidden"],
                bias=c["bias"], B=3, family=family)


def layer_shapes(c):
    """[(IC, H, W, OC, Ho, Wo, kh, kw, sh, sw)] of the three convs (IC without labels), or None when one is empty."""
    out, h, w, ic = [], c["H"], c["W"], c["nA"] + c["nB"]
    for oc, (kh, kw), (sh, sw) in zip(c["C"], c["K"], c["S"]):
        if kh > h or kw > w:
            return None
        ho, wo = (h - kh) // sh + 1, (w - kw) // sw + 1
        out.append((ic, h, w, oc, ho, wo, kh, kw, sh, sw))
        h, w, ic = ho, wo, oc
    return out


def features(c):
    s = layer_shapes(c)[2]
    return s[3] * s[4] * s[5]


# the rollout entries' domain cases, which the inference entries take: the forward's bits are compared there
REUSED = ([from_audio(c) for c in ac.AUDIO + ac.LABELS + ac.LIMIT + ac.REF_FITS]
          + [from_visual(c) for c in vc.VISUAL + vc.LIMIT] + [from_map(c) for c in mc.LAYOUTS + mc.LIMIT])
# past the inference entries' shared-memory limit: only the training entry takes them
OVER_LIMIT = ([from_audio(c, "over_limit") for c in ac.OVER_LIMIT]
              + [from_visual(c, "over_limit") for c in vc.OVER_LIMIT]
              + [from_map(c, "over_limit") for c in mc.OVER_LIMIT])

FWD = [
    # CS_FWD rows B Ho Wo of conv3 (a 1 x 1 output) 1, 127, 128 and 129 around the 128-row tile; OC 1, 31, 32 and 33
    # around the 32-channel tile; K = IC KH KW of 1 (conv1 1 x 1 over one channel), 15 (conv2 3 x 5 over one channel;
    # conv3 3 x 5 over one channel), 16 (conv1 2 x 4 over two) and 17 (conv1 1 x 1 over 17)
    case("fwd_rows1_oc1_k1_k15", "map", 1, 5, 7, (1, 1, 31), ((1, 1), (3, 5), (3, 3)), ((1, 1), (1, 1), (1, 1)), 3, B=1,
         family="fwd"),
    case("fwd_rows127_oc31", "map", 1, 5, 7, (31, 32, 33), ((1, 1), (1, 1), (5, 7)), UNIT, 4, B=127,
         family="fwd"),
    case("fwd_rows128_oc32_k16_k15", "map", 2, 4, 8, (32, 1, 33), ((2, 4), (1, 1), (3, 5)), UNIT, 2, B=128,
         family="fwd"),
    case("fwd_rows129_oc33_k17", "map", 17, 3, 3, (33, 2, 32), ((1, 1), (3, 3), (1, 1)), UNIT, 33, B=129,
         family="fwd"),
    # K = 2047 (conv2 over 2047 channels, 1 x 1) and K = 2048 (conv3 over 128 channels, 4 x 4)
    case("fwd_k2047", "map", 1, 3, 3, (2047, 3, 2), ((1, 1), (1, 1), (1, 1)), UNIT, 5, B=2, family="fwd"),
    case("fwd_k2048", "map", 2, 6, 6, (4, 128, 3), ((1, 1), (1, 1), (4, 4)), UNIT, 5, B=2, family="fwd"),
]

DW = [
    # rows B H W of every (1 x 1, stride 1) layer: 2047, 2048, 2049, 4096 and 4097 give 1, 1, 2, 2 and 3 chunks of
    # 2048, the last partial where 2048 does not divide
    case("dw_rows2047", "map", 1, 23, 89, (4, 3, 2), UNIT, UNIT, 5, B=1, family="dw"),
    case("dw_rows2048", "map", 1, 32, 64, (4, 3, 2), UNIT, UNIT, 5, B=1, family="dw"),
    case("dw_rows2049", "map", 1, 3, 683, (4, 3, 2), UNIT, UNIT, 5, B=1, family="dw"),
    case("dw_rows4096", "map", 2, 32, 32, (4, 3, 2), UNIT, UNIT, 5, B=4, family="dw"),
    case("dw_rows4097", "map", 1, 17, 241, (4, 3, 2), UNIT, UNIT, 5, B=1, family="dw"),
    # K = 127, 128 and 129 (conv2 over 127 channels 1 x 1, 8 channels 4 x 4, 43 channels 1 x 3): 1, 1 and 2 row tiles
    case("dw_k127", "map", 1, 6, 6, (127, 5, 2), ((1, 1), (1, 1), (2, 2)), UNIT, 3, B=3, family="dw"),
    case("dw_k128", "map", 1, 9, 9, (8, 5, 2), ((1, 1), (4, 4), (2, 2)), UNIT, 3, B=3, family="dw"),
    case("dw_k129", "map", 1, 6, 9, (43, 5, 2), ((1, 1), (1, 3), (2, 2)), UNIT, 3, B=3, family="dw"),
]


def _dx(name, at, IC, K, S, H, W, OC=5, B=3):
    """A DX geometry (kernel K, stride S, IC input channels, an H x W layer input) on conv2 (``at`` = 1) or conv3
    (``at`` = 2); the other layers 1 x 1 at stride 1."""
    Ks, Ss, Cs = [(1, 1)] * 3, [(1, 1)] * 3, [4, 4, 3]
    Ks[at], Ss[at], Cs[at - 1], Cs[at] = K, S, IC, OC
    return case(name, "map", 2, H, W, Cs, Ks, Ss, 3, B=B, family="dx")


DX = [g for at in (1, 2) for g in (
    # kernel divisible by the stride (4 / 2), and not (5 / 2), with sh != sw elsewhere
    _dx(f"dx{at}_k4s2", at, 32, (4, 4), (2, 2), 10, 10),
    _dx(f"dx{at}_k5s2", at, 31, (5, 5), (2, 2), 11, 12),
    # a kernel smaller than the stride (2 / 3): classes rh = 2 have Jh = 0 (and rw = 2 Jw = 0); input rows 2, 5, 8, 9
    # and columns likewise never read
    _dx(f"dx{at}_k2s3_unread", at, 33, (2, 2), (3, 3), 10, 10),
    # a stride larger than the layer input (5 > 3 rows, 7 > 4 columns): classes with Qh = 0 or Qw = 0
    _dx(f"dx{at}_stride_over_input", at, 32, (2, 1), (5, 7), 3, 4),
    # sh != sw, non-square kernel, one not divisible
    _dx(f"dx{at}_k3x4_s2x1", at, 33, (3, 4), (2, 1), 9, 8),
    # KX = OC ceil(KH / SH) ceil(KW / SW) = 2048: 128 channels through a 4 x 4 kernel at stride 1
    _dx(f"dx{at}_kx2048", at, 4, (4, 4), (1, 1), 6, 6, OC=128, B=2),
)]

LABEL_COUNTS = (0, 1, 21, 256)
LABEL_LAYOUT = dict(H=16, W=12, C=(8, 6, 4), K=((4, 3), (3, 3), (2, 2)), S=((2, 1), (2, 2), (1, 1)), hidden=7)
INPUTS = ([dict(case(f"labels{n}_{kind}_{scale:g}", "audio", 2, NL=n, label_stride=n + 3, B=4, family="inputs",
                     **LABEL_LAYOUT), labels=(kind, scale))
           for n in LABEL_COUNTS for kind, scale in (ac.LABEL_KINDS if n else ac.LABEL_KINDS[:1])]
          # SAVi's 21 one-hot labels at an input seed whose ReLU inputs all lie clear of 0 (end to end and routing)
          + [dict(case("route_labels21", "audio", 2, NL=21, B=4, family="inputs", **LABEL_LAYOUT),
                  labels=("one_hot", 1.0), seed=33)]
          + [case(f"visual_{a}rgb_{b}depth", "visual", a, 20, 24, (6, 5, 4), ((4, 4), (3, 3), (2, 2)),
                  ((2, 2), (1, 2), (1, 1)), 6, nB=b, B=3, family="inputs")
             for a, b in ((3, 0), (0, 1), (3, 1), (3, 2), (9, 3))]
          + [case(f"map_c{c}", "map", c, 14, 13, (5, 4, 3), ((3, 3), (3, 2), (2, 2)), ((2, 2), (1, 1), (1, 1)), 5,
                  B=3, family="inputs") for c in range(1, 9)])

# biases and flags on one small layout
FLAG_LAYOUT = dict(kind="map", nA=2, H=12, W=11, C=(6, 5, 4), K=((3, 3), (3, 2), (2, 2)), S=((2, 1), (1, 2), (1, 1)),
                   hidden=6, B=4)
FLAGS = ([case(f"no_bias{i}", bias=tuple(j != i for j in range(4)), family="flags", **FLAG_LAYOUT) for i in range(4)]
         + [case(f"relu{r1}{r2}{r3}_lin{lr}", relu=(r1, r2, r3), lin_relu=lr, family="flags", **FLAG_LAYOUT)
            for r1 in (0, 1) for r2 in (0, 1) for r3 in (0, 1) for lr in (0, 1)])

# batch sizes on a small layout; 65536 is refused
SMALL_LAYOUT = dict(kind="map", nA=1, H=8, W=8, C=(4, 4, 2), K=((3, 3), (2, 2), (2, 2)), S=((1, 1), (2, 2), (1, 1)),
                    hidden=4)
BATCHES = [case(f"batch{b}", B=b, family="batch", **SMALL_LAYOUT) for b in (1, 2, 17, 65535)]

# the non-finite and exact-zero inputs: one env per case, on the flag layout and an audio layout with 21 labels
INPUT_LAYOUT = case("nonfinite", family="inputs", **FLAG_LAYOUT)
LABEL_INPUT_LAYOUT = case("nonfinite_labels", "audio", 2, NL=21, label_stride=24, B=4, family="inputs",
                          **LABEL_LAYOUT)

# the forward workspace: conv1's output at float 0, conv2's after it, each region a multiple of 4 floats
def round4(n):
    return (n + 3) // 4 * 4


def saved_offsets(c, B=None):
    """(offset, shape) in floats of conv1's and conv2's outputs in the forward workspace (``cs_plan``'s a1, a2)."""
    B = c["B"] if B is None else B
    s1, s2 = layer_shapes(c)[:2]
    return [(0, (B, s1[3], s1[4], s1[5])), (round4(B * s1[3] * s1[4] * s1[5]), (B, s2[3], s2[4], s2[5]))]


# limits as accepted / refused pairs, checked through ssb_conv_stack_train_workspace_bytes (nothing is allocated)
LIMITS = [
    (case("k2048", "map", 128, 4, 4, (1, 1, 1), ((4, 4), (1, 1), (1, 1)), UNIT, 1, family="limit"), True),
    (case("k2049", "map", 2049, 1, 1, (1, 1, 1), UNIT, UNIT, 1, family="limit"), False),
    (case("kx2048", "map", 1, 4, 4, (1, 128, 1), ((1, 1), (4, 4), (1, 1)), UNIT, 1, family="limit"), True),
    (case("kx2049", "map", 1, 1, 1, (1, 1, 2049), UNIT, UNIT, 1, family="limit"), False),
    (case("labels256", "audio", 2, 4, 4, (1, 1, 1), UNIT, UNIT, 1, NL=256, label_stride=300, family="limit"), True),
    (case("labels257", "audio", 2, 4, 4, (1, 1, 1), UNIT, UNIT, 1, NL=257, label_stride=300, family="limit"), False),
    (case("b65535", "map", 1, 1, 1, (1, 1, 1), UNIT, UNIT, 1, B=65535, family="limit"), True),
    (case("b65536", "map", 1, 1, 1, (1, 1, 1), UNIT, UNIT, 1, B=65536, family="limit"), False),
    # B H W (the channels-last observation's pixels): 32768 x 65535 = 2^31 - 32768, 32768 x 65537 > 2^31 - 1
    (case("bhw_in", "visual", 1, 1, 65535, (1, 1, 1), UNIT, UNIT, 1, B=32768, family="limit"), True),
    (case("bhw_over", "visual", 1, 1, 65537, (1, 1, 1), UNIT, UNIT, 1, B=32768, family="limit"), False),
    # a layer's B C H W input (conv1's two map channels) and output (conv1's two channels), within 2^31 - 1 (65535 x 2 x
    # 16384 = 2^31 - 32768) and past it, with B H W itself far below
    (case("bchw_input_in", "map", 2, 1, 16384, (1, 1, 1), UNIT, UNIT, 1, B=65535, family="limit"), True),
    (case("bchw_input_over", "map", 2, 1, 16385, (1, 1, 1), UNIT, UNIT, 1, B=65535, family="limit"), False),
    (case("bchw_output_in", "map", 1, 1, 16384, (2, 1, 1), UNIT, UNIT, 1, B=65535, family="limit"), True),
    (case("bchw_output_over", "map", 1, 1, 16385, (2, 1, 1), UNIT, UNIT, 1, B=65535, family="limit"), False),
    # B hidden: 65535 x 32768 = 2^31 - 32768, and 65535 x 32769 > 2^31 - 1 (2^31 - 1 itself is prime)
    (case("bhidden_in", "map", 1, 1, 1, (1, 1, 1), UNIT, UNIT, 32768, B=65535, family="limit"), True),
    (case("bhidden_over", "map", 1, 1, 1, (1, 1, 1), UNIT, UNIT, 32769, B=65535, family="limit"), False),
    # the two grid edges of the backward: conv2's / conv3's dX at SH SW = 65535 (the last grid z) and 65536, and the
    # Linear's dW at hidden = 4194240 (grid y 65535) and 4194241 (65536)
    (case("stride_area65535_conv2", "map", 1, 1, 1, (1, 1, 1), UNIT, ((1, 1), (3, 21845), (1, 1)), 1,
          family="limit"), True),
    (case("stride_area65536_conv2", "map", 1, 1, 1, (1, 1, 1), UNIT, ((1, 1), (256, 256), (1, 1)), 1,
          family="limit"), False),
    (case("stride_area65536_conv3", "map", 1, 1, 1, (1, 1, 1), UNIT, ((1, 1), (1, 1), (256, 256)), 1,
          family="limit"), False),
    (case("hidden4194240", "map", 1, 1, 1, (1, 1, 1), UNIT, UNIT, 4194240, B=1, family="limit"), True),
    (case("hidden4194241", "map", 1, 1, 1, (1, 1, 1), UNIT, UNIT, 4194241, B=1, family="limit"), False),
]
GRID_EDGES = ("stride_area65536_conv2", "stride_area65536_conv3", "hidden4194241")

# rollout cases the training entry refuses (conv3's KX = C3 ceil(KH / SH) ceil(KW / SW) or K past 2048): the patched
# module runs the original for them
TRAIN_REFUSED = ("f256", "f257", "limit_conv3_slice", "over_conv3_slice")
# every case that runs on the GPU against float64
RUN = [c for c in REUSED + OVER_LIMIT + FWD + DW + DX + INPUTS + FLAGS + BATCHES[:3] if c["name"] not in TRAIN_REFUSED]
REFUSED = [c for c in REUSED + OVER_LIMIT if c["name"] in TRAIN_REFUSED]


def make_params(c, seed=0):
    """(w1, b1, w2, b2, w3, b3, w_lin, b_lin) of a case on the CPU in float32 (torch's default init), absent biases
    None, present ones in [-0.1, 0.1] so that every ReLU clips."""
    g = torch.Generator().manual_seed(seed)
    out, ic = [], c["nA"] + c["nB"] + c["NL"]
    for oc, (kh, kw), b in zip(c["C"], c["K"], c["bias"]):
        s = (ic * kh * kw) ** -0.5
        out.append((torch.rand((oc, ic, kh, kw), generator=g) * 2 - 1) * s)
        out.append(torch.rand(oc, generator=g) * 0.2 - 0.1 if b else None)
        ic = oc
    F = features(c)
    out.append((torch.rand((c["hidden"], F), generator=g) * 2 - 1) * F ** -0.5)
    out.append(torch.rand(c["hidden"], generator=g) * 0.2 - 0.1 if c["bias"][3] else None)
    return out


def make_inputs(c, B=None, seed=None):
    """(x, depth, labels) of a case on the CPU in float32: a spectrogram in [0, 3), RGB in [0, 255), depth and maps in
    [0, 1), labels as a (B, NL) view of rows of ``label_stride`` floats whose other columns are NaN (never read), of
    the case's ("labels") kind, else soft in [-1, 1); drawn from the case's ``seed`` (default 1)."""
    B = c["B"] if B is None else B
    g = torch.Generator().manual_seed(c.get("seed", 1) if seed is None else seed)
    H, W = c["H"], c["W"]
    depth = labels = None
    if c["kind"] == "audio":
        x = torch.rand((B, H, W, 2), generator=g) * 3.0
    elif c["kind"] == "visual":
        x = torch.floor(torch.rand((B, H, W, c["nA"]), generator=g) * 255.0) if c["nA"] else None
        depth = torch.rand((B, H, W, c["nB"]), generator=g) if c["nB"] else None
    else:
        x = torch.rand((B, H, W, c["nA"]), generator=g)
    if c["NL"]:
        kind, scale = c.get("labels", ("soft", 1.0))
        NL = c["NL"]
        if kind == "one_hot":
            lab = torch.nn.functional.one_hot(torch.randint(0, NL, (B,), generator=g), NL).float()
        elif kind == "zero":
            lab = torch.zeros(B, NL)
        elif kind == "negative":
            lab = -torch.rand((B, NL), generator=g)
        else:
            lab = torch.rand((B, NL), generator=g) * 2.0 - 1.0
        buf = torch.full((B, c["label_stride"]), float("nan"))
        buf[:, :NL] = lab * scale
        labels = buf[:, :NL]
    return x, depth, labels

# the cases held to float64 autograd end to end: no ReLU input within float32 rounding of 0 (the host file checks)
END_TO_END = ("fwd_rows1_oc1_k1_k15", "fwd_k2048", "dw_rows2047", "dw_rows2048", "dw_rows2049", "dw_rows4097",
              "dw_k129", "dx1_k4s2", "dx1_k2s3_unread", "dx1_stride_over_input", "dx1_k3x4_s2x1", "dx2_k2s3_unread",
              "dx2_stride_over_input", "dx2_k3x4_s2x1", "dx2_kx2048", "labels0_one_hot_1", "labels256_soft_0.001",
              "map_c1", "map_c2", "visual_kernel_is_input", "route_labels21", "map_f257", "relu000_lin0",
              "relu010_lin0", "relu100_lin0", "no_bias2", "no_bias3", "batch1", "batch2", "batch17")
