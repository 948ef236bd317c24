"""A numpy model, in float64, of the equations ``ssb_conv_stack_train_forward_batch`` / ``_backward_batch`` compute
for ``Conv2d ReLU Conv2d ReLU Conv2d Flatten Linear ReLU`` (include/ssb200.h): the forward from the observation (the
spectrogram with SAVi's labels as constant conv1 channels, RGB / 255 then depth, or a map); the backward in the
kernels' order and form: the Linear's ReLU mask (the gradient passes where !(out <= 0)), dW_lin = g^T F, dF = g W_lin,
then per conv dW / db summed over (env, pixel) rows in chunks of 2048, dX as a gather over the taps of each input
pixel's residue class (ih mod SH, iw mod SW) masked by the ReLU below, and a label channel's tap gradients all
sum_n labels[n][c] sum_pos g1[n][oc][pos].

Also the golden cases of tests/golden/make_conv_stack_golden.py: :func:`case_inputs` regenerates their inputs from
seeds, and :func:`grad_summary` is what the fixture stores of a gradient."""
import numpy as np
import torch

RCHUNK = 2048


def cnn_input(kind, x, depth=None, labels=None):
    """The channels-first network input: 'audio' the ears (labels apart), 'visual' RGB / 255 then depth, 'map' x."""
    parts = []
    if kind == "visual":
        if x is not None:
            parts.append(np.transpose(x, (0, 3, 1, 2)) / 255.0)
        if depth is not None:
            parts.append(np.transpose(depth, (0, 3, 1, 2)))
    else:
        parts.append(np.transpose(x, (0, 3, 1, 2)))
    return np.concatenate(parts, axis=1)


def im2col(a, KH, KW, SH, SW):
    """(N Ho Wo, C KH KW) rows of (env, output pixel), columns (c, kh, kw)."""
    N, C, H, W = a.shape
    Ho, Wo = (H - KH) // SH + 1, (W - KW) // SW + 1
    cols = np.empty((N, Ho, Wo, C, KH, KW))
    for kh in range(KH):
        for kw in range(KW):
            cols[:, :, :, :, kh, kw] = np.transpose(a[:, :, kh:kh + SH * (Ho - 1) + 1:SH,
                                                      kw:kw + SW * (Wo - 1) + 1:SW], (0, 2, 3, 1))
    return cols.reshape(N * Ho * Wo, C * KH * KW), Ho, Wo


def conv(a, w, b, stride, bias_rows=None):
    """Conv2d of a channels-first a; ``bias_rows`` (N, OC) replaces b per env (the label fold)."""
    N = a.shape[0]
    OC, _, KH, KW = w.shape
    cols, Ho, Wo = im2col(a, KH, KW, *stride)
    y = cols @ w.reshape(OC, -1).T
    y = y.reshape(N, Ho, Wo, OC)
    if bias_rows is not None:
        y = y + bias_rows[:, None, None, :]
    elif b is not None:
        y = y + b
    return np.transpose(y, (0, 3, 1, 2))


def relu(v):
    return np.where(v > 0, v, np.where(np.isnan(v), v, 0.0))



def mask(g, act):
    """torch's threshold_backward on the ReLU output: 0 where act <= 0, else g (NaN passes)."""
    return np.where(act <= 0, 0.0, g)


def forward(kind, x, params, strides, depth=None, labels=None, flags=(1, 1, 0), lin_relu=1):
    """-> (a1, a2, features, out) for ``params`` = (w1, b1, w2, b2, w3, b3, w_lin, b_lin), any bias None;
    ``flags`` the three convs' ReLU flags, ``lin_relu`` the Linear's."""
    w1, b1, w2, b2, w3, b3, wl, bl = params
    a0 = cnn_input(kind, x, depth)
    lbias = None
    if labels is not None:                        # the label channels: a per-env conv1 bias
        L = labels.shape[1]
        lbias = (0.0 if b1 is None else b1[None, :]) + labels @ w1[:, 2:2 + L].sum(axis=(2, 3)).T
        w1 = w1[:, :2]
    act = lambda v, f: relu(v) if f else v                                 # noqa: E731
    a1 = act(conv(a0, w1, b1, strides[0], lbias), flags[0])
    a2 = act(conv(a1, w2, b2, strides[1]), flags[1])
    a3 = act(conv(a2, w3, b3, strides[2]), flags[2])
    feat = a3.reshape(a3.shape[0], -1)
    y = feat @ wl.T + (0.0 if bl is None else bl)
    return a1, a2, feat, act(y, lin_relu)


def _weight_grad(a_in, g, KH, KW, stride):
    """dW (OC, C KH KW) and db (OC,) of one conv, summed over rows in chunks of RCHUNK, chunks in order."""
    cols, _, _ = im2col(a_in, KH, KW, *stride)
    gr = np.transpose(g, (0, 2, 3, 1)).reshape(-1, g.shape[1])
    dw, db = 0.0, 0.0
    for r0 in range(0, gr.shape[0], RCHUNK):
        dw = dw + gr[r0:r0 + RCHUNK].T @ cols[r0:r0 + RCHUNK]
        db = db + gr[r0:r0 + RCHUNK].sum(axis=0)
    return dw, db


def _input_grad(g, w, in_shape, stride):
    """dX of one conv as a gather: input pixel (ih, iw) of residue (rh, rw) sums the taps kh = rh + SH jh,
    kw = rw + SW jw whose output pixel (qh - jh, qw - jw) exists."""
    N, C, H, W = in_shape
    OC, _, KH, KW = w.shape
    SH, SW = stride
    Ho, Wo = g.shape[2:]
    dx = np.zeros(in_shape)
    for rh in range(SH):
        for rw in range(SW):
            Qh, Qw = (H - rh + SH - 1) // SH, (W - rw + SW - 1) // SW
            for jh in range(max(0, (KH - rh + SH - 1) // SH)):
                for jw in range(max(0, (KW - rw + SW - 1) // SW)):
                    kh, kw = rh + SH * jh, rw + SW * jw
                    q0h, q1h = jh, min(Qh, jh + Ho)
                    q0w, q1w = jw, min(Qw, jw + Wo)
                    if q1h <= q0h or q1w <= q0w:
                        continue
                    part = np.einsum("nohw,oc->nchw", g[:, :, :q1h - q0h, :q1w - q0w], w[:, :, kh, kw])
                    dx[:, :, rh + SH * q0h:rh + SH * (q1h - 1) + 1:SH, rw + SW * q0w:rw + SW * (q1w - 1) + 1:SW] += part
    return dx


def backward(kind, x, params, strides, dout, depth=None, labels=None, flags=(1, 1, 0), lin_relu=1):
    """The eight parameter gradients of sum(out * dout)."""
    acts = forward(kind, x, params, strides, depth, labels, flags, lin_relu)
    return backward_given(kind, x, params, strides, dout, acts, depth, labels, masks(acts, flags, lin_relu))


def masks(acts, flags=(1, 1, 0), lin_relu=1):
    """Where the gradient passes each ReLU (conv1, conv2, conv3, Linear) of the activations ``acts`` (a1, a2, features,
    out): !(act <= 0) where the flag is set, everywhere where it is not."""
    return [np.ones(a.shape, bool) if not f else ~(np.asarray(a) <= 0)
            for a, f in zip(acts, tuple(flags) + (lin_relu,))]


def backward_given(kind, x, params, strides, dout, acts, depth=None, labels=None, keep=None):
    """The backward from given activations ``acts`` (a1, a2, features, out) and ReLU pass masks ``keep``
    (:func:`masks`): the kernels' equations with the forward taken as given.  With |x|, |params|, |labels|, |dout|,
    |acts| and the masks of the real activations it is the bound sum_terms |product| of every gradient."""
    w1, b1, w2, b2, w3, b3, wl, bl = params
    a1, a2, feat, _ = acts
    k1, k2, k3, ko = keep
    g = np.where(ko, dout, 0.0)
    dwl, dbl = g.T @ feat, g.sum(axis=0)
    H3, W3 = (a2.shape[2] - w3.shape[2]) // strides[2][0] + 1, (a2.shape[3] - w3.shape[3]) // strides[2][1] + 1
    g3 = np.where(k3, g @ wl, 0.0).reshape(feat.shape[0], w3.shape[0], H3, W3)
    dw3, db3 = _weight_grad(a2, g3, *w3.shape[2:], strides[2])
    g2 = np.where(k2, _input_grad(g3, w3, a2.shape, strides[2]), 0.0)
    dw2, db2 = _weight_grad(a1, g2, *w2.shape[2:], strides[1])
    g1 = np.where(k1, _input_grad(g2, w2, a1.shape, strides[1]), 0.0)
    a0 = cnn_input(kind, x, depth)
    dw1, db1 = _weight_grad(a0, g1, *w1.shape[2:], strides[0])
    dw1 = dw1.reshape((w1.shape[0], a0.shape[1]) + w1.shape[2:])
    if labels is not None:                        # every tap of label channel c: sum_n labels[n][c] sum_pos g1
        s = g1.sum(axis=(2, 3))
        lab = (labels.T @ s).T
        dw1 = np.concatenate([dw1, np.broadcast_to(lab[:, :, None, None], (w1.shape[0], labels.shape[1])
                                                   + w1.shape[2:])], axis=1)
    return [dw1, db1, dw2.reshape(w2.shape), db2, dw3.reshape(w3.shape), db3, dwl, dbl]


# golden cases: name -> (kind, spec), spec (H, W, C) of audio / map inputs or (n_rgb, n_depth, H, W) of visual ones
HIDDEN, N = 8, 4
CASES = {
    "avnav_audio16k": ("audio", (65, 26, 2)),
    "avnav_audio44k": ("audio", (65, 69, 2)),
    "savi_audio_category": ("audio_category", (65, 26, 2)),
    "visual_rgbd": ("visual", (3, 1, 36, 36)),
    "visual_depth": ("visual", (0, 1, 36, 36)),
    "visual_rgb": ("visual", (3, 0, 36, 36)),
    "map_gm": ("gm", (200, 200, 2)),
    "map_am": ("am", (20, 20, 1)),
}
FULL = 512            # gradients with at most this many elements are stored whole
SAMPLES, PROJ = 256, 32


def case_inputs(name):
    """(observations, dout) of golden case ``name``: float64 tensors holding float32 values, the first input's
    element [-1, 0, 0, 0] NaN, and the seeded upstream gradient of the N - 1 finite rows."""
    from avnav_models import visual_obs
    from map_cnn_models import map_obs
    i = list(CASES).index(name)
    kind, spec = CASES[name]
    g = torch.Generator().manual_seed(70 + i)
    if kind.startswith("audio"):
        obs = {"audiogoal": torch.rand((N,) + spec, generator=g, dtype=torch.float64) * 3}
        if kind == "audio_category":
            obs["category"] = torch.nn.functional.one_hot(torch.randint(0, 21, (N,), generator=g), 21).double()
        first = "audiogoal"
    elif kind == "visual":
        n_rgb, n_depth, H, W = spec
        obs = {k: v.double() for k, v in visual_obs(N, H, W, n_rgb, n_depth, seed=80 + i).items()}
        first = "rgb" if n_rgb else "depth"
    else:
        H, W, C = spec
        obs = {kind: map_obs(N, H, W, C, seed=80 + i, kind=kind).double()}
        first = kind
    obs = {k: v.float().double() for k, v in obs.items()}
    obs[first][-1, 0, 0, 0] = float("nan")
    return obs, torch.randn((N - 1, HIDDEN), generator=g, dtype=torch.float64)


def _probe(name, j, n):
    g = torch.Generator().manual_seed(1000 + 16 * list(CASES).index(name) + j)
    idx = torch.randperm(n, generator=g)[:SAMPLES].numpy()
    return idx, torch.randn((PROJ, n), generator=g, dtype=torch.float64).numpy()


def grad_summary(name, j, grad):
    """What the fixture keeps of gradient ``j`` of case ``name``: {"": the whole tensor} when it has at most FULL
    elements, else {"_sample": SAMPLES seeded elements, "_proj": PROJ seeded Gaussian projections of all of them}."""
    flat = np.asarray(grad, np.float64).reshape(-1)
    if flat.size <= FULL:
        return {"": flat}
    idx, P = _probe(name, j, flat.size)
    return {"_sample": flat[idx], "_proj": P @ flat}


def check_grad(name, j, grad, golden, rel):
    """Assert that ``grad`` agrees with the fixture's summary of gradient ``j``: each stored value within ``rel`` of
    its scale (the tensor's largest element; for a projection, sum_i |P_i| |grad_i|)."""
    flat = np.asarray(grad, np.float64).reshape(-1)
    key = f"{name}/g{j}"
    if key in golden:
        ref = golden[key]
        assert ref.shape == flat.shape and np.abs(flat - ref).max() <= rel * np.abs(ref).max(), key
        return
    idx, P = _probe(name, j, flat.size)
    sample = golden[key + "_sample"]
    assert np.abs(flat[idx] - sample).max() <= rel * np.abs(flat).max(), key + "_sample"
    scale = np.abs(P) @ np.abs(flat)
    assert (np.abs(P @ flat - golden[key + "_proj"]) <= rel * scale).all(), key + "_proj"
