"""Cases, seeded parameters, the reference loss and a numpy float64 model of the kernels of SAVi's audio-goal predictor
training (ssb_resnet18_train_*) for tests/golden/audiogoal_train_golden.npz.

The model follows the kernels' equations rather than autograd's: BatchNorm normalises with the batch mean and biased
variance per channel (training) or the running statistics (eval), and its backward is dz = gamma rstd (dS - sum dS / N
- x^ sum dS x^ / N) over every row, a row with a zero upstream gradient included; the ReLU gradient is taken on the
saved output; the maxpool routes each window's gradient to its first maximum in row-major order and each stem pixel
gathers the windows that picked it; AdaptiveAvgPool2d's backward spreads dY / (H4 W4); conv gradients are the padded
dW and gather-form dX of tests/smt_resnet_train_models.py."""
import numpy as np
import torch

from smt_resnet_train_models import _conv, _conv_dw, _conv_dx, _geometry

# name: (H, W, n_out, B, mode, steps); every case with B > 1 has row 1 silent and row 2 scaled by 1e-3
CASES = {
    "s26_o23_b7": (65, 26, 23, 7, "train", 2),
    "s69_o21_b1": (65, 69, 21, 1, "train", 1),
    "s26_o2_b64": (65, 26, 2, 64, "train", 1),
    "s69_o23_b7_eval": (65, 69, 23, 7, "eval", 1),
}
PARAM_SEED = 110
MOMENTUM = 0.1
FULL = 64                 # tensors up to this many elements are stored whole
SAMPLES, PROJ = 16, 8


def tv_net(n_out):
    """AudioGoalPredictor's predictor: torchvision's resnet18 with a 2-channel stem and fc = Linear(512, n_out)."""
    import torchvision
    m = torchvision.models.resnet18(weights=None)
    m.conv1 = torch.nn.Conv2d(2, 64, kernel_size=7, stride=2, padding=3, bias=False)
    m.fc = torch.nn.Linear(512, n_out)
    return m


def set_params(net, seed=PARAM_SEED):
    """Seeded parameters and running statistics in the order of belief_nets.resnet18_params / resnet18_buffers, so
    the reference class and the stand-in get the same values: convs at He scale, gamma around 1, beta around 0, fc
    weight / sqrt(in) and bias 0.1, running means around 0 and variances in [0.5, 1.5)."""
    from soundspaces_b200.belief_nets import resnet18_buffers, resnet18_params
    g = torch.Generator().manual_seed(seed)
    rnd = lambda shape: torch.randn(shape, generator=g, dtype=torch.float64)       # noqa: E731
    with torch.no_grad():
        for i, p in enumerate(resnet18_params(net)):
            if i < 20:
                fan_in = p.shape[1] * p.shape[2] * p.shape[3]
                p.copy_(rnd(p.shape) * (2.0 / fan_in) ** 0.5)
            elif i < 40:
                p.copy_(1.0 + 0.3 * rnd(p.shape))
            elif i < 60:
                p.copy_(0.2 * rnd(p.shape))
            elif i == 60:
                p.copy_(rnd(p.shape) / p.shape[1] ** 0.5)
            else:
                p.copy_(0.1 * rnd(p.shape))
        bufs = resnet18_buffers(net)
        for t in bufs[:20]:
            t.copy_(0.3 * rnd(t.shape))
        for t in bufs[20:40]:
            t.copy_(0.5 + torch.rand(t.shape, generator=g, dtype=torch.float64))
        for t in bufs[40:]:
            t.zero_()
    for _, n in _pairs(net):
        n.momentum = MOMENTUM
    return net


def _pairs(net):
    from soundspaces_b200.belief_nets import conv_norm_pairs
    return conv_norm_pairs(net)


def case_inputs(name, step=0):
    """(spectrogram (B, H, W, 2), targets (B, 3): label, x, y) in float32, from the case's seed and step."""
    H, W, n_out, B, _, _ = CASES[name]
    g = torch.Generator().manual_seed(1000 + 17 * sum(map(ord, name)) + step)
    x = torch.rand((B, H, W, 2), generator=g) * 3.0
    if B > 1:
        x[1] = 0.0
        x[2] *= 1e-3
    gts = torch.cat([torch.randint(0, 21, (B, 1), generator=g).float(), torch.randn((B, 2), generator=g) * 5.0], 1)
    return x, gts


def reference_loss(pred, gts):
    """audiogoal_trainer.py:113-124: CrossEntropy on the 21 label logits and MSE on the last two outputs, whichever
    the predictor has."""
    n_out = pred.shape[1]
    ce, mse = torch.nn.functional.cross_entropy, torch.nn.functional.mse_loss
    if n_out == 23:
        return ce(pred[:, :-2], gts[:, 0].long()) + mse(pred[:, -2:], gts[:, -2:])
    if n_out == 21:
        return ce(pred, gts[:, 0].long())
    return mse(pred, gts[:, -2:])


def torch_step(net, x, gts):
    """pred and the 62 parameter gradients of the reference loss through ``net`` (its own dtype and mode)."""
    from soundspaces_b200.belief_nets import resnet18_params
    dt = next(net.parameters()).dtype
    net.zero_grad(set_to_none=True)
    pred = net(x.to(dt).permute(0, 3, 1, 2))
    reference_loss(pred, gts.to(dt)).backward()
    return pred.detach(), [p.grad.detach().clone() for p in resnet18_params(net)]


def _probe(key, n):
    r = np.random.default_rng(sum(map(ord, key)))
    return r.choice(n, size=SAMPLES, replace=False), r.standard_normal((PROJ, n))


def _segments(key, tensors):
    """Per tensor j, the stored summary under ``<key><j>``: the elements when at most FULL, else SAMPLES seeded
    elements then PROJ seeded Gaussian projections."""
    segs = []
    for j, t in enumerate(tensors):
        flat = np.asarray(t, np.float64).reshape(-1)
        if flat.size <= FULL:
            segs.append(("full", flat, None))
        else:
            idx, P = _probe(f"{key}{j}", flat.size)
            segs.append(("sample", flat, idx))
            segs.append(("proj", flat, P))
    return segs


def summary(key, tensors):
    """The fixture vector of ``tensors``: every tensor's summary, concatenated (one array keeps the file small)."""
    return np.concatenate([f if kind == "full" else (f[a] if kind == "sample" else a @ f)
                           for kind, f, a in _segments(key, tensors)])


def check(key, tensors, golden, rel):
    """``tensors`` against the fixture vector ``golden[key]``: each stored value within ``rel`` of its tensor's scale
    (the largest element; for a projection, sum_i |P_i| |t_i|)."""
    ref, o = golden[key], 0
    for n, (kind, f, a) in enumerate(_segments(key, tensors)):
        got = f if kind == "full" else (f[a] if kind == "sample" else a @ f)
        want = ref[o:o + got.size]
        o += got.size
        scale = np.abs(a) @ np.abs(f) if kind == "proj" else np.abs(f).max()
        assert (np.abs(got - want) <= rel * scale).all(), f"{key}: segment {n} ({kind})"
    assert o == ref.size, key


def record(name, step, pred, grads, stats):
    """The fixture entries of one step: logits, the 62 gradients, the 40 running statistics after the step."""
    return {f"{name}/{step}/pred": np.asarray(pred, np.float64),
            f"{name}/{step}/g": summary(f"{name}/{step}/g", grads),
            f"{name}/{step}/s": summary(f"{name}/{step}/s", stats)}


# ---------------------------------------------------------------------------------------------------------------
# numpy model of the kernels
# ---------------------------------------------------------------------------------------------------------------
def _bn(z, gamma, beta, eps, training, rm, rv, momentum):
    """-> (out, mean, rstd, new running mean, new running var), per channel over (B, H, W)."""
    if training:
        mean = z.mean((0, 2, 3))
        var = ((z - mean[None, :, None, None]) ** 2).mean((0, 2, 3))
        N = z.size // z.shape[1]
        rm = (1 - momentum) * rm + momentum * mean
        rv = (1 - momentum) * rv + momentum * var * N / (N - 1)
    else:
        mean, var = rm, rv
    rstd = 1.0 / np.sqrt(var + eps)
    xh = (z - mean[None, :, None, None]) * rstd[None, :, None, None]
    return xh * gamma[None, :, None, None] + beta[None, :, None, None], (mean, rstd), rm, rv


def _bn_bwd(ds, z, st, gamma, training):
    """-> (dz, dgamma, dbeta): dz = gamma rstd (dS - sum dS / N - x^ sum dS x^ / N), the sums over every row and
    pixel of the channel (0 in eval mode)."""
    mean, rstd = st
    xh = (z - mean[None, :, None, None]) * rstd[None, :, None, None]
    sb = ds.sum((0, 2, 3))
    sg = (ds * xh).sum((0, 2, 3))
    N = z.size // z.shape[1]
    k = (gamma * rstd)[None, :, None, None]
    if not training:
        return k * ds, sg, sb
    return k * (ds - sb[None, :, None, None] / N - xh * sg[None, :, None, None] / N), sg, sb


def _maxpool(y):
    """MaxPool2d(3, 2, 1) -> (out, arg): arg is the window index 3 dh + dw of the first maximum in row-major order."""
    Bn, C, H, W = y.shape
    Ho, Wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    yp = np.pad(y, ((0, 0), (0, 0), (1, 1), (1, 1)), constant_values=-np.inf)
    win = np.stack([yp[:, :, dh:dh + 2 * (Ho - 1) + 1:2, dw:dw + 2 * (Wo - 1) + 1:2]
                    for dh in range(3) for dw in range(3)], 0)
    arg = win.argmax(0)                               # numpy's argmax: the first maximum
    return np.take_along_axis(win, arg[None], 0)[0], arg


def _maxpool_bwd(g, arg, H, W):
    """Gather form: stem pixel (ih, iw) sums dY over the windows (oh, ow) holding it whose argmax it is."""
    Ho, Wo = g.shape[2:]
    dx = np.zeros(g.shape[:2] + (H, W))
    for ih in range(H):
        for oh in range(ih // 2, min(Ho - 1, (ih + 1) // 2) + 1):
            dh = ih - 2 * oh + 1
            for iw in range(W):
                for ow in range(iw // 2, min(Wo - 1, (iw + 1) // 2) + 1):
                    hit = arg[:, :, oh, ow] == dh * 3 + (iw - 2 * ow + 1)
                    dx[:, :, ih, iw] += np.where(hit, g[:, :, oh, ow], 0.0)
    return dx


def tv_geometry():
    """(ks, stride, pad) per conv in module order, and the blocks as (c1, c2, cd or -1): the SMT network's layout with
    torchvision's stride-2 stem."""
    convs, blocks = _geometry()
    return [(7, 2, 3)] + [c[:3] for c in convs[1:]], blocks


def numpy_model(params, stats, eps, momentum, training, x, gts):
    """pred, the 62 gradients of the reference loss and the 40 running statistics after the call, in float64, by the
    kernels' equations.  ``params`` / ``stats``: numpy arrays in resnet18_params / resnet18_buffers order (fc bias
    present; the first 40 buffers)."""
    x = np.asarray(x, np.float64)
    Wt, Gm, Bt, fw, fb = params[:20], params[20:40], params[40:60], params[60], params[61]
    rm, rv = list(stats[:20]), list(stats[20:40])
    convs, blocks = tv_geometry()
    spec = x.transpose(0, 3, 1, 2)
    Z, S, Y = {}, {}, {}

    def norm(i, z):
        out, S[i], rm[i], rv[i] = _bn(z, Gm[i], Bt[i], eps[i], training, rm[i], rv[i], momentum)
        return out
    Z[0] = _conv(spec, Wt[0], 2, 3)
    Y[0] = np.maximum(norm(0, Z[0]), 0)
    pooled, arg = _maxpool(Y[0])
    xin, cur = {}, pooled
    for c1, c2, cd in blocks:
        xin[c1] = cur
        _, s, p = convs[c1]
        Z[c1] = _conv(cur, Wt[c1], s, p)
        Y[c1] = np.maximum(norm(c1, Z[c1]), 0)
        Z[c2] = _conv(Y[c1], Wt[c2], 1, 1)
        y = norm(c2, Z[c2])
        if cd >= 0:
            Z[cd] = _conv(cur, Wt[cd], 2, 0)
            y = y + norm(cd, Z[cd])
        else:
            y = y + cur
        Y[c2] = np.maximum(y, 0)
        cur = Y[c2]
    P4 = cur.shape[2] * cur.shape[3]
    F = cur.mean((2, 3))
    pred = F @ fw.T + fb
    pt = torch.tensor(pred, requires_grad=True)
    reference_loss(pt, torch.as_tensor(np.asarray(gts, np.float64))).backward()
    g = pt.grad.numpy()
    grads = [None] * 62
    grads[60] = g.T @ F
    grads[61] = g.sum(0)
    G = np.broadcast_to((g @ fw)[:, :, None, None] / P4, cur.shape)
    for c1, c2, cd in reversed(blocks):
        dS = G * (Y[c2] > 0)
        dz2, grads[20 + c2], grads[40 + c2] = _bn_bwd(dS, Z[c2], S[c2], Gm[c2], training)
        grads[c2] = _conv_dw(dz2, Y[c1], 3, 1, 1)
        dY1 = _conv_dx(dz2, Wt[c2], *Y[c1].shape[2:], 1, 1)
        dz1, grads[20 + c1], grads[40 + c1] = _bn_bwd(dY1 * (Y[c1] > 0), Z[c1], S[c1], Gm[c1], training)
        _, s, p = convs[c1]
        grads[c1] = _conv_dw(dz1, xin[c1], 3, s, p)
        if cd >= 0:
            dzd, grads[20 + cd], grads[40 + cd] = _bn_bwd(dS, Z[cd], S[cd], Gm[cd], training)
            grads[cd] = _conv_dw(dzd, xin[c1], 1, 2, 0)
            other = _conv_dx(dzd, Wt[cd], *xin[c1].shape[2:], 2, 0)
        else:
            other = dS
        G = _conv_dx(dz1, Wt[c1], *xin[c1].shape[2:], s, p) + other
    dY0 = _maxpool_bwd(G, arg, *Y[0].shape[2:])
    dz0, grads[20], grads[40] = _bn_bwd(dY0 * (Y[0] > 0), Z[0], S[0], Gm[0], training)
    grads[0] = _conv_dw(dz0, spec, 7, 2, 3)
    return pred, grads, rm + rv
