"""Cases, seeded parameters and a numpy float64 model of the backward of SAVi's online location predictor
(ssb_smt_resnet18_train_backward_batch) for tests/golden/smt_resnet_train_golden.npz.

The model follows the kernels' equations rather than autograd's: it lists the live rows (upstream gradient not all
zero) and works on those only; the ReLU gradient is taken on the saved output (threshold_backward); GroupNorm's
backward is dz = rstd (gamma dS - (A + x^ Bs) / E) per (row, group) from the forward's statistics; a block's
gradient splits into the main branch and the identity or downsample branch; dX of a padded, strided conv is the
gather form (input pixel (ih, iw) collects output (oh, ow) with oh s = ih + pad - kh); the stem's label channels get
their weight gradient from per-row tap sums times the labels, never from a broadcast label image."""
import numpy as np
import torch

from belief_nets_models import network_input

HW = (65, 26)
B = 4                     # row 1 silent, row 2 scaled by 1e-3
CASES = {"smt2": 0, "smt23": 21}
PARAM_SEED = 90
FULL = 512                # gradients up to this many elements are stored whole
SAMPLES, PROJ = 48, 12


def set_params(net, seed=PARAM_SEED):
    """Seeded parameters in the order of belief_nets.smt_resnet18_params, so the reference class and the stand-in
    get the same values: convs at He scale, gamma around 1, beta around 0, fc weight / sqrt(in) and bias 0.1."""
    from soundspaces_b200.belief_nets import smt_resnet18_params
    g = torch.Generator().manual_seed(seed)
    ps = smt_resnet18_params(net)
    with torch.no_grad():
        for i, p in enumerate(ps):
            if i < 20:
                fan_in = p.shape[1] * p.shape[2] * p.shape[3]
                p.copy_(torch.randn(p.shape, generator=g, dtype=torch.float64).to(p.dtype) * (2.0 / fan_in) ** 0.5)
            elif i < 40:
                p.copy_(1.0 + 0.3 * torch.randn(p.shape, generator=g, dtype=torch.float64).to(p.dtype))
            elif i < 60:
                p.copy_(0.2 * torch.randn(p.shape, generator=g, dtype=torch.float64).to(p.dtype))
            elif i == 60:
                p.copy_(torch.randn(p.shape, generator=g, dtype=torch.float64).to(p.dtype) / p.shape[1] ** 0.5)
            else:
                p.copy_(0.1 * torch.randn(p.shape, generator=g, dtype=torch.float64).to(p.dtype))
    return net


def case_inputs(name):
    """(spectrogram (B, H, W, 2), labels (B, L) or None, targets (B, 2)) in float32, from the case's seed."""
    n = CASES[name]
    g = torch.Generator().manual_seed(100 + n)
    x = torch.rand((B, HW[0], HW[1], 2), generator=g) * 3.0
    x[1] = 0.0
    x[2] *= 1e-3
    labels = torch.nn.functional.one_hot(torch.randint(0, n, (B,), generator=g), n).float() if n else None
    gts = torch.randn((B, 2), generator=g) * 5.0
    return x, labels, gts


def masked_mse(pred, x, gts):
    """train_belief_predictor's loss (ppo_trainer.py:375-381)."""
    masks = (torch.sum(torch.reshape(x, (x.shape[0], -1)), dim=1, keepdim=True) != 0).to(pred.dtype)
    return torch.nn.functional.mse_loss(masks.expand_as(pred) * pred, masks.expand_as(gts) * gts)


def torch_grads(net, x, labels, gts):
    """pred and the 62 parameter gradients of the masked MSE through ``net`` in its own dtype."""
    from soundspaces_b200.belief_nets import smt_resnet18_params
    dt = next(net.parameters()).dtype
    xd, ld, gd = x.to(dt), None if labels is None else labels.to(dt), gts.to(dt)
    net.zero_grad(set_to_none=True)
    pred = net(network_input(xd, ld))
    masked_mse(pred, xd, gd).backward()
    return pred.detach(), [p.grad.detach().clone() for p in smt_resnet18_params(net)]


def _probe(name, j, n):
    r = np.random.default_rng(sum(map(ord, name)) * 1000 + j)
    return r.choice(n, size=SAMPLES, replace=False), r.standard_normal((PROJ, n))


def grad_summary(name, j, grad):
    flat = np.asarray(grad, np.float64).reshape(-1)
    if flat.size <= FULL:
        return {"": flat}
    idx, P = _probe(name, j, flat.size)
    return {"_sample": flat[idx], "_proj": P @ flat}


def check_grad(name, j, grad, golden, rel):
    """``grad`` against the fixture's summary of gradient j: each stored value within ``rel`` of its scale (the
    largest element; for a projection, sum_i |P_i| |grad_i|)."""
    flat = np.asarray(grad, np.float64).reshape(-1)
    key = f"{name}/g{j}"
    if key in golden:
        ref = golden[key]
        assert ref.shape == flat.shape and np.abs(flat - ref).max() <= rel * np.abs(ref).max(), key
        return
    idx, P = _probe(name, j, flat.size)
    s = golden[key + "_sample"]
    assert np.abs(flat[idx] - s).max() <= rel * np.abs(flat).max(), key + "_sample"
    scale = np.abs(P) @ np.abs(flat)
    assert (np.abs(P @ flat - golden[key + "_proj"]) <= rel * scale).all(), key + "_proj"


# ---------------------------------------------------------------------------------------------------------------
# numpy model of the kernels
# ---------------------------------------------------------------------------------------------------------------
def _geometry():
    """Per conv (module order): (ks, stride, pad, kind) with kind 'stem', 'c1', 'c2' or 'ds'; and the blocks as
    (c1, c2, cd or -1)."""
    convs, blocks, i = [(7, 1, 3, "stem")], [], 1
    for s in range(4):
        for b in range(2):
            stride = 2 if s and b == 0 else 1
            convs += [(3, stride, 1, "c1"), (3, 1, 1, "c2")]
            if stride == 2:
                convs.append((1, 2, 0, "ds"))
            blocks.append((i, i + 1, i + 2 if stride == 2 else -1))
            i += 3 if stride == 2 else 2
    return convs, blocks


def _conv(x, w, s, p):
    Bn, _, H, W = x.shape
    k = w.shape[2]
    Ho, Wo = (H + 2 * p - k) // s + 1, (W + 2 * p - k) // s + 1
    xp = np.pad(x, ((0, 0), (0, 0), (p, p), (p, p)))
    out = np.zeros((Bn, w.shape[0], Ho, Wo))
    for kh in range(k):
        for kw in range(k):
            out += np.einsum("oi,bihw->bohw", w[:, :, kh, kw], xp[:, :, kh:kh + s * (Ho - 1) + 1:s,
                                                                    kw:kw + s * (Wo - 1) + 1:s])
    return out


def _conv_dw(dz, x, k, s, p):
    Ho, Wo = dz.shape[2:]
    xp = np.pad(x, ((0, 0), (0, 0), (p, p), (p, p)))
    dw = np.zeros((dz.shape[1], x.shape[1], k, k))
    for kh in range(k):
        for kw in range(k):
            dw[:, :, kh, kw] = np.einsum("bohw,bihw->oi", dz, xp[:, :, kh:kh + s * (Ho - 1) + 1:s,
                                                                   kw:kw + s * (Wo - 1) + 1:s])
    return dw


def _conv_dx(dz, w, H, W, s, p):
    """Gather form: dX[b][ic][ih][iw] = sum over (oc, kh, kw) of W[oc][ic][kh][kw] dz[b][oc][oh][ow] where
    oh s = ih + p - kh and ow s = iw + p - kw land on the output grid."""
    Ho, Wo = dz.shape[2:]
    k = w.shape[2]
    dx = np.zeros((dz.shape[0], w.shape[1], H, W))
    ih, iw = np.arange(H), np.arange(W)
    for kh in range(k):
        th = ih + p - kh
        okh = (th >= 0) & (th % s == 0) & (th // s < Ho)
        for kw in range(k):
            tw = iw + p - kw
            okw = (tw >= 0) & (tw % s == 0) & (tw // s < Wo)
            g = dz[:, :, np.clip(th // s, 0, Ho - 1)][:, :, :, np.clip(tw // s, 0, Wo - 1)]
            g = g * (okh[:, None] & okw[None, :])
            dx += np.einsum("oi,bohw->bihw", w[:, :, kh, kw], g)
    return dx


def _gn(z, gamma, beta, eps, G=16):
    Bn, C, H, W = z.shape
    zg = z.reshape(Bn, G, -1)
    mean = zg.mean(2, keepdims=True)
    rstd = 1.0 / np.sqrt(((zg - mean) ** 2).mean(2, keepdims=True) + eps)
    xh = ((zg - mean) * rstd).reshape(z.shape)
    return xh * gamma[None, :, None, None] + beta[None, :, None, None], (mean, rstd)


def _gn_bwd(ds, z, st, gamma, G=16):
    """-> (dz, dgamma, dbeta): dz = rstd (gamma dS - (A + x^ Bs) / E) with A = sum_c gamma_c dbeta_c and
    Bs = sum_c gamma_c dgamma_c over the group's channels (per row)."""
    Bn, C = z.shape[:2]
    mean, rstd = st
    xh = ((z.reshape(Bn, G, -1) - mean) * rstd).reshape(z.shape)
    db_row = ds.sum((2, 3))                       # per-row partials, as the kernel keeps them
    dg_row = (ds * xh).sum((2, 3))
    A = (gamma * db_row).reshape(Bn, G, -1).sum(2)
    Bs = (gamma * dg_row).reshape(Bn, G, -1).sum(2)
    E = z[0].size // G
    Ab = np.repeat(A, C // G, axis=1)[:, :, None, None]
    Bb = np.repeat(Bs, C // G, axis=1)[:, :, None, None]
    rs = np.repeat(rstd.reshape(Bn, G), C // G, axis=1)[:, :, None, None]
    dz = rs * (gamma[None, :, None, None] * ds - (Ab + xh * Bb) / E)
    return dz, dg_row.sum(0), db_row.sum(0)


def numpy_model(params, eps, x, labels, gts):
    """pred and the 62 gradients of the masked MSE, in float64, by the kernels' equations.  ``params``: numpy
    arrays in smt_resnet18_params order (fc bias present)."""
    x = np.asarray(x, np.float64)
    lab = None if labels is None else np.asarray(labels, np.float64)
    W, Gm, Bt, fw, fb = params[:20], params[20:40], params[40:60], params[60], params[61]
    convs, blocks = _geometry()
    spec = x.transpose(0, 3, 1, 2)
    inp = spec if lab is None else np.concatenate(
        [spec, np.broadcast_to(lab[:, :, None, None], lab.shape + spec.shape[2:])], 1)
    Z, S, Y = {}, {}, {}
    Z[0] = _conv(inp, W[0], 1, 3)
    y, S[0] = _gn(Z[0], Gm[0], Bt[0], eps[0])
    Y[0] = np.maximum(y, 0)
    xin = {}
    cur = Y[0]
    for c1, c2, cd in blocks:
        xin[c1] = cur
        k, s, p, _ = convs[c1]
        Z[c1] = _conv(cur, W[c1], s, p)
        y, S[c1] = _gn(Z[c1], Gm[c1], Bt[c1], eps[c1])
        Y[c1] = np.maximum(y, 0)
        Z[c2] = _conv(Y[c1], W[c2], 1, 1)
        y, S[c2] = _gn(Z[c2], Gm[c2], Bt[c2], eps[c2])
        if cd >= 0:
            Z[cd] = _conv(cur, W[cd], 2, 0)
            yd, S[cd] = _gn(Z[cd], Gm[cd], Bt[cd], eps[cd])
            y = y + yd
        else:
            y = y + cur
        Y[c2] = np.maximum(y, 0)
        cur = Y[c2]
    F = cur.reshape(cur.shape[0], -1)
    pred = F @ fw.T + fb
    n = pred.size
    mask = (x.reshape(x.shape[0], -1).sum(1, keepdims=True) != 0).astype(np.float64)
    g = 2.0 * mask * (mask * pred - mask * np.asarray(gts, np.float64)) / n
    live = np.nonzero((g != 0).any(1))[0]       # the compacted rows every later step works on
    g = g[live]

    def rows(d):
        return {k: (v[live] if not isinstance(v, tuple) else tuple(a[live] for a in v)) for k, v in d.items()}
    Z, S, Y, xin = rows(Z), rows(S), rows(Y), rows(xin)
    grads = [None] * 62
    grads[60] = g.T @ F[live]
    grads[61] = g.sum(0)
    G = (g @ fw).reshape(cur[live].shape)
    for c1, c2, cd in reversed(blocks):
        dS = G * (Y[c2] > 0)
        dz2, grads[20 + c2], grads[40 + c2] = _gn_bwd(dS, Z[c2], S[c2], Gm[c2])
        grads[c2] = _conv_dw(dz2, Y[c1], 3, 1, 1)
        dY1 = _conv_dx(dz2, W[c2], *Y[c1].shape[2:], 1, 1)
        dz1, grads[20 + c1], grads[40 + c1] = _gn_bwd(dY1 * (Y[c1] > 0), Z[c1], S[c1], Gm[c1])
        k, s, p, _ = convs[c1]
        grads[c1] = _conv_dw(dz1, xin[c1], 3, s, p)
        if cd >= 0:
            dzd, grads[20 + cd], grads[40 + cd] = _gn_bwd(dS, Z[cd], S[cd], Gm[cd])
            grads[cd] = _conv_dw(dzd, xin[c1], 1, 2, 0)
            other = _conv_dx(dzd, W[cd], *xin[c1].shape[2:], 2, 0)
        else:
            other = dS
        G = _conv_dx(dz1, W[c1], *xin[c1].shape[2:], s, p) + other
    dz0, grads[20], grads[40] = _gn_bwd(G * (Y[0] > 0), Z[0], S[0], Gm[0])
    dw0 = np.zeros_like(W[0])
    dw0[:, :2] = _conv_dw(dz0, spec[live], 7, 1, 3)
    if lab is not None:
        H, Wd = spec.shape[2:]
        taps = np.zeros(dz0.shape[:2] + (7, 7))      # per-row sums over the outputs whose tap lies inside the image
        for kh in range(7):
            for kw in range(7):
                taps[:, :, kh, kw] = dz0[:, :, max(0, 3 - kh):min(H, H + 3 - kh),
                                         max(0, 3 - kw):min(Wd, Wd + 3 - kw)].sum((2, 3))
        dw0[:, 2:] = np.einsum("bl,bokw->olkw", lab[live], taps)
    grads[0] = dw0
    return pred, grads
