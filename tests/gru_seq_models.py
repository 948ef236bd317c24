"""Models of ``RNNStateEncoder.seq_forward`` (ss_baselines/av_nav/models/rnn_state_encoder.py:92-143) for the tests of
``ssb_gru_seq_*``:

- ``RNNStateEncoder``: a stand-in written from the reference's computation (split the sequence at the steps where
  some env's mask is 0, mask the carried state at each piece's first step, one ``nn.GRU`` call per piece);
  tests/golden/gru_seq_golden.npz pins it to the reference class in float64.
- ``segment_starts``, ``forward``, ``backward``: float64 numpy of exactly what the kernels compute, the device-side
  segment rule, the forward with its saved state (h_prev, r, z, n, W_hn h_prev + b_hn) and the explicit BPTT.
- ``CASES`` / ``case_inputs``: the golden's shapes and seeded inputs and mask patterns.
"""
import numpy as np
import torch

from avnav_models import RNNStateEncoder as _StepEncoder

# name: (T, N, I, Hd)
CASES = {
    "no_zero": (6, 3, 10, 8),        # no zero past t = 0 (one segment); t = 0 has zeros and ones
    "one_zero": (5, 3, 7, 6),        # exactly one zero step: the reference's scalar .item() branch
    "many_zeros": (9, 4, 12, 8),     # zeros at t = 2, 3 (consecutive), 6 and T - 1
    "all_zero": (4, 3, 6, 5),        # every mask 0: every step a segment start
    "fractional": (7, 3, 8, 6),      # fractional masks at segment starts (applied) and elsewhere (not applied)
    "single_env": (6, 1, 5, 4),      # N = 1
    "two_steps": (2, 4, 6, 4),       # T = 2
    "odd": (5, 3, 13, 7),            # odd Hd, I not a multiple of 4
}


def case_masks(name):
    T, N = CASES[name][:2]
    m = np.ones((T, N))
    if name == "no_zero":
        m[0] = [0, 1, 1]
    elif name == "one_zero":
        m[2, 1] = 0
    elif name == "many_zeros":
        m[2, 0] = m[3, 3] = m[6, 1] = m[8, 2] = 0
    elif name == "all_zero":
        m[:] = 0
    elif name == "fractional":
        m[0] = [0.5, 0.25, 1.0]        # t = 0: applied
        m[3] = [0.0, 0.5, 1.0]         # a segment start: 0.5 applied to env 1
        m[5] = [1.0, 1.0, 0.7]         # no zero at t = 5: 0.7 not applied
    elif name == "single_env":
        m[3, 0] = 0
    elif name == "two_steps":
        m[1, 2] = 0
    elif name == "odd":
        m[2, 0] = 0
        m[0, 1] = 0
    return m.reshape(T * N, 1)


def case_inputs(name, dtype=torch.float64):
    """(x, h0, masks, g_out, g_h_last) of a case, seeded by its position in CASES."""
    T, N, I, Hd = CASES[name]
    g = torch.Generator().manual_seed(60 + list(CASES).index(name))
    x = torch.randn(T * N, I, generator=g, dtype=torch.float64)
    h0 = torch.randn(1, N, Hd, generator=g, dtype=torch.float64)
    g_out = torch.randn(T * N, Hd, generator=g, dtype=torch.float64)
    g_h = torch.randn(1, N, Hd, generator=g, dtype=torch.float64)
    masks = torch.from_numpy(case_masks(name))
    return tuple(t.to(dtype) for t in (x, h0, masks, g_out, g_h))


class RNNStateEncoder(_StepEncoder):
    """tests/avnav_models.py's stand-in plus ``seq_forward`` (GRU only) and the reference's ``forward`` dispatch."""

    def seq_forward(self, x, hidden_states, masks):
        N = hidden_states.size(1)
        T = x.size(0) // N
        x = x.view(T, N, x.size(1))
        m = masks.view(T, N)
        # one host read of the done steps per call, as the reference makes
        bounds = [0] + [t + 1 for t in (m[1:] == 0.0).any(dim=-1).nonzero().squeeze(-1).cpu().tolist()] + [T]
        h, outs = hidden_states, []
        for a, b in zip(bounds[:-1], bounds[1:]):
            y, h = self.rnn(x[a:b], m[a].view(1, -1, 1) * h)
            outs.append(y)
        return torch.cat(outs, dim=0).view(T * N, -1), h

    def forward(self, x, hidden_states, masks):
        if x.size(0) == hidden_states.size(1):
            return self.single_forward(x, hidden_states, masks)
        return self.seq_forward(x, hidden_states, masks)


def segment_starts(masks, T, N):
    """(T,) bool: t = 0, or some env's mask at t equals 0.0 (NaN does not)."""
    m = np.asarray(masks, np.float64).reshape(T, N)
    s = (m == 0.0).any(axis=1)
    s[0] = True
    return s


def _sigmoid(a):
    return 1.0 / (1.0 + np.exp(-a))


def forward(x, h0, masks, w_ih, w_hh, b_ih, b_hh):
    """-> (out (T N, Hd), h_last (1, N, Hd), saved (5, T N, Hd)), float64."""
    Hd = w_hh.shape[1]
    N = h0.size // Hd
    T = x.shape[0] // N
    seg = segment_starts(masks, T, N)
    m = np.asarray(masks, np.float64).reshape(T, N)
    gi = (x @ w_ih.T + b_ih).reshape(T, N, 3 * Hd)
    h = np.asarray(h0, np.float64).reshape(N, Hd)
    out = np.empty((T, N, Hd))
    saved = np.empty((5, T, N, Hd))
    for t in range(T):
        hp = m[t][:, None] * h if seg[t] else h
        gh = hp @ w_hh.T + b_hh
        r = _sigmoid(gi[t, :, :Hd] + gh[:, :Hd])
        z = _sigmoid(gi[t, :, Hd:2 * Hd] + gh[:, Hd:2 * Hd])
        n = np.tanh(gi[t, :, 2 * Hd:] + r * gh[:, 2 * Hd:])
        h = (1 - z) * n + z * hp
        out[t] = h
        saved[:, t] = hp, r, z, n, gh[:, 2 * Hd:]
    return out.reshape(T * N, Hd), h.reshape(1, N, Hd), saved.reshape(5, T * N, Hd)


def backward(x, masks, w_ih, w_hh, saved, g_out, g_h_last):
    """Explicit BPTT from ``forward``'s saved state -> (dx, dh0, dw_ih, dw_hh, db_ih, db_hh), float64.  g_out /
    g_h_last may be None (zero)."""
    Hd = w_hh.shape[1]
    TN = x.shape[0]
    sv = saved.reshape(5, TN, Hd)
    N = (g_h_last.size // Hd) if g_h_last is not None else None
    if N is None:
        raise ValueError("backward needs g_h_last (zeros for none) to know N")
    T = TN // N
    seg = segment_starts(masks, T, N)
    m = np.asarray(masks, np.float64).reshape(T, N)
    hp, r, z, n, ghn = (sv[i].reshape(T, N, Hd) for i in range(5))
    go = np.zeros((T, N, Hd)) if g_out is None else np.asarray(g_out).reshape(T, N, Hd)
    carry = np.asarray(g_h_last).reshape(N, Hd).copy()
    dgi = np.empty((T, N, 3 * Hd))
    dgh = np.empty((T, N, 3 * Hd))
    for t in range(T - 1, -1, -1):
        dh = carry + go[t]
        dn = dh * (1 - z[t])
        dz = dh * (hp[t] - n[t])
        dan = dn * (1 - n[t] ** 2)
        dar = dan * ghn[t] * r[t] * (1 - r[t])
        daz = dz * z[t] * (1 - z[t])
        dgi[t] = np.concatenate([dar, daz, dan], axis=1)
        dgh[t] = np.concatenate([dar, daz, dan * r[t]], axis=1)
        dhp = dh * z[t] + dgh[t] @ w_hh
        carry = m[t][:, None] * dhp if seg[t] else dhp
    dgi, dgh = dgi.reshape(TN, 3 * Hd), dgh.reshape(TN, 3 * Hd)
    return (dgi @ w_ih, carry.reshape(1, N, Hd), dgi.T @ x, dgh.T @ sv[0], dgi.sum(0), dgh.sum(0))


def make_encoder(I, Hd, params=None, dtype=torch.float64):
    enc = RNNStateEncoder(I, Hd).to(dtype)
    if params is not None:
        with torch.no_grad():
            for p, v in zip((enc.rnn.weight_ih_l0, enc.rnn.weight_hh_l0, enc.rnn.bias_ih_l0, enc.rnn.bias_hh_l0),
                            params):
                p.copy_(torch.as_tensor(v))
    return enc


def gru_params(enc):
    r = enc.rnn
    return r.weight_ih_l0, r.weight_hh_l0, r.bias_ih_l0, r.bias_hh_l0
