"""Host side of the fused ``RNNStateEncoder.seq_forward`` (``soundspaces_b200.rnn``, ``ssb_gru_seq_*``): the stand-in
and the float64 model of the kernels pinned to the reference's golden data and to torch's autograd, the segment rule,
and the qualification, fallback and patching logic.  No GPU needed."""
import os

import numpy as np
import pytest
import torch

import gru_seq_models as gm
from soundspaces_b200 import rnn as srnn

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "gru_seq_golden.npz")
GRADS = ("dx", "dh0", "dw_ih", "dw_hh", "db_ih", "db_hh")


@pytest.fixture(scope="module")
def golden():
    with np.load(GOLDEN) as z:
        return {k: z[k] for k in z.files}


def _case(golden, name):
    return {k.split("/", 1)[1]: v for k, v in golden.items() if k.startswith(name + "/")}


def _close(a, b, tol=1e-12):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    assert a.shape == b.shape
    assert np.abs(a - b).max() <= tol * max(1.0, np.abs(b).max())


@pytest.mark.parametrize("name", list(gm.CASES))
def test_golden_holds_the_cases(golden, name):
    c = _case(golden, name)
    assert tuple(c["config"]) == gm.CASES[name]
    x, h0, masks, g_out, g_h = gm.case_inputs(name)
    for k, v in (("x", x), ("h0", h0), ("masks", masks), ("g_out", g_out), ("g_h_last", g_h)):
        assert np.array_equal(c[k], v.numpy()), k


@pytest.mark.parametrize("name", list(gm.CASES))
def test_stand_in_matches_reference_golden(golden, name):
    c = _case(golden, name)
    T, N, I, Hd = gm.CASES[name]
    enc = gm.make_encoder(I, Hd, (c["w_ih"], c["w_hh"], c["b_ih"], c["b_hh"]))
    x = torch.tensor(c["x"], requires_grad=True)
    h0 = torch.tensor(c["h0"], requires_grad=True)
    out, h_last = enc(x, h0, torch.tensor(c["masks"]))
    ((out * torch.tensor(c["g_out"])).sum() + (h_last * torch.tensor(c["g_h_last"])).sum()).backward()
    _close(out.detach(), c["out"])
    _close(h_last.detach(), c["h_last"])
    got = [x.grad, h0.grad] + [p.grad for p in gm.gru_params(enc)]
    for k, g in zip(GRADS, got):
        _close(g, c[k])


@pytest.mark.parametrize("name", list(gm.CASES))
def test_kernel_model_matches_reference_golden(golden, name):
    c = _case(golden, name)
    params = (c["w_ih"], c["w_hh"], c["b_ih"], c["b_hh"])
    out, h_last, saved = gm.forward(c["x"], c["h0"], c["masks"], *params)
    _close(out, c["out"])
    _close(h_last, c["h_last"])
    grads = gm.backward(c["x"], c["masks"], c["w_ih"], c["w_hh"], saved, c["g_out"], c["g_h_last"])
    for k, g in zip(GRADS, grads):
        _close(g, c[k])


def test_kernel_model_matches_autograd_at_a_larger_shape():
    T, N, I, Hd = 23, 6, 17, 11
    g = torch.Generator().manual_seed(5)
    enc = gm.RNNStateEncoder(I, Hd).double()
    with torch.no_grad():
        for p in enc.parameters():
            p.copy_(torch.randn(p.shape, generator=g, dtype=torch.float64) * 0.3)
    x = torch.randn(T * N, I, generator=g, dtype=torch.float64, requires_grad=True)
    h0 = torch.randn(1, N, Hd, generator=g, dtype=torch.float64, requires_grad=True)
    masks = (torch.rand(T * N, 1, generator=g, dtype=torch.float64) > 0.1).double()
    masks[::7] *= 0.5                                       # fractional values, some at segment starts
    g_out = torch.randn(T * N, Hd, generator=g, dtype=torch.float64)
    g_h = torch.randn(1, N, Hd, generator=g, dtype=torch.float64)
    out, h_last = enc(x, h0, masks)
    ((out * g_out).sum() + (h_last * g_h).sum()).backward()
    params = [p.detach().numpy() for p in gm.gru_params(enc)]
    m_out, m_h, saved = gm.forward(x.detach().numpy(), h0.detach().numpy(), masks.numpy(), *params)
    _close(m_out, out.detach())
    _close(m_h, h_last.detach())
    grads = gm.backward(x.detach().numpy(), masks.numpy(), params[0], params[1], saved, g_out.numpy(), g_h.numpy())
    for k, a, b in zip(GRADS, grads, [x.grad, h0.grad] + [p.grad for p in gm.gru_params(enc)]):
        _close(a, b, 1e-11)


def test_kernel_model_takes_missing_output_gradients_as_zero(golden):
    c = _case(golden, "many_zeros")
    params = (c["w_ih"], c["w_hh"], c["b_ih"], c["b_hh"])
    _, _, saved = gm.forward(c["x"], c["h0"], c["masks"], *params)
    zero_h = np.zeros_like(c["g_h_last"])
    a = gm.backward(c["x"], c["masks"], c["w_ih"], c["w_hh"], saved, None, c["g_h_last"])
    b = gm.backward(c["x"], c["masks"], c["w_ih"], c["w_hh"], saved, np.zeros_like(c["g_out"]), c["g_h_last"])
    for u, v in zip(a, b):
        assert np.array_equal(u, v)
    only_out = gm.backward(c["x"], c["masks"], c["w_ih"], c["w_hh"], saved, c["g_out"], zero_h)
    assert np.abs(only_out[0]).max() > 0


def test_segment_rule():
    m = np.array([[0.5, 1.0], [1.0, 0.3], [0.0, 1.0], [0.0, 0.0], [1.0, np.nan], [-0.0, 1.0]])
    assert gm.segment_starts(m.reshape(-1, 1), 6, 2).tolist() == [True, False, True, True, False, True]


def test_fractional_masks_are_applied_only_at_segment_starts(golden):
    """Masking every step differs from the reference exactly when a fractional mask lies off a segment start."""
    c = _case(golden, "fractional")
    T, N, I, Hd = gm.CASES["fractional"]
    params = (c["w_ih"], c["w_hh"], c["b_ih"], c["b_hh"])
    out, _, _ = gm.forward(c["x"], c["h0"], c["masks"], *params)
    _close(out, c["out"])
    seg = gm.segment_starts(c["masks"], T, N)
    assert seg.tolist() == [True, False, False, True, False, False, False]
    m = c["masks"].reshape(T, N)
    assert (m[~seg] != 1.0).any() and (m[seg] % 1.0 != 0).any()
    enc = gm.make_encoder(I, Hd, params)
    with torch.no_grad():
        h = torch.tensor(c["h0"])
        ys = []
        for t in range(T):                                  # mask applied at every step
            y, h = enc.rnn(torch.tensor(c["x"]).view(T, N, I)[t:t + 1], torch.tensor(m[t]).view(1, N, 1) * h)
            ys.append(y)
        every_step = torch.cat(ys).view(T * N, Hd).numpy()
    rows = slice(5 * N + 2, 5 * N + 3)                       # env 2 at t = 5, whose 0.7 is not applied
    assert np.abs(every_step[rows] - c["out"][rows]).max() > 1e-3
    assert np.abs(every_step[:5 * N] - c["out"][:5 * N]).max() < 1e-12


# qualification and patching --------------------------------------------------------------------------------------

def _dense_cpu(t, device):
    return isinstance(t, torch.Tensor) and t.device == device and t.dtype == torch.float32 and t.is_contiguous()


def _args(T=3, N=2, I=5, Hd=4):
    enc = gm.RNNStateEncoder(I, Hd)
    return enc, torch.randn(T * N, I), torch.randn(1, N, Hd), torch.ones(T * N, 1)


def test_gru_seq_error_on_the_cpu_names_the_device():
    enc, x, h, m = _args()
    assert "contiguous CUDA float32" in srnn.gru_seq_error(enc, x, h, m)


def test_gru_seq_error_reasons(monkeypatch):
    """Every reason, with the device check relaxed to the CPU so the shape checks behind it are reached."""
    monkeypatch.setattr(srnn, "_dense", _dense_cpu)
    enc, x, h, m = _args()
    assert srnn.gru_seq_error(enc, x, h, m) == ""
    lstm = gm.RNNStateEncoder(5, 4, rnn_type="LSTM")
    assert "LSTM is not nn.GRU" in srnn.gru_seq_error(lstm, x, h, m)
    two = gm.RNNStateEncoder(5, 4, num_layers=2)
    assert "num_layers is 2" in srnn.gru_seq_error(two, x, h, m)
    assert "x is not a tensor" in srnn.gru_seq_error(enc, x.numpy(), h, m)
    cases = {
        "x is not": (x.double(), h, m),
        "hidden_states is not": (x, h.double(), m),
        "masks is not": (x, h, m.double()),
        "x has shape": (x[:, :4].contiguous(), h, m),
        "hidden_states has shape": (x, h[0], m),
        "not T * N": (x[:5].contiguous(), h, m[:5].contiguous()),
        "masks hold": (x, h, m[:5].contiguous()),
    }
    for want, (a, b, c) in cases.items():
        assert want in srnn.gru_seq_error(enc, a, b, c), want
    # T = 1 is single_forward's shape, not a sequence
    assert "T >= 2" in srnn.gru_seq_error(enc, x[:2].contiguous(), h, m[:2].contiguous())
    assert "N=0" in srnn.gru_seq_error(enc, x, torch.zeros(1, 0, 4), m)
    with torch.no_grad():
        enc.rnn.weight_hh_l0.data = enc.rnn.weight_hh_l0.data.t().contiguous().t()
    assert "weight_hh_l0 is not" in srnn.gru_seq_error(enc, x, h, m)


def test_gru_seq_error_limits_grad_masks_and_autocast(monkeypatch):
    monkeypatch.setattr(srnn, "_dense", _dense_cpu)
    enc, x, h, m = _args(T=srnn.MAX_STEPS + 1, N=1, I=2, Hd=2)
    assert "the library takes" in srnn.gru_seq_error(enc, x, h, m)
    enc, x, h, m = _args(T=2, N=srnn.MAX_ENVS + 1, I=2, Hd=2)
    assert "the library takes" in srnn.gru_seq_error(enc, x, h, m)
    enc, x, h, m = _args(T=2, N=1, I=2, Hd=srnn.MAX_HIDDEN + 1)
    assert "the library takes" in srnn.gru_seq_error(enc, x, h, m)
    enc, x, h, m = _args()
    assert srnn.gru_seq_error(enc, x, h, m.requires_grad_(True)) == "masks require grad"
    monkeypatch.setattr(torch, "is_autocast_enabled", lambda device_type=None: True)
    assert srnn.gru_seq_error(enc, x, h, m.detach()) == "autocast is on"


def _fresh_class():
    return type("RNNStateEncoder", (gm.RNNStateEncoder,), {})


def test_plain_patch_leaves_seq_forward_alone():
    cls = _fresh_class()
    seq = cls.seq_forward
    srnn.patch_rnn_state_encoder(cls)
    assert cls.seq_forward is seq and not hasattr(cls.seq_forward, "_ssb_original")
    assert hasattr(cls.single_forward, "_ssb_original")


def test_sequence_patch_is_idempotent_and_keeps_originals():
    cls = _fresh_class()
    single, seq = cls.single_forward, cls.seq_forward
    srnn.patch_rnn_state_encoder(cls)
    srnn.patch_rnn_state_encoder(cls, sequence=True)           # the flag after a plain patch
    assert cls.seq_forward._ssb_original is seq and cls.single_forward._ssb_original is single
    srnn.patch_rnn_state_encoder(cls, sequence=True)
    srnn.patch_rnn_state_encoder(cls)
    assert cls.seq_forward._ssb_original is seq and cls.single_forward._ssb_original is single
    assert cls.seq_forward.__doc__ == seq.__doc__


def test_patched_seq_forward_on_the_cpu_runs_the_original(golden):
    c = _case(golden, "many_zeros")
    T, N, I, Hd = gm.CASES["many_zeros"]
    cls = _fresh_class()
    srnn.patch_rnn_state_encoder(cls, sequence=True)
    enc = cls(I, Hd).double()
    ref = gm.make_encoder(I, Hd)
    for dst in (enc, ref):
        with torch.no_grad():
            for p, v in zip(gm.gru_params(dst), (c["w_ih"], c["w_hh"], c["b_ih"], c["b_hh"])):
                p.copy_(torch.tensor(v))
    args = [torch.tensor(c[k]) for k in ("x", "h0", "masks")]
    out, h = enc(*args)
    want, h_want = ref(*args)
    assert torch.equal(out, want) and torch.equal(h, h_want)
    _close(out.detach(), c["out"])
