"""Host side of SAVi's scene memory transformer: the stand-in against the reference's float64 golden outputs, the
structural checks of ``soundspaces_b200.smt`` and every single deviation they refuse, the inputs
``fused_single_forward`` hands back to the module, the patch, and the ctypes layout of ``ssb_smt_params``.  No GPU."""
import copy
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

torch = pytest.importorskip("torch")
nn = torch.nn

from smt_models import SMTStandIn, make_inputs, make_smt  # noqa: E402
from soundspaces_b200 import _lib, smt  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CPU = torch.device("cpu")
GOLDEN = os.path.join(ROOT, "tests", "golden", "smt_golden.npz")


def golden_cases():
    with np.load(GOLDEN) as z:
        data = {k: z[k] for k in z.files}
    names = sorted({k.split("/")[0] for k in data})
    cases = {}
    for n in names:
        D, pi, d, nhead, pre, goal = (int(v) for v in data[f"{n}/config"])
        m = SMTStandIn(D, nhead, d, 0.0, None if pi < 0 else pi, bool(pre)).double().eval()
        m.load_state_dict({k[len(n) + 3:]: torch.from_numpy(v) for k, v in data.items() if k.startswith(f"{n}/w/")})
        cases[n] = (m, torch.from_numpy(data[f"{n}/x"]), torch.from_numpy(data[f"{n}/memory"]),
                    torch.from_numpy(data[f"{n}/masks"]), torch.from_numpy(data[f"{n}/goal"]) if goal else None,
                    torch.from_numpy(data[f"{n}/out"]))
    return cases


def test_stand_in_reproduces_the_reference():
    cases = golden_cases()
    assert len(cases) == 8
    for name, (m, x, memory, masks, goal, want) in cases.items():
        with torch.no_grad():
            got = m.single_forward(x, memory, masks, goal)
        err = (got - want).abs().max().item()
        assert err <= 1e-12 * max(1.0, want.abs().max().item()), f"{name}: {err:.3g}"


def test_accepts_the_stand_in():
    assert smt.smt_layout_error(make_smt()) == ""
    assert smt.smt_layout_error(make_smt(), CPU) == ""
    assert smt.smt_layout_error(make_smt(D=40, pose_index=None, d_model=64, nhead=4)) == ""
    m = make_smt()
    m.train()                                      # dropout 0: the trainer's rollouts run in training mode
    assert smt.smt_layout_error(m) == ""
    assert smt.smt_layout_error(make_smt(dropout=0.1).eval()) == ""


def _set(m, path, value):
    *parent, last = path.split(".")
    for p in parent:
        m = m[int(p)] if p.isdigit() else getattr(m, p)
    if last.isdigit():
        m[int(last)] = value
    else:
        setattr(m, last, value)


def _encoder_layer(**kw):
    args = dict(d_model=256, nhead=8, dim_feedforward=256, dropout=0.0)
    args.update(kw)
    return nn.TransformerEncoderLayer(**args)


DEVIATIONS = {
    "norm_first": lambda m: _set(m, "transformer.encoder.layers.0", _encoder_layer(norm_first=True)),
    "gelu": lambda m: _set(m, "transformer.decoder.layers.0",
                           nn.TransformerDecoderLayer(256, 8, 256, 0.0, activation="gelu")),
    "batch_first": lambda m: _set(m, "transformer.encoder.layers.0", _encoder_layer(batch_first=True)),
    "two_encoder_layers": lambda m: m.transformer.encoder.layers.append(_encoder_layer()),
    "dropout_in_training": lambda m: setattr(m.transformer.encoder.layers[0].dropout1, "p", 0.1),
    "mha_dropout_in_training": lambda m: setattr(m.transformer.decoder.layers[0].multihead_attn, "dropout", 0.1),
    "no_final_norm": lambda m: _set(m, "transformer.encoder.norm", None),
    "bias_free_mha": lambda m: _set(m, "transformer.encoder.layers.0.self_attn", nn.MultiheadAttention(256, 8, bias=False)),
    "add_bias_kv": lambda m: _set(m, "transformer.decoder.layers.0.self_attn", nn.MultiheadAttention(256, 8, add_bias_kv=True)),
    "add_zero_attn": lambda m: _set(m, "transformer.decoder.layers.0.multihead_attn",
                                    nn.MultiheadAttention(256, 8, add_zero_attn=True)),
    "fusion_without_relu": lambda m: _set(m, "fusion_encoder.1", nn.Tanh()),
    "fusion_width": lambda m: _set(m, "fusion_encoder.0", nn.Linear(276, 256)),
    "pose_encoder_width": lambda m: _set(m, "pose_encoder", nn.Linear(5, 8)),
    "ff_width": lambda m: _set(m, "transformer.encoder.layers.0.linear1", nn.Linear(256, 512)),
    "layer_norm_not_affine": lambda m: _set(m, "transformer.decoder.norm", nn.LayerNorm(256, elementwise_affine=False)),
    "d_not_multiple_of_nhead": lambda m: setattr(m.transformer, "nhead", 7),
    "float64_parameters": lambda m: m.double(),
}


@pytest.mark.parametrize("name", sorted(DEVIATIONS))
def test_refuses_each_deviation(name):
    m = make_smt()
    m.train()
    DEVIATIONS[name](m)
    assert smt.smt_layout_error(m, CPU) != "", name


def test_parameters_must_be_contiguous_on_the_device():
    m = make_smt()
    assert "parameters" in smt.smt_layout_error(m, torch.device("cuda", 0))
    w = m.fusion_encoder[2].weight
    w.data = w.data.t().contiguous().t()
    assert "contiguous" in smt.smt_layout_error(m, CPU)


def test_fused_single_forward_returns_none_for_what_it_cannot_run():
    m = make_smt()
    x, memory, masks, goal = make_inputs(2, 5)
    with torch.no_grad():
        assert smt.fused_single_forward(m, x, memory, masks, goal) is None            # CPU tensors
    # grad enabled returns None before looking at anything else
    assert smt.fused_single_forward(m, None, None, None) is None
    with torch.no_grad():
        assert smt.fused_single_forward(m, x.double(), memory, masks) is None
        assert smt.fused_single_forward(m, x, memory, masks.bool()) is None
        assert smt.fused_single_forward(m, x, memory[:, :1], masks) is None


class FakeOps:
    def __init__(self):
        self.calls = []

    def smt_state_encoder(self, module, x, memory, masks, goal):
        self.calls.append((x.shape, memory.shape, masks.shape, goal is None))
        return "fused"


class FakeCuda:
    """Lets ``fused_single_forward``'s device checks pass on CPU tensors so its shape / limit logic can be tested."""

    def __init__(self, monkeypatch):
        self.ops = FakeOps()
        monkeypatch.setattr(smt, "_dense", lambda t, dev: isinstance(t, torch.Tensor) and t.dtype == torch.float32
                            and t.is_contiguous())
        from soundspaces_b200 import renderer
        monkeypatch.setattr(renderer.WaveformOps, "get", classmethod(lambda cls, dev: self.ops))


def test_fused_single_forward_limits(monkeypatch):
    fake = FakeCuda(monkeypatch)
    m = make_smt(D=40, pose_index=36, d_model=64, nhead=4)
    with torch.no_grad():
        x, memory, masks, goal = make_inputs(3, 6, D=40, d_model=64, pose_index=36)
        assert smt.fused_single_forward(m, x, memory, masks, goal) == "fused"
        assert smt.fused_single_forward(m, x, memory, masks) == "fused"
        assert smt.fused_single_forward(m, x, memory, masks, goal[:, :10]) is None            # goal width
        assert smt.fused_single_forward(m, x, memory, masks[:, :5]) is None                    # masks width
        assert smt.fused_single_forward(m, x[:, :39].contiguous(), memory[..., :39].contiguous(), masks) is None
        x, memory, masks, _ = make_inputs(2, 1024, D=40, d_model=64, pose_index=36)
        assert smt.fused_single_forward(m, x, memory, masks) is None                           # M + 1 > 1024
        x, memory, masks, _ = make_inputs(2, 1023, D=40, d_model=64, pose_index=36)
        assert smt.fused_single_forward(m, x, memory, masks) == "fused"
        big = make_smt(D=40, pose_index=36, d_model=256, nhead=1)                                 # head dim 256
        x, memory, masks, _ = make_inputs(2, 4, D=40, d_model=256, pose_index=36)
        assert smt.fused_single_forward(big, x, memory, masks) is None
        x, memory, masks, _ = make_inputs(1025, 1, D=40, d_model=64, pose_index=36)
        assert smt.fused_single_forward(m, x, memory, masks) is None                           # B > 1024
    assert len(fake.ops.calls) == 3


def test_patch_installs_is_idempotent_and_falls_back():
    class Enc(SMTStandIn):
        pass

    original = Enc.single_forward
    smt.patch_smt_state_encoder(Enc)
    patched = Enc.single_forward
    assert patched._ssb_original is original
    smt.patch_smt_state_encoder(Enc)
    assert Enc.single_forward._ssb_original is original
    m = make_smt()
    m.__class__ = Enc
    x, memory, masks, goal = make_inputs(2, 5)
    with torch.no_grad():
        want = original(m, x, memory, masks, goal)
        got = m.single_forward(x, memory, masks, goal)            # CPU: the original runs
    assert torch.equal(got, want)
    assert SMTStandIn.single_forward is not Enc.single_forward


def test_params_struct_layout_matches_c(tmp_path):
    src = tmp_path / "layout.c"
    fields = ["pose", "fuse1", "enc_qkv", "enc_norm1", "enc_norm", "dec_sa_qkv", "dec_ff2", "dec_norm1", "dec_norm"]
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "ssb200.h"\n'
                   'int main(void){printf("%zu %zu %zu ", sizeof(ssb_smt_params), sizeof(ssb_linear), sizeof(ssb_layer_norm));'
                   + "".join(f'printf("%zu ", offsetof(ssb_smt_params, {f}));' for f in fields)
                   + 'printf("%zu\\n", offsetof(ssb_layer_norm, eps));return 0;}\n')
    exe = tmp_path / "layout"
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    vals = [int(v) for v in subprocess.check_output([str(exe)]).split()]
    P = _lib.SmtParams
    assert vals == ([C.sizeof(P), C.sizeof(_lib.Linear), C.sizeof(_lib.LayerNorm)]
                    + [getattr(P, f).offset for f in fields] + [_lib.LayerNorm.eps.offset])


def test_params_point_at_the_live_tensors():
    m = make_smt()
    p = smt.smt_params(m, 276)
    enc, dec = m.transformer.encoder.layers[0], m.transformer.decoder.layers[0]
    assert (p.d_in, p.pose_index, p.d_model, p.n_heads, p.pretraining) == (276, 272, 256, 8, 0)
    assert p.enc_qkv.d_weight == enc.self_attn.in_proj_weight.data_ptr()
    assert p.dec_ca_qkv.d_bias == dec.multihead_attn.in_proj_bias.data_ptr()
    assert p.dec_norm.d_gamma == m.transformer.decoder.norm.weight.data_ptr()
    assert p.pose.d_weight == m.pose_encoder.weight.data_ptr()
    assert abs(p.enc_norm2.eps - enc.norm2.eps) < 1e-12
    q = smt.smt_params(make_smt(D=40, pose_index=None, d_model=64, nhead=4, pretraining=True), 40)
    assert (q.pose_index, q.pretraining, q.pose.d_weight) == (-1, 1, None)


def test_scratch_bytes():
    lib = _lib.load_library()
    p = smt.smt_params(make_smt(), 276)
    assert lib.ssb_smt_scratch_bytes(8, 300, C.byref(p)) == 256 + 5 * 8 * 301 * 256 * 4
    assert lib.ssb_smt_scratch_bytes(1024, 3, C.byref(p)) == 4096 + 5 * 1024 * 4 * 256 * 4      # the counts: 4 B bytes
    assert lib.ssb_smt_scratch_bytes(65, 0, C.byref(p)) == 512 + 5 * 65 * 256 * 4
    assert lib.ssb_smt_scratch_bytes(-1, 300, C.byref(p)) == -1
    assert lib.ssb_smt_scratch_bytes(8, 300, None) == -1
