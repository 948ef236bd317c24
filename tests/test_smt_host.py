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


class RecordingLib:
    """Stands in for libssb200 behind a WaveformOps on the CPU: records each ssb_smt_state_encoder_batch call."""

    def __init__(self):
        self.calls = []

    def ssb_smt_scratch_bytes(self, N, M, params):
        return 256

    def ssb_smt_state_encoder_batch(self, handle, N, M, x, memory, masks, goal, params, scratch, out, stream):
        p = params._obj
        self.calls.append((N, M, p.d_in, p.pose_index))
        return 0


class RecordingCtx:
    handle = None
    launch_count = 0

    def __init__(self, lib):
        self.lib = lib

    def check(self, rc, what):
        assert rc == 0, what


def _cpu_ops():
    from soundspaces_b200.renderer import WaveformOps
    ops = WaveformOps.__new__(WaveformOps)
    ops.device = CPU
    ops.lib = RecordingLib()
    ops.ctx = RecordingCtx(ops.lib)
    ops._smt_scratch = {}
    ops._stream = lambda: None
    return ops


def test_smt_state_encoder_refuses_a_width_mismatch():
    """Without pose encoding the library takes x's width D as fusion_encoder[0]'s input width and reads its weight
    with row stride D: for any other width it would read past the weight or compute garbage, so the call raises
    before anything is allocated or launched.  The matching width reaches the library with d_in = D."""
    ops = _cpu_ops()
    m = make_smt(D=64, pose_index=None, d_model=64, nhead=4)
    with torch.no_grad():
        for D in (40, 100):
            x, memory, masks, goal = make_inputs(3, 5, D=D, d_model=64, pose_index=None)
            try:
                ops.smt_state_encoder(m, x, memory, masks, goal)
            except ValueError as e:
                assert "fusion_encoder" in str(e)
            else:
                pytest.fail(f"x of width {D} reached the library as (N, M, d_in, pose_index) {ops.lib.calls}")
        assert ops.lib.calls == [] and ops._smt_scratch == {}
        x, memory, masks, goal = make_inputs(3, 5, D=64, d_model=64, pose_index=None)
        assert ops.smt_state_encoder(m, x, memory, masks, goal).shape == (3, 64)
        p = make_smt(D=40, pose_index=36, d_model=64, nhead=4)          # with pose encoding F = pose index + 16
        x, memory, masks, goal = make_inputs(3, 5, D=40, d_model=64, pose_index=36)
        ops.smt_state_encoder(p, x, memory, masks, goal)
    assert ops.lib.calls == [(3, 5, 64, -1), (3, 5, 40, 36)]


def test_fused_single_forward_hands_narrow_inputs_to_the_library(monkeypatch):
    """D = 1 and 2 without pose encoding are inside the library's limits (the pose index + 4 <= D limit applies only
    with pose encoding)."""
    fake = FakeCuda(monkeypatch)
    with torch.no_grad():
        for D in (1, 2):
            m = make_smt(D=D, pose_index=None, d_model=64, nhead=4)
            x, memory, masks, goal = make_inputs(3, 6, D=D, d_model=64, pose_index=None)
            assert smt.smt_layout_error(m, CPU) == ""
            assert smt.fused_single_forward(m, x, memory, masks, goal) == "fused"
            assert smt.fused_single_forward(m, x, memory, masks) == "fused"
    assert fake.ops.calls == [((3, D), (6, 3, D), (3, 6), g) for D in (1, 2) for g in (False, True)]


# ---------------------------------------------------------------------------
# the tiling of ssb_smt_state_encoder_batch, restated, against the sweep of tests/test_gpu_smt_domain.py
# ---------------------------------------------------------------------------
SMT_RT = 16            # token rows per CTA: fuse, both linears, attention queries, encoder tail
SMT_KT_KEYS = 64       # attention keys per shared-memory tile
NC, KT = 128, 64       # smt_block_linear<16, 2>: output columns per chunk, K per weight tile
DEC_ENVS = 4           # decoder envs per CTA
SMT_WS = 8256


def last_tile(n, tile):
    """(tiles, size of the last one) for n items in tiles of ``tile``."""
    t = -(-n // tile)
    return t, n - (t - 1) * tile


def smt_geometry(c):
    """What each of the six launches of one case meets: per kernel, its GEMMs (N, K), the last query tile's rows for
    each env, the attention's last key tile for each env, d, head dim, B."""
    d, hd = c["d_model"], c["d_model"] // c["nhead"]
    F = c["pose_index"] + 16 if c["pose_index"] is not None else c["D"]
    cnt = [1 if c["pretraining"] else v + 1 for v in c["valid"]]
    return dict(d=d, hd=hd, F=F, B=c["B"], T=c["M"] + 1, cnt=cnt,
                gemms={"fuse": [(d, F), (d, d)], "qkv": [(3 * d, d)], "tail": [(d, d)] * 3, "kv": [(2 * d, d)]})


def smt_smem(g):
    """Dynamic shared memory of each launch (bytes), as the entry sizes it."""
    Fp, Tp, d, hd = (g["F"] + 3) & ~3, (g["T"] + 3) & ~3, g["d"], g["hd"]
    return {"fuse": (SMT_RT * Fp + SMT_RT * d + SMT_WS + SMT_RT + 8) * 4, "linear": (SMT_RT * d + SMT_WS) * 4,
            "attn": (SMT_RT * hd + SMT_KT_KEYS * (hd + 1) + SMT_RT * Tp) * 4, "tail": (3 * SMT_RT * d + SMT_WS) * 4,
            "dec": (4 * DEC_ENVS * d + 8 * Tp) * 4}


def test_smt_tiling_mirror():
    """The mirror's tiles cover their extents exactly, and its largest shared-memory sizes are the ones ssb_create
    opts into (SMT_SMEM_*; the fuse kernel's X tile is sized for D + 16 = 1040 columns, F reaches 1036)."""
    for n in (1, 15, 16, 17, 1023, 1024):
        for tile in (16, 64, 128):
            t, last = last_tile(n, tile)
            assert 0 < last <= tile and (t - 1) * tile + last == n
    top = smt_smem(dict(F=smt.MAX_D_IN + 12, T=smt.MAX_TOKENS, d=smt.MAX_D_MODEL, hd=smt.MAX_HEAD_DIM))
    assert top["linear"] == (SMT_RT * 512 + SMT_WS) * 4 and top["attn"] == (16 * 128 + 64 * 129 + 16 * 1024) * 4
    assert top["fuse"] < (SMT_RT * (1024 + 16) + SMT_RT * 512 + SMT_WS + SMT_RT + 8) * 4 <= 227 * 1024


def test_gpu_sweep_reaches_every_smt_tile_edge():
    """For each kernel: a full and a partial last 128-column tile; one K tile, several, and a short last one; a last
    query tile of 1, 15 and 16 rows; (attention) a last key tile of 1, 63 and 64 keys; d and head dim below 32 and off
    the 32-lane grid; (decoder) a full and a partial 4-env group.  Also the largest shared-memory footprint of each
    launch the entry allows."""
    from smt_domain_cases import sweep
    kernels = ("fuse", "qkv", "attn", "tail", "kv", "dec")
    seen = {k: set() for k in kernels}
    top = {}
    for c in sweep():
        g = smt_geometry(c)
        for k, gemms in g["gemms"].items():
            for N, K in gemms:
                seen[k].add("full columns" if N % NC == 0 else "partial columns")
                kt, last = last_tile(K, KT)
                seen[k].add("one K tile" if kt == 1 else "several K tiles")
                if last < KT:
                    seen[k].add("short K tile" if kt == 1 else "short last K tile")
        for n in g["cnt"]:
            for k in ("fuse", "qkv", "attn", "tail", "kv"):
                seen[k].add(f"rows {last_tile(n, SMT_RT)[1]}")
            seen["attn"].add(f"keys {last_tile(n, SMT_KT_KEYS)[1]}")
            seen["dec"].add(f"lane keys {n % 32}")
        for k in ("tail", "dec"):
            seen[k].add("d < 32" if g["d"] < 32 else "d tail" if g["d"] % 32 else "d on the lanes")
        for k in ("attn", "dec"):
            seen[k].add("hd < 32" if g["hd"] < 32 else "hd tail" if g["hd"] % 32 else "hd on the lanes")
        seen["dec"].add("partial group" if g["B"] % DEC_ENVS else "full group")
        for k, v in smt_smem(g).items():
            top[k] = max(top.get(k, 0), v)
    gemm = {"full columns", "partial columns", "one K tile", "several K tiles", "short K tile", "short last K tile"}
    rows = {"rows 1", "rows 15", "rows 16"}
    for k in ("fuse", "qkv", "tail", "kv"):
        assert gemm | rows <= seen[k], (k, (gemm | rows) - seen[k])
    assert rows | {"keys 1", "keys 63", "keys 64"} <= seen["attn"], seen["attn"]
    lanes = {"d < 32", "d tail", "d on the lanes"}
    heads = {"hd < 32", "hd tail", "hd on the lanes"}
    assert lanes <= seen["tail"] and heads <= seen["attn"]
    assert lanes | heads | {"partial group", "full group", "lane keys 0", "lane keys 1", "lane keys 31"} <= seen["dec"]
    most = smt_smem(dict(F=smt.MAX_D_IN + 12, T=smt.MAX_TOKENS, d=smt.MAX_D_MODEL, hd=smt.MAX_HEAD_DIM))
    assert top == most, (top, most)


def test_gpu_sweep_masks_hold_the_listed_counts():
    """The masks the GPU file builds hold exactly each case's listed valid slots (padding iff 1 - m > 0)."""
    from smt_domain_cases import sweep
    from test_gpu_smt_domain import masks_for
    for c in sweep():
        masks = masks_for(c)
        assert masks.shape == (c["B"], c["M"])
        assert (~((1 - masks) > 0)).sum(1).tolist() == c["valid"], c["name"]
