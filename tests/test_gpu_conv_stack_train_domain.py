"""``ssb_conv_stack_train_forward_batch`` / ``_backward_batch`` across the layer shapes, inputs, gradient requests and
limits their entries accept (tests/conv_stack_train_domain_cases.py), on the GPU:

1. the forward's features and out bit-identical (as int32) to the inference entry of the same input wherever that
   entry takes the case, at the case's B, on a permuted batch and for one env alone; elsewhere within float64's bound;
2. every requested gradient against a float64 backward from the kernel's own saved activations and masks:
   |got - ref64| <= C_BAR * bound elementwise, the bound being the same backward over |W|, |x|, |labels|, |g_out|.
   C_BAR = 1e-4.  Worst err / bound per family, torch's float32 CPU backward (calibrated the same way in
   tests/test_conv_stack_train_domain_host.py::test_calibrated_bars) / these kernels on an NVIDIA H100 80GB HBM3:
   reused 2.6e-7 / 2.5e-7, over_limit 1.7e-7 / 1.8e-7, fwd 1.7e-7 / 1.7e-7, dw 9.3e-8 / 1.1e-7, dx 1.7e-7 / 1.4e-7,
   inputs 1.3e-7 / 1.7e-7, flags 1.1e-7 / 1.4e-7, batch 1.1e-7 / 1.2e-7 (batch includes 65535 envs), so C_BAR
   leaves about 400x headroom over both;
3. the flip-free END_TO_END cases against float64 autograd, each tensor within 1e-5 of its largest value;
4. NaN / +-Inf pixels and a NaN label give float64's NaN and Inf positions, and an all-zero env adds exactly 0;
5. each gradient requested alone or in subsets gives the full request's bits and leaves the other gradients' memory
   (its neighbours in one NaN-filled buffer) untouched, with the launch count of the entry's formula;
6. determinism at 3 dW chunks and at 65535 envs;
7. refusals of both entries return their code and launch nothing;
8. the patched AudioCNN (with and without SAVi's labels), VisualCNN and MapCNN run the library where the workspace
   function accepts the shape and fall back as a whole where it refuses (a layout past the K limit, 65536 envs, the
   two backward grid edges), matching float64 either way."""
import ctypes as C
import math

import numpy as np
import pytest

import conv_stack_models as cm
import conv_stack_train_domain_cases as cases
from test_conv_stack_train_domain_host import (C_BAR, bounded_reference, model_args, torch_grads, torch_input,
                                               torch_net)

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

INVALID, SHAPE = -1, -4


def _ops():
    from soundspaces_b200.renderer import WaveformOps
    return WaveformOps.get("cuda:0")


def _gpu(t):
    if t is None:
        return None
    if t._base is not None and not t.is_contiguous():          # labels: keep the row stride
        return t._base.cuda()[:, :t.shape[1]]
    return t.contiguous().cuda()


def _ptr(t):
    return None if t is None else t.data_ptr()


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


class Call:
    """One case's inputs, parameters and ABI structures on the GPU."""

    def __init__(self, c, params=None, inputs=None, B=None):
        from soundspaces_b200 import _lib
        self.c, self.ops = c, _ops()
        self.lib, self.ctx = self.ops.lib, self.ops.ctx
        self.params_cpu = cases.make_params(c) if params is None else params
        self.inputs_cpu = cases.make_inputs(c, B) if inputs is None else inputs
        self.params = [_gpu(p) for p in self.params_cpu]
        self.x, self.depth, self.labels = (_gpu(t) for t in self.inputs_cpu)
        first = self.inputs_cpu[0] if self.inputs_cpu[0] is not None else self.inputs_cpu[1]
        self.B = first.shape[0]
        kind = {"audio": _lib.CONV_INPUT_SPECTROGRAM, "visual": _lib.CONV_INPUT_VISUAL, "map": _lib.CONV_INPUT_MAP}
        self.inp = _lib.ConvStackInput(d_x=_ptr(self.x), d_depth=_ptr(self.depth), d_labels=_ptr(self.labels),
                                       label_stride=self.labels.stride(0) if self.labels is not None else 0,
                                       kind=kind[c["kind"]], H=c["H"], W=c["W"], channels=c["nA"], n_depth=c["nB"],
                                       n_labels=c["NL"])
        self.layers = (_lib.Conv2dLayer * 3)()
        for i in range(3):
            self.layers[i] = _lib.Conv2dLayer(self.params[2 * i].data_ptr(), _ptr(self.params[2 * i + 1]),
                                              c["C"][i], *c["K"][i], *c["S"][i], c["relu"][i])
        self.F, self.hidden = cases.features(c), c["hidden"]

    def ws(self, backward):
        n = self.lib.ssb_conv_stack_train_workspace_bytes(self.B, C.byref(self.inp), self.layers, self.F, self.hidden,
                                                          backward)
        assert n >= 0
        return torch.empty(max(n, 16), dtype=torch.uint8, device="cuda")

    def forward(self, **kw):
        feat = torch.empty((self.B, self.F), device="cuda")
        out = torch.empty((self.B, self.hidden), device="cuda")
        saved = self.ws(0) if "ws" not in kw else None
        a = dict(B=self.B, inp=C.byref(self.inp), layers=self.layers, lw=self.params[6].data_ptr(),
                 lb=_ptr(self.params[7]), F=self.F, feat=feat.data_ptr(), out=out.data_ptr(), ws=_ptr(saved))
        a.update(kw)
        rc = self.lib.ssb_conv_stack_train_forward_batch(self.ctx.handle, a["B"], a["inp"], a["layers"], a["lw"],
                                                          a["lb"], a["F"], self.hidden, self.c["lin_relu"], a["feat"],
                                                          a["out"], a["ws"], _stream())
        return rc, feat, out, saved

    def inference(self):
        """(rc, features, out) of the rollout entry of the case's kind."""
        feat = torch.empty((self.B, self.F), device="cuda")
        out = torch.empty((self.B, self.hidden), device="cuda")
        c, h = self.c, self.ctx.handle
        common = (self.params[6].data_ptr(), _ptr(self.params[7]), self.hidden, c["lin_relu"], feat.data_ptr(),
                  out.data_ptr(), _stream())
        if c["kind"] == "audio":
            rc = self.lib.ssb_audio_encoder_category_batch(h, self.B, _ptr(self.x), c["H"], c["W"], self.layers,
                                                           _ptr(self.labels), c["NL"], self.inp.label_stride, *common)
        elif c["kind"] == "visual":
            rc = self.lib.ssb_visual_encoder_batch(h, self.B, _ptr(self.x), c["nA"], _ptr(self.depth), c["nB"],
                                                   c["H"], c["W"], self.layers, *common)
        else:
            rc = self.lib.ssb_map_encoder_batch(h, self.B, _ptr(self.x), c["nA"], c["H"], c["W"], self.layers, *common)
        return rc, feat, out

    def backward(self, feat, out, saved, dout, need=(True,) * 8, **kw):
        # all eight gradients back to back in one NaN-filled buffer (each 16-byte aligned): a write outside a
        # requested gradient would land in a neighbour
        offs, total = [], 0
        for p in self.params:
            offs.append(total)
            total += cases.round4(p.numel()) if p is not None else 0
        arena = torch.full((max(total, 4),), float("nan"), device="cuda")
        grads = [arena[o:o + p.numel()].view(p.shape) if p is not None else None for o, p in zip(offs, self.params)]
        use = [g if n else None for g, n in zip(grads, need)]
        dw = (C.c_void_p * 4)(*[_ptr(g) for g in use[0::2]])
        db = (C.c_void_p * 4)(*[_ptr(g) for g in use[1::2]])
        ws = self.ws(1)
        a = dict(B=self.B, d_saved=saved.data_ptr(), ws=ws.data_ptr(), dw=dw, db=db, d_features=feat.data_ptr(),
                 d_grad_out=dout.data_ptr())
        a.update(kw)
        rc = self.lib.ssb_conv_stack_train_backward_batch(self.ctx.handle, a["B"], C.byref(self.inp), self.layers,
                                                           self.params[6].data_ptr(), self.F, self.hidden,
                                                           self.c["lin_relu"], a["d_features"], out.data_ptr(),
                                                           a["d_saved"], a["d_grad_out"], a["ws"], a["dw"], a["db"],
                                                           _stream())
        return rc, grads, use

    def saved_acts(self, saved, feat, out):
        flat = saved.view(torch.float32)
        a = [flat[o:o + math.prod(s)].view(s) for o, s in cases.saved_offsets(self.c, self.B)]
        return [t.double().cpu().numpy() for t in a + [feat, out]]


def same_bits(a, b):
    """Equal as int32 wherever either is not NaN; NaN at the same positions."""
    na, nb = torch.isnan(a), torch.isnan(b)
    return torch.equal(na, nb) and torch.equal(a.view(torch.int32)[~na], b.view(torch.int32)[~nb])


def _dout(c, B):
    g = torch.Generator().manual_seed(2)
    return torch.randn((B, c["hidden"]), generator=g)


def _forward_bound(call):
    """float64 features and out of a case and the bounds of their pre-activations."""
    c = call.c
    kind, xn, pn, strides, dn, ln = model_args(c, call.params_cpu, *call.inputs_cpu)
    acts = cm.forward(kind, xn, pn, strides, dn, ln, c["relu"], c["lin_relu"])
    ab = lambda a: None if a is None else np.abs(a)                         # noqa: E731
    b = cm.forward(kind, ab(xn), [ab(p) for p in pn], strides, ab(dn), ab(ln),
                                                (0, 0, 0), 0)
    return acts[2:], b[2:]


FWD_CASES = cases.RUN + [cases.INPUT_LAYOUT, cases.LABEL_INPUT_LAYOUT]


@pytest.mark.parametrize("c", FWD_CASES, ids=[c["name"] for c in FWD_CASES])
def test_forward_bits(c):
    call = Call(c)
    rc, feat, out, _ = call.forward()
    assert rc == 0
    irc, ifeat, iout = call.inference()
    if c["family"] == "reused":                                 # the rollout entry takes these: the same bits
        assert irc == 0
    elif c["family"] == "over_limit":                           # past its shared-memory limit
        assert irc == SHAPE
    if irc == 0:
        assert same_bits(feat, ifeat) and same_bits(out, iout)
    else:                                                       # a shape only the training entry takes
        assert irc == SHAPE
        (f64, o64), (fb, ob) = _forward_bound(call)
        assert (np.abs(feat.double().cpu().numpy() - f64) <= C_BAR * fb + 1e-30).all()
        assert (np.abs(out.double().cpu().numpy() - o64) <= C_BAR * ob + 1e-30).all()
    if call.B > 1:
        perm = torch.randperm(call.B, generator=torch.Generator().manual_seed(4))
        pin = tuple(None if t is None else t[perm] for t in call.inputs_cpu)
        if c["NL"]:                                              # the permuted labels keep their row stride
            buf = torch.full((call.B, c["label_stride"]), float("nan"))
            buf[:, :c["NL"]] = pin[2]
            pin = (pin[0], pin[1], buf[:, :c["NL"]])
        _, pfeat, pout, _ = Call(c, call.params_cpu, pin).forward()
        perm = perm.cuda()
        assert same_bits(pfeat, feat[perm]) and same_bits(pout, out[perm])
        j = call.B - 1                                           # the last env alone
        one = tuple(None if t is None else t[j:j + 1] for t in call.inputs_cpu)
        if c["NL"]:
            buf = torch.full((1, c["label_stride"]), float("nan"))
            buf[:, :c["NL"]] = one[2]
            one = (one[0], one[1], buf[:, :c["NL"]])
        _, ofeat, oout, _ = Call(c, call.params_cpu, one).forward()
        assert same_bits(ofeat[0], feat[j]) and same_bits(oout[0], out[j])


def test_negative_zero_bias_over_a_zero_env():
    """conv biases of -0.0 and non-positive conv3 weights over an all-zero env: every conv3 product is +0 x w = -0, so
    the env's features are -0 sums, and conv3's K (20, 24) ends in a short 16-wide tile.  A padded step would add
    fmaf(0, 0, .) and turn them into +0; the forward keeps -0, as the inference entry does."""
    for c in (cases.INPUT_LAYOUT, cases.LABEL_INPUT_LAYOUT):
        params = cases.make_params(c)
        for i in (1, 3, 5):
            if params[i] is not None:
                params[i] = torch.full_like(params[i], -0.0)
        params[4] = -params[4].abs()
        x, depth, labels = cases.make_inputs(c)
        x[1] = 0.0
        if labels is not None:
            labels[1] = 0.0
        call = Call(c, params, (x, depth, labels))
        ic3, kh3, kw3 = (cases.layer_shapes(c)[2][j] for j in (0, 6, 7))
        assert ic3 * kh3 * kw3 % cases.BK                                 # conv3's last K tile is short
        _, feat, out, _ = call.forward()
        assert (feat[1] == 0).all() and torch.signbit(feat[1]).all()
        irc, ifeat, iout = call.inference()
        assert irc == 0 and same_bits(feat, ifeat) and same_bits(out, iout)


def _check_bound(call, grads, feat, out, saved, dout, what):
    acts = call.saved_acts(saved, feat, out)
    ref, bound = bounded_reference(call.c, call.params_cpu, call.inputs_cpu, dout, acts)
    for j, (g, r, b) in enumerate(zip(grads, ref, bound)):
        if g is None:
            continue
        err = np.abs(g.double().cpu().numpy() - r)
        assert (err <= C_BAR * b).all(), (what, j, float(np.max(err / np.maximum(b, 1e-300))))


@pytest.mark.parametrize("c", cases.RUN, ids=[c["name"] for c in cases.RUN])
def test_backward_against_float64_bound(c):
    call = Call(c)
    rc, feat, out, saved = call.forward()
    dout = _dout(c, call.B)
    rc2, grads, _ = call.backward(feat, out, saved, dout.cuda())
    assert rc == 0 and rc2 == 0
    _check_bound(call, grads, feat, out, saved, dout, c["name"])


def test_backward_at_65535_envs_and_deterministic():
    c = cases.BATCHES[3]
    call = Call(c)
    _, feat, out, saved = call.forward()
    dout = _dout(c, call.B)
    rc, a, _ = call.backward(feat, out, saved, dout.cuda())
    _, b, _ = call.backward(feat, out, saved, dout.cuda())
    assert rc == 0 and all(same_bits(x, y) for x, y in zip(a, b) if x is not None)
    _check_bound(call, a, feat, out, saved, dout, "batch65535")


def test_three_chunks_deterministic():
    c = next(c for c in cases.DW if c["name"] == "dw_rows4097")
    call = Call(c)
    _, feat, out, saved = call.forward()
    dout = _dout(c, call.B).cuda()
    _, a, _ = call.backward(feat, out, saved, dout)
    _, b, _ = call.backward(feat, out, saved, dout)
    assert all(same_bits(x, y) for x, y in zip(a, b) if x is not None)


E2E = [c for c in cases.RUN if c["name"] in cases.END_TO_END]


@pytest.mark.parametrize("c", E2E, ids=[c["name"] for c in E2E])
def test_end_to_end_against_float64_autograd(c):
    call = Call(c)
    _, feat, out, saved = call.forward()
    dout = _dout(c, call.B)
    _, grads, _ = call.backward(feat, out, saved, dout.cuda())
    acts, ref = torch_grads(c, [None if p is None else p.double() for p in call.params_cpu], *call.inputs_cpu, dout,
                            torch.float64)
    for got, r in zip([feat, out] + grads, acts[2:] + [None if g is None else g.numpy() for g in ref]):
        if r is None:
            continue
        got = got.double().cpu().numpy().reshape(r.shape)
        assert np.abs(got - r).max() <= 1e-5 * max(np.abs(r).max(), 1e-30), c["name"]


@pytest.mark.parametrize("value", [float("nan"), float("inf"), float("-inf"), "label"])
def test_non_finite_inputs_follow_float64(value):
    c = cases.LABEL_INPUT_LAYOUT if value == "label" else cases.INPUT_LAYOUT
    x, depth, labels = cases.make_inputs(c)
    if value == "label":
        labels[1, 3] = float("nan")
    else:
        x[1, 5, 4, 0] = value
    call = Call(c, None, (x, depth, labels))
    _, feat, out, saved = call.forward()
    dout = _dout(c, call.B)
    _, grads, _ = call.backward(feat, out, saved, dout.cuda())
    acts, ref = torch_grads(c, [None if p is None else p.double() for p in call.params_cpu], x, depth, labels, dout,
                            torch.float64)
    for got, r in zip([feat, out] + grads, acts[2:] + [None if g is None else g.numpy() for g in ref]):
        if r is None:
            continue
        got = got.double().cpu().numpy().reshape(r.shape)
        assert np.array_equal(np.isnan(got), np.isnan(r)) and np.array_equal(np.isposinf(got), np.isposinf(r))
        assert np.array_equal(np.isneginf(got), np.isneginf(r))


def test_all_zero_env_adds_exactly_zero():
    c = dict(cases.INPUT_LAYOUT, bias=(True,) * 4)
    params = [torch.zeros_like(p) if i % 2 else p for i, p in enumerate(cases.make_params(c))]
    x, _, _ = cases.make_inputs(c)
    x[-1] = 0.0
    dout = _dout(c, c["B"])
    full = Call(c, params, (x, None, None))
    _, feat, out, saved = full.forward()
    _, g_full, _ = full.backward(feat, out, saved, dout.cuda())
    assert (out[-1] == 0).all()
    part = Call(c, params, (x[:-1], None, None))
    _, pf, po, ps = part.forward()
    _, g_part, _ = part.backward(pf, po, ps, dout[:-1].cuda())
    for a, b in zip(g_full, g_part):
        assert torch.equal(a, b)                                # equal values; -0 may have become +0
    x0 = torch.cat([x[-1:], x[:-1]])                            # first instead of last: within the bound
    first = Call(c, params, (x0, None, None))
    _, f0, o0, s0 = first.forward()
    d0 = torch.cat([dout[-1:], dout[:-1]])
    _, g0, _ = first.backward(f0, o0, s0, d0.cuda())
    _check_bound(first, g0, f0, o0, s0, d0, "zero env first")


def _launches(need, NL):
    wants = [need[2 * i] or need[2 * i + 1] for i in range(4)]
    n = 1 + wants[3]
    lowest = next((i for i in range(3) if wants[i]), 3)
    if lowest < 3:
        n += 1 + (2 - lowest)
        n += sum(2 + (2 if i == 0 and NL and need[0] else 0) for i in range(3) if wants[i])
    return n


REQUESTS = [tuple(j == i for j in range(8)) for i in range(8)] + [
    (True, True) + (False,) * 6, (False, False, False, True) + (False,) * 4, (False,) * 6 + (True, True),
    (False, False) + (True,) * 6]


@pytest.mark.parametrize("c", [cases.INPUT_LAYOUT, cases.LABEL_INPUT_LAYOUT], ids=["map", "labels"])
def test_gradient_requests(c):
    call = Call(c)
    _, feat, out, saved = call.forward()
    dout = _dout(c, call.B).cuda()
    n0 = call.ctx.launch_count
    _, full, _ = call.backward(feat, out, saved, dout)
    assert call.ctx.launch_count - n0 == _launches((True,) * 8, c["NL"]) == (13 if c["NL"] else 11)
    for need in REQUESTS:
        n0 = call.ctx.launch_count
        rc, grads, _ = call.backward(feat, out, saved, dout, need=need)
        assert rc == 0 and call.ctx.launch_count - n0 == _launches(need, c["NL"]), need
        for g, f, n in zip(grads, full, need):                  # requested: the full request's bits; the rest of
            assert same_bits(g, f) if n else torch.isnan(g).all()  # the shared buffer untouched


def test_refusals_launch_nothing():
    c = cases.LABEL_INPUT_LAYOUT
    call = Call(c)
    rc, feat, out, saved = call.forward()
    assert rc == 0
    dout = _dout(c, call.B).cuda()
    lib, h = call.lib, call.ctx.handle
    msg = lambda: lib.ssb_last_error(h).decode()                            # noqa: E731
    n0 = call.ctx.launch_count
    grads = [torch.empty_like(p) for p in call.params]
    arr = lambda gs: (C.c_void_p * 4)(*[_ptr(g) for g in gs])                # noqa: E731
    dw, db = arr(grads[0::2]), arr(grads[1::2])
    none = arr([None] * 4)
    bad = [dict(d_saved=None), dict(d_saved=saved.data_ptr() + 4),                  # NULL or misaligned d_saved
           dict(dw=(C.c_void_p * 4)(grads[0].data_ptr() + 2, None, None, None), db=none),   # misaligned gradient
           dict(dw=arr([grads[0], grads[0], None, None]), db=none),              # over another gradient
           dict(dw=arr([None, None, None, call.params[6]]), db=none),            # over an input
           dict(dw=(C.c_void_p * 4)(call.x.data_ptr(), None, None, None), db=none),
           dict(dw=(C.c_void_p * 4)(saved.data_ptr(), None, None, None), db=none),
           dict(dw=None), dict(db=None), dict(d_features=None), dict(d_grad_out=None)]       # NULL arrays and inputs
    for k, kw in enumerate(bad):
        kw.setdefault("dw", dw)
        kw.setdefault("db", db)
        rc, _, _ = call.backward(feat, out, saved, dout, **kw)
        assert rc == INVALID and "bad arguments" in msg(), k
    ws = call.ws(1)                                             # a gradient over the workspace
    rc, _, _ = call.backward(feat, out, saved, dout, ws=ws.data_ptr(),
                             dw=(C.c_void_p * 4)(ws.data_ptr(), None, None, None), db=arr([None] * 4))
    assert rc == INVALID
    assert call.ctx.launch_count == n0
    rc, _, _ = call.backward(feat, out, saved, dout, B=0)       # B = 0 and no gradient: nothing to launch
    assert rc == 0
    rc, _, _ = call.backward(feat, out, saved, dout, need=(False,) * 8)
    assert rc == 0 and call.ctx.launch_count == n0
    assert call.forward(B=65536)[0] == INVALID and call.forward(F=call.F + 1)[0] == SHAPE
    assert call.ctx.launch_count == n0
    for name in cases.GRID_EDGES:                               # refused before any launch, forward and backward
        e = next(e for e, _ in cases.LIMITS if e["name"] == name)
        g = Call(dict(e, B=1))
        assert g.lib.ssb_conv_stack_train_workspace_bytes(1, C.byref(g.inp), g.layers, g.F, g.hidden, 1) == -1
        n0 = g.ctx.launch_count
        assert g.forward(ws=16)[0] == SHAPE and ("exceeds" in msg() or "residue classes" in msg())
        assert g.ctx.launch_count == n0


def _module(c, params):
    """A stand-in of the case's encoder class (SAVi's AudioCNN with labels, AV-Nav's without; VisualCNN; MapCNN) with
    the case's ``cnn``, and the function that patches its class."""
    from avnav_models import VisualCNN
    from map_cnn_models import MapCNN
    from soundspaces_b200.encoder import patch_audio_cnn, patch_map_cnn, patch_visual_cnn
    from test_encoder_host import reference_classes
    if c["kind"] == "map":
        m, patch = MapCNN(20, 20, c["nA"], 1, map_type="gm"), patch_map_cnn
    elif c["kind"] == "visual":
        m, patch = VisualCNN(c["nA"], c["nB"], 64, 64, 1), patch_visual_cnn
    else:
        AvNav, _, Savi = reference_classes()
        m = (Savi((65, 26, 2), 1, has_distractor_sound=True) if c["NL"] else
             AvNav((65, 26, 2), 1, audiogoal_sensor="audiogoal"))
        patch = lambda cls, training: patch_audio_cnn(cls, category=True, training=training)   # noqa: E731
    m.cnn = torch_net(c, params, torch.float32)[0]
    return m, patch


def _observations(c, x, depth, labels):
    if c["kind"] == "map":
        return {"gm": x}
    if c["kind"] == "visual":
        return {k: v for k, v in (("rgb", x), ("depth", depth)) if v is not None}
    return {"audiogoal": x, **({"category": labels.contiguous()} if labels is not None else {})}


# (case, B, whether the library runs it): map, AV-Nav audio, SAVi audio with 21 labels and RGB-D visual layouts the
# training entry takes; a rollout layout it refuses (conv3's KX past 2048); 65536 envs; the two backward grid edges
ROUTES = [("dx1_k4s2", None, True), ("dw_rows4097", None, True), ("labels0_one_hot_1", None, True),
          ("route_labels21", None, True), ("visual_kernel_is_input", None, True), ("f257", None, False),
          ("batch17", 65536, False), ("stride_area65536_conv2", 3, False), ("stride_area65536_conv3", 3, False),
          ("hidden4194241", 3, False)]


@pytest.mark.parametrize("name,B,fused", ROUTES, ids=[r[0] for r in ROUTES])
def test_patched_module_routes_and_matches_float64(name, B, fused):
    import copy
    from soundspaces_b200.encoder import conv_stack_train_error
    c = next(c for c in cases.RUN + cases.REFUSED + [e for e, _ in cases.LIMITS] if c["name"] == name)
    c = dict(c, B=c["B"] if B is None else B)
    params = cases.make_params(c)
    m, patch = _module(c, params)
    ref = copy.deepcopy(m).double()
    m.__class__ = patch(type("Patched" + type(m).__name__, (type(m),), {}), training=True)
    m.cuda()
    x, depth, labels = cases.make_inputs(c)
    obs = {k: v.cuda() for k, v in _observations(c, x, depth, labels).items()}
    dout = _dout(c, c["B"])
    prev = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    try:
        assert (conv_stack_train_error(m, obs) == "") == fused
        ops = _ops()
        n0 = ops.ctx.launch_count
        out = m(obs)
        assert ops.ctx.launch_count - n0 == ((5 if c["NL"] else 4) if fused else 0)
        n0 = ops.ctx.launch_count
        (out * dout.cuda()).sum().backward()
        assert ops.ctx.launch_count - n0 == ((13 if c["NL"] else 11) if fused else 0)
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = prev
    r = ref.cnn(torch_input(c, x, depth, labels, torch.float64))
    (r * dout.double()).sum().backward()
    # the fused cases are flip-free (END_TO_END); eager float32 on the others may flip a mask or two
    tol = 1e-5 if fused else 1e-3
    assert (out.double().cpu() - r.detach()).abs().max() <= tol * max(r.abs().max().item(), 1e-30)
    for p, q in zip(m.parameters(), ref.parameters()):
        assert (p.grad.double().cpu() - q.grad).abs().max() <= tol * max(q.grad.abs().max().item(), 1e-30)
