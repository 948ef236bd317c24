"""The conv-stack training kernels' domain cases (tests/conv_stack_train_domain_cases.py) on the host: a restatement of
``cs_plan`` and ``cs_launch_gemm`` (workspace sizes, dW chunks, the three grids, dX's residue classes) checked against
``ssb_conv_stack_train_workspace_bytes`` and shown to reach every tile edge, residue class and limit; the numpy model
of the kernels' equations (tests/conv_stack_models.py) against torch float64 autograd on every case; and the error
bars of tests/test_gpu_conv_stack_train_domain.py calibrated on torch's float32 CPU forward and backward."""
import ctypes as C

import numpy as np
import pytest
import torch

import conv_stack_models as cm
import conv_stack_train_domain_cases as cases

GRID_X, GRID_YZ = 2 ** 31 - 1, 65535
# the GPU file's bar: |got - ref64| <= C_BAR bound, elementwise (bound: the same backward over |W|, |x|, |labels|,
# |g_out| with the kernel's masks).  The calibration below holds torch's float32 CPU results to C_BAR / 10.
C_BAR = 1e-4
# a ReLU input closer to 0 than this fraction of its bound (sum |w| |x| + |b|) could round to the other side
FLIP_MARGIN = 1e-4


def _ceil(a, b):
    return -(-a // b)


def plan(c, B=None, grid_limits=True):
    """``cs_plan`` and ``cs_launch_gemm`` of case ``c`` at B envs: None when refused, else a dict of the layers (K, Kw,
    KX, chunks, fwd / dw / dx grids, dx residue classes on demand), F and the workspace sizes in floats.
    ``grid_limits=False`` leaves out the stride-area and hidden refusals, which keep the backward's grids in range."""
    B = c["B"] if B is None else B
    NL, hidden = c["NL"], c["hidden"]
    if B > cases.MAX_B or NL > cases.MAX_LABELS or B * c["H"] * c["W"] > cases.INT32_MAX:
        return None
    layers, ic = [], c["nA"] + c["nB"]
    shapes = cases.layer_shapes(c)
    if shapes is None:
        return None
    for i, (ic, h, w, oc, ho, wo, kh, kw, sh, sw) in enumerate(shapes):
        if grid_limits and i > 0 and sh * sw > cases.MAX_STRIDE_AREA:
            return None
        K, KX = ic * kh * kw, oc * _ceil(kh, sh) * _ceil(kw, sw)
        if (K > cases.MAX_K or (i > 0 and KX > cases.MAX_K) or B * oc * ho * wo > cases.INT32_MAX
                or B * ic * h * w > cases.INT32_MAX):
            return None
        rows = B * ho * wo
        chunks = _ceil(rows, cases.RCHUNK)
        layers.append(dict(IC=ic, H=h, W=w, OC=oc, Ho=ho, Wo=wo, KH=kh, KW=kw, SH=sh, SW=sw, K=K, KX=KX, rows=rows,
                           Kw=(ic + (NL if i == 0 else 0)) * kh * kw, chunks=chunks,
                           fwd=(_ceil(rows, cases.BM), _ceil(oc, cases.BN), 1),
                           dw=(chunks, _ceil(K, cases.BM), _ceil(oc, cases.BN)),
                           dx=(_ceil(B * _ceil(h, sh) * _ceil(w, sw), cases.BM), _ceil(ic, cases.BN), sh * sw)))
    F = cases.features(c)
    if B * hidden > cases.INT32_MAX or (grid_limits and hidden > cases.MAX_HIDDEN):
        return None
    r4 = cases.round4
    L1, L2 = layers[0], layers[1]
    a2 = r4(B * L1["OC"] * L1["Ho"] * L1["Wo"])
    lb = a2 + r4(B * L2["OC"] * L2["Ho"] * L2["Wo"])
    fwd = lb + (r4(B * L1["OC"]) if NL else 0)
    part = max(L["chunks"] * L["OC"] * L["K"] for L in layers)
    partb = max(L["chunks"] * L["OC"] for L in layers)
    dF = r4(B * hidden)
    da2 = dF + r4(B * F)
    da1 = da2 + (lb - a2)
    s = da1 + a2 + r4(part) + r4(partb)
    bwd = s + (r4(B * L1["OC"]) if NL else 0)
    lin = dict(dw=(_ceil(F, cases.GG_BN), _ceil(hidden, cases.GG_BM), 1), df=(_ceil(F, cases.GG_BN),
                                                                               _ceil(B, cases.GG_BM), 1))
    return dict(layers=layers, F=F, fwd_floats=fwd, bwd_floats=bwd, lin=lin)


def classes(L):
    """dX's residue classes (rh, rw, Qh, Qw, Jh, Jw) of a planned layer, as cs_gemm_kernel<CS_DX> derives them."""
    out = []
    for rh in range(L["SH"]):
        for rw in range(L["SW"]):
            Qh, Qw = (L["H"] - rh + L["SH"] - 1) // L["SH"], (L["W"] - rw + L["SW"] - 1) // L["SW"]
            Jh = (L["KH"] - rh + L["SH"] - 1) // L["SH"] if rh < L["KH"] else 0
            Jw = (L["KW"] - rw + L["SW"] - 1) // L["SW"] if rw < L["KW"] else 0
            out.append((rh, rw, Qh, Qw, Jh, Jw))
    return out


def grids(p):
    """Every launch grid of a planned call: the forward's and the backward's with every gradient requested."""
    g = [p["lin"]["dw"], p["lin"]["df"]]
    for i, L in enumerate(p["layers"]):
        g += [L["fwd"], L["dw"]] + ([L["dx"]] if i > 0 else [])
    return g


def lib_args(c, B=None):
    """The ssb_conv_stack_input and layer array of a case with dummy pointers (the workspace function reads none)."""
    from soundspaces_b200 import _lib
    B = c["B"] if B is None else B
    kind = {"audio": _lib.CONV_INPUT_SPECTROGRAM, "visual": _lib.CONV_INPUT_VISUAL, "map": _lib.CONV_INPUT_MAP}
    inp = _lib.ConvStackInput(d_x=16 if c["nA"] else None, d_depth=16 if c["nB"] else None,
                              d_labels=16 if c["NL"] else None, label_stride=c["label_stride"], kind=kind[c["kind"]],
                              H=c["H"], W=c["W"], channels=c["nA"], n_depth=c["nB"], n_labels=c["NL"])
    layers = (_lib.Conv2dLayer * 3)()
    for i in range(3):
        layers[i] = _lib.Conv2dLayer(16, 16 if c["bias"][i] else None, c["C"][i], *c["K"][i], *c["S"][i],
                                     c["relu"][i])
    return B, inp, layers


def lib_bytes(c, backward, B=None):
    from soundspaces_b200 import _lib
    B, inp, layers = lib_args(c, B)
    shapes = cases.layer_shapes(c)
    F = cases.features(c) if shapes else 1
    return _lib.load_library().ssb_conv_stack_train_workspace_bytes(B, C.byref(inp), layers, F, c["hidden"],
                                                                    backward)


EVERY = (cases.RUN + cases.REFUSED + [cases.BATCHES[3], cases.INPUT_LAYOUT, cases.LABEL_INPUT_LAYOUT]
         + [c for c, _ in cases.LIMITS])


def test_restated_plan_matches_library():
    for c in EVERY:
        p = plan(c)
        for backward in (0, 1):
            want = -1 if p is None else 4 * (p["bwd_floats"] if backward else p["fwd_floats"])
            assert lib_bytes(c, backward) == want, (c["name"], backward)
    assert lib_bytes(cases.BATCHES[0], 1, B=65536) == -1
    assert len(cases.REFUSED) == len(cases.TRAIN_REFUSED) and all(plan(c) is None for c in cases.REFUSED)


def test_limit_pairs():
    for c, accepted in cases.LIMITS:
        assert (plan(c) is not None) == accepted, c["name"]
    names = [c["name"] for c, _ in cases.LIMITS]
    for lo, hi in (("k2048", "k2049"), ("kx2048", "kx2049"), ("labels256", "labels257"), ("b65535", "b65536"),
                   ("bhw_in", "bhw_over"), ("bchw_input_in", "bchw_input_over"),
                   ("bchw_output_in", "bchw_output_over"), ("bhidden_in", "bhidden_over"),
                   ("stride_area65535_conv2", "stride_area65536_conv2"), ("hidden4194240", "hidden4194241")):
        assert lo in names and hi in names
    by = {c["name"]: c for c, _ in cases.LIMITS}
    assert by["labels257"]["label_stride"] > 257 and by["labels256"]["label_stride"] > 256
    assert plan(by["k2048"])["layers"][0]["K"] == 2048 and plan(by["kx2048"])["layers"][1]["KX"] == 2048
    # each over-limit shape is refused by the guard it names, the others holding
    assert by["bhw_over"]["B"] * by["bhw_over"]["H"] * by["bhw_over"]["W"] > cases.INT32_MAX
    c = by["bchw_input_over"]
    assert c["B"] * c["H"] * c["W"] <= cases.INT32_MAX < c["B"] * c["nA"] * c["H"] * c["W"]
    c = by["bchw_output_over"]
    assert c["B"] * c["nA"] * c["H"] * c["W"] <= cases.INT32_MAX < c["B"] * c["C"][0] * c["H"] * c["W"]
    assert by["bhidden_over"]["B"] * by["bhidden_over"]["hidden"] > cases.INT32_MAX


def test_grid_edges():
    """Without the stride-area and hidden limits, cs_plan accepted the three GRID_EDGES shapes and the backward's
    launches would have exceeded a grid dimension (dX's z = SH SW, the Linear dW's y = ceil(hidden / 64)): 65536 >
    65535.  The plan refuses them now, and every grid of every accepted case is within the device limits."""
    for c, _ in cases.LIMITS:
        p, loose = plan(c), plan(c, grid_limits=False)
        if c["name"] in cases.GRID_EDGES:
            assert p is None and loose is not None
            assert max(max(g[1], g[2]) for g in grids(loose)) == 65536, c["name"]
    for c in EVERY:
        p = plan(c)
        if p is not None:
            for g in grids(p):
                assert g[0] <= GRID_X and g[1] <= GRID_YZ and g[2] <= GRID_YZ, (c["name"], g)


def _run_plans():
    return [(c, plan(c)) for c in cases.RUN]


def test_cases_reach_every_edge():
    runs = _run_plans()
    assert all(p is not None for _, p in runs)
    Ls = [(i, L) for _, p in runs for i, L in enumerate(p["layers"])]
    rows = {L["rows"] for _, L in Ls}
    assert {1, 127, 128, 129} <= rows                                      # CS_FWD row tiles
    assert {1, 31, 32, 33} <= {L["OC"] for _, L in Ls}                     # CS_FWD / CS_DW channel tiles
    assert {1, 15, 16, 17, 2047, 2048} <= {L["K"] for _, L in Ls}          # K tiles of 16, the K limit
    chunk_rows = {(L["rows"], L["chunks"]) for _, L in Ls}
    assert {(2047, 1), (2048, 1), (2049, 2), (4096, 2), (4097, 3)} <= chunk_rows
    assert {127, 128, 129} <= {L["K"] for _, L in Ls}                      # CS_DW's 128-column tiles
    for at in (1, 2):                                                      # CS_DX in conv2 and in conv3
        dx = [L for i, L in Ls if i == at]
        assert any(L["KH"] % L["SH"] == 0 and L["KH"] > L["SH"] for L in dx)
        assert any(L["KH"] % L["SH"] and L["KH"] > L["SH"] for L in dx)
        assert any(any(j[4] == 0 for j in classes(L)) and any(j[5] == 0 for j in classes(L)) for L in dx)
        assert any(any(j[2] == 0 for j in classes(L)) and any(j[3] == 0 for j in classes(L)) for L in dx)
        assert any(L["SH"] != L["SW"] for L in dx)
        unread = lambda n, k, s, o: set(range(n)) - {s * q + t for q in range(o) for t in range(k)}  # noqa: E731
        assert any(unread(L["H"], L["KH"], L["SH"], L["Ho"]) and unread(L["W"], L["KW"], L["SW"], L["Wo"])
                   for L in dx)
        assert {31, 32, 33} <= {L["IC"] for L in dx}
        assert 2048 in {L["KX"] for L in dx}
    got = {(c["NL"], c.get("labels")) for c, _ in runs if c["kind"] == "audio"}
    for n in cases.LABEL_COUNTS[1:]:
        assert all((n, k) in got for k in cases.ac.LABEL_KINDS)
    assert all(c["label_stride"] > c["NL"] for c, _ in runs if c["name"].startswith("labels") and c["NL"])
    assert 0 in {n for n, _ in got}
    vis = {(c["nA"], c["nB"]) for c, _ in runs if c["kind"] == "visual"}
    assert {(3, 0), (0, 1), (3, 1), (3, 2), (9, 3)} <= vis
    assert set(range(1, 9)) <= {c["nA"] for c, _ in runs if c["kind"] == "map"}
    flags = {(c["bias"], c["relu"], c["lin_relu"]) for c, _ in runs}
    for i in range(4):
        assert any(not b[i] for b, _, _ in flags)
    assert {(r, lr) for _, r, lr in flags} >= {((a, b, d), e) for a in (0, 1) for b in (0, 1) for d in (0, 1)
                                              for e in (0, 1)}
    assert [c["B"] for c in cases.BATCHES] == [1, 2, 17, 65535] and plan(cases.BATCHES[3]) is not None
    assert plan(cases.BATCHES[0], B=65536) is None


def test_saved_offsets_follow_the_plan():
    for c in cases.RUN:
        p = plan(c)
        (o1, s1), (o2, s2) = cases.saved_offsets(c)
        assert o1 == 0 and o2 == cases.round4(int(np.prod(s1))) and o2 + np.prod(s2) <= p["fwd_floats"]


# --- the numpy model against float64 autograd, and the calibration ---------------------------------------------

def torch_net(c, params, dtype):
    """``cnn`` of a case as a torch Sequential of ``dtype`` holding ``params``."""
    mods, ic = [], c["nA"] + c["nB"] + c["NL"]
    convs = []
    for i, (oc, k, s) in enumerate(zip(c["C"], c["K"], c["S"])):
        conv = torch.nn.Conv2d(ic, oc, k, s, bias=c["bias"][i])
        convs.append(conv)
        mods += [conv] + ([torch.nn.ReLU()] if c["relu"][i] else [])
        ic = oc
    lin = torch.nn.Linear(cases.features(c), c["hidden"], bias=c["bias"][3])
    mods += [torch.nn.Flatten(), lin] + ([torch.nn.ReLU()] if c["lin_relu"] else [])
    net = torch.nn.Sequential(*mods).to(dtype)
    with torch.no_grad():
        for m, (w, b) in zip(convs + [lin], zip(params[0::2], params[1::2])):
            m.weight.copy_(w)
            if b is not None:
                m.bias.copy_(b)
    return net, convs + [lin]


def torch_input(c, x, depth, labels, dtype):
    parts = []
    if c["kind"] == "visual":
        if x is not None:
            parts.append(x.to(dtype).permute(0, 3, 1, 2) / 255.0)
        if depth is not None:
            parts.append(depth.to(dtype).permute(0, 3, 1, 2))
    else:
        parts.append(x.to(dtype).permute(0, 3, 1, 2))
    if labels is not None and labels.shape[1]:
        B, _, H, W = parts[0].shape
        parts.append(labels.to(dtype)[:, :, None, None].expand(B, labels.shape[1], H, W))
    return torch.cat(parts, 1)


def torch_grads(c, params, x, depth, labels, dout, dtype):
    """torch autograd of a case in ``dtype``: (activations (a1, a2, features, out), the eight gradients)."""
    net, layers = torch_net(c, params, dtype)
    a, acts = torch_input(c, x, depth, labels, dtype), []
    for conv, f in zip(layers[:3], c["relu"]):
        a = torch.relu(conv(a)) if f else conv(a)
        acts.append(a)
    acts[2] = acts[2].flatten(1)
    out = layers[3](acts[2])
    acts.append(torch.relu(out) if c["lin_relu"] else out)
    (acts[3] * dout.to(dtype)).sum().backward()
    g = []
    for m, b in zip(layers, c["bias"]):
        g += [m.weight.grad, m.bias.grad if b else None]
    return [t.detach().double().numpy() for t in acts], g


def model_args(c, params, x, depth, labels):
    n = lambda t: None if t is None else t.double().numpy()                 # noqa: E731
    strides = [tuple(s) for s in c["S"]]
    return c["kind"], n(x), [n(p) for p in params], strides, n(depth), n(labels)


def dout_of(c, B=None, seed=2):
    g = torch.Generator().manual_seed(seed)
    return torch.randn((c["B"] if B is None else B, c["hidden"]), generator=g)


def bounded_reference(c, params, inputs, dout, acts):
    """The float64 backward from given activations with their masks, and its bound: the same backward over |W|, |x|,
    |labels|, |g_out| and |activations| with the same masks."""
    kind, xn, pn, strides, dn, ln = model_args(c, params, *inputs)
    keep = cm.masks(acts, c["relu"], c["lin_relu"])
    d = dout.double().numpy() if isinstance(dout, torch.Tensor) else dout
    ref = cm.backward_given(kind, xn, pn, strides, d, acts, dn, ln, keep)
    ab = lambda a: None if a is None else np.abs(a)                         # noqa: E731
    bound = cm.backward_given(kind, ab(xn), [ab(p) for p in pn], strides, np.abs(d), [np.abs(a) for a in acts],
                              ab(dn), ab(ln), keep)
    return ref, bound


def flip_margin(c, params, inputs):
    """min over the ReLU inputs of |v| / bound(v) (bound: the forward over |W|, |x| and |labels|), inf without ReLUs;
    an input whose bound is 0 is exactly 0 in any precision and counts as no flip."""
    kind, xn, pn, strides, dn, ln = model_args(c, params, *inputs)
    ab = lambda a: None if a is None else np.abs(a)                         # noqa: E731
    pre = cm.forward(kind, xn, pn, strides, dn, ln, (0, 0, 0), 0)
    pre_b = cm.forward(kind, ab(xn), [ab(p) for p in pn], strides, ab(dn), ab(ln), (0, 0, 0), 0)
    m = np.inf
    for v, b, f in zip(pre, pre_b, tuple(c["relu"]) + (c["lin_relu"],)):
        if f:
            m = min(m, float(np.min(np.where(b > 0, np.abs(v) / np.where(b > 0, b, 1), np.inf))))
    return m


def reference(c, B=None):
    """A case's float32 inputs and float64 model results on them: activations and gradients."""
    params = cases.make_params(c)
    inputs = cases.make_inputs(c, B)
    dout = dout_of(c, B)
    kind, xn, pn, strides, dn, ln = model_args(c, params, *inputs)
    acts = cm.forward(kind, xn, pn, strides, dn, ln, c["relu"], c["lin_relu"])
    grads = cm.backward_given(kind, xn, pn, strides, dout.double().numpy(), acts, dn, ln,
                              cm.masks(acts, c["relu"], c["lin_relu"]))
    return dict(params=params, inputs=inputs, dout=dout, acts=acts, grads=grads)


HOST_CASES = cases.RUN


@pytest.mark.parametrize("c", HOST_CASES, ids=[c["name"] for c in HOST_CASES])
def test_model_matches_float64_autograd(c):
    r = reference(c)
    acts, g = torch_grads(c, [None if p is None else p.double() for p in r["params"]], *r["inputs"], r["dout"],
                          torch.float64)
    for got, ref in zip(r["acts"], acts):
        assert np.abs(got.reshape(ref.shape) - ref).max() <= 1e-12 * max(np.abs(ref).max(), 1e-30), c["name"]
    for j, (got, ref) in enumerate(zip(r["grads"], g)):
        if ref is None:
            continue
        ref = ref.numpy()
        assert np.abs(got - ref).max() <= 1e-11 * max(np.abs(ref).max(), 1e-300), (c["name"], j)


def calibrate(c):
    """max over the gradients of |torch float32 - float64| / bound, the float64 backward and its bound taken from
    torch's float32 activations and masks (what the GPU file does with the kernel's): the backward's own error."""
    params, inputs, dout = cases.make_params(c), cases.make_inputs(c), dout_of(c)
    acts, g32 = torch_grads(c, params, *inputs, dout, torch.float32)
    ref, bound = bounded_reference(c, params, inputs, dout, acts)
    worst = 0.0
    for got, r, b in zip(g32, ref, bound):
        if got is not None:
            err = np.abs(got.double().numpy() - r)
            worst = max(worst, float(np.max(np.where(b > 0, err / np.where(b > 0, b, 1), np.where(err > 0, np.inf,
                                                                                                    0)))))
    return worst


def test_calibrated_bars():
    """torch's float32 CPU backward is within C_BAR / 10 of float64 relative to the bound on every case."""
    worst = {}
    for c in HOST_CASES:
        ratio = calibrate(c)
        worst[c["family"]] = max(worst.get(c["family"], 0.0), ratio)
        assert ratio <= C_BAR / 10, (c["name"], ratio)
    print({k: f"{v:.2e}" for k, v in sorted(worst.items())})
    assert set(worst) == {"reused", "over_limit", "fwd", "dw", "dx", "inputs", "flags", "batch"}


def test_end_to_end_cases_are_flip_free():
    """No ReLU input of the end-to-end cases lies within FLIP_MARGIN of its bound from 0, so float32 rounding cannot
    flip a mask there and the GPU file can hold them to float64 autograd."""
    for c in cases.RUN:
        if c["name"] in cases.END_TO_END:
            assert flip_margin(c, cases.make_params(c), cases.make_inputs(c)) > FLIP_MARGIN, c["name"]
