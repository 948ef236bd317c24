"""The float32 image ``ssb_smt_cnn_batch`` documents (tests/smt_cnn_models.py: prep_image_f32) against torch's own area
resize, and the cases of tests/test_gpu_smt_cnn_domain.py (tests/smt_cnn_domain_cases.py) against what the entry
accepts: every bin shape, crop origin, resize limit, stem K split and head layout is reached by at least one case.
Also the float32 calibration of the GPU file's accuracy bar.  No GPU."""
import copy
import os
import re

import numpy as np
import pytest

torch = pytest.importorskip("torch")
F = torch.nn.functional

import smt_cnn_domain_cases as cases  # noqa: E402
from smt_cnn_models import CROP, SMTCNN, bins, observations, prep_image_f32, resize_crop64, set_params  # noqa: E402
from soundspaces_b200 import encoder  # noqa: E402
from test_belief_nets_host import RN_TK, rn_layer  # noqa: E402

RGB_MUL = np.float32(1) / np.float32(255)      # torch's CUDA x / 255.0: a multiply by the float32 reciprocal
MAX_RESIZED = 64 * 1024


def stem(C):
    """The SMTCNN stem's layer: rn_geometry(true, C, 64, 64)'s Conv2d(C, 16, 7, 1, 3)."""
    return rn_layer(C, 16, 7, 1, 3, CROP, CROP)


def _obs(m, B, seed):
    """The GPU file's observation for one input: integer RGB in [0, 255] or depth in k / 1000."""
    o = observations(B, m["H"], m["W"], seed, rgb=m["C"] if m["scale"] else 0, depth=0 if m["scale"] else m["C"])
    return o["rgb" if m["scale"] else "depth"]


def _geom(m):
    return m["rh"], m["rw"], m["cy"], m["cx"]


def _area_f32(x, m):
    """torch's CPU float32 F.interpolate(mode="area") of the scaled observation, cropped.  The input is made
    channels-first contiguous: torch's vectorised channels-last CPU path divides by the bin's area in one step."""
    x = x.permute(0, 3, 1, 2).contiguous()
    if m["scale"]:
        x = x * RGB_MUL
    rh, rw, cy, cx = _geom(m)
    return F.interpolate(x, size=(rh, rw), mode="area")[..., cy:cy + CROP, cx:cx + CROP]


# ------------------------------------------------------------------------------------------------ the emulator
def _inputs():
    for c in cases.fused_cases():
        for k, m in enumerate(c["inputs"]):
            yield f"{c['name']}/{k}", m


@pytest.mark.parametrize("name,m", list(_inputs()), ids=lambda v: v if isinstance(v, str) else "")
def test_emulator_matches_torch_area_resize_bit_for_bit(name, m):
    """The documented order (rounded product, row-by-row sum, / height, / width) is torch's CPU area resize bit for
    bit, and within float32 rounding of the float64 area-matrix stand-in."""
    x = _obs(m, 2, seed=len(name))
    got = torch.from_numpy(prep_image_f32(x.numpy(), RGB_MUL if m["scale"] else 1, *_geom(m)))
    assert got.shape == (2, m["C"], CROP, CROP)
    assert torch.equal(got, _area_f32(x, m)), name
    ref = resize_crop64(x.permute(0, 3, 1, 2).double() / (255.0 if m["scale"] else 1.0), *_geom(m))
    (r0, r1), (c0, c1) = (bins(m["H"], m["rh"], m["cy"]), bins(m["W"], m["rw"], m["cx"]))
    terms = int((r1 - r0).max() * (c1 - c0).max())          # a float32 sum of n terms: n + 3 roundings at most
    assert (got.double() - ref).abs().max().item() <= 2.0 ** -24 * (terms + 3) * ref.abs().max().item(), name


def test_emulator_rounds_each_product():
    """A contracted multiply-add (the product left unrounded) gives a different image wherever a bin is wider than one
    pixel, so the bit-exact tests can tell the two apart."""
    x = observations(2, 128, 128, 0, rgb=3, depth=0)["rgb"].numpy()
    want = prep_image_f32(x, RGB_MUL, 64, 64, 0, 0)
    fused = np.zeros_like(want)
    for dy in range(2):
        for dx in range(2):
            p = x[:, dy::2, dx::2, :].transpose(0, 3, 1, 2).astype(np.float64) * np.float64(RGB_MUL)
            fused = (fused.astype(np.float64) + p).astype(np.float32)      # fma: one rounding per add
    fused = fused / np.float32(2) / np.float32(2)
    assert (fused != want).sum() > 1000
    depth = observations(2, 128, 128, 0, rgb=0, depth=1)["depth"].numpy()
    assert np.array_equal(prep_image_f32(depth, 1, 64, 64, 0, 0),
                          F.avg_pool2d(torch.from_numpy(depth).permute(0, 3, 1, 2), 2).numpy())


def test_emulator_ignores_unread_pixels():
    """NaN / Inf outside every bin of the crop never reach the image."""
    for H, W in cases.UNREAD_SHAPES:
        m = cases.modality(H, W, 2, 1)
        x = _obs(m, 2, seed=1).numpy()
        bad = x.copy()
        rows, cols = _read_window(m)
        mask = np.ones((H, W), bool)
        mask[rows[0]:rows[1], cols[0]:cols[1]] = False
        assert mask.any(), (H, W)
        for v in (np.nan, np.inf):
            bad[:, mask, :] = v
            assert np.array_equal(prep_image_f32(bad, RGB_MUL, *_geom(m)), prep_image_f32(x, RGB_MUL, *_geom(m)))


def _read_window(m):
    """([row0, row1), [col0, col1)): the input pixels the crop's bins read."""
    h0, h1 = bins(m["H"], m["rh"], m["cy"])
    w0, w1 = bins(m["W"], m["rw"], m["cx"])
    return (int(h0[0]), int(h1[-1])), (int(w0[0]), int(w1[-1]))


# ------------------------------------------------------------------------------------------------ coverage
def test_every_case_is_accepted():
    """Every input passes the entry's shape checks; the reference-geometry ones pass encoder.crop_inside too."""
    names = [c["name"] for c in cases.fused_cases() + [cases.IDENTITY_CASE, cases.MAX_B_CASE]]
    assert len(names) == len(set(names))
    for c in cases.fused_cases() + [cases.IDENTITY_CASE, cases.MAX_B_CASE]:
        assert 1 <= len(c["inputs"]) <= 2 and 1 <= c["B"] <= 1024, c["name"]
        for m in c["inputs"]:
            assert 1 <= m["H"] <= 1024 and 1 <= m["W"] <= 1024 and m["C"] >= 1 and m["n_out"] >= 1, c["name"]
            assert CROP <= m["rh"] <= MAX_RESIZED and CROP <= m["rw"] <= MAX_RESIZED, c["name"]
            assert encoder.crop_inside(*_geom(m)), c["name"]
    for c in cases.SHAPE_CASES + cases.PAIR_CASES:
        for m in c["inputs"]:
            assert _geom(m) == encoder.resize_center_crop_geometry(m["H"], m["W"]), c["name"]
    for H, W in cases.UNREAD_SHAPES + [cases.SHARED_PIXEL_SHAPE]:
        assert (H, W) in cases.SHAPES


def _edges(m):
    """The resize / crop edges one input reaches."""
    out = set()
    H, W, rh, rw, cy, cx = m["H"], m["W"], m["rh"], m["rw"], m["cy"], m["cx"]
    out.add("square" if H == W else "landscape" if W > H else "portrait")
    if cy > 0 and cx == 0:
        out.add("crop_y > 0 = crop_x")
    if cx > 0 and cy == 0:
        out.add("crop_x > 0 = crop_y")
    for n_in, n_out, c, axis in ((H, rh, cy, "rows"), (W, rw, cx, "columns")):
        lo, hi = bins(n_in, n_out, c)
        out.add(f"{axis} bins {sorted(set((hi - lo).tolist()))}")
        if n_out > n_in and (lo[1:] < hi[:-1]).any():
            out.add("overlapping upsampling bins")
        if n_out == MAX_RESIZED:
            out.add(f"{axis} resized to {MAX_RESIZED}")
        if c == n_out - CROP and n_out > CROP:
            out.add(f"{axis}: crop at the far edge")
        if c >= 16336:
            out.add("crop offset >= 16336")
        if lo[0] > 0 or hi[-1] < n_in:
            out.add(f"unread {axis}")
    if (H, W) in ((1, 1), (2, 2)):
        out.add(f"{H} x {W} input")
    if (cy, cx) != (rh // 2 - CROP // 2, rw // 2 - CROP // 2):
        out.add("crop not centred")
    if (rh, rw, cy, cx) != encoder.resize_center_crop_geometry(H, W):
        out.add("geometry no reference expression gives")
    return out


def test_cases_reach_every_resize_and_crop_edge():
    seen = set()
    for c in cases.fused_cases():
        for m in c["inputs"]:
            seen |= _edges(m)
    want = {"square", "landscape", "portrait", "crop_y > 0 = crop_x", "crop_x > 0 = crop_y",
            "overlapping upsampling bins", f"rows resized to {MAX_RESIZED}", f"columns resized to {MAX_RESIZED}",
            "rows: crop at the far edge", "columns: crop at the far edge", "crop offset >= 16336", "unread rows",
            "unread columns", "1 x 1 input", "2 x 2 input", "crop not centred", "geometry no reference expression gives"}
    for w in ([1], [1, 2], [2], [2, 3], [3], [4, 5], [8], [8, 9], [16], [16, 17]):
        want |= {f"rows bins {w}", f"columns bins {w}"}
    want |= {"rows bins [5]", "columns bins [4]"}
    assert want <= seen, sorted(want - seen)
    # every square and oblong shape of the issue is there, each only once
    assert sorted(cases.SHAPES) == sorted(set(cases.SHAPES))
    assert {(m, m) for m in (1, 2, 3, 7, 31, 33, 63, 65, 127, 129, 255, 1000, 1023, 1024)} <= set(cases.SHAPES)


def test_unread_and_shared_pixel_shapes():
    """The containment shapes leave rows or columns unread (both orientations and both 65536-long resizes), and the
    shared-pixel shape has a pixel two bins read along each axis."""
    kinds = set()
    for H, W in cases.UNREAD_SHAPES:
        m = cases.modality(H, W, 1, 0)
        (r0, r1), (c0, c1) = _read_window(m)
        assert (r0, r1) != (0, H) or (c0, c1) != (0, W), (H, W)
        kinds |= _edges(m) & {"landscape", "portrait", f"rows resized to {MAX_RESIZED}",
                              f"columns resized to {MAX_RESIZED}"}
    assert len(kinds) == 4, kinds
    H, W = cases.SHARED_PIXEL_SHAPE
    m = cases.modality(H, W, 1, 0)
    for n_in, n_out, c in ((H, m["rh"], m["cy"]), (W, m["rw"], m["cx"])):
        lo, hi = bins(n_in, n_out, c)
        assert n_out > n_in and (lo[1:] < hi[:-1]).any()


def test_restated_stem_split():
    """The stem's layer as ssb_smt_cnn_batch builds it (rn_geometry(true, C, 64, 64): Conv2d(C, 16, 7, 1, 3)), and its
    K split for C = 1 .. 8."""
    src = open(os.path.join(os.path.dirname(encoder.__file__), "csrc", "ssb200.cu")).read()
    assert "rn_geometry(true, in.C, CNN_CROP, CNN_CROP, L[k])" in src
    assert "L[0] = rn_layer(ic, width[0], 7, smt ? 1 : 2, 3, H, W);" in src
    assert re.search(r"#define RN_TK 16\b", src) and RN_TK == 16
    got = {C: stem(C)["S"] for C in range(1, 9)}
    assert got == {1: 1, 2: 1, 3: 2, 4: 3, 5: 4, 6: 4, 7: 4, 8: 4}
    assert stem(2)["K"] == 98 and stem(2)["K"] % RN_TK
    assert stem(4)["K"] - (stem(4)["S"] - 1) * stem(4)["kps"] == 36
    assert [stem(C)["K"] - 3 * stem(C)["kps"] for C in (5, 6, 7, 8)] == [53, 54, 55, 56]


def test_cases_reach_every_channel_count_split_and_head():
    seen, pairs = set(), set()
    for c in cases.fused_cases():
        ms = c["inputs"]
        for m in ms:
            seen.add((m["C"], m["scale"]))
            L = stem(m["C"])
            seen.add(f"S={L['S']}")
            if L["K"] % L["kps"] and L["S"] > 1:
                seen.add("short last range")
            if L["S"] == 1 and L["K"] % RN_TK:
                seen.add("S=1 partial K tile")
            seen.add(f"n_out={m['n_out']}")
            if not m["bias"]:
                seen.add("no bias")
        if len(ms) == 2:
            s0, s1 = stem(ms[0]["C"])["S"], stem(ms[1]["C"])["S"]
            pairs.add("S0>S1" if s0 > s1 else "S0<S1" if s0 < s1 else "S0=S1")
            if ms[0]["C"] == ms[1]["C"] and (ms[0]["H"], ms[0]["W"]) != (ms[1]["H"], ms[1]["W"]):
                pairs.add("equal C, different geometry")
            if ms[0]["n_out"] != ms[1]["n_out"]:
                pairs.add("different n_out")
            if ms[0]["bias"] != ms[1]["bias"]:
                pairs.add("one fc without a bias")
        else:
            pairs.add("one input")
    want = {(C, s) for C in cases.CHANNELS for s in (0, 1)}
    want |= {"S=1", "S=2", "S=3", "S=4", "short last range", "S=1 partial K tile", "no bias"}
    want |= {f"n_out={n}" for n in (1, 64, 100, 257)}
    assert want <= seen, sorted(map(str, want - seen))
    assert {"S0>S1", "S0<S1", "S0=S1", "equal C, different geometry", "different n_out", "one fc without a bias",
            "one input"} <= pairs, pairs
    ident = cases.IDENTITY_CASE["inputs"]
    assert ident[0]["C"] != ident[1]["C"] and (ident[0]["H"], ident[0]["W"]) != (ident[1]["H"], ident[1]["W"])
    assert max(cases.IDENTITY_BATCHES) < cases.IDENTITY_CASE["B"] and cases.MAX_B_CASE["B"] == 1024


# ------------------------------------------------------------------------------------------------ calibration
def _worst_ratio(c, seed, constant=False):
    """max over envs and inputs of max|f32 - f64| / (1e-4 max|f64|) of torch's CPU forward: the float32 image and
    network against the float64 stand-in."""
    ms = c["inputs"]
    model = set_params(SMTCNN({k: m["C"] for k, m in zip(("rgb", "depth"), ms)},
                              n_out={k: m["n_out"] for k, m in zip(("rgb", "depth"), ms)},
                              no_bias=[k for k, m in zip(("rgb", "depth"), ms) if not m["bias"]]), seed).eval()
    worst = 0.0
    for name, m in zip(("rgb", "depth"), ms):
        x = _obs(m, c["B"], seed)
        if constant:
            x = x[:, :1, :1, :].expand_as(x).contiguous()
        net = getattr(model, f"{name}_encoder")
        img32 = torch.from_numpy(prep_image_f32(x.numpy(), RGB_MUL if m["scale"] else 1, *_geom(m)))
        img64 = resize_crop64(x.permute(0, 3, 1, 2).double() / (255.0 if m["scale"] else 1.0), *_geom(m))
        with torch.no_grad():
            a, b = net(img32), copy.deepcopy(net).double()(img64)
        for e in range(a.shape[0]):
            scale = b[e].abs().max().item()
            worst = max(worst, (a[e].double() - b[e]).abs().max().item() / (1e-4 * scale))
    return worst


def test_float32_calibration(capsys):
    """torch's float32 forward on the CPU against float64 on every case, with the GPU file's inputs: the worst error is
    a small fraction of the 1e-4 bar.  Constant images (the 1 x 1 input, and two cases with each env's first pixel
    everywhere) are measured and reported, not bounded: there GroupNorm subtracts a group mean that sits very close to
    most elements, and torch's float32 forward misses the bar by a few times (the GPU file holds the kernels to it)."""
    worst, constant = {}, {}
    for i, c in enumerate(cases.fused_cases()):
        (constant if c["name"] == "s1x1" else worst)[c["name"]] = _worst_ratio(c, seed=i + 1)
    for i, c in enumerate(cases.PAIR_CASES[:2]):
        constant[c["name"]] = _worst_ratio(c, seed=i + 1, constant=True)
    name, cname = max(worst, key=worst.get), max(constant, key=constant.get)
    with capsys.disabled():
        print(f"\nfloat32 / float64 calibration: worst {worst[name]:.3f} of the 1e-4 bar ({name}); constant images "
              f"{constant[cname]:.3f} ({cname})")
    assert worst[name] <= 0.25, (name, worst[name])
