"""AV-WaN's device maps (ssb_map_update_batch / ssb_map_observe_batch) across the domain their entries accept, bit for
bit against the numpy stand-in mapper_models.MapMirror (pinned to the reference Mapper at every case of
tests/map_domain_cases.py by tests/test_map_domain_host.py).

Besides the crops, the raw device state is compared: ``gmap[slot][:N^2]`` decoded into (N, N, 2) bits, its pad bytes
0, and ``amap`` as uint64 bits.  NaN rule: a NaN acoustic cell is compared for NaN-ness only, because NumPy and CUDA
may carry different NaN payloads; every other value, -0.0 and the infinities included, is compared bit for bit."""
import ctypes as C
import re

import numpy as np
import pytest
import torch

from map_domain_cases import (GEOMETRIES, SSB_E_INVALID_ARG, SSB_E_SHAPE, case_record, cases, initial_state,
                              mirror_case, observe_refusal, rot_xy, table_length, turns, unrot_xy, update_refusal)
from mapper_models import MapMirror
from soundspaces_b200 import _lib, maps
from soundspaces_b200.renderer import WaveformOps

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)


@pytest.fixture(scope="module")
def ops():
    return WaveformOps.get(DEV)


def pitch(g):
    return (g.internal_size ** 2 + 15) & ~15


def cgeo(g, n_slots):
    return _lib.MapGeometry(*g, n_slots)


def state(g, n_slots, gm0=None, am0=None):
    """Device state buffers of n_slots slots, each holding (gm0, am0) when given; no acoustic map: amap is empty and
    its pointer NULL."""
    m = g.acoustic_size
    gmap = torch.zeros((n_slots, pitch(g)), dtype=torch.uint8, device=DEV)
    amap = torch.zeros((n_slots, m, m) if g.acoustic else (0,), dtype=torch.float64, device=DEV)
    if gm0 is not None:
        gmap[:, :g.internal_size ** 2] = torch.from_numpy(encode(gm0).reshape(-1)).to(DEV)
        if g.acoustic:
            amap[:] = torch.from_numpy(am0).to(DEV)
    return gmap, amap


def encode(bits):
    return (bits[..., 0] | (bits[..., 1].astype(np.uint8) << 1)).astype(np.uint8)


def records(recs_and_slots):
    """(RECORD_DTYPE array, ego bytes) of [(slot, mapper_models record)]."""
    rec = np.zeros(len(recs_and_slots), dtype=maps.RECORD_DTYPE)
    ego = bytearray()
    for i, (slot, (_, kind, x, y, o, value, half, bits)) in enumerate(recs_and_slots):
        rec[i] = (slot, kind, x, y, o, 0, value, half, len(ego))
        ego += bits
    return rec, np.frombuffer(bytes(ego) or b"\0", dtype=np.uint8)[:len(ego)]


def check_raw(g, gmap, amap, slot, mirror, what):
    n2 = g.internal_size ** 2
    row = gmap[slot].cpu().numpy()
    assert not row[n2:].any(), f"{what}: pad bytes written"
    assert not (row[:n2] & 0xFC).any(), f"{what}: bits above the two channels"
    assert np.array_equal(row[:n2], encode(mirror.gm).reshape(-1)), f"{what}: geometric map"
    if g.acoustic:
        same_am(amap[slot].cpu().numpy(), mirror.am, what)


def same_am(got, ref, what):
    nan = np.isnan(ref)
    assert np.array_equal(np.isnan(got), nan), f"{what}: NaN cells"
    assert np.array_equal(got.view(np.uint64)[~nan], ref.view(np.uint64)[~nan]), f"{what}: acoustic map"


def same_f32(got, ref, what):
    got, ref = np.asarray(got, np.float32), np.asarray(ref, np.float32)
    assert got.shape == ref.shape, what
    nan = np.isnan(ref)
    assert np.array_equal(np.isnan(got), nan), f"{what}: NaN"
    assert np.array_equal(got.view(np.uint32)[~nan], ref.view(np.uint32)[~nan]), what


def call_update(ops, g, n_slots, gmap_ptr, amap_ptr, rec, ego):
    rc = ops.lib.ssb_map_update_batch(ops.ctx.handle, C.byref(cgeo(g, n_slots)) if g is not None else None, gmap_ptr,
                                      amap_ptr, len(rec), rec.ctypes.data if len(rec) else None,
                                      ego.ctypes.data if ego.size else None, ego.size, ops._stream())
    return rc, ops.lib.ssb_last_error(ops.ctx.handle).decode() if rc else ""


def call_observe(ops, g, n_slots, gmap_ptr, amap_ptr, poses, tables, L, outs):
    """outs: {kind: (pointer, stride)}."""
    poses = np.ascontiguousarray(poses, dtype=np.int32).reshape(-1, 4)
    tables = np.ascontiguousarray(tables, dtype=np.int32)
    a = [outs.get(k, (None, 0)) for k in ("gm", "am", "action_map")]
    rc = ops.lib.ssb_map_observe_batch(ops.ctx.handle, C.byref(cgeo(g, n_slots)), gmap_ptr, amap_ptr, len(poses),
                                       poses.ctypes.data if len(poses) else None, tables.ctypes.data, L,
                                       a[0][0], a[0][1], a[1][0], a[1][1], a[2][0], a[2][1], ops._stream())
    return rc, ops.lib.ssb_last_error(ops.ctx.handle).decode() if rc else ""


def expect_refusal(ops, call, expected, buffers):
    """Run a refused call: its code and message, nothing launched, the buffers unchanged (bit for bit)."""
    before, copies = ops.ctx.launch_count, [b.clone() for b in buffers]
    rc, msg = call()
    assert rc == expected[0], (rc, msg, expected)
    assert re.search(expected[1], msg), (msg, expected)
    assert ops.ctx.launch_count == before
    torch.cuda.synchronize()
    for b, c in zip(buffers, copies):
        assert torch.equal(b.view(torch.uint8), c.view(torch.uint8))


# --- geometry x orientation x edge pose, through both entries and through DeviceMaps.resolve ---
@pytest.mark.parametrize("name", list(GEOMETRIES))
def test_edge_cases_bit_identical_to_the_mirror(ops, name):
    g = GEOMETRIES[name][0]
    gm0, am0 = initial_state(name)
    L, tables = table_length(g), maps.navigable_tables(g)
    ego_rec = (g.ego_size ** 2 * 2 + 7) // 8
    accepted, mirrors = [], []
    probe_g, probe_a = state(g, 1)
    for c in cases(name):
        rec, ego = records([(0, case_record(c))])
        why = update_refusal(g, 1, rec, ego_rec)
        if why:
            expect_refusal(ops, lambda: call_update(ops, g, 1, probe_g.data_ptr(), probe_a.data_ptr(), rec, ego), why,
                           (probe_g, probe_a))
            continue
        accepted.append(c)
        mirrors.append(mirror_case(c, (gm0, am0))[0])
    B = len(accepted)
    gmap, amap = state(g, B, gm0, am0)
    rec, ego = records([(i, case_record(c)) for i, c in enumerate(accepted)])
    before = ops.ctx.launch_count
    ops.map_update(cgeo(g, B), gmap, amap, rec, ego)
    assert ops.ctx.launch_count - before == 1
    for i, c in enumerate(accepted):
        check_raw(g, gmap, amap, i, mirrors[i], f"{c}")
    poses = np.array([(i, c.x, c.y, c.orientation) for i, c in enumerate(accepted)], np.int32)
    S = g.map_size
    gm = torch.empty((B, S, S, 2), dtype=torch.float32, device=DEV)
    am = torch.empty((B, 20, 20, 1), dtype=torch.float32, device=DEV) if g.acoustic else None
    ops.map_observe(cgeo(g, B), gmap, amap, poses, tables, gm, am, None)
    act_ok = [observe_refusal(g, B, poses[i:i + 1], L, tables, kinds=("action_map",)) is None for i in range(B)]
    sel = [i for i in range(B) if act_ok[i]]
    action = torch.empty((len(sel), g.action_size, g.action_size, 1), dtype=torch.float32, device=DEV)
    ops.map_observe(cgeo(g, B), gmap, amap, poses[sel], tables, None, None, action)
    for i in range(B):
        if not act_ok[i]:
            why = observe_refusal(g, B, poses[i:i + 1], L, tables, kinds=("action_map",))
            out = torch.empty((1, g.action_size, g.action_size, 1), device=DEV)
            expect_refusal(ops, lambda: call_observe(ops, g, B, gmap.data_ptr(), amap.data_ptr(), poses[i:i + 1],
                                                     tables, L, {"action_map": (out.data_ptr(), g.action_size ** 2)}),
                           why, (gmap, amap))
    # the same cases through DeviceMaps.resolve: the seeded state written into each env's slot, then its update record
    dm = maps.DeviceMaps(DEV)
    descs = []
    for i, c in enumerate(accepted):
        tok = f"{name}/{c.index}"
        slot = dm._slot(tok, g)
        maps._RECEIVED[tok] = [case_record(c, seq=0)]
        descs.append(tok)
    dm.gmap[:B, :g.internal_size ** 2] = torch.from_numpy(encode(gm0).reshape(-1)).to(DEV)
    if g.acoustic:
        dm.amap[:B] = torch.from_numpy(am0).to(DEV)
    kinds = ("gm", "am") if g.acoustic else ("gm",)
    by = {k: [maps.MapDescriptor(k, t, tuple(poses[i, 1:]), 0, g, None) for i, t in enumerate(descs)] for k in kinds}
    out = dm.resolve(by)
    by_act = {"action_map": [maps.MapDescriptor("action_map", descs[i], tuple(poses[i, 1:]), 0, g, None) for i in sel]}
    out_act = dm.resolve(by_act)["action_map"] if sel else None
    big = g.map_size > 1024                               # 128 MB per crop: compare one env at a time
    gm_h, out_gm = (None, None) if big else (gm.cpu().numpy(), out["gm"].cpu().numpy())
    torch.cuda.synchronize()
    for i, tok in enumerate(descs):                       # the same raw state as the direct call, checked above
        assert dm.slots[tok] == i and torch.equal(dm.gmap[i], gmap[i]), accepted[i]
        if g.acoustic:
            assert torch.equal(dm.amap[i].view(torch.int64), amap[i].view(torch.int64)), accepted[i]
        ref = mirrors[i].observe(tuple(poses[i, 1:]))
        same_f32(gm[i].cpu().numpy() if big else gm_h[i], ref[0], f"{accepted[i]} gm")
        if big:
            assert torch.equal(out["gm"][i].view(torch.int32), gm[i].view(torch.int32)), f"resolve {accepted[i]} gm"
        else:
            same_f32(out_gm[i], ref[0], f"resolve {accepted[i]} gm")
        if g.acoustic:
            same_f32(am[i].cpu().numpy(), ref[1], f"{accepted[i]} am")
            same_f32(out["am"][i].cpu().numpy(), ref[1], f"resolve {accepted[i]} am")
        if act_ok[i]:
            j = sel.index(i)
            same_f32(action[j].cpu().numpy(), ref[2], f"{accepted[i]} action_map")
            same_f32(out_act[j].cpu().numpy(), ref[2], f"resolve {accepted[i]} action_map")
    for tok in descs:
        dm.forget(tok)


# --- record order ---
def _valid_pose(g, rng, m):
    while True:
        x, y, o = int(rng.integers(g.internal_size)), int(rng.integers(g.internal_size)), int(rng.choice([0, 90, 180, 270]))
        if m.update_raises(x, y, o) is None:
            return x, y, o


@pytest.mark.parametrize("name", ["n61_s4", "s8_e5", "s1_e2"])
def test_many_records_per_slot_interleaved_in_one_launch(ops, name):
    g = GEOMETRIES[name][0]
    rng = np.random.default_rng(5)
    n_slots, E = 6, g.ego_size
    probe = MapMirror(g)
    per_slot = []
    for s in range(n_slots):
        recs = []
        for t in range(int(rng.integers(150, 300))):
            if t and t % 97 == 0:
                recs.append((0, maps.RESET, 0, 0, 0, 0.0, 0.0, b""))
                continue
            x, y, o = _valid_pose(g, rng, probe)
            ego = rng.random((E, E, 2)) < 0.4
            v = np.float32(rng.random() * 3) if rng.random() > 0.2 else np.float32(0)
            recs.append((0, maps.UPDATE, x, y, o, float(np.float64(v)), float(np.float64(0.5 * v)),
                         np.packbits(ego).tobytes()))
            if t % 40 == 5:
                # the next record's window covers the cell this one cleared: its obstacle bit is set again
                k = turns(o)
                rx, ry = rot_xy(k, g.internal_size, x, y)
                x2, y2 = unrot_xy(k, g.internal_size, rx, ry + 1)
                if probe.update_raises(x2, y2, o) is None:
                    recs.append((0, maps.UPDATE, x2, y2, o, 1.0, 0.5, np.packbits(np.ones((E, E, 2), bool)).tobytes()))
        per_slot.append(recs)
    # a random interleaving that keeps each slot's order
    order, heads = [], [0] * n_slots
    left = [s for s in range(n_slots) for _ in per_slot[s]]
    rng.shuffle(left)
    for s in left:
        order.append((s, per_slot[s][heads[s]]))
        heads[s] += 1
    gm0, am0 = initial_state(name)
    gmap, amap = state(g, n_slots, gm0, am0)
    rec, ego = records(order)
    before = ops.ctx.launch_count
    ops.map_update(cgeo(g, n_slots), gmap, amap, rec, ego)
    assert ops.ctx.launch_count - before == 1
    one_g, one_a = state(g, n_slots, gm0, am0)
    for i in range(len(rec)):                              # one launch per record
        ops.map_update(cgeo(g, n_slots), one_g, one_a, rec[i:i + 1], ego)
    torch.cuda.synchronize()
    assert torch.equal(gmap, one_g) and torch.equal(amap.view(torch.int64), one_a.view(torch.int64))
    for s in range(n_slots):
        m = MapMirror(g)
        m.gm[:], m.am[:] = gm0, am0
        for r in per_slot[s]:
            m.apply(r)
        check_raw(g, gmap, amap, s, m, f"slot {s}")
        pose = per_slot[s][-1][2:5] if per_slot[s][-1][1] == maps.UPDATE else (g.internal_size // 2,) * 2 + (270,)
        gm = torch.empty((1, g.map_size, g.map_size, 2), device=DEV)
        ops.map_observe(cgeo(g, n_slots), gmap, amap, np.array([(s,) + tuple(pose)]), maps.navigable_tables(g), gm)
        same_f32(gm[0].cpu().numpy(), m.observe(pose)[0], f"slot {s} gm")


# --- acoustic values ---
VALUES = [0.0, -0.0, 1e-45, 1.2e-38, 3.4028235e38, -3.4028235e38, np.inf, -np.inf, np.nan, -2.5, 0.75]


@pytest.mark.parametrize("encoding", [0, 1])
def test_acoustic_values_in_both_encodings(ops, encoding):
    """Every ordered pair of special float32 intensities written to one acoustic cell (the second update averages
    with the first under average_intensity), then a third; float64 cells and float32 crops bit for bit, NaN by
    NaN-ness."""
    g = GEOMETRIES["n60_s5"][0]._replace(encoding=encoding)
    vals = [np.float32(v) for v in VALUES]
    ego = np.packbits(np.zeros((g.ego_size, g.ego_size, 2), bool)).tobytes()
    pose = (32, 30, 270)
    order, mirrors = [], []
    for i, a in enumerate(vals):
        for j, b in enumerate(vals):
            m = MapMirror(g)
            for v in (a, b, vals[(i + j) % len(vals)]):
                r = (0, maps.UPDATE) + pose + (float(np.float64(v)), float(np.float64(0.5 * v)), ego)
                m.apply(r)
                order.append((len(mirrors), r))
            mirrors.append(m)
    B = len(mirrors)
    gmap, amap = state(g, B)
    rec, eg = records(order)
    with np.errstate(all="ignore"):
        ops.map_update(cgeo(g, B), gmap, amap, rec, eg)
    am = torch.empty((B, 20, 20, 1), device=DEV)
    ops.map_observe(cgeo(g, B), gmap, amap, np.array([(b,) + pose for b in range(B)]), maps.navigable_tables(g),
                    None, am)
    got_am, got = amap.cpu().numpy(), am.cpu().numpy()
    for b, m in enumerate(mirrors):
        same_am(got_am[b], m.am, f"slot {b}")
        with np.errstate(all="ignore"):
            same_f32(got[b], m.observe(pose)[1], f"slot {b} am crop")


# --- batch sizes ---
@pytest.mark.parametrize("B", [1, 31, 32, 33, 1024])
def test_batch_sizes_in_shuffled_slot_order(ops, B):
    name = "avwan_avg"
    g = GEOMETRIES[name][0]
    gm0, am0 = initial_state(name)
    probe = MapMirror(g)
    pool = [c for c in cases(name) if probe.update_raises(c.x, c.y, c.orientation) is None
            and observe_refusal(g, 1, [(0, c.x, c.y, c.orientation)], table_length(g), kinds=("action_map",)) is None]
    pool = pool[::max(1, len(pool) // 48)]
    refs = {}
    for c in pool:
        m = mirror_case(c, (gm0, am0))[0]
        refs[c.index] = (m, m.observe((c.x, c.y, c.orientation)))
    rng = np.random.default_rng(B)
    envs = [pool[i % len(pool)] for i in range(B)]
    slots = rng.permutation(B)
    gmap, amap = state(g, B, gm0, am0)
    rec, ego = records([(int(slots[i]), case_record(envs[i])) for i in rng.permutation(B)])
    ops.map_update(cgeo(g, B), gmap, amap, rec, ego)
    poses = np.array([(slots[i], envs[i].x, envs[i].y, envs[i].orientation) for i in range(B)], np.int32)
    outs = {"gm": torch.empty((B, g.map_size, g.map_size, 2), device=DEV), "am": torch.empty((B, 20, 20, 1), device=DEV),
            "action_map": torch.empty((B, 9, 9, 1), device=DEV)}
    before = ops.ctx.launch_count
    ops.map_observe(cgeo(g, B), gmap, amap, poses, maps.navigable_tables(g), outs["gm"], outs["am"], outs["action_map"])
    assert ops.ctx.launch_count - before == 1
    host = {k: v.cpu().numpy() for k, v in outs.items()}
    for i in range(B):
        m, ref = refs[envs[i].index]
        for n, k in enumerate(("gm", "am", "action_map")):
            same_f32(host[k][i], ref[n], f"B={B} env {i} {k}")
        if i < 40:
            check_raw(g, gmap, amap, int(slots[i]), m, f"B={B} env {i}")


def test_65535_envs_on_a_tiny_geometry(ops):
    """B = 65535 (the entries' limit and gridDim.y's) on N = 8, S = 2, E = 1; B = 65536 is refused by both."""
    g = maps.MapGeometry(8, 2, 2, 1, 1, 1, 1)
    B = maps.MAX_SLOTS
    rng = np.random.default_rng(65535)
    probe = MapMirror(g)
    combos = []
    for i in range(64):
        x, y, o = _valid_pose(g, rng, probe)
        v = np.float32(rng.random())
        combos.append((0, maps.UPDATE, x, y, o, float(np.float64(v)), float(np.float64(0.5 * v)),
                       np.packbits(rng.random((1, 1, 2)) < 0.5).tobytes()))
    refs = []
    for r in combos:
        m = MapMirror(g)
        m.apply(r)
        refs.append((m, m.observe(r[2:5])))
    gmap, amap = state(g, B)
    rec, ego = records([(b, combos[b % 64]) for b in range(B)])
    ops.map_update(cgeo(g, B), gmap, amap, rec, ego)
    poses = np.array([(b,) + combos[b % 64][2:5] for b in range(B)], np.int32)
    outs = [torch.full((B, 2, 2, 2), -1.0, device=DEV), torch.full((B, 20, 20, 1), -1.0, device=DEV),
            torch.full((B, 1, 1, 1), -1.0, device=DEV)]
    ops.map_observe(cgeo(g, B), gmap, amap, poses, maps.navigable_tables(g), *outs)
    host = [o.cpu().numpy() for o in outs]
    raw_g, raw_a = gmap.cpu().numpy(), amap.cpu().numpy()
    for b in range(B):
        m, ref = refs[b % 64]
        for n in range(3):
            assert np.array_equal(host[n][b], ref[n]), (b, n)
        if b % 1000 == 0 or b == B - 1:
            assert np.array_equal(raw_g[b, :64], encode(m.gm).reshape(-1)) and not raw_g[b, 64:].any()
            assert np.array_equal(raw_a[b].view(np.uint64), m.am.view(np.uint64))
    big = np.array([(b % B,) + combos[0][2:5] for b in range(B + 1)], np.int32)
    expect_refusal(ops, lambda: call_observe(ops, g, B, gmap.data_ptr(), amap.data_ptr(), big, maps.navigable_tables(g),
                                             4, {"gm": (outs[0].data_ptr(), 8)}), (SSB_E_INVALID_ARG, "B=65536"),
                   (gmap, amap))
    expect_refusal(ops, lambda: call_update(ops, g, B + 1, gmap.data_ptr(), amap.data_ptr(), rec[:1], ego),
                   (SSB_E_INVALID_ARG, "bad geometry"), (gmap, amap))


# --- output subsets and strides ---
@pytest.mark.parametrize("subset", [k for k in range(1, 8)])
@pytest.mark.parametrize("pad", [0, 1, 17])
def test_output_subsets_and_strided_rows_with_canaries(ops, subset, pad):
    name = "n60_s5"
    g = GEOMETRIES[name][0]
    kinds = [k for i, k in enumerate(("gm", "am", "action_map")) if subset >> i & 1]
    gm0, am0 = initial_state(name)
    probe = MapMirror(g)
    pool = [c for c in cases(name) if probe.update_raises(c.x, c.y, c.orientation) is None
            and observe_refusal(g, 1, [(0, c.x, c.y, c.orientation)], table_length(g), kinds=("action_map",)) is None]
    envs = pool[::max(1, len(pool) // 5)][:5]
    B = len(envs)
    gmap, amap = state(g, B, gm0, am0)
    rec, ego = records([(i, case_record(c)) for i, c in enumerate(envs)])
    ops.map_update(cgeo(g, B), gmap, amap, rec, ego)
    rows = {"gm": g.map_size ** 2 * 2, "am": 400, "action_map": g.action_size ** 2}
    bases, views = {}, {}
    for k in kinds:
        stride = rows[k] + pad
        bases[k] = torch.full((B * stride + 23,), -1.0, device=DEV)
        views[k] = bases[k][:B * stride].view(B, stride)[:, :rows[k]]
    poses = np.array([(i, c.x, c.y, c.orientation) for i, c in enumerate(envs)], np.int32)
    rc, msg = call_observe(ops, g, B, gmap.data_ptr(), amap.data_ptr(), poses, maps.navigable_tables(g), table_length(g),
                           {k: (views[k].data_ptr(), rows[k] + pad) for k in kinds})
    assert rc == 0, msg
    for k in kinds:
        h = bases[k].cpu().numpy()
        stride = rows[k] + pad
        for i, c in enumerate(envs):
            ref = mirror_case(c, (gm0, am0))[0].observe((c.x, c.y, c.orientation))[("gm", "am", "action_map").index(k)]
            same_f32(h[i * stride:i * stride + rows[k]], ref.reshape(-1), f"{k} env {i}")
            assert (h[i * stride + rows[k]:(i + 1) * stride] == -1).all(), f"{k}: canary between rows {i}"
        assert (h[B * stride:] == -1).all(), f"{k}: canary after the last env"


# --- slot state across steps ---
def test_device_maps_growth_keeps_every_slot_and_reuses_forgotten_ones(ops):
    name = "n61_s4"
    g = GEOMETRIES[name][0]
    dm = maps.DeviceMaps(DEV)
    probe = MapMirror(g)
    pool = [c for c in cases(name) if probe.update_raises(c.x, c.y, c.orientation) is None]
    mirrors, toks = {}, []

    def step(new):
        descs = []
        for j in range(new):
            c = pool[(len(toks) * 7) % len(pool)]
            tok = f"grow/{len(toks)}"
            toks.append(tok)
            ego = np.packbits(np.random.default_rng(len(toks)).random((g.ego_size, g.ego_size, 2)) < 0.5).tobytes()
            recs = [(0, maps.RESET, 0, 0, 0, 0.0, 0.0, b""), (1, maps.UPDATE, c.x, c.y, c.orientation, 1.5, 0.75, ego)]
            maps._RECEIVED[tok] = recs
            m = MapMirror(g)
            for r in recs:
                m.apply(r)
            mirrors[tok] = m
            descs.append(maps.MapDescriptor("gm", tok, (c.x, c.y, c.orientation), 1, g, None))
        dm.resolve({"gm": descs})

    step(16)
    assert dm.capacity == 16
    for want in (32, 64):
        torch.cuda.synchronize()
        snap = {t: (dm.gmap[dm.slots[t]].clone(), dm.amap[dm.slots[t]].clone()) for t in toks}
        step(want - len(toks))
        assert dm.capacity == want
        for t, (sg, sa) in snap.items():
            assert torch.equal(dm.gmap[dm.slots[t]], sg) and torch.equal(dm.amap[dm.slots[t]].view(torch.int64),
                                                                           sa.view(torch.int64)), t
    for t in toks:
        check_raw(g, dm.gmap, dm.amap, dm.slots[t], mirrors[t], t)
    slot = dm.slots[toks[3]]
    dm.forget(toks[3])
    step(1)
    assert dm.slots[toks[-1]] == slot
    check_raw(g, dm.gmap, dm.amap, slot, mirrors[toks[-1]], "reused slot")
    for t in list(dm.slots):
        dm.forget(t)


# --- refusals ---
def _bad_geometries(g):
    return [g._replace(internal_size=0), g._replace(internal_size=4097), g._replace(stride=0),
            g._replace(stride=g.internal_size + 1), g._replace(map_size=0), g._replace(map_size=4098),
            g._replace(map_size=41), g._replace(action_size=0), g._replace(action_size=257), g._replace(action_size=4),
            g._replace(ego_size=0), g._replace(ego_size=g.internal_size + 1), g._replace(ego_size=256),
            g._replace(encoding=2), g._replace(acoustic=2)]


def _window_poses(g):
    """Poses whose update window leaves the top, the left or the right of the rotated view, in each orientation."""
    n, E = g.internal_size, g.ego_size
    c = n // 2
    for o in (0, 90, 180, 270):
        k = turns(o)
        for rx, ry in ((c, E - 1), (E // 2 - 1, c), (n - E + E // 2 + 1, c)):
            yield unrot_xy(k, n, rx, ry) + (o,)


def test_every_refusal_returns_its_code_and_message_and_changes_nothing(ops):
    g = GEOMETRIES["n61_s4"][0]
    n, N_SLOTS = g.internal_size, 4
    gm0, am0 = initial_state("n61_s4")
    gmap, amap = state(g, N_SLOTS, gm0, am0)
    bufs = (gmap, amap)
    probe = MapMirror(g)
    good = next(c for c in cases("n61_s4") if probe.update_raises(c.x, c.y, c.orientation) is None
                and observe_refusal(g, 1, [(0, c.x, c.y, c.orientation)], table_length(g)) is None)
    base = case_record(good)
    tables, L = maps.navigable_tables(g), table_length(g)
    out = {k: torch.empty(s, device=DEV) for k, s in (("gm", 66 * 66 * 2 + 4), ("am", 404), ("action_map", 13))}

    def upd(rec_tuple, geo=g, n_slots=N_SLOTS, gp=0, ap=0, ego_bytes=None):
        rec, ego = records([(rec_tuple[0], (0,) + rec_tuple[1:])])
        if ego_bytes is not None:
            ego = np.zeros(ego_bytes, np.uint8)
        expected = update_refusal(geo, n_slots, rec, ego.size, gp, ap)
        assert expected is not None, rec_tuple
        expect_refusal(ops, lambda: call_update(ops, geo, n_slots, gmap.data_ptr() + gp, amap.data_ptr() + ap, rec,
                                                ego), expected, bufs)
        return expected

    slot_rec = (0,) + base[1:]
    for bg in _bad_geometries(g):
        assert upd(slot_rec, geo=bg)[1] == "bad geometry"
    for ns in (0, 65536):
        assert upd(slot_rec, n_slots=ns)[1] == "bad geometry"
    assert upd(slot_rec, gp=1)[1] == "bad arguments"
    assert upd(slot_rec, ap=4)[1] == "bad arguments"
    for bad in ((-1,) + base[1:], (N_SLOTS,) + base[1:], (0, 2) + base[2:]):
        assert "bad slot" in upd(bad)[1]
    for o in (-90, 45, 360):
        assert "bad orientation" in upd((0, base[1], base[2], base[3], o) + base[5:])[1]
    ego_rec = (g.ego_size ** 2 * 2 + 7) // 8
    assert "ego offset" in upd(slot_rec, ego_bytes=ego_rec - 1)[1]
    for x, y in ((n, 5), (5, -1)):
        assert upd((0, base[1], x, y) + base[4:])[0] == SSB_E_SHAPE
    for x, y, o in _window_poses(g):
        assert "ego window" in upd((0, base[1], x, y, o) + base[5:])[1]
    # an acoustic cell outside the map because N % s != 0: x or y = 60 at N = 61, s = 4 (M = 15)
    probe = MapMirror(g)
    hits = [(x, y, o) for x in (60,) for y in range(n) for o in (0, 90, 180, 270)
            if probe.update_raises(x, y, o) == "acoustic cell"]
    assert hits
    assert "acoustic cell" in upd((0, base[1]) + hits[0] + base[5:])[1]
    # stride 1: the agent on the last row of the rotated view, and the window ending at column N - 1 or N
    g1 = GEOMETRIES["s1_e2"][0]
    g1map, a1map = state(g1, 1)
    for rx, ry in ((16, 32), (31, 16), (32, 16)):
        for o in (0, 90, 180, 270):
            x, y = unrot_xy(turns(o), 33, rx, ry)
            rec, ego = records([(0, (0, maps.UPDATE, x, y, o, 1.0, 0.5, bytes(1)))])
            expected = update_refusal(g1, 1, rec, 1)
            assert "stride 1" in expected[1]
            expect_refusal(ops, lambda: call_update(ops, g1, 1, g1map.data_ptr(), a1map.data_ptr(), rec, ego), expected,
                           (g1map, a1map))

    # the crops
    pose = (0, good.x, good.y, good.orientation)
    rows = {"gm": 66 * 66 * 2, "am": 400, "action_map": 9}

    def obs(poses, kinds=("gm", "am", "action_map"), geo=g, n_slots=N_SLOTS, tabs=tables, LL=L, strides=None, sp=0,
            op=0, expect=None):
        strides = {k: (strides or {}).get(k, rows[k]) for k in kinds}
        expected = observe_refusal(geo, n_slots, poses, LL, tabs, kinds, strides, sp, op)
        assert expected is not None
        if expect:
            assert expect in expected[1], (expected, expect)
        outs = {k: (out[k].data_ptr() + op, strides[k]) for k in kinds}
        expect_refusal(ops, lambda: call_observe(ops, geo, n_slots, gmap.data_ptr() + sp, amap.data_ptr() + sp,
                                                 poses, tabs, LL, outs), expected, bufs + tuple(out.values()))

    for bg in _bad_geometries(g):
        obs([pose], geo=bg, expect="bad geometry")
    obs([pose], n_slots=65536, expect="bad geometry")
    obs([pose], kinds=("gm",), sp=1, expect="bad arguments")
    obs([pose], kinds=("am",), sp=4, expect="bad arguments")
    obs([pose], kinds=("am",), geo=g._replace(acoustic=0), expect="bad arguments")
    for k in rows:
        obs([pose], kinds=(k,), op=2, expect="bad arguments")
        obs([pose], kinds=(k,), strides={k: rows[k] - 1}, expect="bad arguments")
    obs([pose], kinds=("action_map",), LL=0, tabs=tables[:, :, :0], expect="bad arguments")
    for v in (-1, n):
        t = tables.copy()
        t[3, 1, 5] = v
        obs([pose], kinds=("action_map",), tabs=t, expect=f"navigable table entry {3 * 2 * L + L + 5} ")
    obs([pose, (N_SLOTS,) + pose[1:]], expect="env 1: bad slot")
    obs([(-1,) + pose[1:]], expect="bad slot")
    for o in (-90, 45, 360):
        obs([pose[:3] + (o,)], expect=f"orientation {o}")
    obs([(0, n, 3, 0)], expect="outside")
    obs([(0, 3, -1, 0)], expect="outside")
    obs([(0,) + hits[0]], kinds=("am",), expect="acoustic cell")
    h, s = g.action_size // 2, g.stride
    for o in (0, 90, 180, 270):
        k = turns(o)
        for rx, ry in (((h - 1) * s, n // 2), ((L - h) * s, n // 2), (n // 2, (h - 1) * s), (n // 2, (L - h) * s)):
            if 0 <= rx < n and 0 <= ry < n:
                obs([(0,) + unrot_xy(k, n, rx, ry) + (o,)], kinds=("action_map",), expect="occupancy window")
