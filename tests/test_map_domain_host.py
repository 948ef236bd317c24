"""AV-WaN's device maps at the edges, on the host: the numpy stand-in (mapper_models.MapMirror) against the reference
``Mapper`` recorded over the edge cases and walks of tests/map_domain_cases.py (tests/golden/map_edges_golden.npz),
the restated refusal rules of both entries against what the reference does, and proof that the case list reaches
every seam of the kernels in every orientation."""
import os

import numpy as np
import pytest

from map_domain_cases import (AM_CROP, GEOMETRIES, SSB_E_SHAPE, WALKS, Case, case_record, cases, d16, initial_state,
                              mirror_case, observe_refusal, rot_xy, table_length, turns, update_refusal, walk_inputs)
from mapper_models import MapMirror
from soundspaces_b200 import maps

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "map_edges_golden.npz")
ZERO = bytes(16)


@pytest.fixture(scope="module")
def golden():
    with np.load(GOLDEN) as z:
        return {k: z[k] for k in z.files}


def _record_array(rec, slot=0):
    seq, kind, x, y, o, value, half, bits = rec
    return np.array([(slot, kind, x, y, o, 0, value, half, 0)], dtype=maps.RECORD_DTYPE)


@pytest.mark.parametrize("name", list(GEOMETRIES))
def test_mirror_matches_reference_at_every_edge_case(golden, name):
    g = GEOMETRIES[name][0]
    np.testing.assert_array_equal(maps.navigable_tables(g), golden[f"{name}/tables"])
    raised, action_ok, digests = golden[f"{name}/raised"], golden[f"{name}/action_ok"], golden[f"{name}/digests"]
    cs = cases(name)
    assert len(cs) == len(raised)
    state = initial_state(name)
    full = {int(i) for i in golden[f"{name}/full_cases"]}
    for c in cs:
        mirror, why = mirror_case(c, state)
        assert (why is not None) == bool(raised[c.index]), (c, why)
        if why:
            continue
        dig = [d16(mirror.gm), d16(mirror.am) if g.acoustic else ZERO]
        gm, am, action = mirror.observe((c.x, c.y, c.orientation))
        ok = observe_refusal(g, 1, [(0, c.x, c.y, c.orientation)], table_length(g), kinds=("action_map",)) is None
        assert ok == bool(action_ok[c.index]), c
        dig += [d16(gm), d16(am) if g.acoustic else ZERO, d16(action) if ok else ZERO]
        for i, kind in enumerate(("internal gm", "internal am", "gm", "am", "action_map")):
            assert dig[i] == digests[c.index, i].tobytes(), (c, kind)
        if c.index in full:
            p = f"{name}/full{c.index}/"
            np.testing.assert_array_equal(np.packbits(mirror.gm), golden[p + "gm_internal"])
            np.testing.assert_array_equal(mirror.am, golden[p + "am_internal"])
            np.testing.assert_array_equal(np.packbits(gm > 0.5), golden[p + "gm"])
            np.testing.assert_array_equal(am, golden[p + "am"])
            np.testing.assert_array_equal(action, golden[p + "action_map"])


def walk_records(name, poses, raised_at):
    """The records the patched planner logs over a recorded walk: a reset, then one update per completed step."""
    recs = [(0, maps.RESET, 0, 0, 0, 0.0, 0.0, b"")]
    acoustic = GEOMETRIES[WALKS[name][0]][0].acoustic
    for t, (x, y, o) in enumerate(poses.tolist()):
        _, ego, intensity = walk_inputs(name, t)
        v = (float(np.float64(intensity)), float(np.float64(0.5 * intensity))) if acoustic else (0.0, 0.0)
        recs.append((t + 1, maps.UPDATE, x, y, o) + v + (np.packbits(ego > 0.5).tobytes(),))
    return recs


@pytest.mark.parametrize("name", list(WALKS))
def test_mirror_matches_reference_walks_to_the_edge(golden, name):
    g = GEOMETRIES[WALKS[name][0]][0]
    poses, raised_at, digests = golden[f"{name}/poses"], int(golden[f"{name}/raised_at"]), golden[f"{name}/digests"]
    assert raised_at == len(poses) - 1 >= 5                # every walk ends at an edge, where the reference raises
    mirror = MapMirror(g)
    recs = walk_records(name, poses, raised_at)
    mirror.apply(recs[0])
    for t, rec in enumerate(recs[1:]):
        if t == raised_at:
            with pytest.raises(ValueError, match="raises"):
                mirror.apply(rec)
            break
        mirror.apply(rec)
        gm, am, action = mirror.observe(rec[2:5])
        ok = action.shape == (g.action_size, g.action_size, 1)
        dig = [d16(mirror.gm), d16(mirror.am) if g.acoustic else ZERO, d16(gm), d16(am) if g.acoustic else ZERO,
               d16(action) if ok else ZERO]
        assert [d.tobytes() for d in digests[t]] == dig, (name, t)


def test_restated_refusals_agree_with_the_reference(golden):
    """Every case the reference completes is accepted by the update restatement, every one it raises on is refused
    with SSB_E_SHAPE; the crop restatement accepts gm and am for every completed case and refuses the action map
    exactly where the reference returns a wrongly shaped occupancy map."""
    for name, (g, _) in GEOMETRIES.items():
        L = table_length(g)
        for c in cases(name):
            rec = _record_array(case_record(c))
            ego_bytes = (g.ego_size ** 2 * 2 + 7) // 8
            refusal = update_refusal(g, 1, rec, ego_bytes)
            assert (refusal is not None) == bool(golden[f"{name}/raised"][c.index]), c
            if refusal:
                assert refusal[0] == SSB_E_SHAPE
                continue
            pose = [(0, c.x, c.y, c.orientation)]
            kinds = ("gm", "am") if g.acoustic else ("gm",)
            assert observe_refusal(g, 1, pose, L, maps.navigable_tables(g), kinds=kinds) is None, c
            act = observe_refusal(g, 1, pose, L, maps.navigable_tables(g), kinds=("action_map",))
            assert (act is None) == bool(golden[f"{name}/action_ok"][c.index]), c
            if act:
                assert act[0] == (SSB_E_SHAPE if L else -1)


def test_stride_one_refusal_is_the_reference_index_error():
    """At s = 1 the reference reads row N when ry = N - 1 and column N when the window ends at column N - 1 or N:
    checked over every pose and orientation of a small map against the mirror's rule and the update restatement."""
    for E in (1, 2, 3, 4):
        g = maps.MapGeometry(9, 1, 2, 1, E, 0, 1)
        m = MapMirror(g)
        for o in (0, 90, 180, 270):
            for x in range(9):
                for y in range(9):
                    rx, ry = rot_xy(turns(o), 9, x, y)
                    right = rx - E // 2 + E
                    window = (ry < E and E > 1) or rx < E // 2 or right > 9
                    why = m.update_raises(x, y, o)
                    expect = "window" if window else "stride 1" if (ry == 8 or right >= 8) else None
                    assert why == expect, (E, o, x, y)
                    rec = np.array([(0, maps.UPDATE, x, y, o, 0, 0.0, 0.0, 0)], dtype=maps.RECORD_DTYPE)
                    r = update_refusal(g, 1, rec, 8)
                    assert (r is None) == (why is None)
                    if why == "stride 1":
                        assert "stride 1" in r[1]


# --- coverage: the seams every orientation of the list reaches ---
_MIRRORS = {}


def _features(c: Case):
    """The seams one case reaches: accepted cases name the crops' zero-fill sides, the clearing boundary, the window
    and grid edges; refused ones name the rule that refuses them."""
    g = GEOMETRIES[c.geometry][0]
    n, s, S, E, a = g.internal_size, g.stride, g.map_size, g.ego_size, g.action_size
    L, M, h = table_length(g), g.acoustic_size, a // 2
    k = turns(c.orientation)
    rx, ry = rot_xy(k, n, c.x, c.y)
    f = set()
    if c.geometry not in _MIRRORS:
        _MIRRORS[c.geometry] = MapMirror(g)
    why = _MIRRORS[c.geometry].update_raises(c.x, c.y, c.orientation)
    if why:
        f.add(f"refuse {why}")
        if why == "window":
            f |= {"refuse window top"} if ry < E else set()
            f |= {"refuse window left"} if rx < E // 2 else set()
            f |= {"refuse window right"} if rx - E // 2 + E > n else set()
        if why == "stride 1":
            f.add("refuse stride 1 row" if ry == n - 1 else "refuse stride 1 column")
        return f
    r0, c0 = ry - S // 2, rx - S // 2
    f |= {"gm fill top"} if r0 < 0 else set()
    f |= {"gm fill bottom"} if r0 + S > n else set()
    f |= {"gm fill left"} if c0 < 0 else set()
    f |= {"gm fill right"} if c0 + S > n else set()
    if r0 < 0 and c0 < 0:
        f.add("gm fill corner")
    if r0 >= 0 and c0 >= 0 and r0 + S <= n and c0 + S <= n:
        f.add("gm inside")
    if S > n:
        f.add("gm crop larger than map")
    if S % 32:
        f.add("partial tile")
    if g.acoustic:
        ax, ay = rot_xy(k, M, c.x // s, c.y // s)
        f |= {"am fill top"} if ay < AM_CROP // 2 else set()
        f |= {"am fill bottom"} if ay + AM_CROP // 2 > M else set()
        f |= {"am fill left"} if ax < AM_CROP // 2 else set()
        f |= {"am fill right"} if ax + AM_CROP // 2 > M else set()
        if min(ax, ay) >= AM_CROP // 2 and max(ax, ay) + AM_CROP // 2 <= M:
            f.add("am inside")
        if n % s and (c.x // s == M - 1 or c.y // s == M - 1):
            f.add("am last cell of N // s")
    if s >= 2:
        f |= {"cleared x at N + 1 - s"} if rx == n + 1 - s else set()
        f |= {"kept x at N + 2 - s"} if rx == n + 2 - s else set()
        f |= {"cleared y at N + 1 - s"} if ry == n + 1 - s else set()
        f |= {"kept y at N + 2 - s"} if ry == n + 2 - s else set()
    else:
        f.add("stride 1 accepted")
    f |= {"window top edge"} if ry == E else set()
    f |= {"window left edge"} if rx == E // 2 else set()
    f |= {"window right edge"} if rx == n - E + E // 2 else set()
    if n * n % 16:
        f.add("pitch padding")
    gx, gy = rx // s, ry // s
    if L:
        f |= {"grid x low edge"} if gx == h else set()
        f |= {"grid x high edge"} if gx == L - 1 - h else set()
        f |= {"grid y low edge"} if gy == h else set()
        f |= {"grid y high edge"} if gy == L - 1 - h else set()
        f |= {"refuse grid x low"} if gx == h - 1 else set()
        f |= {"refuse grid x high"} if gx == L - h else set()
        f |= {"refuse grid y low"} if gy == h - 1 else set()
        f |= {"refuse grid y high"} if gy == L - h else set()
    else:
        f.add("empty tables")
    return f


EVERY_ORIENTATION = {
    "gm fill top", "gm fill bottom", "gm fill left", "gm fill right", "gm fill corner", "gm inside",
    "gm crop larger than map", "partial tile",
    "am fill top", "am fill bottom", "am fill left", "am fill right", "am inside", "am last cell of N // s",
    "cleared x at N + 1 - s", "kept x at N + 2 - s", "cleared y at N + 1 - s", "kept y at N + 2 - s",
    "stride 1 accepted", "refuse stride 1 row", "refuse stride 1 column",
    "window top edge", "window left edge", "window right edge",
    "refuse window top", "refuse window left", "refuse window right", "refuse acoustic cell",
    "pitch padding", "grid x low edge", "grid x high edge", "grid y low edge", "grid y high edge",
    "refuse grid x low", "refuse grid x high", "refuse grid y low", "refuse grid y high", "empty tables",
}


def test_case_list_reaches_every_seam_in_every_orientation():
    for name in GEOMETRIES:
        for o in (0, 90, 180, 270):
            assert any(c.orientation == o for c in cases(name)), (name, o)
    for o in (0, 90, 180, 270):
        have = set().union(*(_features(c) for c in (c for name in GEOMETRIES for c in cases(name))
                             if c.orientation == o))
        assert EVERY_ORIENTATION <= have, (o, sorted(EVERY_ORIENTATION - have))
    # the seams of the default geometries themselves, not only of the small ones (with E = 31 > s the window
    # refuses rx at N + 1 - s and gy at a/2 there)
    for name in ("avwan_avg", "mp3d_avg"):
        for o in (0, 90, 180, 270):
            have = set().union(*(_features(c) for c in cases(name) if c.orientation == o))
            need = {"gm fill top", "gm fill bottom", "gm fill left", "gm fill right", "gm inside", "am fill top",
                    "am fill bottom", "am fill left", "am fill right", "cleared y at N + 1 - s",
                    "kept y at N + 2 - s", "grid x low edge", "grid x high edge", "grid y high edge",
                    "refuse window top", "refuse window left", "refuse window right"}
            assert need <= have, (name, o, sorted(need - have))


def test_geometries_reach_every_limit_and_value_class():
    gs = [g for g, _ in GEOMETRIES.values()]
    assert {g.encoding for g in gs if g.acoustic} == {0, 1} and any(not g.acoustic for g in gs)
    assert any(g.map_size > g.internal_size for g in gs) and any(g.map_size == 2 for g in gs)
    assert {32, 64, 34} <= {g.map_size for g in gs}
    assert any(g.internal_size % 2 for g in gs) and any(g.internal_size % g.stride for g in gs)
    assert any(g.internal_size ** 2 % 16 for g in gs)
    assert {1, 255} <= {g.ego_size for g in gs} and any(g.ego_size % 2 == 0 for g in gs)
    assert {1, 255} <= {g.action_size for g in gs}
    assert any(g.stride == 1 for g in gs) and any(2 * g.stride > g.internal_size for g in gs)
    big = [g for g in gs if g.internal_size == maps.MAX_INTERNAL]
    assert big and big[0].map_size == maps.MAX_INTERNAL and table_length(big[0]) == 256
    assert any(g.acoustic_size < AM_CROP for g in gs)
    assert all(g.refusal() is None for g in gs)
