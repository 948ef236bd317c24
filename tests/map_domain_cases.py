"""The domain of AV-WaN's device-map entries (``ssb_map_update_batch`` / ``ssb_map_observe_batch``): geometries chosen
for the seams they exercise, edge poses in all four orientations, the seeded map state every case starts from, and a
restatement of both entries' host refusal rules.

A case is one update record followed by one crop at the same pose, starting from a densely filled internal map (both
channel bits set at random, so that clearing the agent's cell is observable) and an acoustic map that is partly 0.
``tests/golden/make_map_edges_golden.py`` drives the unmodified reference ``Mapper`` over every case and a few seeded
walks; ``tests/test_map_domain_host.py`` pins ``mapper_models.MapMirror`` to that recording and
``tests/test_gpu_map_domain.py`` compares the device with the mirror bit for bit.
"""
import hashlib
import re
from typing import NamedTuple, Optional, Tuple

import numpy as np

from soundspaces_b200.maps import MAX_INTERNAL, MAX_EGO, MAX_SLOTS, RESET, UPDATE, MapGeometry

SSB_E_INVALID_ARG, SSB_E_SHAPE = -1, -4
AM_CROP = 20

# name: (geometry (N, s, S, a, E, encoding, acoustic), why it is in the list)
GEOMETRIES = {
    "n60_s5": (MapGeometry(60, 5, 40, 5, 7, 1, 1), "M = 12 < 20: every am crop is partly off the map"),
    "n61_s4": (MapGeometry(61, 4, 66, 3, 8, 0, 1), "odd N, padded pitch (3721), N % s != 0, S > N, even E"),
    "avwan_avg": (MapGeometry(500, 5, 200, 9, 31, 1, 1), "the AV-WaN default"),
    "avwan_int": (MapGeometry(500, 5, 200, 9, 31, 0, 1), "the AV-WaN default, intensity encoding"),
    "mp3d_avg": (MapGeometry(1200, 10, 400, 9, 31, 1, 1), "the mp3d geometry"),
    "mp3d_int": (MapGeometry(1200, 10, 400, 9, 31, 0, 1), "the mp3d geometry, intensity encoding"),
    "s32": (MapGeometry(96, 3, 32, 5, 9, 0, 1), "S = 32: one whole tile"),
    "s64": (MapGeometry(96, 3, 64, 5, 9, 1, 1), "S = 64: whole tiles"),
    "s34": (MapGeometry(96, 3, 34, 5, 9, 1, 1), "S = 34: one extra row and column of tiles"),
    "s1_e1": (MapGeometry(33, 1, 2, 1, 1, 1, 1), "the smallest values; the stride-1 edge"),
    "s1_e2": (MapGeometry(33, 1, 2, 1, 2, 0, 1), "stride 1 with an even ego map"),
    "max": (MapGeometry(4096, 16, 4096, 255, 31, 1, 1), "the largest internal map and crop, the largest action map"),
    "ego255": (MapGeometry(600, 5, 200, 9, 255, 0, 1), "the largest ego map"),
    "wide_stride": (MapGeometry(20, 11, 10, 1, 3, 1, 1), "s > N / 2: navigable tables of length 0, M = 1"),
    "no_acoustic": (MapGeometry(80, 4, 50, 7, 11, 0, 0), "no acoustic map"),
    "s8_e5": (MapGeometry(64, 8, 24, 3, 5, 1, 1), "s > E: the window fits at rx = N + 2 - s, where the cell is kept"),
}
SEEDS = {name: 7000 + i for i, name in enumerate(GEOMETRIES)}
LIGHT = {"max"}          # only the corner poses: one crop of this geometry is 128 MB


class Case(NamedTuple):
    geometry: str
    index: int
    x: int
    y: int
    orientation: int


def table_length(g: MapGeometry) -> int:
    n, s = g.internal_size, g.stride
    return len(range(int(-int(n / 2) / s), int((n - int(n / 2)) / s)))


def rot_xy(k, n, x, y):
    """transform_coordinates(x, y, 90 k, n, n)."""
    return ((x, y), (y, n - 1 - x), (n - 1 - x, n - 1 - y), (n - 1 - y, x))[k]


def unrot_xy(k, n, rx, ry):
    """The (x, y) that rot_xy sends to (rx, ry)."""
    return ((rx, ry), (n - 1 - ry, rx), (n - 1 - rx, n - 1 - ry), (ry, n - 1 - rx))[k]


def turns(orientation):
    return (orientation - 270) % 360 // 90


def axis_values(g: MapGeometry):
    """Coordinates of the rotated view at the seams of one axis: the map edges, the ego window's edges (ry = E,
    rx = E/2 and N - E + E/2, and one past each), the gm crop's edges, the clearing boundary N + 1 - s / N + 2 - s,
    the occupancy grid's edges (gx or gy at a/2 and L - 1 - a/2, and one past each) and acoustic cells within 10 of
    each side."""
    n, s, S, a, E = g.internal_size, g.stride, g.map_size, g.action_size, g.ego_size
    L, M, h = table_length(g), g.acoustic_size, g.action_size // 2
    v = {n // 2, 0, 1, n - 2, n - 1, E, E - 1, E // 2, E // 2 - 1, n - E + E // 2, n - E + E // 2 + 1,
         S // 2 - 5, S // 2 - 1, S // 2, S // 2 + 1, n - S // 2 - 1, n - S // 2, n - S // 2 + 1, n - S // 2 + 5,
         n + 1 - s, n + 2 - s, h * s, h * s - 1, (L - 1 - h) * s + s - 1, (L - h) * s,
         3 * s, 10 * s - 1, (M - 10) * s, (M - 3) * s}
    return sorted(x for x in v if 0 <= x < n)


def corner_values(g: MapGeometry):
    """A few values per axis whose products reach every corner class: each edge of the window, the crop crossing
    both sides, the clearing boundary."""
    n, s, S, E = g.internal_size, g.stride, g.map_size, g.ego_size
    v = {E // 2, E, S // 2 - 5, n - S // 2 + 5, n + 1 - s, n + 2 - s, n - E + E // 2, n - 1}
    return sorted(x for x in v if 0 <= x < n)


def light_values(g: MapGeometry):
    n, s, a = g.internal_size, g.stride, g.action_size
    h = a // 2
    return sorted({g.ego_size, h * s, n - 1})


def cases(name: str):
    """The list's cases of one geometry: per orientation, each seam value of one axis with the other at N / 2, and
    every pair of corner values (light geometries: pairs of a few values only).  Poses outside the window are kept:
    they are the refusal cases."""
    g = GEOMETRIES[name][0]
    n = g.internal_size
    out, seen = [], set()
    for o in (0, 90, 180, 270):
        k = turns(o)
        if name in LIGHT:
            vals = light_values(g)
            pairs = [(u, v) for u in vals for v in vals]
        else:
            c = n // 2
            pairs = [(v, c) for v in axis_values(g)] + [(c, v) for v in axis_values(g)]
            pairs += [(u, v) for u in corner_values(g) for v in corner_values(g)]
        for rx, ry in pairs:
            x, y = unrot_xy(k, n, rx, ry)
            if (x, y, o) not in seen:
                seen.add((x, y, o))
                out.append(Case(name, len(out), x, y, o))
    return out


def all_cases():
    return [c for name in GEOMETRIES for c in cases(name)]


def initial_state(name: str):
    """The seeded map state every case of a geometry starts from: gm bits (N, N, 2) bool and the float64 acoustic
    map (M, M), 30 % of it 0."""
    g = GEOMETRIES[name][0]
    rng = np.random.default_rng([SEEDS[name], 0])
    gm = rng.random((g.internal_size, g.internal_size, 2)) < 0.5
    m = g.acoustic_size
    am = np.where(rng.random((m, m)) < 0.3, 0.0, rng.random((m, m)) * 3) if g.acoustic else np.zeros((m, m))
    return gm, am


def case_inputs(case: Case):
    """The ego map (E, E, 2) float64 with values 0, 0.25, 0.5, 0.75, 1 and the float32 intensity of a case."""
    g = GEOMETRIES[case.geometry][0]
    rng = np.random.default_rng([SEEDS[case.geometry], 1, case.index])
    levels = np.array([0.0, 0.25, 0.5, 0.75, 1.0])
    ego = rng.choice(levels, size=(g.ego_size, g.ego_size, 2), p=[0.4, 0.1, 0.1, 0.1, 0.3])
    r = rng.random()
    intensity = np.float32(0.0) if r < 0.1 else np.float32(-0.0) if r < 0.15 else np.float32(rng.random() * 3)
    return ego, intensity


def case_record(case: Case, seq=0):
    """The record the patched planner logs for the case's update (mapper_models / maps.MapLog layout)."""
    g = GEOMETRIES[case.geometry][0]
    ego, intensity = case_inputs(case)
    value, half = (float(np.float64(intensity)), float(np.float64(0.5 * intensity))) if g.acoustic else (0.0, 0.0)
    return (seq, UPDATE, case.x, case.y, case.orientation, value, half, np.packbits(ego > 0.5).tobytes())


def d16(a) -> bytes:
    """The first 16 bytes of SHA-256 of an array's bytes (the edge recording's digests)."""
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).digest()[:16]


def mirror_case(case: Case, state=None):
    """(MapMirror after the case's update, None) from ``initial_state``, or (untouched mirror, why the reference
    raises).  ``state``: ``initial_state(case.geometry)`` when the caller already holds it."""
    from mapper_models import MapMirror
    g = GEOMETRIES[case.geometry][0]
    gm0, am0 = state if state is not None else initial_state(case.geometry)
    mirror = MapMirror(g)
    mirror.gm[:] = gm0
    mirror.am[:] = am0
    why = mirror.update_raises(case.x, case.y, case.orientation)
    if why is None:
        mirror.apply(case_record(case))
    return mirror, why


# --- walks: seeded MOVE_FORWARD / TURN_LEFT / TURN_RIGHT sequences on small maps, run until the reference raises ---
WALKS = {  # name: (geometry, seed, max steps)
    "walk_n60": ("n60_s5", 31, 400),
    "walk_n61": ("n61_s4", 32, 400),
    "walk_n96": ("s34", 33, 400),
    "walk_n80": ("no_acoustic", 34, 400),
}


def walk_inputs(name: str, t: int):
    """Action (1 MOVE_FORWARD, 2 TURN_LEFT, 3 TURN_RIGHT; None at t = 0), ego map and float32 intensity of step t."""
    g = GEOMETRIES[WALKS[name][0]][0]
    rng = np.random.default_rng([WALKS[name][1], t])
    action = None if t == 0 else int(rng.choice([1, 2, 3], p=[0.8, 0.1, 0.1]))
    levels = np.array([0.0, 0.25, 0.5, 0.75, 1.0])
    ego = rng.choice(levels, size=(g.ego_size, g.ego_size, 2), p=[0.6, 0.1, 0.1, 0.05, 0.15])
    intensity = np.float32(0.0) if rng.random() < 0.1 else np.float32(rng.random() * 3)
    return action, ego, intensity


# --- a restatement of both entries' host refusals, in the order the entries check them ---
def _geometry_ok(g: MapGeometry, n_slots: int) -> bool:
    n = g.internal_size
    return (1 <= n <= MAX_INTERNAL and 1 <= g.stride <= n and 2 <= g.map_size <= MAX_INTERNAL and g.map_size % 2 == 0
            and 1 <= g.action_size <= MAX_EGO and g.action_size % 2 == 1 and 1 <= g.ego_size <= min(n, MAX_EGO)
            and g.encoding in (0, 1) and g.acoustic in (0, 1) and 1 <= n_slots <= MAX_SLOTS)


def update_refusal(g: MapGeometry, n_slots: int, records, ego_bytes: int,
                   gmap_align: int = 0, amap_align: int = 0) -> Optional[Tuple[int, str]]:
    """(code, message regex) ``ssb_map_update_batch`` refuses ``records`` (rows of maps.RECORD_DTYPE) with, or None.
    ``gmap_align`` / ``amap_align``: the state pointers' offsets from a 256-byte boundary."""
    if not _geometry_ok(g, n_slots):
        return SSB_E_INVALID_ARG, "bad geometry"
    if ego_bytes < 0 or gmap_align % 16 or (g.acoustic and amap_align % 8):
        return SSB_E_INVALID_ARG, "bad arguments"
    n, s, E, m = g.internal_size, g.stride, g.ego_size, g.acoustic_size
    ego_rec = (E * E * 2 + 7) // 8
    for i, r in enumerate(records):
        slot, kind, x, y, o, off = (int(r[f]) for f in ("slot", "kind", "x", "y", "orientation", "ego_offset"))
        if not 0 <= slot < n_slots or kind not in (RESET, UPDATE):
            return SSB_E_INVALID_ARG, f"record {i}: bad slot {slot} or kind {kind}"
        if kind == RESET:
            continue
        if not (0 <= o < 360 and o % 90 == 0) or off < 0 or off > ego_bytes - ego_rec:
            return SSB_E_INVALID_ARG, f"record {i}: bad orientation {o} or ego offset {off}"
        if not (0 <= x < n and 0 <= y < n):
            return SSB_E_SHAPE, f"record {i}: pose \\({x}, {y}\\) outside"
        rx, ry = rot_xy(turns(o), n, x, y)
        if (ry - E < 0 and E > 1) or rx - E // 2 < 0 or rx - E // 2 + E > n:
            return SSB_E_SHAPE, f"record {i}: the {E} x {E} ego window at \\({rx}, {ry}\\).* leaves"
        if s == 1 and (ry == n - 1 or rx - E // 2 + E >= n - 1):
            return SSB_E_SHAPE, f"record {i}: at stride 1 the reference's loop reads past .* at \\({rx}, {ry}\\)"
        if g.acoustic and (x // s >= m or y // s >= m):
            return SSB_E_SHAPE, f"record {i}: acoustic cell \\({x // s}, {y // s}\\) outside"
    return None


def observe_refusal(g: MapGeometry, n_slots: int, poses, L: int, tables=None, kinds=("gm", "am", "action_map"),
                    strides=None, state_align: int = 0, out_align: int = 0) -> Optional[Tuple[int, str]]:
    """(code, message regex) ``ssb_map_observe_batch`` refuses B envs at ``poses`` ((B, 4) slot, x, y, orientation)
    with, or None.  ``strides``: {kind: stride in floats} (default the row size); ``tables``: (4, 2, L) int32."""
    if not _geometry_ok(g, n_slots):
        return SSB_E_INVALID_ARG, "bad geometry"
    n, s, S, a, m = g.internal_size, g.stride, g.map_size, g.action_size, g.acoustic_size
    rows = {"gm": S * S * 2, "am": AM_CROP * AM_CROP, "action_map": a * a}
    strides = {k: (strides or {}).get(k, rows[k]) for k in kinds}
    B = len(poses)
    need_g = "gm" in kinds or "action_map" in kinds
    if (B > MAX_SLOTS or (need_g and state_align % 16) or ("am" in kinds and (not g.acoustic or state_align % 8))
            or any(out_align % 4 or strides[k] < rows[k] for k in kinds)
            or ("action_map" in kinds and L < 1)):
        return SSB_E_INVALID_ARG, "bad arguments"
    if "action_map" in kinds and tables is not None:
        flat = np.asarray(tables).reshape(-1)
        bad = np.flatnonzero((flat < 0) | (flat >= n))
        if len(bad):
            return SSB_E_INVALID_ARG, f"navigable table entry {bad[0]} is {flat[bad[0]]}, outside"
    for b, (slot, x, y, o) in enumerate(np.asarray(poses).tolist()):
        if not 0 <= slot < n_slots or not (0 <= o < 360 and o % 90 == 0):
            return SSB_E_INVALID_ARG, f"env {b}: bad slot {slot} or orientation {o}"
        if not (0 <= x < n and 0 <= y < n):
            return SSB_E_SHAPE, f"env {b}: pose \\({x}, {y}\\) outside"
        if "am" in kinds and (x // s >= m or y // s >= m):
            return SSB_E_SHAPE, f"env {b}: acoustic cell \\({x // s}, {y // s}\\) outside"
        if "action_map" in kinds:
            rx, ry = rot_xy(turns(o), n, x, y)
            gx, gy = rx // s, ry // s
            if gx - a // 2 < 0 or gy - a // 2 < 0 or gx + a // 2 + 1 > L or gy + a // 2 + 1 > L:
                return SSB_E_SHAPE, f"env {b}: the {a} x {a} occupancy window at grid cell \\({gx}, {gy}\\) leaves"
    return None


def message_matches(pattern: str, message: str) -> bool:
    return re.search(pattern, message) is not None
