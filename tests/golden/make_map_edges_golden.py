"""Generate tests/golden/map_edges_golden.npz by driving the UNMODIFIED reference AV-WaN ``Mapper``
(ss_baselines/av_wan/models/mapper.py of an upstream sound-spaces checkout, path in ``SOUNDSPACES_REFERENCE``; loaded
as tests/golden/make_mapper_golden.py loads it, habitat's actions stubbed) over the edge cases of
``tests/map_domain_cases.py`` and a few seeded walks.

    SOUNDSPACES_REFERENCE=<sound-spaces checkout> python tests/golden/make_map_edges_golden.py

Per geometry ``<g>/``: ``tables`` (the reference's ``_rotated_xs`` / ``_rotated_ys`` after ``compute_navigable_xys()``
at the start pose, int32 (4, 2, L)); per case, in ``cases(g)`` order: ``raised`` (``Mapper.update`` raised),
``action_ok`` (the occupancy map had the (a, a) shape, i.e. its window lies inside the grid) and ``digests``
(n, 5, 16): the first 16 bytes of SHA-256 of the internal geometric map after ``> 0.5``, the float64 acoustic map (M, M),
and the float32 ``gm``, ``am`` and ``action_map`` as ``Planner.add_maps_to_observation`` casts them (zeros where they
do not apply: a raising case, no acoustic map, an occupancy window outside the grid).  For a few cases ``full_cases``
the full outputs are stored too (geometric maps bit-packed).

Every case starts from ``initial_state(g)`` (set into the Mapper's maps), sets ``_x``, ``_y``, ``_orientation`` and
calls ``update(None, ego, intensity)`` with ``case_inputs``.  Per walk ``<w>/``: ``poses`` after each completed step,
``raised_at`` (the step whose update raised, or -1) and ``digests`` (steps, 5, 16) as above; a walk starts from a
reset Mapper and turns and moves with the reference's own pose arithmetic.
"""
import logging
import os
import sys
from types import SimpleNamespace as ns

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_mapper_golden import ROOT, load_planner  # noqa: E402  (puts ROOT and tests/ on sys.path)

from map_domain_cases import (GEOMETRIES, WALKS, case_inputs, cases, initial_state, walk_inputs,  # noqa: E402
                              d16 as digest16)

ENC_NAMES = ("intensity", "average_intensity")
FULL_EVERY = {"n60_s5": 97, "n61_s4": 89, "s1_e1": 53}     # geometry: store the full outputs of every k-th case


def d16(a):
    return np.frombuffer(digest16(a), np.uint8)


def make_mapper(Mapper, g):
    gm = ns(INTERNAL_MAP_SIZE=g.internal_size, MAP_SIZE=g.map_size, MAP_RESOLUTION=1.0)
    am = ns(ENCODING=ENC_NAMES[g.encoding], MAP_SIZE=20, MAP_RESOLUTION=float(g.stride))
    m = Mapper(gm, am, ns(MAP_SIZE=g.action_size, MAP_RESOLUTION=float(g.stride)), bool(g.acoustic))
    assert m._stride == g.stride
    m.compute_navigable_xys()
    return m


def outputs(m, g):
    """(digests (5, 16), action_ok, full outputs) of the mapper's current state and pose."""
    zero = np.zeros(16, np.uint8)
    gm_int = m._geometric_map > 0.5
    am_int = np.ascontiguousarray(m._acoustic_map[..., 0]) if g.acoustic else None
    gm = m.get_egocentric_geometric_map().astype(np.float32)
    am = m.get_egocentric_acoustic_map().astype(np.float32) if g.acoustic else None
    om = m.get_egocentric_occupancy_map(size=g.action_size, action_map_res=float(g.stride))
    action_ok = om.shape == (g.action_size, g.action_size)
    action = np.expand_dims(om, -1).astype(np.float32) if action_ok else None
    dig = np.stack([d16(gm_int), d16(am_int) if g.acoustic else zero, d16(gm), d16(am) if g.acoustic else zero,
                    d16(action) if action_ok else zero])
    return dig, action_ok, (gm_int, am_int, gm, am, action)


def run_cases(Mapper, name):
    g = GEOMETRIES[name][0]
    m = make_mapper(Mapper, g)
    tables = np.array([[m._rotated_xs[90 * k], m._rotated_ys[90 * k]] for k in range(4)], np.int32)
    tables = tables.reshape(4, 2, -1)
    gm0, am0 = initial_state(name)
    raised, action_ok, digests, full = [], [], [], {}
    for c in cases(name):
        m._geometric_map = gm0.astype(np.float64)
        if g.acoustic:
            m._acoustic_map = am0[..., None].copy()
        m._x, m._y, m._orientation = c.x, c.y, c.orientation
        ego, intensity = case_inputs(c)
        try:
            m.update(None, ego, intensity)
        except (IndexError, ValueError):
            raised.append(True)
            action_ok.append(False)
            digests.append(np.zeros((5, 16), np.uint8))
            continue
        dig, ok, outs = outputs(m, g)
        raised.append(False)
        action_ok.append(ok)
        digests.append(dig)
        if name in FULL_EVERY and c.index % FULL_EVERY[name] == 0 and ok:
            full[c.index] = outs
    res = {"tables": tables, "raised": np.array(raised), "action_ok": np.array(action_ok),
           "digests": np.array(digests), "full_cases": np.array(sorted(full), np.int32)}
    for i in sorted(full):
        gm_int, am_int, gm, am, action = full[i]
        res[f"full{i}/gm_internal"] = np.packbits(gm_int)
        res[f"full{i}/am_internal"] = am_int
        res[f"full{i}/gm"] = np.packbits(gm > 0.5)
        res[f"full{i}/am"] = am
        res[f"full{i}/action_map"] = action
    return res


def run_walk(Mapper, name):
    geometry, _, steps = WALKS[name]
    g = GEOMETRIES[geometry][0]
    m = make_mapper(Mapper, g)
    poses, digests, raised_at = [], [], -1
    for t in range(steps):
        action, ego, intensity = walk_inputs(name, t)
        try:
            m.update(action, ego, intensity)
        except (IndexError, ValueError):
            poses.append((m._x, m._y, m._orientation))
            raised_at = t
            break
        poses.append((m._x, m._y, m._orientation))
        digests.append(outputs(m, g)[0])
    return {"poses": np.array(poses, np.int32), "raised_at": np.array(raised_at, np.int32),
            "digests": np.array(digests, np.uint8).reshape(-1, 5, 16)}


def main():
    logging.getLogger().setLevel(logging.ERROR)      # the reference warns at every cleared agent cell
    load_planner()
    Mapper = sys.modules["ss_baselines.av_wan.models.mapper"].Mapper
    out = {}
    for name in GEOMETRIES:
        res = run_cases(Mapper, name)
        out.update({f"{name}/{k}": v for k, v in res.items()})
        print(name, "cases", len(res["raised"]), "raised", int(res["raised"].sum()), "action ok",
              int(res["action_ok"].sum()), "full", list(res["full_cases"]))
    for name in WALKS:
        res = run_walk(Mapper, name)
        out.update({f"{name}/{k}": v for k, v in res.items()})
        p = res["poses"]
        print(name, "steps", len(p), "raised at", int(res["raised_at"]), "x", p[:, 0].min(), p[:, 0].max(),
              "y", p[:, 1].min(), p[:, 1].max())
    path = os.path.join(ROOT, "tests", "golden", "map_edges_golden.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
