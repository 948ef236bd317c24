"""Host side of AV-WaN's device maps (soundspaces_b200.maps): the numpy stand-in pinned to the reference recording,
record packing, log draining at pickling time, sequence gaps, structural refusals and CUDA-free workers."""
import multiprocessing as mp
import os
import pickle
import sys
import warnings

import numpy as np
import pytest

from mapper_models import (TRACES, MapMirror, StandInPlanner, digest, drive, geometry, step_inputs, task_config,
                           trace_records)
from soundspaces_b200 import maps

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "mapper_golden.npz")


@pytest.fixture(scope="module")
def golden():
    with np.load(GOLDEN) as z:
        return {k: z[k] for k in z.files}


@pytest.mark.parametrize("name", sorted(TRACES))
def test_stand_in_matches_reference_at_every_step(golden, name):
    config, encoding = TRACES[name][:2]
    mirror = MapMirror(geometry(config, encoding))
    poses, flags, digests = golden[f"{name}/poses"], golden[f"{name}/flags"], golden[f"{name}/digests"]
    full = list(golden[f"{name}/full_steps"])
    for t, recs in enumerate(trace_records(name, poses, flags)):
        for r in recs:
            mirror.apply(r)
        outs = mirror.observe(tuple(int(v) for v in poses[t]))
        for i, kind in enumerate(("gm", "am", "action_map")):
            assert digest(outs[i]) == digests[t, i].tobytes(), f"{name} step {t} {kind}"
        if t in full:
            j = full.index(t)
            np.testing.assert_array_equal(np.packbits(outs[0] > 0.5), golden[f"{name}/gm_bits{j}"])
            np.testing.assert_array_equal(outs[1], golden[f"{name}/am{j}"])
            np.testing.assert_array_equal(outs[2], golden[f"{name}/action_map{j}"])


def test_golden_traces_cover_turns_moves_resets_and_collisions(golden):
    for name in TRACES:
        poses, flags = golden[f"{name}/poses"], golden[f"{name}/flags"]
        assert set(poses[:, 2]) == {0, 90, 180, 270}
        assert len({(x, y) for x, y, _ in poses}) > 3
        assert flags[:, 0].any() and flags[:, 1].any()


def test_record_packing_and_half_dtype_rule():
    g = geometry("avwan", "average_intensity")
    log = maps.MapLog(g)
    ego, _, _, _ = step_inputs(3, 1)

    class M:
        _x, _y, _orientation = 250, 245, 90
    log.update(M, ego, np.float32(0.1))
    seq, kind, x, y, o, value, half, bits = log.pending[-1]
    assert (seq, kind, x, y, o) == (0, maps.UPDATE, 250, 245, 90)
    assert len(bits) == 241                                     # 31 x 31 x 2 bits
    np.testing.assert_array_equal(np.unpackbits(np.frombuffer(bits, np.uint8))[:1922].reshape(31, 31, 2), ego > 0.5)
    assert value == float(np.float32(0.1))
    # NumPy 2 keeps 0.5 * float32 in float32: half is that product widened, not 0.5 * float64(intensity) rounded
    assert isinstance(0.5 * np.float32(0.1), np.float32)
    assert half == float(np.float32(0.5) * np.float32(0.1))
    log.update(M, ego, 0.1)                                     # a Python float stays float64
    assert log.pending[-1][6] == 0.5 * 0.1
    with pytest.raises(ValueError, match="ego maps"):
        log.update(M, np.zeros((31, 30, 2)), 0.0)


def _patched_planner(config="avwan", encoding="average_intensity"):
    class P(StandInPlanner):
        pass
    assert maps.patch_planner(P)
    return P(task_config=task_config(config, encoding), use_acoustic_map=True)


def test_log_drains_at_pickling_time_including_dropped_observations():
    p = _patched_planner()
    steps = list(drive(p, 5, 4))                               # four observations built, none sent
    token = steps[-1]["gm"].token
    kept = pickle.dumps(steps[-1])                              # the fourth is sent: it carries every record so far
    assert p.mapper._b200_map_log.pending == []
    maps._RECEIVED.pop(token, None)
    obs = pickle.loads(kept)
    recs = maps._RECEIVED[token]
    assert [r[0] for r in recs] == list(range(obs["gm"].seq + 1))
    assert recs[0][1] == maps.RESET
    assert maps.contiguous_records(obs["gm"], -1) == recs
    # the other descriptors of the same observation carry nothing more
    assert obs["am"].seq == obs["gm"].seq and obs["action_map"].token == token
    # a terminal observation built and dropped: its records travel with the next pickled one
    dropped = next(drive(p, 5, 1, t0=4))
    p.reset()
    sent = pickle.loads(pickle.dumps(next(drive(p, 5, 1, t0=5))))
    assert sent["gm"].seq > dropped["gm"].seq
    assert [r[0] for r in maps.contiguous_records(sent["gm"], obs["gm"].seq)] == \
        list(range(obs["gm"].seq + 1, sent["gm"].seq + 1))
    maps._RECEIVED.pop(token, None)


def test_in_process_descriptor_reads_and_trims_the_log():
    p = _patched_planner()
    obs = list(drive(p, 6, 3))[-1]
    d = obs["gm"]
    assert d.log is p.mapper._b200_map_log
    recs = maps.contiguous_records(d, -1)
    assert [r[0] for r in recs] == list(range(d.seq + 1))
    d.trim(d.seq)
    assert p.mapper._b200_map_log.pending == []
    assert maps.contiguous_records(d, d.seq) == []


def test_sequence_gap_is_an_error_naming_the_env():
    p = _patched_planner()
    obs = list(drive(p, 7, 3))[-1]
    token = obs["gm"].token
    got = pickle.loads(pickle.dumps(obs))
    del maps._RECEIVED[token][1]
    with pytest.raises(RuntimeError, match=f"env {token}.*record 1 never reached"):
        maps.contiguous_records(got["gm"], -1)
    maps._RECEIVED.pop(token, None)


def _cfg(**over):
    cfg = task_config("avwan", "average_intensity")
    for path, v in over.items():
        obj = cfg.TASK
        parts = path.split("__")
        for q in parts[:-1]:
            obj = getattr(obj, q)
        setattr(obj, parts[-1], v)
    return cfg


@pytest.mark.parametrize("over,why", [
    ({"GEOMETRIC_MAP__MAP_SIZE": 201}, "odd MAP_SIZE"),
    ({"EGOMAP_SENSOR__MAP_SIZE": (31, 29)}, "non-square ego map"),
    ({"ACTION_MAP__MAP_RESOLUTION": 0.55}, "non-integer stride"),
    ({"ACOUSTIC_MAP__ENCODING": "peak"}, "unknown acoustic map encoding"),
    ({"GEOMETRIC_MAP__INTERNAL_MAP_SIZE": 5000}, "past the limits"),
    ({"EGOMAP_SENSOR__MAP_SIZE": 300}, "past the limits"),
    ({"ACTION_MAP__MAP_SIZE": 8}, "even ACTION_MAP.MAP_SIZE"),
])
def test_structural_refusals_keep_the_reference_path(over, why):
    class P(StandInPlanner):
        pass
    assert maps.patch_planner(P)
    cfg = _cfg(**over)
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        try:
            p = P(task_config=cfg, use_acoustic_map=True)
        except ValueError:                     # the stand-in itself raises for an unknown encoding, as the reference
            assert why == "unknown acoustic map encoding"
            return
    assert any(why in str(x.message) for x in w), [str(x.message) for x in w]
    assert not hasattr(p.mapper, "_b200_map_log")
    obs = {"gm": None, "am": None, "action_map": None}
    p.add_maps_to_observation(obs)
    assert all(isinstance(obs[k], np.ndarray) for k in obs)


def test_unknown_encoding_refusal_from_geometry():
    class Mp:
        _action_map_res, _gm_res, _use_acoustic_map, _am_encoding = 0.5, 0.1, True, "peak"

    class Pl:
        mapper = Mp()
    g, why = maps.planner_geometry(Pl(), task_config("avwan", "intensity"))
    assert g is None and "unknown acoustic map encoding" in why


def test_class_without_the_reference_methods_is_left_unpatched():
    class NotAPlanner:
        pass
    with pytest.warns(UserWarning, match="left unpatched"):
        assert not maps.patch_planner(NotAPlanner)
    assert not hasattr(NotAPlanner, "add_maps_to_observation")


def test_patched_planner_without_acoustic_map_refuses_am_as_the_reference():
    class P(StandInPlanner):
        pass
    maps.patch_planner(P)
    p = P(task_config=task_config("avwan", "intensity"), use_acoustic_map=False)
    obs = {"gm": None, "action_map": None}
    p.add_maps_to_observation(obs)
    assert isinstance(obs["gm"], maps.MapDescriptor) and obs["gm"].geometry.acoustic == 0


def test_navigable_tables_restate_compute_navigable_xys():
    for config in ("avwan", "mp3d"):
        g = geometry(config, "intensity")
        t = maps.navigable_tables(g)
        n, s = g.internal_size, g.stride
        assert t.shape == (4, 2, n // s)
        np.testing.assert_array_equal(t[0, 0], np.arange(0, n, s)[: n // s])
        np.testing.assert_array_equal(t[2, 0], np.sort(n - 1 - t[0, 0]))


def _worker(conn, config):
    sys.path[:0] = [os.path.dirname(os.path.abspath(__file__))]
    import torch
    from mapper_models import StandInPlanner as SP, drive as drv, task_config as tc
    from soundspaces_b200 import maps as m

    class P(SP):
        pass
    m.patch_planner(P)
    p = P(task_config=tc(config, "average_intensity"), use_acoustic_map=True)
    payload = [pickle.dumps(o) for o in drv(p, 9, 3)]
    conn.send((payload, torch.cuda.is_initialized()))
    conn.close()


@pytest.mark.parametrize("method", ["fork", "spawn"])
def test_workers_never_touch_cuda(method):
    ctx = mp.get_context(method)
    a, b = ctx.Pipe()
    proc = ctx.Process(target=_worker, args=(b, "avwan"))
    proc.start()
    b.close()
    payload, cuda_used = a.recv()
    proc.join(60)
    assert proc.exitcode == 0 and not cuda_used
    obs = [pickle.loads(x) for x in payload]
    d = obs[-1]["gm"]
    assert maps.contiguous_records(d, -1)[-1][0] == d.seq
    maps._RECEIVED.pop(d.token, None)
