"""AV-WaN's maps on the device (ssb_map_update_batch / ssb_map_observe_batch through soundspaces_b200.maps) against
the numpy stand-in and the reference recording, bit for bit."""
import copy
import os
import pickle

import numpy as np
import pytest
import torch

from mapper_models import (TRACES, MapMirror, StandInPlanner, digest, drive, geometry, task_config, trace_records)
from soundspaces_b200 import maps
from soundspaces_b200.sensors import batch_obs

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "mapper_golden.npz")
KINDS = ("gm", "am", "action_map")


def _desc(kind, token, pose, seq, g, log):
    return maps.MapDescriptor(kind, token, tuple(pose), seq, g, log)


def _logs(name, golden):
    """The trace's geometry, an empty MapLog and, per step, the records the patched planner logs and the pose."""
    config, encoding = TRACES[name][:2]
    g = geometry(config, encoding)
    log = maps.MapLog(g)
    steps = []
    for t, recs in enumerate(trace_records(name, golden[f"{name}/poses"], golden[f"{name}/flags"])):
        steps.append((list(recs), tuple(int(v) for v in golden[f"{name}/poses"][t])))
    return g, log, steps


@pytest.fixture(scope="module")
def golden():
    with np.load(GOLDEN) as z:
        return {k: z[k] for k in z.files}


@pytest.mark.parametrize("name", sorted(TRACES))
def test_every_step_matches_golden_and_stand_in(golden, name):
    g, log, steps = _logs(name, golden)
    dm = maps.DeviceMaps(torch.device("cuda", 0))
    mirror = MapMirror(g)
    digests = golden[f"{name}/digests"]
    for t, (recs, pose) in enumerate(steps):
        log.pending.extend(recs)
        log.seq = recs[-1][0] if recs else log.seq
        for r in recs:
            mirror.apply(r)
        out = dm.resolve({k: [_desc(k, log.token, pose, log.seq, g, log)] for k in KINDS})
        ref = mirror.observe(pose)
        for i, k in enumerate(KINDS):
            got = out[k][0].cpu().numpy()
            assert digest(got) == digests[t, i].tobytes(), f"{name} step {t} {k}"
            assert np.array_equal(got.view(np.uint32), ref[i].view(np.uint32))


def _random_envs(n, seed, config="mp3d", steps=6):
    """n stand-in-driven logs: (geometry, [(log, pose, mirror)])."""
    g = geometry(config, "average_intensity")
    out = []
    for e in range(n):
        p = StandInPlanner(task_config=task_config(config, "average_intensity"), use_acoustic_map=True)
        maps._attach(p.mapper, g)
        for _ in drive(p, seed + e, steps):
            pass
        m = p.mapper
        out.append((m._b200_map_log, (m._x, m._y, m._orientation), m.mirror))
    return g, out


@pytest.mark.parametrize("B", [1, 7, 64, 1024])
def test_bit_identical_across_batch_sizes_and_slot_order(B):
    g, envs = _random_envs(min(B, 64), 100)
    envs = [envs[i % len(envs)] for i in range(B)]
    refs = [m.observe(pose) for _, pose, m in envs]
    dm = maps.DeviceMaps(torch.device("cuda", 0))
    order = np.random.default_rng(B).permutation(B)
    descs = {k: [] for k in KINDS}
    for i in order:
        log, pose, _ = envs[i]
        tok = f"{log.token}/{i}"                       # copies of one env under several tokens, own slots each
        for k in KINDS:
            d = _desc(k, tok, pose, log.seq, g, None)
            descs[k].append(d)
        maps._RECEIVED[tok] = list(log.pending)
    out = dm.resolve(descs)
    for j, i in enumerate(order):
        for n, k in enumerate(KINDS):
            assert np.array_equal(out[k][j].cpu().numpy(), refs[i][n]), (B, j, k)
    for tok in list(dm.slots):
        dm.forget(tok)


def test_outputs_land_in_strided_rollout_slots_and_two_launches_per_step():
    g, envs = _random_envs(5, 200)
    dm = maps.DeviceMaps(torch.device("cuda", 0))
    S = g.map_size
    store = {"gm": torch.full((3, 5, S, S, 2), -1.0, device="cuda"), "am": torch.full((3, 5, 20, 20, 1), -1.0, device="cuda"),
             "action_map": torch.full((3, 5, 9, 9, 1), -1.0, device="cuda")}
    obs = [{k: _desc(k, log.token, pose, log.seq, g, log) for k in KINDS} for log, pose, _ in envs]
    before = dm.ops.ctx.launch_count
    batch = batch_obs(obs, device=torch.device("cuda", 0), out={k: v[1] for k, v in store.items()})
    assert dm.ops.ctx.launch_count - before == 2
    for k in KINDS:
        assert batch[k].data_ptr() == store[k][1].data_ptr()
        assert (store[k][0] == -1).all() and (store[k][2] == -1).all()
    for j, (_, pose, m) in enumerate(envs):
        for n, k in enumerate(KINDS):
            assert np.array_equal(store[k][1, j].cpu().numpy(), m.observe(pose)[n])
    # a step without records launches the crops only
    before = dm.ops.ctx.launch_count
    batch_obs(obs, out={k: v[2] for k, v in store.items()})
    assert dm.ops.ctx.launch_count - before == 1
    assert torch.equal(store["gm"][1], store["gm"][2])


def test_reset_and_slot_reuse_after_forget():
    g, envs = _random_envs(2, 300)
    dm = maps.DeviceMaps(torch.device("cuda", 0))
    (log0, pose0, m0), (log1, pose1, m1) = envs
    dm.resolve({"gm": [_desc("gm", log0.token, pose0, log0.seq, g, log0)]})
    slot = dm.slots[log0.token]
    dm.forget(log0.token)
    out = dm.resolve({"gm": [_desc("gm", log1.token, pose1, log1.seq, g, log1)]})
    assert dm.slots[log1.token] == slot                 # reused: its first record (a reset) clears env 0's maps
    assert np.array_equal(out["gm"][0].cpu().numpy(), m1.observe(pose1)[0])
    log1.reset()
    centre = (g.internal_size // 2, g.internal_size // 2, 270)
    out = dm.resolve({k: [_desc(k, log1.token, centre, log1.seq, g, log1)] for k in KINDS})
    assert not out["gm"].any() and not out["am"].any() and out["action_map"].all()


def test_refusals_launch_nothing_and_gaps_name_the_env():
    g, envs = _random_envs(1, 400)
    log, pose, _ = envs[0]
    dm = maps.DeviceMaps(torch.device("cuda", 0))
    before = dm.ops.ctx.launch_count
    bad = list(log.pending)
    bad[-1] = (bad[-1][0], maps.UPDATE, 5, bad[-1][3], 270) + bad[-1][5:]        # the ego window leaves the map
    tok = "refused-window"
    maps._RECEIVED[tok] = bad
    with pytest.raises(RuntimeError, match="leaves"):
        dm.resolve({"gm": [_desc("gm", tok, pose, log.seq, g, None)]})
    gap = [r for r in log.pending if r[0] != 1]
    maps._RECEIVED["gap"] = gap
    with pytest.raises(RuntimeError, match="env gap"):
        dm.resolve({"gm": [_desc("gm", "gap", pose, log.seq, g, None)]})
    near = (g.internal_size - 3, pose[1], 0)                           # occupancy window leaves the grid
    dm.forget(tok)
    maps._RECEIVED[tok] = [log.pending[0]]
    with pytest.raises(RuntimeError, match="occupancy window"):
        dm.resolve({"action_map": [_desc("action_map", tok, near, 0, g, None)]})
    torch.cuda.synchronize()
    assert dm.ops.ctx.launch_count - before == 1                      # only the last call's (valid) update ran
    for t in list(dm.slots):
        dm.forget(t)


def _worker_obs(conn, seed, steps):
    import sys
    sys.path[:0] = [os.path.dirname(os.path.abspath(__file__))]
    from mapper_models import StandInPlanner as SP, drive as drv, task_config as tc
    from soundspaces_b200 import maps as m

    class P(SP):
        pass
    m.patch_planner(P)
    p, ref = P(task_config=tc("avwan", "average_intensity"), use_acoustic_map=True), \
        SP(task_config=tc("avwan", "average_intensity"), use_acoustic_map=True)
    for a, b in zip(drv(p, seed, steps), drv(ref, seed, steps)):
        conn.send((pickle.dumps(a), {k: b[k] for k in KINDS}))
    conn.close()


def test_end_to_end_workers_batch_obs_and_map_cnn():
    import multiprocessing as mp
    ctx = mp.get_context("spawn")
    pipes, procs = [], []
    for e in range(4):
        a, b = ctx.Pipe()
        pr = ctx.Process(target=_worker_obs, args=(b, 500 + e, 30), daemon=True)
        pr.start()
        b.close()                                     # a worker that dies then ends recv() with EOFError
        pipes.append(a)
        procs.append(pr)
    try:
        _end_to_end(pipes)
    finally:
        for pr in procs:
            pr.terminate()
            pr.join(10)


def _end_to_end(pipes):
    from map_cnn_models import MapCNN
    from soundspaces_b200.encoder import patch_map_cnn
    torch.manual_seed(0)

    class PatchedMapCNN(MapCNN):
        pass
    net = PatchedMapCNN(200, 200, 2, 32, "gm").cuda().eval()
    ref_net = copy.deepcopy(net).double()                 # the MapCNN tests' yardstick: float64 of the same module
    patch_map_cnn(PatchedMapCNN)
    for _ in range(30):
        got = [pipe.recv() for pipe in pipes]
        obs = [pickle.loads(o) for o, _ in got]
        batch = batch_obs(obs, device=torch.device("cuda", 0))
        ref = {k: np.stack([r[k] for _, r in got]) for k in KINDS}
        for k in KINDS:
            assert np.array_equal(batch[k].cpu().numpy(), ref[k]), k
        with torch.no_grad():
            f = net(batch)
            f_ref = PatchedMapCNN.forward._ssb_original(ref_net, {"gm": torch.from_numpy(ref["gm"]).cuda().double()})
        for b in range(f.shape[0]):
            scale = f_ref[b].abs().max().item()
            assert (f[b].double() - f_ref[b]).abs().max().item() <= 1e-4 * scale
