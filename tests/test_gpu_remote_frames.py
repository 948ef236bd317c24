"""Remote env workers' RGB-D frames gathered on the device: ``batch_obs`` on the FrameRefs a worker with
``remote_frames`` sends must be ``torch.equal`` (bitwise, where NaN is involved) to the reference ``batch_obs`` --
``torch.stack(...).float()`` -- of the arrays a worker without the flag sends, with one gather launch per step."""
import ctypes as C
import pickle
import uuid

import numpy as np
import pytest
import torch

from oracle.ref_harness import write_rir
from synth import make_rir, make_source

from soundspaces_b200 import _lib
from soundspaces_b200 import frames as fr
from soundspaces_b200.remote import FrameArray, FrameRef
from soundspaces_b200.renderer import WaveformOps
from soundspaces_b200.replay import ProcessReplayVectorEnv, replay_sim, scene_observations, write_scene_observations
from soundspaces_b200.sensors import batch_obs

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
E_INVALID, E_SHAPE = -1, -4


def _sent(a, key):
    """What the trainer receives for a FrameArray a worker pickles (this process plays both sides)."""
    return pickle.loads(pickle.dumps(FrameArray(a, key), protocol=pickle.HIGHEST_PROTOCOL))


def _reference(arrays):
    return torch.stack([torch.from_numpy(np.ascontiguousarray(a)).float() for a in arrays]).to(DEV)


def _bits_equal(a, b):
    return a.shape == b.shape and torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


def _pool(tag, n_scenes, nodes, h, w, seed):
    """{key: (rgb, depth)} as habitat's sensors return them for every pose of ``n_scenes`` seeded scenes."""
    from soundspaces_b200.replay import visual_observations
    out = {}
    for s in range(n_scenes):
        scene = f"/obs/{tag}/scene{s}.pkl"
        for (node, rot), frame in scene_observations(nodes, h, w, seed=seed + s).items():
            v = visual_observations(frame)
            out[(scene, node, rot)] = (v["rgb"], v["depth"])
    return out


@pytest.mark.parametrize("sensors", [("rgb",), ("depth",), ("rgb", "depth")])
def test_batch_obs_equals_reference_across_scenes(sensors):
    tag = uuid.uuid4().hex
    pool = _pool(tag, 3, 6, 32, 24, seed=11)
    keys = list(pool)
    rng = np.random.default_rng(2)
    ops = WaveformOps.get(DEV)
    for step in range(40):
        scene = 0 if step < 15 else (1 if step < 30 else 2)          # every env changes scene together, twice
        pick = [k for k in keys if k[0].endswith(f"scene{scene}.pkl")]
        chosen = [pick[i] for i in rng.integers(0, len(pick), size=16)]
        obs = [{u: _sent(pool[k][0 if u == "rgb" else 1], k + (u,)) for u in sensors} for k in chosen]
        n0 = ops.ctx.launch_count
        b = batch_obs(obs, device=DEV)
        assert ops.ctx.launch_count - n0 == 1                          # every visual sensor in one launch
        for u in sensors:
            assert isinstance(obs[0][u], FrameRef)
            ref = _reference([pool[k][0 if u == "rgb" else 1] for k in chosen])
            assert b[u].dtype == torch.float32 and b[u].is_cuda and torch.equal(b[u], ref)


def test_depth_special_values_are_copied_bit_for_bit():
    tag = uuid.uuid4().hex
    vals = np.array([0.0, -0.0, 1.0, 10.0, 11.5, 1e30, np.inf, -np.inf, np.nan, 1e-42], np.float32)
    frames = []
    for i in range(5):
        d = np.resize(np.roll(vals, i), (16, 16, 1)).astype(np.float32)
        d.view(np.int32)[0, 0, 0] = 0x7fc00123                        # a NaN with a payload
        frames.append(d)
    obs = [{"depth": _sent(d, (f"/obs/{tag}.pkl", i, 0, "depth"))} for i, d in enumerate(frames)]
    for _ in range(2):                                                # upload step, then a step served from the bank
        b = batch_obs(obs, device=DEV)
        assert _bits_equal(b["depth"], _reference(frames))
        obs = [{"depth": FrameRef(o["depth"].key, np.float32, (16, 16, 1))} for o in obs]


def test_a_small_bank_evicts_and_uploads_again():
    tag = uuid.uuid4().hex
    shape = (12, 10, 3)
    store = fr.FrameStore.get(DEV, "rgb", np.uint8, shape, max_bank_bytes=6 * 360)
    rng = np.random.default_rng(4)
    pool = {(f"/obs/{tag}.pkl", n, 0, "rgb"): rng.integers(0, 256, size=shape, dtype=np.uint8) for n in range(20)}
    keys = list(pool)
    for step in range(60):
        chosen = [keys[i] for i in rng.integers(0, 20, size=4)]
        obs = [{"rgb": _sent(pool[k], k)} for k in chosen]
        b = batch_obs(obs, device=DEV)
        assert torch.equal(b["rgb"], _reference([pool[k] for k in chosen]))
    assert store.capacity == 6 and store.stats["evictions"] > 20 and store.stats["hits"] > 0


def test_out_slots_with_strided_rows_and_non_contiguous_slots():
    tag = uuid.uuid4().hex
    pool = _pool(tag, 1, 4, 8, 8, seed=5)
    chosen = list(pool)[:10]
    obs = [{"rgb": _sent(pool[k][0], k + ("rgb",)), "depth": _sent(pool[k][1], k + ("depth",))} for k in chosen]
    big = torch.full((10, 8 * 8 * 3 + 20), -7.0, device=DEV)
    rgb_slot = big[:, : 8 * 8 * 3].view(10, 8, 8, 3)                 # rows 212 floats apart
    depth_store = torch.full((3, 10, 8, 8, 2), -7.0, device=DEV)
    depth_slot = depth_store[1][..., :1]                              # not contiguous within a row: copied in
    b = batch_obs(obs, device=DEV, out={"rgb": rgb_slot, "depth": depth_slot})
    assert b["rgb"].data_ptr() == rgb_slot.data_ptr() and torch.equal(rgb_slot, _reference([pool[k][0] for k in chosen]))
    assert bool((big[:, 8 * 8 * 3:] == -7.0).all())
    assert torch.equal(depth_slot, _reference([pool[k][1] for k in chosen]))
    assert bool((depth_store[1][..., 1:] == -7.0).all()) and bool((depth_store[0] == -7.0).all())


def test_mixed_values_take_the_plain_path_with_the_same_result():
    tag = uuid.uuid4().hex
    pool = _pool(tag, 1, 3, 8, 8, seed=6)
    chosen = list(pool)[:6]
    obs = [{"rgb": _sent(pool[k][0], k + ("rgb",)) if i % 2 else pool[k][0]} for i, k in enumerate(chosen)]
    assert torch.equal(batch_obs(obs, device=DEV)["rgb"], _reference([pool[k][0] for k in chosen]))


def test_one_env_and_no_envs():
    tag = uuid.uuid4().hex
    a = np.random.default_rng(8).integers(0, 256, size=(5, 7, 3), dtype=np.uint8)  # rows too short for 16-byte units
    b = batch_obs([{"rgb": _sent(a, (f"/obs/{tag}.pkl", 0, 0, "rgb"))}], device=DEV)
    assert torch.equal(b["rgb"], _reference([a]))
    assert batch_obs([], device=DEV) == {}
    ops = WaveformOps.get(DEV)
    bank = torch.zeros((2, 4), dtype=torch.uint8, device=DEV)
    n0 = ops.ctx.launch_count
    ops.frame_gather(0, [(bank, None, torch.empty((0, 4), device=DEV), [], [])])
    assert ops.ctx.launch_count == n0


def test_frame_steps_do_not_synchronise():
    tag = uuid.uuid4().hex
    pool = _pool(tag, 1, 4, 16, 16, seed=9)
    keys = list(pool)
    rng = np.random.default_rng(1)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for step in range(20):
            chosen = [keys[i] for i in rng.integers(0, len(keys), size=8)]
            obs = [{"rgb": _sent(pool[k][0], k + ("rgb",)), "depth": _sent(pool[k][1], k + ("depth",))}
                   for k in chosen]
            b = batch_obs(obs, device=DEV)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert torch.equal(b["rgb"], _reference([pool[k][0] for k in chosen]))


def test_gather_entry_refuses_bad_arguments():
    ops = WaveformOps.get(DEV)
    lib, h = ops.lib, ops.ctx.handle
    stream = C.c_void_p(torch.cuda.current_stream(DEV).cuda_stream)
    bank = torch.zeros((4, 64), dtype=torch.float32, device=DEV)
    stage = torch.zeros((2, 64), dtype=torch.float32, device=DEV)
    dst = torch.zeros((3, 64), dtype=torch.float32, device=DEV)
    idx = (C.c_int32 * 3)(0, 1, -1)
    fill = (C.c_int32 * 2)(2, 3)

    def sensor(**kw):
        f = dict(d_bank=bank.data_ptr(), d_stage=stage.data_ptr(), d_dst=dst.data_ptr(), h_index=C.addressof(idx),
                 h_fill=C.addressof(fill), row_elems=64, bank_rows=4, dst_stride=64, n_fill=2, dtype=1)
        f.update(kw)
        return (_lib.FrameSensor * 1)(_lib.FrameSensor(**f))

    def call(n_sensors=1, N=3, **kw):
        return lib.ssb_frame_gather_batch(h, n_sensors, sensor(**kw), N, stream)

    n0 = ops.ctx.launch_count
    assert call(n_sensors=0) == E_INVALID
    assert call(n_sensors=5) == E_INVALID
    assert lib.ssb_frame_gather_batch(h, 1, None, 3, stream) == E_INVALID
    assert call(N=-1) == E_INVALID
    assert call(N=257) == E_SHAPE
    assert call(dtype=2) == E_INVALID                                   # unsupported dtype
    assert call(row_elems=0) == E_INVALID
    assert call(bank_rows=0) == E_INVALID
    assert call(dst_stride=63) == E_INVALID                            # rows would overlap
    assert call(n_fill=4) == E_INVALID                                 # more staged rows than envs
    assert call(bank_rows=1 << 45) == E_SHAPE
    assert call(d_bank=None) == E_INVALID
    assert call(d_dst=None) == E_INVALID
    assert call(h_index=None) == E_INVALID
    assert call(d_stage=None) == E_INVALID
    assert call(h_fill=None) == E_INVALID
    assert call(d_dst=dst.data_ptr() + 2) == E_INVALID                  # misaligned float32
    assert call(d_bank=bank.data_ptr() + 2) == E_INVALID
    assert call(d_stage=stage.data_ptr() + 2) == E_INVALID
    bad = (C.c_int32 * 3)(0, 4, -1)                                     # past the bank
    assert call(h_index=C.addressof(bad)) == E_INVALID
    bad = (C.c_int32 * 3)(0, 1, -3)                                     # past the staged rows
    assert call(h_index=C.addressof(bad)) == E_INVALID
    bad = (C.c_int32 * 3)(0, 2, -1)                                     # reads a row the call fills
    assert call(h_index=C.addressof(bad)) == E_INVALID
    badf = (C.c_int32 * 2)(2, 4)                                        # fill past the bank
    assert call(h_fill=C.addressof(badf)) == E_INVALID
    badf = (C.c_int32 * 2)(3, 3)                                        # one row filled twice
    assert call(h_fill=C.addressof(badf)) == E_INVALID
    assert call(d_dst=bank.data_ptr() + 4 * 64) == E_INVALID            # destination inside the bank
    assert call(d_stage=bank.data_ptr()) == E_INVALID                   # staged rows inside the bank it fills
    two = (_lib.FrameSensor * 2)(sensor()[0], sensor()[0])
    assert lib.ssb_frame_gather_batch(h, 2, two, 3, stream) == E_INVALID   # two sensors, one destination
    assert ops.ctx.launch_count == n0                                   # all decided before any launch
    assert call() == 0 and ops.ctx.launch_count == n0 + 1
    torch.cuda.synchronize()


@pytest.mark.parametrize("episode_steps", [25])
def test_process_workers_match_workers_without_the_flag(tmp_path, episode_steps):
    """Worker processes with and without ``remote_frames`` on the same actions, auto-reset included: the trainer's
    visual batches are equal, in the same ``batch_obs`` call as the audio descriptors."""
    sr, side, n_envs, steps = 16000, 3, 8, 200
    root = str(tmp_path)
    for ai, az in enumerate((0, 90, 180, 270)):
        for n in range(side * side):
            write_rir(root, "replica", "scene", az, n, 0, sr, make_rir(50 * ai + n, 1500 + 100 * n))
    path = write_scene_observations(str(tmp_path / "obs" / "replica" / "scene.pkl"),
                                    scene_observations(side * side, 32, 32, seed=12))
    clip = make_source(0, sr)
    base = [(sr, "scene", side, root, "c.wav", clip, 0, e % (side * side), 90 * (e % 4), "remote", 10 ** 6, path)
            for e in range(n_envs)]
    actions = np.random.default_rng(7).choice([1, 1, 2, 3], size=(steps, n_envs))
    ops = WaveformOps.get(DEV)
    with ProcessReplayVectorEnv(replay_sim, [a + (True,) for a in base], episode_steps=episode_steps) as on, \
            ProcessReplayVectorEnv(replay_sim, [a + (False,) for a in base], episode_steps=episode_steps) as off:
        obs_on, obs_off = on.observe(), off.observe()
        sizes = []
        for step in range(steps + 1):
            assert isinstance(obs_on[0]["rgb"], FrameRef) and type(obs_off[0]["rgb"]) is np.ndarray
            b_on = batch_obs(obs_on, device=DEV)
            n0 = ops.ctx.launch_count
            frames_only = batch_obs([{k: o[k] for k in ("rgb", "depth")} for o in obs_on], device=DEV)
            assert ops.ctx.launch_count - n0 == 1
            b_off = batch_obs(obs_off, device=DEV)
            for u in ("rgb", "depth", "spectrogram"):
                assert torch.equal(b_on[u], b_off[u]), (step, u)
            for u in ("rgb", "depth"):
                assert torch.equal(frames_only[u], b_off[u])
            if step < steps:
                b0, c0 = on.bytes_received, off.bytes_received
                obs_on, obs_off = on.step(actions[step]), off.step(actions[step])
                sizes.append((on.bytes_received - b0, off.bytes_received - c0))
    steady = np.array(sizes[-50:], dtype=np.float64).sum(axis=0)
    assert steady[0] < 0.25 * steady[1], steady                        # keys instead of 7 KiB of frames per env
