"""Remote env workers' RGB-D frames (``patch_simulator(..., deferred="remote", remote_frames=True)``): the worker side
(FrameArray, pickling once per key, where the substitution happens) and the trainer's host half of the frame store
(LRU order, re-upload on a miss, unknown keys), all without CUDA."""
import pickle
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from synth import make_source

from soundspaces_b200 import frames as fr
from soundspaces_b200 import remote
from soundspaces_b200.remote import FrameArray, FrameRef, frame_data
from soundspaces_b200.replay import (MOVE_FORWARD, TURN_LEFT, FrameReplaySim, ProcessReplayVectorEnv, ReplayScene,
                                     replay_sim, scene_observations, visual_observations, write_scene_observations)
from soundspaces_b200.simulator import frame_observations, patch_simulator

SR = 16000


def _asnumpy(v):
    # EgoMap's conversion (soundspaces/tasks/nav.py:395-415): anything but an ndarray or a tensor is refused
    if torch.is_tensor(v):
        return v.cpu().numpy()
    if isinstance(v, np.ndarray):
        return v
    raise ValueError("Invalid input")


def _key(tag):
    return (f"/obs/{tag}.pkl", 3, 90, "rgb")


def test_frame_array_is_the_array_it_wraps():
    a = np.random.default_rng(0).integers(0, 256, size=(8, 8, 3), dtype=np.uint8)
    f = FrameArray(a, _key("same"))
    assert isinstance(f, np.ndarray) and f.frame_key == _key("same")
    assert np.array_equal(f, a) and f.dtype == a.dtype and f.shape == a.shape
    assert _asnumpy(f) is f and np.array_equal(_asnumpy(f), a)
    # views and results of operations are not the keyed frame: they carry no key and pickle as plain arrays
    for derived in (f[:, :, :2], f * 2, f.copy(), f.astype(np.float32)):
        assert getattr(derived, "frame_key", None) is None
        assert type(pickle.loads(pickle.dumps(derived))) is np.ndarray


def test_first_pickle_carries_the_data_later_ones_only_the_key():
    a = np.random.default_rng(1).random((64, 64, 1), dtype=np.float32)
    key = _key("first")
    first = pickle.dumps(FrameArray(a, key), protocol=pickle.HIGHEST_PROTOCOL)
    later = [pickle.dumps(FrameArray(a, key), protocol=pickle.HIGHEST_PROTOCOL) for _ in range(3)]
    assert len(first) > a.nbytes
    assert all(len(p) < 300 for p in later), [len(p) for p in later]      # 16 KiB frame, a key of a few dozen bytes
    ref = pickle.loads(first)
    assert isinstance(ref, FrameRef) and ref.key == key and ref.dtype == np.float32 and ref.shape == a.shape
    assert np.array_equal(np.asarray(ref), a)
    for p in later:
        r = pickle.loads(p)
        assert r.data is None and np.array_equal(np.asarray(r), a)      # from this process's frame dict


def test_an_observation_built_and_dropped_does_not_count_as_shipped():
    a = np.arange(48, dtype=np.uint8).reshape(4, 4, 3)
    key = _key("dropped")
    FrameArray(a, key)                              # the terminal step's observation under auto_reset_done: never sent
    ref = pickle.loads(pickle.dumps(FrameArray(a, key)))
    assert ref.data is not None and np.array_equal(ref.data, a)


def test_unknown_frame_raises_naming_the_key():
    ref = FrameRef(_key("never-sent"), np.uint8, (4, 4, 3))
    with pytest.raises(RuntimeError, match="never-sent"):
        frame_data(ref)
    with pytest.raises(RuntimeError, match="never-sent"):
        np.asarray(ref)
    with pytest.raises(RuntimeError, match="never-sent"):          # checked before the store is touched
        fr.gather({"rgb": [ref]}, "cpu")


class _RefSim:
    """The slice of ``SoundSpacesSim`` the frame wrapper reads, with the reference's reset / step shape: the frame comes
    from ``_frame_cache`` (or from habitat-sim without rendered observations), the sensors process it."""

    def __init__(self, rendered=True, cache=None):
        self.config = SimpleNamespace(USE_RENDERED_OBSERVATIONS=rendered)
        self._frame_cache = scene_observations(4, 8, 8, seed=3) if cache is None else cache
        self._receiver_position_index, self._rotation_angle = 0, 0
        self._prev_sim_obs = None
        self.current_scene_observation_file = "/obs/replica/room.pkl"

    def _get_sim_observation(self):
        frame = self._frame_cache.get((self._receiver_position_index, self._rotation_angle))
        if frame is None:                      # habitat-sim's render: not from the cache
            return {"rgb": np.zeros((8, 8, 4), np.uint8), "depth": np.zeros((8, 8), np.float32)}
        return frame

    def reset(self):
        self._prev_sim_obs = self._get_sim_observation()
        return {**visual_observations(self._prev_sim_obs), "pointgoal": np.zeros(2, np.float32)}

    def step(self, action):
        self._rotation_angle = (self._rotation_angle + 90) % 360
        self._prev_sim_obs = self._get_sim_observation()
        return {**visual_observations(self._prev_sim_obs), "pointgoal": np.zeros(2, np.float32)}


def test_patch_wraps_reset_and_step_and_keys_the_cached_frames():
    class Sim(_RefSim):
        pass
    original = Sim.step
    patch_simulator(Sim, deferred="remote", remote_frames=True)
    patch_simulator(Sim, deferred="remote", remote_frames=True)          # patching twice wraps once
    assert Sim.step.__wrapped__ is original
    sim = Sim()
    obs = sim.reset()
    plain = visual_observations(sim._frame_cache[(0, 0)])
    for uuid in ("rgb", "depth"):
        assert type(obs[uuid]) is FrameArray and np.array_equal(obs[uuid], plain[uuid])
        assert obs[uuid].frame_key == ("/obs/replica/room.pkl", 0, 0, uuid)
    assert type(obs["pointgoal"]) is np.ndarray                          # not a sim sensor of the frame
    obs = sim.step(TURN_LEFT)
    assert obs["depth"].frame_key == ("/obs/replica/room.pkl", 0, 90, "depth")
    patch_simulator(Sim, deferred="remote")                              # off again: the reference's own methods
    assert Sim.step is original and type(Sim().reset()["rgb"]) is np.ndarray


def test_flag_needs_remote_mode_and_leaves_other_sims_plain():
    for deferred in (False, True):
        with pytest.raises(ValueError, match="remote_frames"):
            patch_simulator(type("S", (_RefSim,), {}), deferred=deferred, remote_frames=True)
    with pytest.raises(ValueError, match="remote_frames"):
        replay_sim(SR, "s", 2, "/r", "c.wav", make_source(0, SR), 0, deferred=True, remote_frames=True)

    class Off(_RefSim):
        pass
    patch_simulator(Off, deferred="remote")
    assert type(Off().reset()["rgb"]) is np.ndarray

    class Rendered(_RefSim):
        pass
    patch_simulator(Rendered, deferred="remote", remote_frames=True)
    live = Rendered(rendered=False)                                      # habitat-sim renders: no key
    assert type(live.reset()["rgb"]) is np.ndarray
    missing = Rendered(cache={(0, 0): scene_observations(1, 8, 8)[(0, 0)]})
    missing.reset()
    assert type(missing.step(TURN_LEFT)["rgb"]) is np.ndarray             # (0, 90) is not in _frame_cache

    class Continuous(_RefSim):
        pass
    patch_simulator(Continuous, continuous=True, deferred="remote", remote_frames=True)
    assert type(Continuous().reset()["rgb"]) is np.ndarray and not getattr(Continuous.reset, "_b200_frames", False)
    assert frame_observations(SimpleNamespace(b200_remote_frames=False), {"rgb": 1}) == {"rgb": 1}


def _model_step(model, cap, keys):
    """LRU of a bank with ``cap`` rows as a list, least recently used first."""
    for k in dict.fromkeys(keys):
        if k in model:
            model.remove(k)
            model.append(k)
    for k in dict.fromkeys(keys):
        if k not in model:
            if len(model) == cap:
                model.pop(0)
            model.append(k)


def test_store_plan_matches_a_numpy_model_of_the_bank():
    rng = np.random.default_rng(5)
    frames = {k: rng.integers(0, 256, size=12, dtype=np.uint8) for k in range(40)}
    store = fr.FrameStore("cpu", "rgb", np.uint8, (12,), max_bank_bytes=7 * 12)
    assert store.capacity == 7
    bank = np.zeros((7, 12), np.uint8)
    model = []
    for step in range(300):
        n = int(rng.integers(1, 6))
        keys = [int(k) for k in rng.integers(0, 12 if step < 150 else 40, size=n)]
        index, fill, staged = store.plan(keys)
        _model_step(model, 7, keys)
        assert list(store._rows) == model
        assert len(set(staged)) == len(staged)
        stage = np.stack([frames[k] for k in staged]) if staged else np.zeros((0, 12), np.uint8)
        reads = {i for i in index if i >= 0}
        assert not reads & set(fill) and len(set(fill)) == len(fill)    # what the kernel refuses never happens
        got = np.stack([bank[i] if i >= 0 else stage[-1 - i] for i in index])
        bank[fill] = stage
        assert np.array_equal(got, np.stack([frames[k] for k in keys]))
        for k, row in store._rows.items():
            assert np.array_equal(bank[row], frames[k])                 # every resident row holds its frame
    assert store.stats["evictions"] > 0 and store.stats["hits"] > 0


def test_a_step_with_more_frames_than_the_bank_regrows_it():
    store = fr.FrameStore("cpu", "depth", np.float32, (4,), max_bank_bytes=2 * 16)
    index, fill, staged = store.plan([1, 2, 3, 1])
    assert store.capacity == 3 and store.stats["regrown"] == 1
    assert staged == [1, 2, 3] and index == [-1, -2, -3, -1] and sorted(fill) == [0, 1, 2]


def test_process_workers_ship_each_frame_once(tmp_path):
    """A few steps of two forkserver workers: once every pose's frames have crossed, a step pickles keys only."""
    cache = scene_observations(4, 32, 32, seed=7)
    path = write_scene_observations(str(tmp_path / "replica" / "room.pkl"), cache)
    clip = make_source(0, SR)
    args = [(SR, "room", 2, str(tmp_path), "c.wav", clip, 3, e, 0, "remote", 10 ** 6, path, True) for e in range(2)]
    trace = [TURN_LEFT] * 8 + [MOVE_FORWARD, TURN_LEFT, TURN_LEFT, MOVE_FORWARD] * 2 + [TURN_LEFT] * 8
    with ProcessReplayVectorEnv(replay_sim, args) as envs:
        obs = envs.observe()
        sizes = []
        for a in trace:
            b0 = envs.bytes_received
            obs = envs.step([a, a])
            sizes.append(envs.bytes_received - b0)
            for o in obs:
                assert isinstance(o["rgb"], FrameRef) and o["rgb"].shape == (32, 32, 3)
                assert isinstance(o["depth"], FrameRef) and o["depth"].dtype == np.float32
                sim_key = o["rgb"].key
                want = visual_observations(cache[(sim_key[1], sim_key[2])])
                assert np.array_equal(np.asarray(o["rgb"]), want["rgb"])
                assert np.array_equal(np.asarray(o["depth"]), want["depth"], equal_nan=True)
    frame_bytes = 32 * 32 * 3 + 32 * 32 * 4
    assert max(sizes[:4]) > frame_bytes                                  # new poses: the data travels
    assert sizes[-1] < frame_bytes // 4                                  # every pose seen: keys only


def test_frame_replay_sim_in_process_returns_frame_arrays(tmp_path):
    path = write_scene_observations(str(tmp_path / "replica" / "s.pkl"), scene_observations(4, 8, 8))
    sim = FrameReplaySim(None, ReplayScene("s", 2), "c.wav", make_source(0, SR), 0, deferred="remote", sr=SR,
                         frames=path)
    obs = sim.reset()
    assert type(obs["rgb"]) is FrameArray and obs["rgb"].frame_key == (path, 0, 0, "rgb")
    obs = sim.step(TURN_LEFT)
    assert obs["depth"].frame_key == (path, 0, 90, "depth")
    assert remote._FRAMES is fr._FRAMES
