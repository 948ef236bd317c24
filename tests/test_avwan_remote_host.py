"""AV-WaN's Intensity in remote deferred mode, worker side (no GPU): the sensor returns the waveform request, the
patched planner logs it in the map records, and nothing in the worker converts it or touches CUDA."""
import os
import pickle
import subprocess
import warnings

import numpy as np
import pytest
import torch

from avwan_remote_envs import IntensityPlanner, MapNavReplayEnv
from mapper_models import StandInPlanner, drive, step_inputs, task_config
from oracle.ref_harness import write_rir
from synth import make_rir, make_source

from soundspaces_b200.maps import UPDATE, MapDescriptor, patch_planner
from soundspaces_b200.remote import WAVEFORM, IntensityRequest, RemoteAudioRequest
from soundspaces_b200.replay import ReplayScene, ReplaySim
from soundspaces_b200.sensors import Intensity
from soundspaces_b200.simulator import INTENSITY_REMOTE_ERROR, patch_simulator

SR = 16000
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _tree(root):
    for az in (0, 90, 180, 270):
        for n in range(9):
            for s in (0, 1):
                write_rir(root, "replica", "scene", az, n, s, SR, make_rir(n + 10 * s, 800))


def _sim(root, clip, deferred="remote"):
    sim = ReplaySim(None, ReplayScene("scene", 3, rir_root=root), "c.wav", clip, 0, 4, 0, deferred=deferred, sr=SR)
    sim.b200_remote_intensity = True
    return sim


def test_intensity_returns_the_waveform_request_and_memoises(tmp_path):
    clip = make_source(2, 3 * SR)                              # a 3-s clip: _audio_index advances on a memo miss
    sim = _sim(str(tmp_path), clip)
    sensor = Intensity(sim=sim, config=None)
    seen, indices = {}, []
    for a in [0, 2, 2, 3, 3, 1, 2, 2, 2, 2]:
        if a:
            sim.step(a)
        key = (sim._source_position_index, sim._receiver_position_index, sim.azimuth_angle)
        before = sim._audio_index
        v = sensor.get_observation()
        assert isinstance(v, list) and len(v) == 1 and isinstance(v[0], IntensityRequest)
        d = v[0].request
        assert isinstance(d, RemoteAudioRequest) and d.kind == WAVEFORM
        assert d.hit == (key in seen) and sim._audiogoal_cache[key] is (seen.get(key) or d)
        if key in seen:
            assert sim._audio_index == before and d.offset == seen[key].offset
        else:
            assert sim._audio_index == (before + 1) % 3 and d.offset == before * SR
            seen[key] = d
        indices.append(sim._audio_index)
    assert len(seen) < 10 and len(set(indices)) > 1
    assert not torch.cuda.is_initialized()


def test_the_opt_in_is_a_patch_simulator_keyword():
    class Sim:
        pass
    patch_simulator(Sim, deferred="remote", remote_intensity=True)
    assert Sim.b200_remote_intensity is True
    class Plain:
        pass
    patch_simulator(Plain, deferred="remote")
    assert Plain.b200_remote_intensity is False
    with pytest.raises(ValueError, match="remote_intensity"):
        patch_simulator(type("In", (), {}), deferred=True, remote_intensity=True)
    assert "in-process envs" in INTENSITY_REMOTE_ERROR and "remote_intensity=True" in INTENSITY_REMOTE_ERROR


def test_converting_in_the_building_process_raises(tmp_path):
    q = Intensity(sim=_sim(str(tmp_path), make_source(0, SR)), config=None).get_observation()[0]
    for convert in (float, np.asarray, lambda x: np.float64(0.5) * x):
        with pytest.raises(RuntimeError, match="trainer"):
            convert(q)
    assert pickle.loads(pickle.dumps(q)).received and not q.received
    assert not torch.cuda.is_initialized()


def _drive_pair(root, encoding, seed=21, steps=6, episode_steps=None):
    """The remote env and a float-fed twin: same seeds, the twin's Intensity replaced by the float32 intensities of
    step_inputs.  Returns both envs and their per-step observations' records."""
    clip = make_source(5, SR)
    env = MapNavReplayEnv("discrete", SR, root, clip, seed, "remote", encoding=encoding, episode_steps=episode_steps)
    twin = MapNavReplayEnv("discrete", SR, root, clip, seed, "remote", encoding=encoding, episode_steps=episode_steps)
    fixed = iter(range(10 ** 6))

    class FloatIntensity:
        def get_observation(self, **_):
            return [float(step_inputs(seed, next(fixed))[3])]
    twin.sensors["intensity"] = FloatIntensity()
    return env, twin


def test_records_carry_requests_and_match_a_float_fed_run(tmp_path):
    root = str(tmp_path)
    _tree(root)
    for encoding in ("intensity", "average_intensity"):
        env, twin = _drive_pair(root, encoding, episode_steps=3)
        got, want = [], []
        for step in range(7):
            o1, o2 = (env.reset(), twin.reset()) if step == 0 else (env.step(), twin.step())
            for kind in ("gm", "am", "action_map"):
                assert isinstance(o1[kind], MapDescriptor) and o1[kind].pose == o2[kind].pose
            got += env.planner.mapper._b200_map_log.drain()
            want += twin.planner.mapper._b200_map_log.drain()
        assert len(got) == len(want) > 10 and env.updates == twin.updates
        n_req = 0
        for a, b in zip(got, want):
            assert a[:5] == b[:5] and a[7] == b[7]
            if a[1] == UPDATE:
                assert isinstance(a[5], IntensityRequest) and a[6] is None
                n_req += 1
        assert n_req > 10
    assert not torch.cuda.is_initialized()


def test_pickled_records_carry_the_requests_once_and_no_samples_after_the_first_send(tmp_path):
    root = str(tmp_path)
    _tree(root)
    env = MapNavReplayEnv("discrete", SR, root, make_source(8, SR), 3, "remote", episode_steps=4)
    sizes, first = [], pickle.dumps(env.reset())
    for _ in range(12):
        obs = env.step()
        data = pickle.dumps(obs, protocol=pickle.HIGHEST_PROTOCOL)
        back = pickle.loads(data)
        sizes.append(len(data))
        recs = back["gm"].pending()
        assert back["intensity"][0].received
        reqs = [r[5] for r in recs if r[1] == UPDATE]
        assert all(isinstance(q, IntensityRequest) and q.request.clip.samples is None for q in reqs)
        if reqs and not obs["collision"][0]:
            assert reqs[-1] is back["intensity"][0]             # one object: the trainer resolves it once
    assert len(first) > 4 * SR and max(sizes) < 4 * SR / 2          # the clip's samples travelled once


def test_refused_geometry_with_an_acoustic_map_names_the_reason(tmp_path):
    class Refused(StandInPlanner):
        pass
    patch_planner(Refused)
    tc = task_config("avwan", "intensity")
    tc.TASK.GEOMETRIC_MAP.MAP_SIZE = 201                       # odd: the device path refuses it
    q = Intensity(sim=_sim(str(tmp_path), make_source(0, SR)), config=None).get_observation()[0]
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        acoustic = Refused(task_config=tc, use_acoustic_map=True)
        plain = Refused(task_config=tc, use_acoustic_map=False)
    ego = step_inputs(1, 1)[0]
    with pytest.raises(RuntimeError, match="odd MAP_SIZE 201"):
        acoustic.mapper.update(1, ego, q)
    assert plain.mapper.update(1, ego, q) == ([], [])


def test_without_an_acoustic_map_the_records_carry_no_intensity(tmp_path):
    q = Intensity(sim=_sim(str(tmp_path), make_source(0, SR)), config=None).get_observation()[0]
    p = IntensityPlanner(task_config=task_config("avwan", "intensity"), use_acoustic_map=False)
    p.set_action(1)
    p.update_map_and_graph({"collision": np.array([False]), "intensity": [q], "ego_map": step_inputs(2, 1)[0]})
    recs = p.mapper._b200_map_log.drain()
    assert recs[-1][1] == UPDATE and recs[-1][5:7] == (0.0, 0.0)


def test_float_intensities_still_take_the_host_path():
    p = IntensityPlanner(task_config=task_config("avwan", "average_intensity"), use_acoustic_map=True)
    obs = list(drive(p, 7, 5))
    assert isinstance(obs[-1]["am"], MapDescriptor)
    recs = [r for r in p.mapper._b200_map_log.drain() if r[1] == UPDATE]
    assert recs and all(isinstance(r[5], float) and isinstance(r[6], float) for r in recs)


def test_workers_never_initialise_cuda(tmp_path):
    """A remote MapNav loop in a fresh interpreter started like a spawn worker: torch imported, CUDA untouched."""
    root = str(tmp_path)
    _tree(root)
    code = ("import sys, pickle, torch\n"
            f"sys.path[:0] = [{os.path.join(ROOT, 'tests')!r}, {ROOT!r}]\n"
            "from avwan_remote_envs import MapNavReplayEnv\n"
            "from synth import make_source\n"
            f"env = MapNavReplayEnv('discrete', {SR}, {root!r}, make_source(1, {SR}), 5, 'remote', episode_steps=3)\n"
            "pickle.dumps(env.reset())\n"
            "for _ in range(6): pickle.dumps(env.step())\n"
            "print(torch.cuda.is_initialized())\n")
    out = subprocess.run([os.sys.executable, "-c", code], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stderr
    assert out.stdout.strip().splitlines()[-1] == "False"


def test_record_struct_layout_matches_c(tmp_path):
    """The reserved field the device-intensity entry reads sits where RECORD_DTYPE puts it."""
    from soundspaces_b200.maps import RECORD_DTYPE
    src = tmp_path / "l.c"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "ssb200.h"\nint main(void){printf("%zu %zu %zu %zu\\n",'
                   'sizeof(ssb_map_record), offsetof(ssb_map_record, reserved), offsetof(ssb_map_record, intensity),'
                   'offsetof(ssb_map_record, half));return 0;}\n')
    exe = tmp_path / "l"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    got = [int(v) for v in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    f = RECORD_DTYPE.fields
    assert got == [RECORD_DTYPE.itemsize, f["reserved"][1], f["intensity"][1], f["half"][1]]
