"""Generate tests/golden/mapper_golden.npz by driving the UNMODIFIED reference AV-WaN ``Planner`` and ``Mapper`` of an
upstream sound-spaces checkout (path in ``SOUNDSPACES_REFERENCE``, as for the other oracle fixtures):
ss_baselines/av_wan/models/planner.py and mapper.py, with habitat's ``HabitatSimActions`` stubbed (networkx is real).

    SOUNDSPACES_REFERENCE=<sound-spaces checkout> python tests/golden/make_mapper_golden.py

Each trace of ``tests/mapper_models.TRACES`` (the AV-WaN default geometry -- internal 500, MAP_SIZE 200, stride 5 --
and the mp3d one -- 1200, 400, stride 10 -- in both acoustic-map encodings) runs the env's reset flow at step 0 and
after every episode end, and otherwise ``plan`` (towards a seeded action-map goal) then ``update_map_and_graph`` with
the step's ego map, collision flag and float32 intensity, then ``add_maps_to_observation``.  Stored per trace
``<name>/``: ``poses`` (the mapper's pose after every step), ``flags`` (collided, reset), ``digests`` (SHA-256 of the
float32 gm, am and action_map bytes at every step), and at two steps ``full_steps`` the full outputs (gm bit-packed:
its values are 0 and 1).
"""
import importlib.util
import os
import sys
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from mapper_models import ACTION, TRACES, digest, step_inputs, task_config  # noqa: E402
from oracle.ref_harness import REFERENCE_ROOT  # noqa: E402


def _stub(name, **attrs):
    m = types.ModuleType(name)
    m.__dict__.update(attrs)
    m.__path__ = []
    sys.modules[name] = m
    return m


def load_planner():
    if not REFERENCE_ROOT:
        sys.exit("set SOUNDSPACES_REFERENCE to a sound-spaces checkout")

    class HabitatSimActions:
        STOP, MOVE_FORWARD, TURN_LEFT, TURN_RIGHT = 0, 1, 2, 3

    for pkg in ("habitat", "habitat.sims", "habitat.sims.habitat_simulator", "ss_baselines", "ss_baselines.av_wan",
                "ss_baselines.av_wan.models"):
        _stub(pkg)
    _stub("habitat.sims.habitat_simulator.actions", HabitatSimActions=HabitatSimActions)
    mods = {}
    for name in ("mapper", "planner"):
        spec = importlib.util.spec_from_file_location(
            f"ss_baselines.av_wan.models.{name}",
            os.path.join(REFERENCE_ROOT, "ss_baselines", "av_wan", "models", f"{name}.py"))
        mods[name] = importlib.util.module_from_spec(spec)
        sys.modules[spec.name] = mods[name]
        spec.loader.exec_module(mods[name])
    return mods["planner"].Planner


def run_trace(Planner, name):
    config, encoding, seed, steps = TRACES[name]
    np.random.seed(seed)                                   # Planner.plan draws its random turns from np.random
    rng = np.random.default_rng(seed + 1000)
    planner = Planner(task_config=task_config(config, encoding), use_acoustic_map=True, masking=False)
    poses, flags, digests, outs = [], [], [], []
    obs = None
    for t in range(steps):
        ego, collided, reset, intensity = step_inputs(seed, t)
        if reset:
            planner.reset()
        elif t > 0:
            g = int(rng.integers(ACTION * ACTION - 1))
            goal = planner.get_map_coordinates(g + (g >= ACTION * ACTION // 2))   # the centre index means STOP
            planner.plan(obs, goal, stop=False)
        obs = {"ego_map": ego, "depth": np.zeros((4, 4, 1), np.float32),
               "collision": np.array([collided and not reset]), "intensity": np.array([intensity]),
               "gm": None, "am": None, "action_map": None}
        planner.update_map_and_graph(obs)
        planner.add_maps_to_observation(obs)
        m = planner.mapper
        poses.append((m._x, m._y, m._orientation))
        flags.append((collided, reset))
        digests.append([np.frombuffer(digest(obs[k]), np.uint8) for k in ("gm", "am", "action_map")])
        outs.append({k: obs[k] for k in ("gm", "am", "action_map")})
    full = [steps // 2, steps - 1]
    res = {"poses": np.array(poses, np.int32), "flags": np.array(flags, bool), "digests": np.array(digests),
           "full_steps": np.array(full, np.int32)}
    for i, s in enumerate(full):
        gm = outs[s]["gm"]
        assert np.all((gm == 0) | (gm == 1))
        res[f"gm_bits{i}"] = np.packbits(gm > 0.5)
        res[f"am{i}"] = outs[s]["am"]
        res[f"action_map{i}"] = outs[s]["action_map"]
    return res


def main():
    Planner = load_planner()
    out = {}
    for name in TRACES:
        for k, v in run_trace(Planner, name).items():
            out[f"{name}/{k}"] = v
        poses = out[f"{name}/poses"]
        print(name, "steps", len(poses), "x range", poses[:, 0].min(), poses[:, 0].max(), "y range",
              poses[:, 1].min(), poses[:, 1].max(), "orientations", sorted(set(poses[:, 2])), "resets", int(out[f"{name}/flags"][:, 1].sum()))
    path = os.path.join(ROOT, "tests", "golden", "mapper_golden.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
