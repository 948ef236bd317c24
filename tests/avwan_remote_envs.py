"""AV-WaN's MapNavEnv step as the remote-intensity tests run it, in worker processes or in process.

``MapNavReplayEnv.step`` mirrors ``MapNavEnv.step`` (ss_baselines/av_wan/mapnav_env.py): up to PREDICTION_INTERVAL
low-level steps, each one a simulator step, the sensor suite's observation and ``Planner.update_map_and_graph``; a
seeded waypoint check ends the loop early; ``add_maps_to_observation`` on the last observation.  The planner is the
stand-in of tests/mapper_models.py reading ``observation['intensity'][0]`` exactly as planner.py:59 does."""
import pickle
import traceback

import numpy as np
import torch

from mapper_models import StandInPlanner, step_inputs, task_config
from soundspaces_b200.maps import patch_planner
from soundspaces_b200.replay import ReplayScene, ReplaySim
from soundspaces_b200.sensors import AudioGoalSensor, Intensity

PREDICTION_INTERVAL = 10


def to_array(x):
    """ss_baselines/av_wan/models/mapper.py:19-24."""
    return x.cpu().numpy() if torch.is_tensor(x) else x


class IntensityPlanner(StandInPlanner):
    def update_map_and_graph(self, observation):
        collided = to_array(observation["collision"][0])
        intensity = to_array(observation["intensity"][0]) if "intensity" in observation else None   # planner.py:59
        if not collided:
            return self.mapper.update(self._prev_action, to_array(observation["ego_map"]), intensity)
        return None


patch_planner(IntensityPlanner)


def make_sim(kind, sr, root, clip, seed, deferred, service=None):
    """``kind``: "discrete", "distractor" or "continuous"."""
    if kind == "continuous":
        from remote_envs import ContinuousReplaySim
        sim = ContinuousReplaySim(sr, clip, seed, True, deferred)
    else:
        sim = ReplaySim(service, ReplayScene("scene", 3, rir_root=root), f"s{len(clip) // sr}.wav", clip, 0,
                        seed % 9, 90 * (seed % 4), deferred=deferred, duration=40, sr=sr)
        if kind == "distractor":
            sim.config.AUDIO.HAS_DISTRACTOR_SOUND = True
            sim._current_distractor_sound = "d.wav"
            sim._source_sound_dict["d.wav"] = clip[::-1].copy()
            sim._distractor_position_index = 1
    if deferred == "remote":
        sim.b200_remote_intensity = True
    return sim


class MapNavReplayEnv:
    def __init__(self, kind, sr, root, clip, seed, deferred, encoding="average_intensity", order=("intensity",),
                 episode_steps=None, service=None):
        self.sim = make_sim(kind, sr, root, clip, seed, deferred, service)
        cls = {"intensity": Intensity, "audiogoal": AudioGoalSensor}
        self.sensors = {u: cls[u](sim=self.sim, config=None) for u in order}
        self.planner = IntensityPlanner(task_config=task_config("avwan", encoding), use_acoustic_map=True)
        self.seed, self.t, self.episode_steps, self.steps = seed, 0, episode_steps, 0
        self.rng = np.random.default_rng(seed + 500)
        self.updates = []                                   # what Mapper.update returned, per low-level step

    def _observe(self, t):
        ego, collided, _, _ = step_inputs(self.seed, t)
        obs = {u: s.get_observation(observations=None, episode=None) for u, s in self.sensors.items()}
        obs.update(ego_map=ego, collision=np.array([collided]), gm=None, am=None, action_map=None)
        return obs

    def reset(self):
        if hasattr(self.sim, "reset"):
            self.sim.reset()                                # a new episode from the start pose, memo dicts kept
        self.sim._episode_step_count = 0
        self.planner.reset()
        self.steps = 0
        obs = self._observe(self.t)
        self.t += 1
        self.planner.update_map_and_graph(obs)
        self.planner.add_maps_to_observation(obs)
        return obs

    def step(self, _action=None):
        for _ in range(PREDICTION_INTERVAL):
            a = int(self.rng.integers(1, 4))
            self.sim.step(a)
            self.planner.set_action(a)
            obs = self._observe(self.t)
            self.t += 1
            self.updates.append(self.planner.update_map_and_graph(obs))
            if self.rng.random() < 0.2:                     # waypoint reached
                break
        self.planner.add_maps_to_observation(obs)
        self.steps += 1
        if self.episode_steps and self.steps >= self.episode_steps:
            obs = self.reset()                              # auto_reset_done: the terminal observation is dropped
        return obs


def _worker(conn, args, kwargs):
    try:
        env = MapNavReplayEnv(*args, **kwargs)
        conn.send_bytes(pickle.dumps(None))
        while True:
            cmd = conn.recv()
            if cmd == "close":
                return
            try:
                if cmd == "reset":
                    res = env.reset()
                elif cmd == "step":
                    res = env.step()
                else:
                    res = {"cuda_initialized": torch.cuda.is_initialized()}
                conn.send_bytes(pickle.dumps(res, protocol=pickle.HIGHEST_PROTOCOL))
            except Exception:                               # noqa: BLE001 - reported to the parent
                conn.send_bytes(pickle.dumps(RuntimeError(traceback.format_exc())))
    except (EOFError, KeyboardInterrupt):
        pass
    except Exception:                                       # noqa: BLE001
        conn.send_bytes(pickle.dumps(RuntimeError(traceback.format_exc())))
    finally:
        conn.close()


class ProcessMapNavEnvs:
    """One worker process per env; ``bytes_received`` counts the pickled observations.  ``close`` joins them all."""

    def __init__(self, configs, start_method="forkserver"):
        import multiprocessing as mp
        ctx = mp.get_context(start_method)
        self.conns, self.procs, self.bytes_received, self.sizes = [], [], 0, []
        try:
            for args, kwargs in configs:
                parent, child = ctx.Pipe()
                p = ctx.Process(target=_worker, args=(child, args, kwargs), daemon=True)
                p.start()
                child.close()
                self.conns.append(parent)
                self.procs.append(p)
            for c in self.conns:
                self._recv(c)
        except BaseException:
            self.close()
            raise

    def _recv(self, conn):
        data = conn.recv_bytes()
        self.bytes_received += len(data)
        self.sizes.append(len(data))
        res = pickle.loads(data)
        if isinstance(res, RuntimeError):
            raise res
        return res

    def _all(self, cmd):
        for c in self.conns:
            c.send(cmd)
        return [self._recv(c) for c in self.conns]

    def reset(self):
        return self._all("reset")

    def step(self):
        return self._all("step")

    def report(self):
        return self._all("report")

    def close(self):
        for c in self.conns:
            try:
                c.send("close")
            except (OSError, ValueError):
                pass
        for p in self.procs:
            p.join(timeout=30)
            if p.is_alive():
                p.terminate()
                p.join()
        for c in self.conns:
            c.close()
        self.conns, self.procs = [], []

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()
