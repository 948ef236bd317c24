"""A numpy stand-in of AV-WaN's device maps (soundspaces_b200.maps records, ssb_map_update_batch /
ssb_map_observe_batch), written from the behaviour of the reference ``Mapper`` (ss_baselines/av_wan/models/mapper.py)
rather than from the CUDA code, plus the seeded traces tests/golden/make_mapper_golden.py drives the reference with.

The golden file stores, per trace, the seed, the mapper's pose after every step, the collided and reset flags, and
SHA-256 digests of the reference's three outputs; ego maps and intensities are regenerated here from the seed."""
import hashlib
from types import SimpleNamespace

import numpy as np

from soundspaces_b200.maps import RESET, UPDATE, MapGeometry, navigable_tables

# name: (INTERNAL_MAP_SIZE, MAP_SIZE, GEOMETRIC_MAP.MAP_RESOLUTION, ACTION_MAP.MAP_RESOLUTION) -> stride 5 / 10
CONFIGS = {"avwan": (500, 200, 0.1, 0.5), "mp3d": (1200, 400, 0.1, 1.0)}
EGO, ACTION = 31, 9
TRACES = {  # name: (config, encoding, seed, steps)
    "avwan_avg": ("avwan", "average_intensity", 11, 120),
    "avwan_int": ("avwan", "intensity", 12, 120),
    "mp3d_avg": ("mp3d", "average_intensity", 13, 120),
    "mp3d_int": ("mp3d", "intensity", 14, 120),
}


def task_config(config, encoding):
    n, s, gm_res, am_res = CONFIGS[config]
    ns = SimpleNamespace
    return ns(TASK=ns(GEOMETRIC_MAP=ns(INTERNAL_MAP_SIZE=n, MAP_SIZE=s, MAP_RESOLUTION=gm_res),
                      ACOUSTIC_MAP=ns(ENCODING=encoding, MAP_SIZE=20, MAP_RESOLUTION=am_res),
                      ACTION_MAP=ns(MAP_SIZE=ACTION, MAP_RESOLUTION=am_res),
                      EGOMAP_SENSOR=ns(MAP_SIZE=EGO, MAP_RESOLUTION=gm_res)))


def geometry(config, encoding, acoustic=1):
    n, s, gm_res, am_res = CONFIGS[config]
    return MapGeometry(n, int(am_res / gm_res), s, ACTION, EGO, {"intensity": 0, "average_intensity": 1}[encoding],
                       acoustic)


def step_inputs(seed, t):
    """The ego map (values 0, 0.25, 0.5, 0.75, 1 so that the > 0.5 threshold matters), collided and reset flags, and
    the float32 intensity of step t of a trace (t = 0 is the episode's first observation)."""
    rng = np.random.default_rng([seed, t])
    levels = np.array([0.0, 0.25, 0.5, 0.75, 1.0])
    ego = np.stack([rng.choice(levels, size=(EGO, EGO), p=[0.93, 0.02, 0.02, 0.01, 0.02]),     # sparse obstacles
                    rng.choice(levels, size=(EGO, EGO), p=[0.3, 0.1, 0.1, 0.1, 0.4])], axis=-1)
    collided = bool(t > 0 and rng.random() < 0.15)
    reset = bool(t > 0 and rng.random() < 0.04)
    r = rng.random()
    intensity = np.float32(0.0) if r < 0.1 else np.float32(-0.0) if r < 0.15 else np.float32(rng.random() * 3)
    return ego, collided, reset, intensity


def digest(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).digest()


class MapMirror:
    """One env's maps kept as the device keeps them: channel bits of the geometric map and the float64 acoustic map."""

    def __init__(self, g: MapGeometry):
        self.g = g
        self.tables = navigable_tables(g)
        self.gm = np.zeros((g.internal_size, g.internal_size, 2), dtype=bool)
        self.am = np.zeros((g.acoustic_size, g.acoustic_size), dtype=np.float64)

    @staticmethod
    def turns(orientation):
        return (orientation - 270) % 360 // 90

    def update_raises(self, x, y, o):
        """Why the reference's ``Mapper.update`` raises for an update to pose (x, y, o) (of a valid orientation), or
        None: the ego window leaves the map (a broadcast ValueError; with E = 1 at ry = 0 the window's rows [-1, 0)
        are an empty slice the one-row ego map broadcasts into, so nothing is written and nothing raises), at stride 1
        its loop reads row or column N (IndexError: with new_top = min(ry + 1, N) it visits row new_top, with
        new_right = min(right + 1, N) column new_right), or the acoustic cell lies outside the M x M map (IndexError)."""
        g, n = self.g, self.g.internal_size
        if not (0 <= x < n and 0 <= y < n):
            return "pose"
        rx, ry = ((x, y), (y, n - 1 - x), (n - 1 - x, n - 1 - y), (n - 1 - y, x))[self.turns(o)]
        right = rx - g.ego_size // 2 + g.ego_size
        if (ry - g.ego_size < 0 and g.ego_size > 1) or rx - g.ego_size // 2 < 0 or right > n:
            return "window"
        if g.stride == 1 and (ry == n - 1 or right >= n - 1):
            return "stride 1"
        if g.acoustic and (x // g.stride >= g.acoustic_size or y // g.stride >= g.acoustic_size):
            return "acoustic cell"
        return None

    def apply(self, rec):
        seq, kind, x, y, o, value, half, bits = rec
        g = self.g
        if kind == RESET:
            self.gm[:] = False
            self.am[:] = 0.0
            return
        assert kind == UPDATE
        why = self.update_raises(x, y, o)
        if why:
            raise ValueError(f"the reference's Mapper.update raises at pose ({x}, {y}, {o}): {why}")
        k = self.turns(o)
        ego = np.unpackbits(np.frombuffer(bits, dtype=np.uint8))[:g.ego_size * g.ego_size * 2]
        ego = ego.reshape(g.ego_size, g.ego_size, 2).astype(bool)
        view = np.rot90(self.gm, k)                        # a view: writes land in self.gm
        n = g.internal_size
        rx, ry = ((x, y), (y, n - 1 - x), (n - 1 - x, n - 1 - y), (n - 1 - y, x))[k]
        top, left = ry - g.ego_size, rx - g.ego_size // 2
        if top >= 0:
            view[top:ry, left:left + g.ego_size] |= ego
        if rx <= n + 1 - g.stride and ry <= n + 1 - g.stride:      # the reference's loop visits the agent's node
            self.gm[y, x, 0] = False
        if g.acoustic:
            c = (y // g.stride, x // g.stride)
            if g.encoding == 0 or self.am[c] == 0:
                self.am[c] = value
            else:
                self.am[c] = np.float64(half) + 0.5 * self.am[c]

    def observe(self, pose):
        x, y, o = pose
        g, n, k = self.g, self.g.internal_size, self.turns(o)
        S, m = g.map_size, g.acoustic_size
        view = np.rot90(self.gm, k)
        rx, ry = ((x, y), (y, n - 1 - x), (n - 1 - x, n - 1 - y), (n - 1 - y, x))[k]
        gm = np.zeros((S, S, 2), dtype=np.float32)
        r0, c0 = ry - S // 2, rx - S // 2
        rs, cs = slice(max(r0, 0), min(r0 + S, n)), slice(max(c0, 0), min(c0 + S, n))
        gm[rs.start - r0:rs.stop - r0, cs.start - c0:cs.stop - c0] = view[rs, cs]
        am = np.zeros((20, 20, 1), dtype=np.float32)
        if g.acoustic:
            av = np.rot90(self.am, k)
            ax, ay = x // g.stride, y // g.stride
            ax, ay = ((ax, ay), (ay, m - 1 - ax), (m - 1 - ax, m - 1 - ay), (m - 1 - ay, ax))[k]
            r0, c0 = ay - 10, ax - 10
            rs, cs = slice(max(r0, 0), min(r0 + 20, m)), slice(max(c0, 0), min(c0 + 20, m))
            am[rs.start - r0:rs.stop - r0, cs.start - c0:cs.stop - c0, 0] = av[rs, cs].astype(np.float32)
        xs, ys = self.tables[k]
        gx, gy = rx // g.stride, ry // g.stride
        h = g.action_size // 2
        grid = view[np.ix_(ys[gy - h:gy + h + 1], xs[gx - h:gx + h + 1])][..., 0]
        action = (1.0 - grid.astype(np.float64)).astype(np.float32)[..., None]
        return gm, am, action


def trace_records(name, poses, flags):
    """The records the patched planner logs over a golden trace, per step: ``poses[t]`` the mapper's pose after step
    t, ``flags[t]`` = (collided, reset).  Step 0 follows the constructor's reset."""
    config, encoding, seed, steps = TRACES[name]
    seq, out = 0, []
    first = [(0, RESET, 0, 0, 0, 0.0, 0.0, b"")]
    for t in range(steps):
        ego, collided, reset, intensity = step_inputs(seed, t)
        recs = first if t == 0 else []
        if reset:
            seq += 1
            recs.append((seq, RESET, 0, 0, 0, 0.0, 0.0, b""))
        if not collided or reset:
            seq += 1
            x, y, o = (int(v) for v in poses[t])
            recs.append((seq, UPDATE, x, y, o, float(np.float64(intensity)), float(np.float64(0.5 * intensity)),
                         np.packbits(ego > 0.5).tobytes()))
        out.append(recs)
    return out


class StandInMapper:
    """The reference ``Mapper``'s pose bookkeeping and attributes, with its maps kept by a :class:`MapMirror` (the
    planner's graph is left out).  Actions: 1 MOVE_FORWARD, 2 TURN_LEFT, 3 TURN_RIGHT as HabitatSimActions."""

    def __init__(self, gm_config, am_config, action_map_config, use_acoustic_map):
        self._internal_gm_size = gm_config.INTERNAL_MAP_SIZE
        self._gm_size = gm_config.MAP_SIZE
        self._gm_res = gm_config.MAP_RESOLUTION
        self._use_acoustic_map = use_acoustic_map
        self._am_encoding = am_config.ENCODING
        self._action_map_res = action_map_config.MAP_RESOLUTION
        self._stride = int(self._action_map_res / self._gm_res)
        self._action_size = action_map_config.MAP_SIZE
        self.reset()

    def reset(self):
        n = self._internal_gm_size
        self._x = self._y = int(n / 2)
        self._orientation = 270
        g = MapGeometry(n, self._stride, self._gm_size, self._action_size, EGO,
                        {"intensity": 0}.get(self._am_encoding, 1), int(bool(self._use_acoustic_map)))
        self.mirror = MapMirror(g)

    def update(self, prev_action, ego_map, intensity):
        if prev_action == 1:
            self._x += int(self._stride * np.cos(np.deg2rad(self._orientation)))
            self._y += int(self._stride * np.sin(np.deg2rad(self._orientation)))
        elif prev_action == 2:
            self._orientation = (self._orientation - 90) % 360
        elif prev_action == 3:
            self._orientation = (self._orientation + 90) % 360
        v = (float(np.float64(intensity)), float(np.float64(0.5 * intensity))) if self._use_acoustic_map else (0.0, 0.0)
        self.mirror.apply((0, UPDATE, self._x, self._y, self._orientation) + v +
                          (np.packbits(np.asarray(ego_map) > 0.5).tobytes(),))
        return [], []


class StandInPlanner:
    """The reference ``Planner``'s constructor, reset, map update and ``add_maps_to_observation`` over
    :class:`StandInMapper`; ``plan`` is replaced by ``set_action``."""

    def __init__(self, task_config=None, use_acoustic_map=False, model_dir=None, masking=True):
        t = task_config.TASK
        self.mapper = StandInMapper(t.GEOMETRIC_MAP, t.ACOUSTIC_MAP, t.ACTION_MAP, use_acoustic_map)
        self._action_map_size = t.ACTION_MAP.MAP_SIZE
        self.reset()

    def reset(self):
        self._prev_action = None
        self.mapper.reset()

    def set_action(self, action):
        self._prev_action = action

    def update_map_and_graph(self, observation):
        if not np.asarray(observation["collision"])[0]:
            intensity = np.asarray(observation["intensity"])[0] if "intensity" in observation else None
            self.mapper.update(self._prev_action, observation["ego_map"], intensity)

    def add_maps_to_observation(self, observation):
        m = self.mapper
        gm, am, action = m.mirror.observe((m._x, m._y, m._orientation))
        for k, v in (("gm", gm), ("am", am), ("action_map", action)):
            if k in observation:
                observation[k] = v


def drive(planner, seed, steps, t0=0):
    """Run a stand-in or reference-shaped planner over ``steps`` seeded steps (episode ends included) and yield each
    step's observation dict after ``add_maps_to_observation``."""
    rng = np.random.default_rng(seed + 1000)
    for t in range(t0, t0 + steps):
        ego, collided, reset, intensity = step_inputs(seed, t)
        if reset:
            planner.reset()
        elif t > 0:
            planner.set_action(int(rng.integers(1, 4)))
        obs = {"ego_map": ego, "collision": np.array([collided and not reset]), "intensity": np.array([intensity]),
               "gm": None, "am": None, "action_map": None}
        planner.update_map_and_graph(obs)
        planner.add_maps_to_observation(obs)
        yield obs
