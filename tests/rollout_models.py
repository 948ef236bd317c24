"""Stand-ins for the reference's PPO rollout storage (ss_baselines/common/rollout_storage.py, savi/models/
rollout_storage.py) and ``PPO.get_advantages`` (av_nav/ppo/ppo.py, savi/ppo/ppo.py), written from the computation
they perform, and the seeded scripts that drive them.  tests/golden/make_rollout_golden.py runs the scripts on the
unmodified reference classes; test_rollout_host.py checks that these stand-ins reproduce that golden bit for bit, and
test_gpu_rollout.py runs them eagerly on the device next to the patched copies.

The stand-ins keep the reference's attribute names, shapes, dtypes and float32 operation order (the GAE loop rounds
every product and sum on its own), which is all the patched methods rely on."""
from __future__ import annotations

import types
from collections import defaultdict

import numpy as np
import torch

EPS_PPO = 1e-5


class ActionSpace:          # recognised by class name, as the reference does
    pass


class Box:
    def __init__(self, shape):
        self.shape = tuple(shape)


def spaces(shapes):
    return types.SimpleNamespace(spaces={k: Box(s) for k, s in shapes.items()})


class _Storage:
    """What the two reference storages share: the tensors, ``to`` and ``compute_returns`` over ``rows`` steps."""

    def _alloc(self, num_steps, num_envs, observation_space, action_space, hidden, layers, masks_init):
        S, N = num_steps, num_envs
        self.observations = {k: torch.zeros(S + 1, N, *sp.shape) for k, sp in observation_space.spaces.items()}
        self.recurrent_hidden_states = torch.zeros(S + 1, layers, N, hidden)
        self.rewards = torch.zeros(S, N, 1)
        self.value_preds = torch.zeros(S + 1, N, 1)
        self.returns = torch.zeros(S + 1, N, 1)
        self.action_log_probs = torch.zeros(S, N, 1)
        discrete = type(action_space).__name__ == "ActionSpace"
        width = 1 if discrete else action_space.shape[0]
        dtype = torch.long if discrete else torch.float32
        self.actions = torch.zeros(S, N, width, dtype=dtype)
        self.prev_actions = torch.zeros(S + 1, N, width, dtype=dtype)
        self.masks = masks_init(S + 1, N, 1)
        self.num_steps = S
        self.step = 0

    def _tensors(self):
        return ["recurrent_hidden_states", "rewards", "value_preds", "returns", "action_log_probs", "actions",
                "prev_actions", "masks"]

    def to(self, device):
        self.observations = {k: v.to(device) for k, v in self.observations.items()}
        for name in self._tensors():
            setattr(self, name, getattr(self, name).to(device))

    def _write_step(self, observations, hidden, actions, log_probs, values, rewards, masks):
        t = self.step
        for k, v in observations.items():
            self.observations[k][t + 1].copy_(v)
        self.recurrent_hidden_states[t + 1].copy_(hidden)
        self.actions[t].copy_(actions)
        self.prev_actions[t + 1].copy_(actions)
        self.action_log_probs[t].copy_(log_probs)
        self.value_preds[t].copy_(values)
        self.rewards[t].copy_(rewards)
        self.masks[t + 1].copy_(masks)

    def _returns(self, rows, next_value, use_gae, gamma, tau):
        r, v, m, ret = self.rewards, self.value_preds, self.masks, self.returns
        if not use_gae:
            ret[rows] = next_value
            for t in range(rows - 1, -1, -1):
                ret[t] = ret[t + 1] * gamma * m[t + 1] + r[t]
            return
        v[rows] = next_value
        gae = 0
        for t in range(rows - 1, -1, -1):
            delta = r[t] + gamma * v[t + 1] * m[t + 1] - v[t]
            gae = delta + gamma * tau * m[t + 1] * gae
            ret[t] = gae + v[t]

    def _batches(self, advantages, num_mini_batch, rows, extra):
        N = self.rewards.size(1)
        assert N >= num_mini_batch, (
            "Trainer requires the number of processes ({}) to be greater than or equal to the number of trainer "
            "mini batches ({}).".format(N, num_mini_batch))
        nb = N // num_mini_batch
        perm = torch.randperm(N)
        flat = lambda x, cols: x[:rows].index_select(1, cols).reshape(rows * nb, *x.shape[2:])  # noqa: E731
        for start in range(0, N, nb):
            cols = perm[start:start + nb].to(self.rewards.device)
            obs = defaultdict(list)
            for k, v in self.observations.items():
                obs[k] = flat(v, cols)
            out = (obs, self.recurrent_hidden_states[0].index_select(1, cols), flat(self.actions, cols),
                   flat(self.prev_actions, cols), flat(self.value_preds, cols), flat(self.returns, cols),
                   flat(self.masks, cols), flat(self.action_log_probs, cols), flat(advantages, cols))
            yield out + extra(cols, rows, nb)

    def _restart(self, src, extra=()):
        for v in list(self.observations.values()) + [self.recurrent_hidden_states, self.masks, self.prev_actions,
                                                     *extra]:
            v[0].copy_(v[src])


class CommonRolloutStorage(_Storage):
    """common/rollout_storage.py: ``step`` wraps at ``num_steps``; masks start at 1."""

    def __init__(self, num_steps, num_envs, observation_space, action_space, recurrent_hidden_state_size,
                 num_recurrent_layers=1):
        self._alloc(num_steps, num_envs, observation_space, action_space, recurrent_hidden_state_size,
                    num_recurrent_layers, torch.ones)

    def insert(self, observations, recurrent_hidden_states, actions, action_log_probs, value_preds, rewards, masks):
        self._write_step(observations, recurrent_hidden_states, actions, action_log_probs, value_preds, rewards, masks)
        self.step = (self.step + 1) % self.num_steps

    def after_update(self):
        self._restart(-1)

    def compute_returns(self, next_value, use_gae, gamma, tau):
        self._returns(self.rewards.size(0), next_value, use_gae, gamma, tau)

    def recurrent_generator(self, advantages, num_mini_batch):
        return self._batches(advantages, num_mini_batch, self.num_steps, lambda cols, rows, nb: ())


class ExternalMemory:
    """savi/models/rollout_storage.py's ``ExternalMemory``: ``total`` slots, ``capacity`` valid per env."""

    def __init__(self, num_envs, total_size, capacity, dim, num_copies=1):
        self.total_size, self.capacity, self.dim = total_size, capacity, dim
        self.masks = torch.zeros(num_envs, total_size)
        self.memory = torch.zeros(total_size, num_copies, num_envs, dim)
        self.idx = 0

    def insert(self, em_features, not_done_masks):
        self.memory[self.idx].copy_(em_features.unsqueeze(0))
        held = self.masks.sum(1)
        assert not torch.any(held > self.capacity)
        self.masks[held == self.capacity, self.idx - self.capacity] = 0.0
        self.masks[:, self.idx] = 1.0
        self.masks *= not_done_masks
        self.idx = (self.idx + 1) % self.total_size

    def to(self, device):
        self.masks = self.masks.to(device)
        self.memory = self.memory.to(device)


class ExternalMemoryVaried(ExternalMemory):
    """A memory with its own ``insert`` (the reference's per-env variant): the patched storage leaves it alone."""

    def insert(self, em_features, not_done_masks):
        raise NotImplementedError


class SaviRolloutStorage(_Storage):
    """savi/models/rollout_storage.py: ``step`` counts up to ``num_steps``; masks start at 0; an external memory."""

    def __init__(self, num_steps, num_envs, observation_space, action_space, recurrent_hidden_state_size,
                 use_external_memory, external_memory_size, external_memory_capacity, external_memory_dim,
                 num_recurrent_layers=1):
        self._alloc(num_steps, num_envs, observation_space, action_space, recurrent_hidden_state_size,
                    max(1, num_recurrent_layers), torch.zeros)
        self.use_external_memory = use_external_memory
        self.em_size, self.em_capacity, self.em_dim = external_memory_size, external_memory_capacity, external_memory_dim
        self.em_masks = torch.zeros(num_steps + 1, num_envs, external_memory_size)
        self.em = ExternalMemory(num_envs, external_memory_size, external_memory_capacity, external_memory_dim,
                                 num_copies=num_steps + 1) if use_external_memory else None

    def to(self, device):
        super().to(device)
        self.em_masks = self.em_masks.to(device)
        if self.use_external_memory:
            self.em.to(device)

    def insert(self, observations, recurrent_hidden_states, actions, action_log_probs, value_preds, rewards,
               not_done_masks, em_features):
        self._write_step(observations, recurrent_hidden_states, actions, action_log_probs, value_preds, rewards,
                         not_done_masks)
        if self.use_external_memory:
            self.em.insert(em_features, not_done_masks)
            self.em_masks[self.step + 1].copy_(self.em.masks)
        self.step += 1

    def after_update(self):
        self._restart(self.step, [self.em_masks] if self.use_external_memory else [])
        self.step = 0

    def compute_returns(self, next_value, use_gae, gamma, tau):
        self._returns(self.step, next_value, use_gae, gamma, tau)

    def recurrent_generator(self, advantages, num_mini_batch):
        def memory(cols, rows, nb):
            if not self.use_external_memory:
                return None, None
            store = self.em.memory[:, :rows].index_select(2, cols).reshape(-1, rows * nb, self.em_dim)
            return store, self.em_masks[:rows].index_select(1, cols).reshape(rows * nb, -1)
        return self._batches(advantages, num_mini_batch, self.step, memory)


class PPO:
    """``PPO.get_advantages`` of av_nav/ppo/ppo.py and savi/ppo/ppo.py."""

    def __init__(self, use_normalized_advantage=True):
        self.use_normalized_advantage = use_normalized_advantage

    def get_advantages(self, rollouts):
        advantages = rollouts.returns[:-1] - rollouts.value_preds[:-1]
        if not self.use_normalized_advantage:
            return advantages
        return (advantages - advantages.mean()) / (advantages.std() + EPS_PPO)


# ---------------------------------------------------------------------------------------------------------------------
# seeded scripts.  name: dict(kind, N, S, sensors, layers, hidden, [em (size, capacity, dim)], rollouts, done_p, seed)
SCRIPTS = {
    "common": dict(kind="common", N=4, S=7, sensors={"spectrogram": (3, 2, 2), "depth": (4, 2, 1), "pointgoal": (2,)},
                   layers=1, hidden=5, rollouts=2, done_p=0.25, seed=1),
    "common_wan": dict(kind="common", N=4, S=6, sensors={"spectrogram": (2, 3, 2), "gm": (3, 3, 2), "am": (2, 2, 1),
                                                          "action_map": (3, 3, 1)},
                       layers=2, hidden=3, rollouts=2, done_p=0.3, seed=2),
    "savi": dict(kind="savi", N=4, S=6, sensors={"spectrogram": (2, 2, 2), "rgb": (2, 3, 3), "category": (3,)},
                 layers=1, hidden=4, em=(11, 5, 3), rollouts=2, done_p=0.15, seed=3),
    "savi_no_memory": dict(kind="savi", N=4, S=5, sensors={"depth": (2, 2, 1)}, layers=1, hidden=3, em=(9, 4, 2),
                           use_em=False, rollouts=2, done_p=0.3, seed=4),
}
MINI_BATCHES = (1, 2, 4)
GAE = {True: (0.99, 0.95), False: (0.98, 0.0)}
GENERATOR_SEEDS = (101, 102, 103)


def make_storage(script, classes, device="cpu"):
    """A storage of ``script`` from ``classes`` (dict common=, savi=), moved to ``device``."""
    sp, act = spaces(script["sensors"]), ActionSpace()
    if script["kind"] == "common":
        st = classes["common"](script["S"], script["N"], sp, act, script["hidden"], script["layers"])
    else:
        size, cap, dim = script["em"]
        st = classes["savi"](script["S"], script["N"], sp, act, script["hidden"], script.get("use_em", True), size,
                             cap, dim, script["layers"])
    st.to(device)
    return st


def step_inputs(script, g):
    """One step's insert arguments from the numpy generator ``g`` (CPU tensors, float32 / int64; numpy's generator
    draws the same numbers on every machine)."""
    N = script["N"]
    f32 = lambda *shape: torch.from_numpy(g.standard_normal(shape, dtype=np.float32))  # noqa: E731
    obs = {k: f32(N, *s) for k, s in script["sensors"].items()}
    hidden = f32(script["layers"], N, script["hidden"])
    actions = torch.from_numpy(g.integers(0, 4, (N, 1), dtype=np.int64))
    log_probs = -torch.from_numpy(g.random((N, 1), dtype=np.float32))
    values = f32(N, 1)
    rewards = f32(N, 1) * 0.5
    masks = torch.from_numpy((g.random((N, 1)) >= script["done_p"]).astype(np.float32))
    args = [obs, hidden, actions, log_probs, values, rewards, masks]
    if script["kind"] == "savi":
        args.append(f32(N, script["em"][2]))
    return args


def to_device(args, device, host=False):
    """``args`` on ``device``; with ``host`` the observations, rewards and masks stay on the CPU, as the stock AV-Nav
    and AV-WaN trainers pass them (``batch_obs(observations)`` without a device, CPU-built rewards and masks)."""
    out = []
    for i, a in enumerate(args):
        if isinstance(a, dict):
            out.append({k: v if host else v.to(device) for k, v in a.items()})
        elif host and i in (5, 6):
            out.append(a)
        else:
            out.append(a.to(device))
    return out


def _np(t):
    """A numpy copy of ``t`` (``.numpy()`` of a CPU tensor would share, and follow, the storage's memory)."""
    return t.detach().cpu().numpy().copy()


def state(st):
    """Every tensor of a storage, by name, as CPU numpy."""
    d = {f"obs_{k}": v for k, v in st.observations.items()}
    for name in ("recurrent_hidden_states", "rewards", "value_preds", "returns", "action_log_probs", "actions",
                 "prev_actions", "masks"):
        d[name] = getattr(st, name)
    if getattr(st, "use_external_memory", False):
        d.update(em_memory=st.em.memory, em_masks_mem=st.em.masks, em_masks=st.em_masks)
    return {k: _np(v) for k, v in d.items()}


def batch_arrays(batch):
    """A minibatch tuple as {name: numpy}."""
    names = ("hidden", "actions", "prev_actions", "value_preds", "returns", "masks", "log_probs", "adv",
             "em_store", "em_masks")
    d = {f"obs_{k}": v for k, v in batch[0].items()}
    d.update({n: t for n, t in zip(names, batch[1:]) if t is not None})
    return {k: _np(v) for k, v in d.items()}


def run_script(script, classes, ppo_cls, use_gae, device="cpu", host=False, on_insert=None):
    """Run ``script`` and return {key: numpy}: per rollout r, the state after its last insert (``r/state/*``), the
    returns (``r/returns``, ``r/value_preds``), the advantages (``r/adv``), every minibatch of every entry of
    MINI_BATCHES after ``torch.manual_seed``, stacked (``r/mb{m}/*``), four draws of torch's RNG after each generator
    (``r/mb{m}/rng``) and the state after ``after_update``.
    ``on_insert(storage)`` runs after every insert."""
    g = np.random.default_rng(script["seed"])
    st = make_storage(script, classes, device)
    first = step_inputs(script, g)[0]
    for k, v in first.items():
        st.observations[k][0].copy_(v.to(device))
    gamma, tau = GAE[use_gae]
    ppo = ppo_cls.__new__(ppo_cls)
    ppo.use_normalized_advantage = True
    out = {}
    for r in range(script["rollouts"]):
        for _ in range(script["S"]):
            st.insert(*to_device(step_inputs(script, g), device, host))
            if on_insert is not None:
                on_insert(st)
        out.update({f"{r}/state/{k}": v for k, v in state(st).items()})
        next_value = torch.from_numpy(g.standard_normal((script["N"], 1), dtype=np.float32)).to(device)
        st.compute_returns(next_value, use_gae, gamma, tau)
        out[f"{r}/returns"] = _np(st.returns)
        out[f"{r}/value_preds"] = _np(st.value_preds)
        adv = ppo.get_advantages(st)
        out[f"{r}/adv"] = _np(adv)
        for m, seed in zip(MINI_BATCHES, GENERATOR_SEEDS):
            torch.manual_seed(seed)
            batches = [batch_arrays(batch) for batch in st.recurrent_generator(adv, m)]
            out.update({f"{r}/mb{m}/{k}": np.stack([b[k] for b in batches]) for k in batches[0]})
            out[f"{r}/mb{m}/rng"] = torch.randint(2 ** 62, (4,)).numpy()   # where the generator left torch's RNG
        st.after_update()
        out.update({f"{r}/after/{k}": v for k, v in state(st).items()})
    return out


def golden_key(name, use_gae):
    return f"{name}/{'gae' if use_gae else 'plain'}"


def advantages64(returns, value_preds):
    """The normalised advantages in float64 from float32 returns and value predictions."""
    a = returns[:-1].astype(np.float64) - value_preds[:-1].astype(np.float64)
    return (a - a.mean()) / (a.std(ddof=1) + EPS_PPO)
