"""PPO's rollout storage on the device: ``RolloutStorage.insert``, ``compute_returns``, ``recurrent_generator`` and
``after_update`` of ss_baselines/common/rollout_storage.py (AV-Nav, AV-WaN) and savi/models/rollout_storage.py (SAVi,
with its ``ExternalMemory``), and ``PPO.get_advantages`` (av_nav/ppo/ppo.py, savi/ppo/ppo.py), each in one launch.

    from soundspaces_b200.rollout import patch_rollout_storage, patch_external_memory, patch_ppo
    patch_rollout_storage(RolloutStorage)    # ss_baselines.common.rollout_storage / savi.models.rollout_storage
    patch_external_memory(ExternalMemory)    # savi.models.rollout_storage (the evaluation loop's memory)
    patch_ppo(PPO)                           # ss_baselines.av_nav.ppo.ppo / savi.ppo.ppo

One launch per ``insert`` (``ssb_rollout_insert_batch``: every slot copy, SAVi's memory update, and rewards / masks
that arrive on the host staged through a pinned ring, with no stream synchronisation), one per ``compute_returns``
(``ssb_rollout_returns_batch``: the returns, bit-identical to the eager loop, and the normalised advantages
``get_advantages`` then takes), one per minibatch and one per ``after_update`` (``ssb_rollout_gather_batch``).  The
reference asserts at every SAVi insert that no memory row holds more than ``capacity`` entries; the patched storage
counts such rows in a device status word instead and reads it once per rollout, in ``compute_returns``, which raises
the reference's ``AssertionError`` there (naming the env rows and the first step), not at the insert that overflowed.
Storage that does not qualify (:func:`rollout_layout_error`) and calls whose arguments do not run the original.
"""
from __future__ import annotations

import inspect
import math
from collections import defaultdict

import torch

MAX_FIELDS = 32         # the kernels' limits (include/ssb200.h, ssb_rollout_*)
MAX_COLS = 256
MAX_ENVS = 65535
MAX_STEPS = 4096
MAX_MEMORY = 16384
MAX_SENSORS = MAX_FIELDS - 10    # a minibatch's fields: the sensors, the hidden state, 7 more, the memory and its masks


def _ops(device):
    from .renderer import WaveformOps
    return WaveformOps.get(device)


def _unwrap(fn):
    return getattr(fn, "_ssb_original", fn)


def _slot(t, k):
    """Byte address of ``t[k]`` of a contiguous tensor."""
    return t.data_ptr() + k * t.stride(0) * t.element_size()


def _slot_bytes(t):
    return t.stride(0) * t.element_size()


def _memory_error(em, N, device) -> str:
    """Why SAVi's ``em`` is not an ``ExternalMemory`` whose insert the kernel runs; ``""`` when it is."""
    base = next((c for c in type(em).__mro__ if c.__name__ == "ExternalMemory"), None)
    if base is None or _unwrap(type(em).insert) is not _unwrap(base.__dict__["insert"]):
        return f"its memory is {type(em).__name__}, whose insert is its own"
    if type(em.idx) is not int:
        return f"its memory's idx is {type(em.idx).__name__}, not int"
    mem, masks = em.memory, em.masks
    for name, t in (("em.memory", mem), ("em.masks", masks)):
        if not (isinstance(t, torch.Tensor) and t.device == device and t.dtype == torch.float32 and t.is_contiguous()):
            return f"{name} is not a contiguous float32 tensor on {device}"
    if mem.ndim != 4 or masks.ndim != 2 or mem.shape[2] != N or tuple(masks.shape) != (N, mem.shape[0]):
        return f"em.memory {tuple(mem.shape)} and em.masks {tuple(masks.shape)} do not hold {N} envs"
    if mem.shape[0] > MAX_MEMORY or not 0 <= em.capacity <= mem.shape[0]:
        return (f"a memory of {mem.shape[0]} slots and capacity {em.capacity}, the kernel takes at most {MAX_MEMORY} "
                "slots and a capacity within them")
    return ""


def rollout_layout_error(storage) -> str:
    """Why ``storage`` is not a reference ``RolloutStorage`` the kernels run; ``""`` when it is.  The layout is
    recognised by its tensors: SAVi's (``use_external_memory``, ``em``, ``em_masks``, ``step`` counting up) or
    the common one (``step`` wrapping at ``num_steps``).  It qualifies when every tensor is contiguous on one CUDA
    device, the float fields are float32, and N, num_steps and the sensor count are within the kernels' limits."""
    rhs = getattr(storage, "recurrent_hidden_states", None)
    if isinstance(rhs, torch.Tensor) and not rhs.is_cuda:
        return "the storage is on the CPU"
    return _layout_error(storage, rhs.device if isinstance(rhs, torch.Tensor) else None)


def _layout_error(storage, device) -> str:
    """:func:`rollout_layout_error`'s checks with every tensor on ``device``."""
    obs = getattr(storage, "observations", None)
    rhs = getattr(storage, "recurrent_hidden_states", None)
    if not isinstance(obs, dict) or not isinstance(rhs, torch.Tensor):
        return "no observations dict or recurrent_hidden_states tensor"
    S = storage.num_steps
    if rhs.ndim != 4 or rhs.shape[0] != S + 1:
        return f"recurrent_hidden_states has shape {tuple(rhs.shape)}, expected ({S + 1}, layers, N, hidden)"
    N = rhs.shape[2]
    named = [("recurrent_hidden_states", rhs, S + 1)] + [(f"observations[{k!r}]", v, S + 1) for k, v in obs.items()]
    named += [("rewards", storage.rewards, S), ("value_preds", storage.value_preds, S + 1),
              ("returns", storage.returns, S + 1), ("action_log_probs", storage.action_log_probs, S),
              ("actions", storage.actions, S), ("prev_actions", storage.prev_actions, S + 1),
              ("masks", storage.masks, S + 1)]
    if getattr(storage, "use_external_memory", False):
        named.append(("em_masks", storage.em_masks, S + 1))
    for name, t, rows in named:
        if not isinstance(t, torch.Tensor) or t.device != device:
            return f"{name} is not a tensor on {device}"
        if not t.is_contiguous():
            return f"{name} is not contiguous"
        if t.ndim < 2 or t.shape[0] != rows or t.shape[1] != N and name != "recurrent_hidden_states":
            return f"{name} has shape {tuple(t.shape)}, expected ({rows}, {N}, ...)"
    for name in ("rewards", "value_preds", "returns", "action_log_probs", "masks"):
        t = getattr(storage, name)
        if t.dtype != torch.float32 or tuple(t.shape) != (t.shape[0], N, 1):
            return f"{name} is not float32 ({t.shape[0]}, {N}, 1)"
    if storage.actions.dtype != storage.prev_actions.dtype or storage.actions.shape[2:] != storage.prev_actions.shape[2:]:
        return "actions and prev_actions differ in dtype or shape"
    if N > MAX_ENVS or S > MAX_STEPS or S < 1 or len(obs) > MAX_SENSORS:
        return (f"N={N}, num_steps={S} and {len(obs)} sensors, the kernels take at most {MAX_ENVS} envs, {MAX_STEPS} "
                f"steps and {MAX_SENSORS} sensors")
    if getattr(storage, "use_external_memory", False):
        err = _memory_error(storage.em, N, device)
        if err:
            return err
        em = storage.em
        if em.memory.shape[1] != S + 1 or tuple(storage.em_masks.shape) != (S + 1, N, em.memory.shape[0]) \
                or storage.em_masks.dtype != torch.float32:
            return "em.memory or em_masks does not have num_steps + 1 float32 copies of the memory"
    return ""


def _layout_key(storage):
    """What :func:`rollout_layout_error`'s verdict depends on that can change without an in-place edit: the objects
    the storage holds (kept alive in the cache, so their ids cannot be reused) and their data pointers."""
    obs = getattr(storage, "observations", None)
    em = getattr(storage, "em", None)
    objs = [obs, em, getattr(em, "memory", None), getattr(em, "masks", None), getattr(storage, "em_masks", None)]
    objs += [getattr(storage, n, None) for n in ("recurrent_hidden_states", "rewards", "value_preds", "returns",
                                                  "action_log_probs", "actions", "prev_actions", "masks")]
    if isinstance(obs, dict):
        objs += list(obs.values())
    ptrs = tuple(o.data_ptr() if isinstance(o, torch.Tensor) else None for o in objs)
    extra = (getattr(storage, "num_steps", None), getattr(storage, "use_external_memory", None), type(em),
             type(getattr(em, "idx", None)), getattr(em, "capacity", None), getattr(type(em), "insert", None))
    return objs, ptrs, extra


def _cached_layout_error(storage) -> str:
    """:func:`rollout_layout_error`, re-evaluated only when :func:`_layout_key` changes.  In-place changes of a held
    tensor's shape, strides, dtype or device (``resize_``, ``t_``) are not seen: the reference never makes them."""
    objs, ptrs, extra = _layout_key(storage)
    cached = storage.__dict__.get("_ssb_layout")
    if (cached is not None and len(cached[0]) == len(objs) and all(a is b for a, b in zip(cached[0], objs))
            and cached[1] == ptrs and cached[2] == extra):
        return cached[3]
    err = rollout_layout_error(storage)
    storage.__dict__["_ssb_layout"] = (objs, ptrs, extra, err)
    return err


def _is_savi(storage) -> bool:
    return hasattr(storage, "use_external_memory")


def _dense_like(t, store, drop=1) -> bool:
    """``t`` can be copied as bytes into ``store`` from ``store``'s device (:func:`_source` 0)."""
    return _source(t, store, drop) == 0


def _source(t, store, drop=1):
    """How ``t`` is copied as bytes into ``store`` with its first ``drop`` dims indexed: 0 from the device, 1 from the
    host (a CPU tensor, staged by the library), None when it cannot be (not a contiguous tensor of that shape and of
    ``store``'s dtype on ``store``'s device or the CPU)."""
    if not (isinstance(t, torch.Tensor) and t.dtype == store.dtype and t.shape == store.shape[drop:]
            and t.is_contiguous()):
        return None
    if t.device == store.device:
        return 0
    return 1 if t.device.type == "cpu" else None


def _status(holder, N, device):
    st = getattr(holder, "_ssb_em_status", None)
    if st is None or st.numel() != N + 1 or st.device != device:
        st = torch.zeros(N + 1, dtype=torch.int32, device=device)
        holder._ssb_em_status = st
    return st


def _overflow_error(status_list, what, steps=True):
    """The reference's ``assert(not torch.any(self.masks.sum(1) > self.capacity))`` from a status word read back."""
    rows = [e for e, s in enumerate(status_list[1:]) if s]
    where = f" (first at step {min(status_list[1 + e] for e in rows) - 1})" if steps else ""
    return AssertionError(f"{what}: the external memory of env rows {rows} held more than its capacity{where}")


def _insert(self, signature, args, kwargs):
    """The patched ``insert``'s launch, or False when the call must run the original."""
    savi = _is_savi(self)
    if savi and self.step >= self.num_steps:
        return False
    n_args = len(signature.parameters) - 1
    values = args if not kwargs and len(args) == n_args else list(signature.bind(self, *args, **kwargs).arguments.values())[1:]
    observations, hidden, actions, log_probs, values_, rewards, masks = values[:7]
    em_features = values[7] if savi else None
    rhs = self.recurrent_hidden_states
    device, N, step = rhs.device, rhs.shape[2], self.step
    fields = []
    for sensor, t in observations.items():
        slot = self.observations.get(sensor)
        where = None if slot is None else _source(t, slot)
        if where is None:
            return False
        if t.data_ptr() != _slot(slot, step + 1):      # rendered in place: nothing to copy, as copy_ does
            fields.append((t.data_ptr(), _slot(slot, step + 1), _slot_bytes(slot), 0, 0, 1, 1, where))
    for t, slot, k in ((hidden, rhs, step + 1), (actions, self.actions, step), (actions, self.prev_actions, step + 1),
                       (log_probs, self.action_log_probs, step), (values_, self.value_preds, step),
                       (rewards, self.rewards, step), (masks, self.masks, step + 1)):
        where = _source(t, slot)
        if where is None:
            return False
        fields.append((t.data_ptr(), _slot(slot, k), _slot_bytes(slot), 0, 0, 1, 1, where))
    memory = None
    if savi and self.use_external_memory:
        em = self.em
        if not _dense_like(em_features, em.memory, 2):
            return False
        fields.append((em_features.data_ptr(), _slot(em.memory, em.idx), _slot_bytes(em.memory[0]), 0, 0, 1,
                       em.memory.shape[1], 0))
        memory = dict(masks=em.masks, not_done=masks, em_masks_out=self.em_masks[step + 1],
                      status=_status(self, N, device), capacity=em.capacity, idx=em.idx, step=step)
    _ops(device).rollout_insert(N, [f for f in fields if f[2] > 0], memory=memory)
    if memory is not None:
        self.em.idx = (self.em.idx + 1) % self.em.memory.shape[0]
    self.step = step + 1 if savi else (step + 1) % self.num_steps
    return True


def _rows(self) -> int:
    """Steps a rollout holds: ``num_steps`` in common, ``step`` in SAVi."""
    return self.step if _is_savi(self) else self.num_steps


def patch_rollout_storage(cls):
    """Replace ``insert``, ``compute_returns``, ``recurrent_generator`` and ``after_update`` of a reference
    ``RolloutStorage`` class in place; the originals stay reachable as ``._ssb_original`` and patching twice changes
    nothing.  Each method runs the original for storage that does not qualify (:func:`rollout_layout_error`), and
    ``insert`` / ``compute_returns`` / ``recurrent_generator`` also for arguments that do not: tensors not of the
    slot's shape and dtype, contiguous on the storage's device (rewards and masks may be float32 CPU tensors),
    a ``next_value`` not float32 (N, 1) there, or advantages not contiguous there."""
    orig_insert = _unwrap(cls.insert)
    orig_returns = _unwrap(cls.compute_returns)
    orig_generator = _unwrap(cls.recurrent_generator)
    orig_after = _unwrap(cls.after_update)
    insert_signature = inspect.signature(orig_insert)

    def insert(self, *args, **kwargs):
        self.__dict__.pop("_ssb_advantages", None)
        if _cached_layout_error(self) or not _insert(self, insert_signature, args, kwargs):
            return orig_insert(self, *args, **kwargs)

    def compute_returns(self, next_value, use_gae, gamma, tau):
        self.__dict__.pop("_ssb_advantages", None)
        status = getattr(self, "_ssb_em_status", None)
        if status is not None and getattr(self, "use_external_memory", False):
            st = status.tolist()                        # the patched storage's one host read per rollout
            if st[0]:
                status.zero_()                          # raise once per overflow, not at every later rollout
                raise _overflow_error(st, "RolloutStorage.insert")
        vp = self.value_preds
        if (_cached_layout_error(self) or not isinstance(next_value, torch.Tensor) or next_value.device != vp.device
                or next_value.dtype != torch.float32 or not next_value.is_contiguous()
                or next_value.numel() != vp.shape[1]):
            return orig_returns(self, next_value, use_gae, gamma, tau)
        S, N = self.rewards.shape[0], vp.shape[1]
        adv = torch.empty((S, N, 1), dtype=torch.float32, device=vp.device)
        _ops(vp.device).rollout_returns(self.rewards, vp, self.returns, self.masks, next_value, _rows(self), use_gae,
                                        gamma, tau, adv=adv, normalize=True)
        self._ssb_advantages = (adv, vp.data_ptr(), vp._version, self.returns.data_ptr(), self.returns._version)

    def recurrent_generator(self, advantages, num_mini_batch):
        num_processes = self.rewards.size(1)
        T = _rows(self)
        if (_cached_layout_error(self) or num_mini_batch < 1 or num_processes % num_mini_batch
                or num_processes // num_mini_batch > MAX_COLS or T < 1
                or not isinstance(advantages, torch.Tensor) or advantages.device != self.rewards.device
                or not advantages.is_contiguous() or advantages.ndim < 2 or advantages.shape[0] < T
                or advantages.shape[1] != num_processes):
            yield from orig_generator(self, advantages, num_mini_batch)
            return
        assert num_processes >= num_mini_batch, (
            "Trainer requires the number of processes ({}) "
            "to be greater than or equal to the number of "
            "trainer mini batches ({}).".format(num_processes, num_mini_batch)
        )
        num_envs_per_batch = num_processes // num_mini_batch
        perm = torch.randperm(num_processes).tolist()
        savi = _is_savi(self)
        em = self.use_external_memory if savi else False
        ops = _ops(self.rewards.device)
        for start_ind in range(0, num_processes, num_envs_per_batch):
            nb = num_envs_per_batch
            fields, outs = [], []

            def take(src, rows, outer=1, o_stride=0, shape=None):
                """src[:rows, cols] of a (steps, N, ...) tensor as a fresh (rows * nb, ...) tensor."""
                row_bytes = math.prod(src.shape[2:]) * src.element_size()
                out = torch.empty(shape or (rows * nb,) + tuple(src.shape[2:]), dtype=src.dtype, device=src.device)
                fields.append((src.data_ptr(), out.data_ptr(), row_bytes, _slot_bytes(src), o_stride, rows, outer))
                outs.append(out)
                return out

            observations_batch = defaultdict(list)
            for sensor, t in self.observations.items():
                observations_batch[sensor] = take(t, T)
            rhs = self.recurrent_hidden_states        # rhs[0, :, cols] -> (layers, nb, hidden)
            hidden_batch = take(rhs[0], 1, outer=rhs.shape[1], o_stride=rhs.stride(1) * rhs.element_size(),
                                shape=(rhs.shape[1], nb, rhs.shape[3]))
            actions_batch = take(self.actions, T)
            prev_actions_batch = take(self.prev_actions, T)
            value_preds_batch = take(self.value_preds, T)
            return_batch = take(self.returns, T)
            masks_batch = take(self.masks, T)
            old_action_log_probs_batch = take(self.action_log_probs, T)
            adv_targ = take(advantages, T)
            em_store_batch = em_masks_batch = None
            if em:
                mem = self.em.memory                  # memory[:, :T, cols] -> (total, T * nb, dim)
                em_store_batch = take(mem[0], T, outer=mem.shape[0], o_stride=_slot_bytes(mem),
                                      shape=(mem.shape[0], T * nb, mem.shape[3]))
                em_masks_batch = take(self.em_masks, T)
            ops.rollout_gather(fields, nb, perm[start_ind:start_ind + nb], num_processes)
            out = (observations_batch, hidden_batch, actions_batch, prev_actions_batch, value_preds_batch,
                   return_batch, masks_batch, old_action_log_probs_batch, adv_targ)
            yield out + (em_store_batch, em_masks_batch) if savi else out

    def after_update(self):
        self.__dict__.pop("_ssb_advantages", None)
        if _cached_layout_error(self):
            return orig_after(self)
        savi = _is_savi(self)
        src = self.step if savi else self.num_steps
        slots = list(self.observations.values()) + [self.recurrent_hidden_states, self.masks, self.prev_actions]
        if savi and self.use_external_memory:
            slots.append(self.em_masks)
        fields = [(_slot(t, src), t.data_ptr(), _slot_bytes(t), 0, 0, 1, 1) for t in slots if src != 0]
        if fields:
            _ops(self.masks.device).rollout_gather(fields, 1)
        if savi:
            self.step = 0

    for name, fn, orig in (("insert", insert, orig_insert), ("compute_returns", compute_returns, orig_returns),
                           ("recurrent_generator", recurrent_generator, orig_generator),
                           ("after_update", after_update, orig_after)):
        fn._ssb_original = orig
        fn.__doc__ = orig.__doc__
        setattr(cls, name, fn)
    return cls


def patch_external_memory(cls):
    """Replace ``cls.insert`` of SAVi's ``ExternalMemory`` in place (the evaluation loop's memory,
    savi/ppo/ppo_trainer.py:844); the original stays reachable as ``cls.insert._ssb_original`` and patching twice
    changes nothing.  One launch writes the features into every copy at ``idx`` and updates the masks; it then reads
    the status word (one host sync; the reference makes two) and raises the reference's ``AssertionError``, without
    advancing ``idx``, when a row held more than ``capacity`` entries.  Unlike the reference, which asserts before it
    touches the masks, the memory is then left with the features at ``idx`` AND every row's masks updated (the
    overflowing rows included); the status word is cleared, so the next call raises only for a new overflow.
    Memories that do not qualify, features not a contiguous float32 (N, dim) tensor on the memory's device, or masks
    not a contiguous float32 (N, 1) tensor there or on the CPU run the original."""
    original = _unwrap(cls.insert)

    def insert(self, em_features, not_done_masks):
        mem = self.memory
        if not (isinstance(mem, torch.Tensor) and mem.is_cuda):
            return original(self, em_features, not_done_masks)
        N, device = mem.shape[2] if mem.ndim == 4 else -1, mem.device
        if (_memory_error(self, N, device) or not _dense_like(em_features, mem, 2)
                or _source(not_done_masks, self.masks[:, :1], 0) is None):
            return original(self, em_features, not_done_masks)
        status = _status(self, N, device)
        fields = [(em_features.data_ptr(), _slot(mem, self.idx), _slot_bytes(mem[0]), 0, 0, 1, mem.shape[1], 0)]
        memory = dict(masks=self.masks, not_done=not_done_masks, em_masks_out=None, status=status,
                      capacity=self.capacity, idx=self.idx, step=0)
        _ops(device).rollout_insert(N, fields, memory=memory)
        st = status.tolist()
        if st[0]:
            status.zero_()
            raise _overflow_error(st, "ExternalMemory.insert", steps=False)
        self.idx = (self.idx + 1) % self.total_size

    insert._ssb_original = original
    insert.__doc__ = original.__doc__
    cls.insert = insert
    return cls


def patch_ppo(cls):
    """Replace ``cls.get_advantages`` of a reference ``PPO`` in place; the original stays reachable as
    ``cls.get_advantages._ssb_original`` and patching twice changes nothing.  With normalised advantages, it returns
    those the patched ``compute_returns`` wrote (once: a second call computes them afresh) when the storage has not
    changed since, computes them in one launch
    of ``ssb_rollout_returns_batch`` for other storage whose returns and value predictions are contiguous float32
    (S + 1, N, 1) CUDA tensors, and runs the original otherwise.  DD-PPO's ``_get_advantages_distributed``, set on
    the instance, shadows this class attribute and keeps working unchanged."""
    original = _unwrap(cls.get_advantages)

    def get_advantages(self, rollouts):
        if not self.use_normalized_advantage:
            return original(self, rollouts)
        ret, vp = rollouts.returns, rollouts.value_preds
        cached = getattr(rollouts, "_ssb_advantages", None)
        if cached is not None:
            del rollouts._ssb_advantages                # handed out once: a caller's in-place edit changes no cache
            if cached[1:] == (vp.data_ptr(), vp._version, ret.data_ptr(), ret._version):
                return cached[0]
        ok = all(isinstance(t, torch.Tensor) and t.is_cuda and t.dtype == torch.float32 and t.is_contiguous()
                 and t.ndim == 3 and t.shape[2] == 1 for t in (ret, vp))
        if not (ok and ret.shape == vp.shape and ret.device == vp.device and 2 <= ret.shape[0] <= MAX_STEPS + 1
                and ret.shape[1] <= MAX_ENVS):
            return original(self, rollouts)
        S, N = ret.shape[0] - 1, ret.shape[1]
        adv = torch.empty((S, N, 1), dtype=torch.float32, device=ret.device)
        _ops(ret.device).rollout_returns(None, vp, ret, None, None, 0, False, 0.0, 0.0, adv=adv, normalize=True,
                                         scan=False)
        return adv

    get_advantages._ssb_original = original
    get_advantages.__doc__ = original.__doc__
    cls.get_advantages = get_advantages
    return cls
