"""Trainer side of ``remote_frames``: the RGB and depth frames remote env workers send once, kept in device banks and
gathered into a step's visual batch with one launch.

With ``patch_simulator(..., deferred="remote", remote_frames=True)`` a worker pickles each rendered frame's data the
first time and only its key afterwards (:class:`~soundspaces_b200.remote.FrameArray`); the trainer receives
:class:`~soundspaces_b200.remote.FrameRef` s, and every frame that carried data lands in the process's host dict
(``remote._FRAMES``), which keeps every frame received.  A :class:`FrameStore` per (device, uuid, dtype, shape) keeps
a device bank of those frames in the sensor's own dtype (uint8 RGB, float32 depth) with least-recently-used eviction
under a byte cap; a frame that is not resident is uploaded again from the host dict, so a frame a worker believes it
has shipped is never lost.  :func:`gather` resolves a step: one batched host-to-device copy of the step's misses
(none on a step without misses), then ONE ``ssb_frame_gather_batch`` launch for every visual sensor, writing the
float32 ``(N, H, W, C)`` batch -- or the rollout slots named by ``out``.
"""
from __future__ import annotations

from collections import OrderedDict
from typing import Dict, List, Optional, Sequence

import numpy as np
import torch

from . import _lib
from .remote import _FRAMES, FrameRef, frame_data

DEFAULT_BANK_BYTES = 2 << 30


class FrameStore:
    """Device bank of one visual sensor's frames.  :meth:`plan` is the host half of a step (bank rows, LRU order,
    eviction), :func:`gather` the device half.  The bank holds ``max(1, max_bank_bytes // row_bytes)`` rows, and at
    least the distinct frames of one step: a step that needs more drops every resident frame and starts a bank that
    large (``stats["regrown"]``)."""

    _instances: Dict[tuple, "FrameStore"] = {}

    def __init__(self, device, uuid: str, dtype, shape, max_bank_bytes: int = DEFAULT_BANK_BYTES):
        self.device = torch.device(device)
        self.uuid, self.dtype, self.shape = uuid, np.dtype(dtype), tuple(int(x) for x in shape)
        if self.dtype not in _lib.FRAME_DTYPES:
            raise ValueError(f"sensor {uuid!r}: frames of dtype {self.dtype} are not gathered on the device "
                             "(uint8 and float32 are)")
        self.row_elems = int(np.prod(self.shape, dtype=np.int64))
        self.row_bytes = self.row_elems * self.dtype.itemsize
        self.max_bank_bytes = int(max_bank_bytes)
        self.capacity = max(1, self.max_bank_bytes // max(1, self.row_bytes))
        self.bank: Optional[torch.Tensor] = None       # (capacity, row_elems), allocated on first use
        self._rows: "OrderedDict[tuple, int]" = OrderedDict()      # key -> bank row, least recently used first
        self._free: List[int] = list(range(self.capacity - 1, -1, -1))
        self.stats = {"hits": 0, "misses": 0, "evictions": 0, "regrown": 0}

    @classmethod
    def get(cls, device, uuid: str, dtype, shape, max_bank_bytes: Optional[int] = None) -> "FrameStore":
        key = (str(torch.device(device)), uuid, np.dtype(dtype).str, tuple(shape))
        inst = cls._instances.get(key)
        if inst is None:
            inst = cls._instances[key] = cls(device, uuid, dtype, shape,
                                             DEFAULT_BANK_BYTES if max_bank_bytes is None else max_bank_bytes)
        elif max_bank_bytes is not None and int(max_bank_bytes) != inst.max_bank_bytes:
            raise ValueError(f"FrameStore for {key} already exists with max_bank_bytes={inst.max_bank_bytes}, "
                             f"asked for {max_bank_bytes}")
        return inst

    def resident(self, key) -> bool:
        return key in self._rows

    def plan(self, keys: Sequence[tuple]):
        """Bank rows for one step's frame keys (one per env): ``(index, fill, staged)`` -- ``index[i]`` the bank row
        env i reads, or ``-1 - j`` for the j-th staged frame; ``fill[j]`` the bank row staged frame j is written to;
        ``staged`` the keys to upload, in staging order.  The step's resident keys become the most recently used
        before any row is given away, so eviction never takes a frame the step reads."""
        distinct = dict.fromkeys(keys)                     # first-use order
        if len(distinct) > self.capacity:
            self.capacity = len(distinct)
            self.bank = None
            self._rows.clear()
            self._free = list(range(self.capacity - 1, -1, -1))
            self.stats["regrown"] += 1
        for k in distinct:
            if k in self._rows:
                self._rows.move_to_end(k)
        index, fill, staged = [], [], {}
        for k in keys:
            j = staged.get(k)
            if j is None:
                row = self._rows.get(k)
                if row is not None:
                    self.stats["hits"] += 1
                    index.append(row)
                    continue
                j = staged[k] = len(fill)
                if self._free:
                    row = self._free.pop()
                else:
                    _, row = self._rows.popitem(last=False)
                    self.stats["evictions"] += 1
                fill.append(row)
                self._rows[k] = row
                self.stats["misses"] += 1
            index.append(-1 - j)
        return index, fill, list(staged)


def _align16(n: int) -> int:
    return (n + 15) & ~15


def _row_contiguous(t: torch.Tensor, n: int, shape) -> bool:
    return (t.dtype == torch.float32 and tuple(t.shape) == (n,) + tuple(shape) and (n == 0 or t[0].is_contiguous())
            and t.stride(0) >= max(1, int(np.prod(shape))))


def gather(by_sensor: Dict[str, List[FrameRef]], device, out: Optional[Dict[str, torch.Tensor]] = None,
           max_bank_bytes: Optional[int] = None) -> Dict[str, torch.Tensor]:
    """The step's visual batch: ``{uuid: (N, *shape) float32 CUDA tensor}`` for sensors whose values are all
    :class:`FrameRef`, written into ``out[uuid]`` when given (a rollout slot; any row stride).  Every frame must be
    resident or in the host dict (``RuntimeError`` naming the key otherwise, checked before any state changes).  One
    host-to-device copy uploads every sensor's misses, then one launch gathers every sensor (up to
    ``_lib.FRAME_MAX_SENSORS`` per launch)."""
    device = torch.device(device)
    jobs, res = [], {}
    for uuid, refs in by_sensor.items():
        n = len(refs)
        if n == 0:
            raise ValueError(f"sensor {uuid!r}: no frames to gather")
        r0 = refs[0]
        if any(r.dtype != r0.dtype or r.shape != r0.shape for r in refs):
            raise ValueError(f"sensor {uuid!r}: one step's frames must share one dtype and shape")
        if n > _lib.FRAME_MAX_N:
            raise ValueError(f"sensor {uuid!r}: {n} envs in one step, the frame gather takes at most "
                             f"{_lib.FRAME_MAX_N}")
        store = FrameStore.get(device, uuid, r0.dtype, r0.shape, max_bank_bytes)
        for r in refs:
            if not store.resident(r.key):
                frame_data(r)                                  # raises when the frame never reached this process
        jobs.append((uuid, store, refs))
    plans = [store.plan([r.key for r in refs]) for _, store, refs in jobs]
    # one pinned staging buffer for every sensor's misses, one copy to the device
    offsets, total = [], 0
    for (_, store, _), (_, _, staged) in zip(jobs, plans):
        offsets.append(total)
        total += _align16(len(staged) * store.row_bytes)
    stage_dev = None
    if total:
        host = torch.empty(total, dtype=torch.uint8, pin_memory=True)
        hv = host.numpy()
        for (_, store, _), (_, _, staged), off in zip(jobs, plans, offsets):
            for j, k in enumerate(staged):
                a = _FRAMES.get(k)
                if a is None:
                    a = next(r.data for r in by_sensor[store.uuid] if r.key == k)
                o = off + j * store.row_bytes
                hv[o: o + store.row_bytes] = np.ascontiguousarray(a, dtype=store.dtype).reshape(-1).view(np.uint8)
        stage_dev = host.to(device, non_blocking=True)
    launch: Dict[int, list] = {}
    for (uuid, store, refs), (index, fill, staged), off in zip(jobs, plans, offsets):
        if store.bank is None:
            store.bank = torch.empty((store.capacity, store.row_elems), dtype=getattr(torch, store.dtype.name),
                                     device=device)
        n = len(refs)
        dst = out.get(uuid) if out else None
        direct = dst is not None and dst.device == device and _row_contiguous(dst, n, store.shape)
        t = dst if direct else torch.empty((n,) + store.shape, dtype=torch.float32, device=device)
        stage = None
        if staged:
            stage = stage_dev[off: off + len(staged) * store.row_bytes].view(store.bank.dtype).view(len(staged), -1)
        launch.setdefault(n, []).append((store.bank, stage, t.view(n, store.row_elems), index, fill))
        res[uuid] = (t, dst if dst is not None and not direct else None)
    ops = _ops(device)
    for n, group in launch.items():                      # one launch per step: every sensor has one value per env
        for q0 in range(0, len(group), _lib.FRAME_MAX_SENSORS):
            ops.frame_gather(n, group[q0: q0 + _lib.FRAME_MAX_SENSORS])
    result = {}
    for uuid, (t, dst) in res.items():
        result[uuid] = dst.copy_(t) if dst is not None else t
    return result


def _ops(device):
    from .renderer import WaveformOps
    return WaveformOps.get(device)
