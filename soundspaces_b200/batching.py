"""Batching behind the per-env Habitat sensor API (SURVEY.md 7 "Batching across a per-env API", 8(b)).

Habitat calls ``Sensor.get_observation`` once per env (``ss_baselines/common/sync_vector_env.py:186-199``); the
reference renders inside that call, one env at a time.  Here the call only ENQUEUES a request and returns a
:class:`DeferredObservation` -- a ``(slot, generation)`` handle into a device ring owned by the
:class:`AudioObservationBatcher` -- and the whole step's requests are rendered by ONE ``render`` when the first
handle is resolved, normally by ``sensors.batch_obs`` (the replacement of ``ss_baselines/common/utils.py:126-153``),
which returns the ``(N, 65, T', 2)`` CUDA view of the ring without a copy.

Ownership (SURVEY.md 8(b)): the ring belongs to the batcher; a row stays valid until its slot is reused, which
happens after ``capacity`` further rows.  Handles that are still referenced at that point (the memoised
observations in a simulator's ``_spectrogram_cache``, simulator.py:696-699) are detached first -- they take a
private copy of their row -- so a handle NEVER shows another observation's data.
"""
from __future__ import annotations

import contextlib
import weakref
from typing import List, Optional, Sequence

import numpy as np
import torch

from .remote import WAVEFORM
from .renderer import AudioRequest


class DeferredObservation:
    """Handle to one env's ``(65, T', 2)`` spectrogram: pending until its batcher flushes, then a device row.

    ``resolve()`` gives the CUDA tensor; ``np.asarray(handle)`` / ``handle.numpy()`` give the host array the
    reference's sensor would have returned (compat: this forces a flush and one device->host copy); pickling
    (multiprocess ``habitat.VectorEnv`` workers) materialises the host array the same way."""

    __slots__ = ("_batcher", "slot", "generation", "_row", "shape", "__weakref__")
    dtype = np.dtype(np.float32)

    def __init__(self, batcher, slot: int, generation: int, shape):
        self._batcher, self.slot, self.generation, self._row, self.shape = batcher, slot, generation, None, tuple(shape)

    @property
    def pending(self) -> bool:
        return self._row is None and self.generation > self._batcher.flushed_generation

    def resolve(self) -> torch.Tensor:
        if self._row is not None:                      # detached (private copy)
            return self._row
        b = self._batcher
        if self.generation > b.flushed_generation:
            b.flush()
        return b.ring[self.slot]

    def detach(self):
        """Take a private copy of the row (called by the batcher before the slot is reused)."""
        if self._row is None:
            self._row = self.resolve().clone()
        return self

    def numpy(self) -> np.ndarray:
        return self.resolve().cpu().numpy()

    def __array__(self, dtype=None, copy=None):
        a = self.numpy()
        return a.astype(dtype) if dtype is not None and a.dtype != dtype else a

    def __reduce__(self):
        return (np.asarray, (self.numpy(),))


class AudioObservationBatcher:
    """Queue of one step's audio requests + the device ring their spectrograms are rendered into."""

    def __init__(self, service, capacity: int = 1024):
        self.service = service
        self.renderer = service.renderer
        self.capacity = int(capacity)
        self.ring: Optional[torch.Tensor] = None       # (capacity, 65, T', 2), allocated on first flush
        self._owners: List[Optional[weakref.ref]] = [None] * self.capacity
        self._pending: List[tuple] = []                # (handle, request, crossfade_from)
        self._next = 0                                 # next free slot
        self.generation = 1                            # generation of the handles being enqueued now
        self.flushed_generation = 0
        self.flushes = 0

    # ------------------------------------------------------------------ enqueue
    def enqueue(self, request: AudioRequest, crossfade_from: Optional[AudioRequest] = None) -> DeferredObservation:
        if len(self._pending) >= self.capacity:
            self.flush()
        if self._next + len(self._pending) >= self.capacity:       # keep a step's rows contiguous: wrap to slot 0
            if self._pending:
                self.flush()
            self._next = 0
        slot = self._next + len(self._pending)
        old = self._owners[slot]
        if old is not None:
            h = old()
            if h is not None and h._row is None:
                h.detach()                              # still referenced (memoised): give it its own copy first
        handle = DeferredObservation(self, slot, self.generation, self.renderer.spec_shape)
        self._owners[slot] = weakref.ref(handle)
        self._pending.append((handle, request, crossfade_from))
        return handle

    # -------------------------------------------------------------------- flush
    def flush(self, out: Optional[torch.Tensor] = None):
        """Render every pending request with ONE launch chain.  ``out``: render straight into this
        ``(n_pending, 65, T', 2)`` CUDA tensor instead of the ring (rollout-storage slot, SURVEY.md N2); the ring
        rows are then filled by one device copy so that the handles stay valid."""
        if not self._pending:
            return None
        r = self.renderer
        if self.ring is None:
            self.ring = torch.zeros((self.capacity,) + r.spec_shape, dtype=torch.float32, device=r.device)
        pending, self._pending = self._pending, []
        n = len(pending)
        s0 = pending[0][0].slot
        rows = self.ring[s0: s0 + n]
        target = out if out is not None else rows
        reqs = [p[1] for p in pending]
        fades = [p[2] for p in pending]
        if any(f is not None for f in fades):          # continuous simulator with CROSSFADE (continuous_simulator.py:422-424)
            with r.transient_windows():
                target.copy_(r.render_crossfade(reqs, fades))
        elif any(q.rir_array is not None or q.wrap or q.offset % r.sr for q in reqs):
            with r.transient_windows():                # per-step RIRs / sample offsets: nothing worth keeping in the pool
                with r._inline_rirs(reqs):
                    r.execute(r.prepare(reqs), out=target)
        else:
            r.execute(r.prepare(reqs), out=target)
        if out is not None:
            rows.copy_(out)
        # between steps: LRU clock, landed prefetches, bank compaction (the requests above already hold their bank
        # ids, so this must not run before they have been turned into launches)
        self.service.maybe_trim()
        self._next = s0 + n
        self.flushed_generation = self.generation
        self.generation += 1
        self.flushes += 1
        return target

    # ------------------------------------------------------------------ resolve
    def gather(self, handles: Sequence[DeferredObservation], out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """``(N, 65, T', 2)`` CUDA tensor of the given handles' rows: flushes once if needed; when the handles are
        the consecutive rows of one flush (the normal step) the result is a VIEW of the ring -- no copy at all."""
        n = len(handles)
        if n == 0:
            return torch.empty((0,) + self.renderer.spec_shape, dtype=torch.float32, device=self.renderer.device)
        pend = [h for h in handles if h._row is None and h.generation > self.flushed_generation]
        if pend:
            all_pending_in_order = (out is not None and len(pend) == n == len(self._pending)
                                    and all(p[0] is h for p, h in zip(self._pending, handles)))
            self.flush(out=out if all_pending_in_order else None)
            if all_pending_in_order:
                return out
        if all(h._row is None for h in handles):
            s0 = handles[0].slot
            if all(h.slot == s0 + i for i, h in enumerate(handles)):
                view = self.ring[s0: s0 + n]
                return view if out is None else out.copy_(view)
            idx = torch.tensor([h.slot for h in handles], device=self.ring.device)
            res = self.ring.index_select(0, idx)
        else:
            res = torch.stack([h.resolve() for h in handles], dim=0)
        return res if out is None else out.copy_(res)


def _device_index(idx, device) -> torch.Tensor:
    """A host index list on the device through pinned memory: no blocking copy, so a step never waits on the host."""
    t = torch.tensor(idx, dtype=torch.int64)
    return t.pin_memory().to(device, non_blocking=True) if torch.device(device).type == "cuda" else t.to(device)


class RemoteObservations:
    """Trainer side of remote deferred mode (:mod:`soundspaces_b200.remote`): turns the workers' descriptors into
    requests against this service's banks -- RIR files are read here, by the service's reader pool -- and keeps the
    rows their memo references resolve to.

    The table maps ``(env token, generation, memo id)`` to what the original descriptor resolved to: a
    :class:`DeferredObservation` for spectrograms (the ring's detach-before-reuse rule keeps it valid), a private
    ``(2, sr)`` row for waveforms, or a ``(1,)`` intensity for a waveform resolved only as AV-WaN's intensity (a
    waveform lookup that finds one renders from the keys and keeps the row).  A new generation of an env drops the
    entries of the previous one.  A memo reference whose original never reached this trainer (a vector env with
    ``auto_reset_done`` drops the terminal step's observation) is rendered from the keys it carries, like the original
    would have been, and counted in :attr:`unseen_hits`; one whose original is in the step being resolved
    (:attr:`arriving`, set by ``batch_obs``) is rendered from its keys too, but is not counted."""

    INTENSITY_CHUNK = 256                              # waveforms rendered at once by intensities()

    def __init__(self, service):
        self.service = service
        self._memo = {}                                # env token -> (generation, {memo id: handle or row})
        self.unseen_hits = 0
        self.arriving = set()                          # (env, generation, memo id) of originals this step still resolves

    @staticmethod
    def of(d) -> "RemoteObservations":
        """The table of the trainer's service a descriptor names."""
        from .simulator import AudioRenderService
        sr, device, pad_mode = d.service
        key = (int(sr), str(torch.device(device)), pad_mode)
        if key not in AudioRenderService._instances and not torch.cuda.is_available():
            raise RuntimeError("a RemoteAudioRequest is rendered by the trainer process that owns the GPU; this process "
                               "has no CUDA device (env workers in remote mode hand descriptors to batch_obs)")
        return AudioRenderService.get(sr, device, pad_mode=pad_mode).remote

    def _lookup(self, d):
        """What a memo reference's original resolved to, or None when the original never reached this trainer."""
        gen, rows = self._memo.get(d.env, (None, {}))
        found = rows.get(d.memo_id) if gen == d.generation else None
        if found is None and (d.env, d.generation, d.memo_id) not in self.arriving:
            self.unseen_hits += 1
        return found

    def _keep(self, d, value):
        if d.memo_id < 0:
            return
        gen, rows = self._memo.get(d.env, (None, None))
        if gen != d.generation:
            rows = {}
            self._memo[d.env] = (d.generation, rows)
        rows[d.memo_id] = value

    def spectrogram(self, d) -> DeferredObservation:
        """Enqueue one spectrogram descriptor on the service's batcher (a memo reference costs no render)."""
        if d.hit:
            h = self._lookup(d)
            if h is not None:
                return h
        req, prev = self.service.requests(d)
        h = self.service.batcher.enqueue(req, crossfade_from=prev)
        self._keep(d, h)
        return h

    def waveforms(self, descs) -> torch.Tensor:
        """``(N, 2, sr)`` CUDA tensor of waveform descriptors: the step's requests go through ONE ``convolve``."""
        r = self.service.renderer
        self.service.maybe_trim()                      # between steps, before any bank id is handed out
        res = torch.zeros((len(descs), 2, r.sr), dtype=torch.float32, device=r.device)
        fresh = []
        for i, d in enumerate(descs):
            row = self._lookup(d) if d.hit else None
            if row is not None and row.ndim == 2:
                res[i] = row
                continue
            fresh.append((i, d))                       # new, unseen, or kept only as an intensity: render the keys
        self._render(res, fresh)
        for i, d in fresh:
            self._keep(d, res[i].clone())
        return res

    def _render(self, res: torch.Tensor, fresh):
        """Render the ``(row, descriptor)`` pairs into the zeroed rows of ``res`` with ONE ``convolve`` (or cross-fade);
        silent descriptors keep their zero rows."""
        svc, r = self.service, self.service.renderer
        idx, reqs, prevs = [], [], []
        for i, d in fresh:
            if not d.silent:
                req, prev = svc.requests(d)
                idx.append(i)
                reqs.append(req)
                prevs.append(prev)
        if reqs:
            transient = any(q.rir_array is not None or q.wrap or q.offset % r.sr for q in reqs)
            with r.transient_windows() if transient else contextlib.nullcontext():
                if any(p is not None for p in prevs):  # continuous simulator with CROSSFADE
                    wave = r.render_crossfade(reqs, prevs, want_wave=True)[1]
                else:
                    wave = r.convolve(reqs)
                res[_device_index(idx, r.device)] = wave

    def intensities(self, descs) -> torch.Tensor:
        """``(N,)`` CUDA float32 intensities of :class:`~soundspaces_b200.remote.IntensityRequest` s (AV-WaN's
        ``Intensity``, avwan_sensors.py:91-100), computed without reading anything back to the host.

        A descriptor resolved before (this step's map records and its ``intensity`` sensor share the object) reuses its
        value; a memo reference reuses the kept scalar, or reduces the kept ``(2, sr)`` row of a waveform sensor.  The
        rest are rendered as :meth:`waveforms` renders them, in chunks of at most :attr:`INTENSITY_CHUNK` waveforms so
        the transient ``(M, 2, sr)`` buffer stays bounded, and reduced by ``ssb_intensity_batch`` (one CTA per
        waveform: a value does not depend on the batch).  The memo keeps a scalar for an original resolved only as an
        intensity, never a row."""
        r = self.service.renderer
        self.service.maybe_trim()
        n = len(descs)
        parts, src = [], [None] * n                    # src[i]: (part, index) the value of descs[i] comes from
        work = []                                      # (i, descriptor): a waveform to reduce
        rows = {}                                      # position in work -> kept (2, sr) row to reduce
        originals = {}                                 # memo key -> position in work of an original in this call
        for i, q in enumerate(descs):
            d = q.request
            if q.value is not None:
                parts.append(q.value)
                src[i] = len(parts) - 1
                continue
            key = (d.env, d.generation, d.memo_id)
            if d.hit and d.memo_id >= 0 and key in originals:
                src[i] = ("work", originals[key])
                continue
            found = self._lookup(d) if d.hit else None
            if found is not None and found.ndim == 1:
                parts.append(found)
                src[i] = len(parts) - 1
                continue
            if found is not None:
                rows[len(work)] = found
            elif d.memo_id >= 0:
                originals[key] = len(work)
            src[i] = ("work", len(work))
            work.append((i, d))
        values = torch.empty(len(work), dtype=torch.float32, device=r.device)
        for c0 in range(0, len(work), self.INTENSITY_CHUNK):
            chunk = work[c0: c0 + self.INTENSITY_CHUNK]
            wave = torch.zeros((len(chunk), 2, r.sr), dtype=torch.float32, device=r.device)
            for j, (i, d) in enumerate(chunk):
                if c0 + j in rows:
                    wave[j] = rows[c0 + j]
            self._render(wave, [(j, d) for j, (i, d) in enumerate(chunk) if c0 + j not in rows])
            values[c0: c0 + len(chunk)] = r.intensity(wave)
        for w, (i, d) in enumerate(work):
            if w not in rows:
                self._keep(d, values[w: w + 1])
        if not parts and src == [("work", k) for k in range(n)]:
            out = values
        else:
            index = [len(parts) + s[1] if isinstance(s, tuple) else s for s in src]
            out = torch.cat(parts + [values]).index_select(0, _device_index(index, r.device))
        for i, q in enumerate(descs):
            q.value = out[i: i + 1]
        return out

    def numpy(self, d) -> np.ndarray:
        """Host copy of one descriptor's observation (flushes the pending step)."""
        if d.kind == WAVEFORM:
            return self.waveforms([d])[0].cpu().numpy()
        return self.spectrogram(d).numpy()
