"""AV-WaN with env workers in remote deferred mode and ``remote_intensity``: workers send waveform requests inside the
map records and the ``intensity`` observation, the trainer renders, reduces and applies them on the device.  Every
map crop, the raw float64 acoustic map state and the ``(N, 1)`` intensity batch must be bit-identical to in-process
deferred mode on the same traces, and the workers must never create a CUDA context."""
import warnings

import numpy as np
import pytest
import torch

from avwan_remote_envs import MapNavReplayEnv, ProcessMapNavEnvs
from oracle import audio_oracle as ao
from oracle.ref_harness import write_rir
from synth import make_rir, make_source

from soundspaces_b200 import _lib
from soundspaces_b200._lib import C
from soundspaces_b200.maps import RECORD_DTYPE, UPDATE, DeviceMaps
from soundspaces_b200.renderer import WaveformOps
from soundspaces_b200.sensors import batch_obs
from soundspaces_b200.simulator import AudioRenderService

pytestmark = pytest.mark.gpu

SR, STEPS = 16000, 14
SSB_E_INVALID_ARG, SSB_E_SHAPE = -1, -4                       # include/ssb200.h
MAPS = ("gm", "am", "action_map")
HOST_SENSORS = ("ego_map", "collision")                      # host arrays: the reference's stack and copy


def _tree(root):
    for az in (0, 90, 180, 270):
        for n in range(9):
            for s in (0, 1):
                write_rir(root, "replica", "scene", az, n, s, SR, make_rir(40 * s + 4 * n + az // 90, 1500 + 200 * n))


def _configs(encoding):
    """One encoding per run: the device maps of one step share one geometry."""
    one, three = make_source(0, SR), make_source(1, 3 * SR)
    return [  # (kind, clip, seed, encoding, episode_steps)
        ("discrete", one, 1, encoding, None),
        ("discrete", three, 2, encoding, None),
        ("discrete", one, 3, encoding, 4),                    # auto-reset: terminal observations are dropped
        ("discrete", three, 4, encoding, 5),
        ("distractor", one, 5, encoding, None),               # no memo
        ("continuous", one, 6, encoding, None),               # inline RIRs, cross-fade, silent after DURATION
    ]


def _run(envs, n, key_order, counters=None, syncs=None):
    """Per step: the batch, each env's raw acoustic map and the step's launch counts; ``syncs`` collects the host
    synchronisations torch reports inside batch_obs."""
    syncs = [] if syncs is None else syncs
    svc = AudioRenderService.get(SR, "cuda:0")
    out = []
    obs = envs.reset()
    for step in range(STEPS + 1):
        obs = [{k: o[k] for k in key_order if k in o} | {k: v for k, v in o.items() if k not in key_order}
               for o in obs]
        maps_ops = WaveformOps.get("cuda:0")
        l_maps, l_r = maps_ops.ctx.launch_count, svc.renderer.ctx.launch_count
        if counters is not None:
            counters.clear()
        if counters is not None and step > 0:                  # the remote run: no host synchronisation once the
            torch.cuda.set_sync_debug_mode("warn")              # clips are resident
        try:
            with warnings.catch_warnings(record=True) as caught:
                warnings.simplefilter("always")
                b = batch_obs(obs, device=torch.device("cuda"), skip_list=HOST_SENSORS)
        finally:
            torch.cuda.set_sync_debug_mode("default")
        syncs.extend(f"step {step}: {w.filename}:{w.lineno}" for w in caught
                     if "called a synchronizing CUDA operation" in str(w.message))
        dm = DeviceMaps.get("cuda:0", obs[0]["gm"].geometry)
        amap = torch.stack([dm.amap[dm.slots[o["gm"].token]] for o in obs]).cpu().numpy()
        launches = (maps_ops.ctx.launch_count - l_maps, svc.renderer.ctx.launch_count - l_r, dict(counters or {}))
        out.append(({k: v.cpu().numpy() for k, v in b.items()}, amap, launches))
        if step < STEPS:
            obs = envs.step()
    return out


class _InProcess:
    def __init__(self, configs, root, order):
        svc = AudioRenderService.get(SR, "cuda:0")
        self.envs = [MapNavReplayEnv(k, SR, root, clip, seed, True, encoding=enc, order=order, episode_steps=ep,
                                     service=svc) for k, clip, seed, enc, ep in configs]

    def reset(self):
        return [e.reset() for e in self.envs]

    def step(self):
        return [e.step() for e in self.envs]


def _exempt_rendering(monkeypatch, svc):
    """The renderer's own calls synchronise by design (a plain synchronous copy of each render's request array,
    renderer._upload_requests; bank and pool upkeep).  The sync check below covers what this path adds around them:
    the intensity bookkeeping and reduction, the map update and the crops."""
    r = svc.renderer
    for obj, name in ((r, "convolve"), (r, "render_crossfade"), (svc, "requests"), (svc, "maybe_trim")):
        fn = getattr(obj, name)

        def quiet(*a, _fn=fn, **k):
            mode = torch.cuda.get_sync_debug_mode()
            torch.cuda.set_sync_debug_mode("default")
            try:
                return _fn(*a, **k)
            finally:
                torch.cuda.set_sync_debug_mode(mode)
        monkeypatch.setattr(obj, name, quiet)


def _count(monkeypatch, r, counters):
    """Count the renderer's outermost calls (render_crossfade renders through convolve)."""
    depth = [0]
    for name in ("convolve", "render_crossfade", "intensity"):
        fn = getattr(r, name)

        def wrapped(*a, _fn=fn, _name=name, **k):
            if depth[0] == 0:
                counters[_name] = counters.get(_name, 0) + 1
            depth[0] += 1
            try:
                return _fn(*a, **k)
            finally:
                depth[0] -= 1
        monkeypatch.setattr(r, name, wrapped)


@pytest.mark.parametrize("encoding,order,key_order", [
    ("intensity", ("intensity",), ("intensity", "gm")),
    ("average_intensity", ("intensity",), ("gm", "am", "action_map", "intensity")),
    ("average_intensity", ("audiogoal", "intensity"), ("audiogoal", "intensity")),
    ("intensity", ("audiogoal", "intensity"), ("intensity", "gm", "audiogoal")),
])
def test_remote_intensity_equals_in_process(tmp_path, monkeypatch, encoding, order, key_order):
    root = str(tmp_path)
    _tree(root)
    configs = _configs(encoding)
    svc = AudioRenderService.get(SR, "cuda:0")
    counters = {}
    _exempt_rendering(monkeypatch, svc)
    _count(monkeypatch, svc.renderer, counters)
    unseen = svc.remote.unseen_hits
    args = [((k, SR, root, clip, seed, "remote"), dict(encoding=enc, order=order, episode_steps=ep))
            for k, clip, seed, enc, ep in configs]
    with ProcessMapNavEnvs(args) as envs:
        syncs = []
        got = _run(envs, len(configs), key_order, counters, syncs)
        assert all(r["cuda_initialized"] is False for r in envs.report())
    dropped = svc.remote.unseen_hits - unseen
    monkeypatch.undo()
    want = _run(_InProcess(configs, root, order), len(configs), key_order)

    for step, ((b, amap, (l_maps, l_r, calls)), (b_ref, amap_ref, _)) in enumerate(zip(got, want)):
        for k in MAPS + ("intensity",):
            assert b[k].dtype == np.float32 and np.array_equal(b[k], b_ref[k]), (step, k)
        assert b["intensity"].shape == (len(configs), 1)
        assert np.array_equal(amap.view(np.uint64), amap_ref.view(np.uint64)), step
        if "audiogoal" in b:
            assert np.array_equal(b["audiogoal"], b_ref["audiogoal"]), step
            for e in range(len(configs)):
                ref = ao.intensity(b["audiogoal"][e])
                assert np.isclose(b["intensity"][e, 0], ref, rtol=1e-5, atol=1e-12), (step, e)
        # one update and one crop; one intensity launch per chunk (one chunk here) and one render for it, plus the
        # audiogoal sensor's
        assert l_maps == 2, step
        assert calls.get("intensity", 0) <= 1 and calls.get("convolve", 0) + calls.get("render_crossfade", 0) <= \
            calls.get("intensity", 0) + ("audiogoal" in b), (step, calls)
    assert sum(g[2][2].get("intensity", 0) for g in got) > STEPS // 2
    assert dropped > 0                                        # references whose originals were dropped, rendered
    assert not syncs, syncs[:3]


def test_descriptor_resolves_in_the_trainer(tmp_path):
    root = str(tmp_path)
    _tree(root)
    args = [(("discrete", SR, root, make_source(2, SR), 7, "remote"), dict(order=("audiogoal", "intensity")))]
    with ProcessMapNavEnvs(args) as envs:
        o = envs.reset()[0]
    assert np.isclose(float(o["intensity"][0]), ao.intensity(np.asarray(o["audiogoal"])), rtol=1e-5, atol=1e-12)


def test_chunks_bound_the_render(tmp_path, monkeypatch):
    """More requests than one chunk: the values equal one render of them all, chunk after chunk."""
    root = str(tmp_path)
    _tree(root)
    svc = AudioRenderService.get(SR, "cuda:0")
    monkeypatch.setattr(type(svc.remote), "INTENSITY_CHUNK", 3)
    args = [(("distractor", SR, root, make_source(3, SR), s, "remote"), {}) for s in range(2)]
    with ProcessMapNavEnvs(args) as envs:
        envs.reset()
        obs = envs.step()
    recs = [r for o in obs for r in o["gm"].pending() if r[1] == UPDATE]
    assert len(recs) > 3
    n0 = svc.renderer.ctx.launch_count
    b = batch_obs(obs, device=torch.device("cuda"))
    assert svc.renderer.ctx.launch_count > n0
    descs = [r[5] for r in recs]
    wave = svc.remote.waveforms([q.request for q in descs])
    want = svc.renderer.intensity(wave)
    got = torch.cat([q.value for q in descs])
    assert torch.equal(got, want)
    assert torch.equal(b["intensity"][:, 0], torch.stack([o["intensity"][0].value[0] for o in obs]))


def _entry_args(g, n=1):
    rec = np.zeros(n, dtype=RECORD_DTYPE)
    rec[0] = (0, UPDATE, 250, 250, 270, 0, 0.0, 0.0, 0)
    return rec


def test_device_intensity_entry_refuses_before_launch():
    g = _lib.MapGeometry(500, 5, 200, 9, 31, 0, 1, 2)
    ops = WaveformOps.get("cuda:0")
    gmap = torch.zeros((2, (500 * 500 + 15) & ~15), dtype=torch.uint8, device="cuda")
    amap = torch.zeros((2, 100, 100), dtype=torch.float64, device="cuda")
    ego = np.zeros(((31 * 31 * 2 + 7) // 8,), dtype=np.uint8)
    vals = torch.tensor([0.25, 0.5], device="cuda")
    lib, ctx = ops.lib, ops.ctx

    def call(rec, ptr, n):
        rec = np.ascontiguousarray(rec)
        return lib.ssb_map_update_device_intensity_batch(ctx.handle, C.byref(g), gmap.data_ptr(),
                                                         amap.data_ptr(), len(rec), rec.ctypes.data, ego.ctypes.data,
                                                         ego.size, ptr, n, None)
    before = ctx.launch_count
    for idx, ptr, n in ((-1, vals.data_ptr(), 2), (2, vals.data_ptr(), 2), (0, None, 2), (0, vals.data_ptr() + 2, 2),
                        (0, vals.data_ptr(), -1)):
        rec = _entry_args(g)
        rec["reserved"] = idx
        assert lib.ssb_map_update_device_intensity_batch is not None
        assert call(rec, ptr, n) == SSB_E_INVALID_ARG, (idx, ptr, n)
    rec = _entry_args(g)
    rec["slot"] = 5
    assert call(rec, vals.data_ptr(), 2) == SSB_E_INVALID_ARG
    rec = _entry_args(g)
    rec["x"] = 600
    assert call(rec, vals.data_ptr(), 2) == SSB_E_SHAPE
    torch.cuda.synchronize()
    assert ctx.launch_count == before
    rec = _entry_args(g)
    rec["reserved"] = 1
    assert call(rec, vals.data_ptr(), 2) == 0
    torch.cuda.synchronize()
    assert ctx.launch_count == before + 1 and amap[0, 50, 50].item() == 0.5


def test_float64_half_of_a_subnormal_product():
    """The entry computes half = 0.5 * (double)v, as a worker does on the Python float the sensor returns; the
    reference's np.float32 product would flush 0.5 v to a float32 subnormal."""
    g = _lib.MapGeometry(500, 5, 200, 9, 31, 1, 1, 1)
    ops = WaveformOps.get("cuda:0")
    gmap = torch.zeros((1, (500 * 500 + 15) & ~15), dtype=torch.uint8, device="cuda")
    amap = torch.zeros((1, 100, 100), dtype=torch.float64, device="cuda")
    cell = 1e-38
    amap[0, 50, 50] = cell
    v = np.nextafter(np.finfo(np.float32).tiny, np.float32(1))    # 0.5 v rounds as a float32 subnormal
    ego = np.zeros(((31 * 31 * 2 + 7) // 8,), dtype=np.uint8)
    rec = _entry_args(g)
    ops.map_update_device_intensity(g, gmap, amap, rec, ego, torch.tensor([v], device="cuda"))
    got = amap[0, 50, 50].item()
    assert got == 0.5 * float(v) + 0.5 * cell
    assert got != float(np.float32(0.5) * v) + 0.5 * cell
