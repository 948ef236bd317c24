"""ssb_render_batch refuses what ssb_convolve_batch and ssb_spectrogram_batch refuse, on the host and before any
launch, at every batch size: also at B >= 64, where it splits the batch over internal streams.  A plan is accepted
only as ssb_make_plan makes it."""
import ctypes as C

import pytest

from synth import make_rir, make_source
from test_gpu_parity import renderer

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

SR, B = 16000, 128                # 128 envs: two internal streams (the context default) of 64


def _batch(silent):
    """The N = 4096 plan's renderer and B prepared requests.  Silent requests read neither the RIR bank nor the
    RIR-spectrum scratch."""
    from soundspaces_b200 import AudioRequest
    r = renderer(SR, 9000, log2n=12)
    sid = r.add_source(make_source(31, SR))
    rids = r.add_rirs([make_rir(3100 + i, 9000 - 700 * i) for i in range(4)])
    batch = r.prepare([AudioRequest(rir=rids[i % 4], source=sid, silent=silent) for i in range(B)])
    assert batch.plan.log2n == 12
    return r, batch


def _render(r, batch, plan=None, bank_offset=0, pad_mode=None):
    plan = batch.plan if plan is None else plan
    hs, wave = r._scratch(B, plan)
    spec = torch.empty((B,) + r.spec_shape, dtype=torch.float32, device="cuda")
    return r.lib.ssb_render_batch(r.ctx.handle, C.byref(plan), B, batch.reqs_dev.data_ptr(),
                                  r._bank.data_ptr() + bank_offset, r._xpool.data_ptr(), hs.data_ptr(), wave.data_ptr(),
                                  SR, r.pad_mode if pad_mode is None else pad_mode, spec.data_ptr(), r._stream())


def test_render_refuses_bad_pad_mode_before_any_launch():
    r, batch = _batch(silent=False)
    before = r.ctx.launch_count
    assert _render(r, batch) == 0
    assert r.ctx.launch_count == before + 6          # per stream: fwd_rir, the cluster kernel, spectrogram
    before = r.ctx.launch_count
    assert _render(r, batch, pad_mode=7) == -1       # SSB_E_INVALID_ARG
    assert b"pad_mode=7" in r.lib.ssb_last_error(r.ctx.handle)
    assert r.ctx.launch_count == before
    torch.cuda.synchronize()


def test_render_refuses_misaligned_rir_bank_before_any_launch():
    r, batch = _batch(silent=True)
    before = r.ctx.launch_count
    assert _render(r, batch, bank_offset=4) == -1    # float2 taps: 8-byte alignment
    assert b"aligned" in r.lib.ssb_last_error(r.ctx.handle)
    assert r.ctx.launch_count == before
    torch.cuda.synchronize()


def test_convolve_refuses_edited_h_elems_per_env():
    from soundspaces_b200._lib import Plan
    r, batch = _batch(silent=True)
    plan = Plan.from_buffer_copy(batch.plan)
    plan.h_elems_per_env //= 2                       # every other field as ssb_make_plan made it
    hs, wave = r._scratch(B, batch.plan)
    before = r.ctx.launch_count
    rc = r.lib.ssb_convolve_batch(r.ctx.handle, C.byref(plan), B, batch.reqs_dev.data_ptr(), r._bank.data_ptr(),
                                  r._xpool.data_ptr(), hs.data_ptr(), wave.data_ptr(), SR, r._stream())
    assert rc == -1
    assert b"invalid plan" in r.lib.ssb_last_error(r.ctx.handle)
    assert r.ctx.launch_count == before
    assert _render(r, batch, plan=plan) == -1
    assert r.ctx.launch_count == before
    torch.cuda.synchronize()
