"""The render path's spectrogram skips the envs whose waveform the convolution leaves all zero (silent, no term with
taps, nothing to output).  Their columns must still hold exactly what the transform of that zero waveform gives, +0.0,
and every other env must be untouched: the whole batch is compared bit for bit against each env's waveform run on its
own through ssb_spectrogram_batch, which has no requests and transforms every env."""
import numpy as np
import pytest

from synth import make_rir, make_source

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

NCHW = 0x100
KINDS = ("live", "silent", "zero_rir", "no_output", "distractor_only", "short", "silent_with_rir")
DEAD = {"silent", "zero_rir", "no_output", "silent_with_rir"}


def _requests(sr, n, ids, sid, did):
    from soundspaces_b200 import AudioRequest
    reqs = []
    for i in range(n):
        kind, rir = KINDS[i % len(KINDS)], ids[i % len(ids)]
        if kind in ("live", "no_output"):
            reqs.append(AudioRequest(rir=rir, source=sid))
        elif kind == "silent":
            reqs.append(AudioRequest(rir=-1, source=sid, silent=True))
        elif kind == "silent_with_rir":
            reqs.append(AudioRequest(rir=rir, source=sid, silent=True))
        elif kind == "zero_rir":
            reqs.append(AudioRequest(rir=-1, source=sid))
        elif kind == "distractor_only":           # the goal term has no taps, the distractor term does
            reqs.append(AudioRequest(rir=-1, source=sid, distractor_rir=rir, distractor_source=did))
        else:                                     # live, but zero past out_samples
            reqs.append(AudioRequest(rir=rir, source=sid, out_samples=sr // 3 + 17))
    return reqs


@pytest.mark.parametrize("pad_mode", ["reflect", "constant"])
@pytest.mark.parametrize("channels_first", [False, True], ids=["nhwc", "nchw"])
@pytest.mark.parametrize("sr", [16000, 44100])
def test_dead_envs_bit_identical(sr, channels_first, pad_mode):
    from soundspaces_b200 import BatchedAudioRenderer
    from soundspaces_b200.renderer import PreparedBatch
    n, taps = 70, sr // 2                         # 70 envs: two sub-batches on the default two internal streams
    r = BatchedAudioRenderer(sr, taps, device="cuda:0", n_terms=2, pad_mode=pad_mode)
    sid = r.add_source(make_source(0, sr))
    did = r.add_source(make_source(1, 2 * sr))
    ids = r.add_rirs([make_rir(i, taps - 37 * i) for i in range(5)])
    batch = r.prepare(_requests(sr, n, ids, sid, did))
    # out_samples = 0 is refused by prepare(); the library's entry takes it, so build that request directly
    reqs = batch.reqs_host.copy()
    kinds = [KINDS[i % len(KINDS)] for i in range(n)]
    reqs["out_samples"][[k == "no_output" for k in kinds]] = 0
    batch = PreparedBatch(n, reqs, r._upload_requests(reqs), batch.plan)

    spec, wave = r.execute(batch, want_wave=True, channels_first=channels_first)
    torch.cuda.synchronize()
    wave = wave.clone()
    dead = np.array([k in DEAD for k in kinds])
    live = ~dead
    assert not wave[torch.from_numpy(dead).cuda()].any()          # the convolution wrote the zero waveform
    assert wave[torch.from_numpy(live).cuda()].abs().amax(dim=(1, 2)).gt(0).all()

    # each env alone, through the entry without requests
    pad = {"reflect": 0, "constant": 1}[pad_mode] | (NCHW if channels_first else 0)
    want = torch.empty_like(spec)
    for i in range(n):
        r.ctx.check(r.lib.ssb_spectrogram_batch(r.ctx.handle, 1, wave[i].data_ptr(), sr, sr, pad,
                                                want[i].data_ptr(), r._stream()), "ssb_spectrogram_batch")
    torch.cuda.synchronize()
    got, want = spec.cpu().numpy(), want.cpu().numpy()
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
    assert not got[dead].view(np.uint32).any()                     # +0.0, sign bit included
    assert (got[live].reshape(live.sum(), -1) > 0).any(axis=1).all()
