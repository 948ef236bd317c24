"""Small run of every kernel for compute-sanitizer (memcheck / racecheck / synccheck)."""
import sys, os
sys.path.insert(0, os.getcwd()); sys.path.insert(0, os.path.join(os.getcwd(), "tests"))
import numpy as np, torch
from synth import make_rir, make_source
from soundspaces_b200 import AudioRequest, BatchedAudioRenderer
for log2n in (12, 13, 14):
    for mode in (0, 1):
        sr = 16000
        r = BatchedAudioRenderer(sr, 20000, n_terms=2, log2n=log2n)
        r.set_conv_mode(mode); r.set_streams(1)
        s1 = r.add_source(make_source(1, sr)); s2 = r.add_source(make_source(2, 3 * sr))
        ids = r.add_rirs([make_rir(i, L) for i, L in enumerate((100, 4097, 9000, 20000))] + [None])
        reqs = [AudioRequest(rir=ids[0], source=s1), AudioRequest(rir=ids[1], source=s2, offset=sr),
                AudioRequest(rir=ids[2], source=s2, offset=2 * sr, distractor_rir=ids[1], distractor_source=s1),
                AudioRequest(rir=ids[3], source=s2, offset=8000, out_samples=4000, wrap=True),
                AudioRequest(rir=ids[4], source=s1), AudioRequest(rir=ids[0], source=s1, silent=True)]
        spec, wave = r.render(reqs, want_wave=True)
        r.render_crossfade(reqs[:2], [reqs[1], None])
        r.intensity(wave)
        torch.cuda.synchronize()
r = BatchedAudioRenderer(16000, 4096)
r.sh_decode(torch.randn(2, 1500, 9), [10.0, 200.0])          # direct form
r.sh_decode(torch.randn(2, 7600, 9), [10.0, 200.0])          # overlap-save FFT form
r.set_streams(2)
sid = r.add_source(make_source(3, 16000))
ids = r.add_rirs([make_rir(i, 3000) for i in range(64)])
r.render([AudioRequest(rir=i, source=sid) for i in ids])
r.set_chunks(2)
spec, wave = r.render([AudioRequest(rir=i, source=sid, silent=(i % 9 == 0)) for i in ids], want_wave=True)   # 2 streams x 2 chunks
r.set_chunks(1)
for pm in ("reflect", "constant"):                                       # log-mel extension kernel, both pad modes / powers
    rm = BatchedAudioRenderer(16000, 1024, pad_mode=pm)
    for n_mels, power in ((64, 2), (13, 1), (1, 2)):
        rm.logmel(wave[:5].clone(), n_mels=n_mels, power=power)
torch.cuda.synchronize()
# single-block plan: the 65536-point cluster kernel (named group barriers, in-place staging, DSMEM combine) + its
# source-spectrum kernel: short / long (> 16384 taps: q2 loop) / zero RIRs, offsets, wrap, truncated outputs, silent
for sr in (16000, 44100):
    rb = BatchedAudioRenderer(sr, min(48000, 65536 - sr + 1), prefer_block64=True)
    s1 = rb.add_source(make_source(1, sr)); s2 = rb.add_source(make_source(2, 3 * sr))
    ids = rb.add_rirs([make_rir(i, L) for i, L in enumerate((100, 4097, 16384, min(48000, 65536 - sr + 1)))] + [None])
    reqs = [AudioRequest(rir=ids[0], source=s1), AudioRequest(rir=ids[1], source=s2, offset=sr),
            AudioRequest(rir=ids[3], source=s2, offset=2 * sr), AudioRequest(rir=ids[2], source=s2, offset=8000, out_samples=4000, wrap=True),
            AudioRequest(rir=ids[4], source=s1), AudioRequest(rir=ids[0], source=s1, silent=True)]
    batch = rb.prepare(reqs)
    assert batch.plan.log2n == 16
    rb.execute(batch, want_wave=True)
    torch.cuda.synchronize()
# fused first layer of the audio encoder (SURVEY N2)
from soundspaces_b200.renderer import WaveformOps
for shape, k, st in (((3, 65, 69, 2), 8, 4), ((3, 65, 26, 2), 5, 2)):
    conv = torch.nn.Conv2d(2, 32, k, st).cuda()
    WaveformOps.get("cuda:0").audio_conv1(torch.rand(shape, device="cuda"), conv)
torch.cuda.synchronize()
# the whole audio encoder (cluster conv kernel + linear kernel) at B = 16, both encoder variants, hidden 512 and 100
sys.path.insert(0, os.path.join(os.getcwd(), "tests"))
from test_encoder_host import make_cnn
for shape in ((16, 65, 26, 2), (16, 65, 69, 2)):
    for c3, hidden in ((64, 512), (32, 100)):
        WaveformOps.get("cuda:0").audio_encoder(torch.rand(shape, device="cuda"), make_cnn(shape[1:], c3, hidden).cuda())
torch.cuda.synchronize()
# SAVi's encoder with a distractor sound (category folded into conv1's bias), labels as a strided column slice
for shape in ((16, 65, 26, 2), (16, 65, 69, 2)):
    wide = torch.rand((16, 40), device="cuda")
    WaveformOps.get("cuda:0").audio_encoder(torch.rand(shape, device="cuda"), make_cnn(shape[1:], 64, 128, in_ch=23).cuda(),
                                            category=wide[:, 5:26])
torch.cuda.synchronize()
# the SAVi belief update at B = 8 and 129, both observation sizes, silent rows and dones
import belief_oracle as bo
for B, shape in ((8, (65, 26, 2)), (129, (65, 69, 2))):
    seq = bo.make_sequence(B, 3, B, loc_cols=23)
    st = [torch.zeros((B, 2), device="cuda"), torch.zeros(B, dtype=torch.uint8, device="cuda"),
          torch.zeros((B, 21), device="cuda"), torch.zeros(B, dtype=torch.uint8, device="cuda")]
    for t in range(3):
        WaveformOps.get("cuda:0").belief_update(
            torch.from_numpy(bo.make_spectrograms(seq["silent"][t], shape, t)).cuda(), list(seq["dones"][t]), 0.5, False,
            pose=torch.from_numpy(seq["pose"][t]).cuda(), loc_pred=torch.from_numpy(seq["loc_pred"][t]).cuda(),
            last_pg=st[0], loc_valid=st[1], loc_out=torch.empty((B, 2), device="cuda"),
            label_pred=torch.from_numpy(seq["label_pred"][t]).cuda(), last_label=st[2], label_valid=st[3],
            cat_out=torch.empty((B, 21), device="cuda"))
torch.cuda.synchronize()
# the belief-predictor ResNet-18s: torchvision (both observation sizes) and SMT with 2 and 23 channels (labels as a
# strided column slice), B = 3 and 17
from belief_nets_models import make_net
for B in (3, 17):
    for shape in ((B, 65, 26, 2), (B, 65, 69, 2)):
        WaveformOps.get("cuda:0").resnet18(torch.rand(shape, device="cuda"), make_net("tv21").cuda())
    x = torch.rand((B, 65, 26, 2), device="cuda")
    WaveformOps.get("cuda:0").smt_resnet18(x, make_net("smt2").cuda())
    WaveformOps.get("cuda:0").smt_resnet18(x, make_net("smt23").cuda(), torch.rand((B, 30), device="cuda")[:, 4:25])
torch.cuda.synchronize()
# SAVi's visual encoder at an odd B: RGB-D with unequal sizes (downsampling, overlapping bins), RGB alone, and depth
# upsampled from 48 x 48
from smt_cnn_models import SMTCNN, observations, set_params
m = set_params(SMTCNN({"rgb": 3, "depth": 1}), 1).cuda().eval()
o = {"rgb": observations(5, 96, 128, 0, depth=0)["rgb"].cuda(), "depth": observations(5, 100, 100, 1, rgb=0)["depth"].cuda()}
WaveformOps.get("cuda:0").smt_cnn(o["rgb"], o["depth"], m.rgb_encoder, m.depth_encoder)
WaveformOps.get("cuda:0").smt_cnn(o["rgb"], None, m.rgb_encoder, None)
WaveformOps.get("cuda:0").smt_cnn(None, observations(5, 48, 48, 2, rgb=0)["depth"].cuda(), None, m.depth_encoder)
torch.cuda.synchronize()
# the scene memory transformer: pose encoding on and off, goal and none, a wrapped ring and only the current token
from smt_models import make_inputs, make_smt
for kw, goal, masks in ((dict(), True, None), (dict(D=40, pose_index=None, d_model=64, nhead=4), False, None),
                        (dict(D=40, pose_index=36, d_model=64, nhead=2), True, torch.zeros(5, 9))):
    m = make_smt(**kw).cuda()
    x, mem, mk, g = (t.cuda() if t is not None else None
                     for t in make_inputs(5, 9, D=kw.get("D", 276), d_model=kw.get("d_model", 256),
                                          pose_index=kw.get("pose_index", 272), goal=goal, masks=masks))
    WaveformOps.get("cuda:0").smt_state_encoder(m, x, mem, mk, g)
    # its training forward and backward (ssb_smt_state_encoder_train_*) on the same inputs
    out, ws = WaveformOps.get("cuda:0").smt_train_forward(m, x, mem, mk, g)
    WaveformOps.get("cuda:0").smt_train_backward(m, x, mem, mk, g, ws, torch.ones_like(out))
torch.cuda.synchronize()
# the AV-Nav visual encoder (RGB, depth, RGB-D; strides 4/2/2 and 4/2/1; 128 x 128, non-square, the smallest input)
# and the GRU state-encoder step (av_nav and odd widths, B past one 16-env tile)
from avnav_models import VisualCNN
for variant, n_rgb, n_depth, H, W in (("av_nav", 3, 1, 128, 128), ("av_wan", 0, 1, 128, 72), ("savi", 3, 0, 36, 36)):
    vm = VisualCNN(n_rgb, n_depth, H, W, 512, variant).cuda()
    WaveformOps.get("cuda:0").visual_encoder(torch.rand((3, H, W, n_rgb), device="cuda") * 255 if n_rgb else None,
                                             torch.rand((3, H, W, n_depth), device="cuda") if n_depth else None, vm.cnn)
for I, Hd, B in ((1024, 512, 17), (1026, 64, 3), (33, 100, 1)):
    gru = torch.nn.GRU(I, Hd).cuda()
    WaveformOps.get("cuda:0").gru_step(torch.randn(B, I, device="cuda"), torch.randn(B, Hd, device="cuda"),
                                       (torch.arange(B, device="cuda") % 2).float()[:, None], gru)
torch.cuda.synchronize()
# AV-WaN's map encoder at an odd B: a non-reference layout of the generic instance (C2 = 3, so ranks 3 - 7 hold no
# conv2 channel and the conv3 gather has three owners; sh != sw in every layer) and MapCNN on the 200 x 200 x 2 map
import map_cnn_domain_cases as mcases
from map_cnn_models import MapCNN, map_obs
c = mcases.LAYOUTS[3]
WaveformOps.get("cuda:0").map_encoder(map_obs(3, c["H"], c["W"], c["C"], 0, "dense").cuda(), mcases.make_cnn(c).cuda())
WaveformOps.get("cuda:0").map_encoder(map_obs(3, 200, 200, 2, 1, "gm").cuda(), MapCNN(200, 200, 2, 512).cuda().cnn)
torch.cuda.synchronize()
hs = r.make_host_session(8, 3000, want_wave=True, n_chunks=2)
hs.h_rir.numpy()[:] = np.stack([make_rir(i, 3000) for i in range(8)]); hs.set_requests(sid); hs.run(); hs.run()
torch.cuda.synchronize()
# orders 0 to 3, several azimuths per input: direct form (forced) and FFT form, both accumulator groupings
for K in (1, 4, 9, 16):
    r.lib.ssb_set_debug(r.ctx.handle, 32)
    r.sh_decode_angles(torch.randn(2, 1500, K), [0.0, 90.0, 37.5])
    r.lib.ssb_set_debug(r.ctx.handle, 0)
    r.sh_decode_angles(torch.randn(2, 7600, K), [10.0])
    r.sh_decode_angles(torch.randn(2, 7600, K), [10.0, 200.0, 0.0, 90.0, 45.0])
    # partial azimuth groups alone (A = 2) and behind a full one (A = 7), at a third block holding one output
    r.sh_decode_angles(torch.randn(2, 7425, K), [10.0, 200.0])
    r.sh_decode_angles(torch.randn(2, 7425, K), [10.0, 200.0, 0.0, 90.0, 45.0, -90.0, 450.0])
torch.cuda.synchronize()
# AV-WaN's device maps: an edge geometry (odd N, padded pitch, S > N) at its far corners in the odd quarter turns, and
# one launch of a few hundred records for two slots, interleaved, with a reset in the middle
from map_domain_cases import GEOMETRIES, case_record, cases
from mapper_models import MapMirror
from soundspaces_b200 import _lib as L, maps
g = GEOMETRIES["n61_s4"][0]
ok = [c for c in cases("n61_s4") if c.orientation in (0, 180) and MapMirror(g).update_raises(c.x, c.y, c.orientation)
      is None]
ops = WaveformOps.get("cuda:0")
gmap = torch.zeros((2, (61 * 61 + 15) & ~15), dtype=torch.uint8, device="cuda")
amap = torch.zeros((2, 15, 15), dtype=torch.float64, device="cuda")
recs = [(i % 2, case_record(c)) for i, c in enumerate(ok * 2)]
recs.insert(len(recs) // 2, (1, (0, maps.RESET, 0, 0, 0, 0.0, 0.0, b"")))
rec = np.zeros(len(recs), maps.RECORD_DTYPE)
ego = b""
for i, (slot, (_, kind, x, y, o, v, h, bits)) in enumerate(recs):
    rec[i] = (slot, kind, x, y, o, 0, v, h, len(ego))
    ego += bits
ops.map_update(L.MapGeometry(*g, 2), gmap, amap, rec, np.frombuffer(ego, np.uint8))
far = [c for c in ok if c.x > 50 or c.y > 50][:8]
poses = np.array([(i % 2, c.x, c.y, c.orientation) for i, c in enumerate(far)], np.int32)
ops.map_observe(L.MapGeometry(*g, 2), gmap, amap, poses, maps.navigable_tables(g),
                torch.empty((len(far), 66, 66, 2), device="cuda"), torch.empty((len(far), 20, 20, 1), device="cuda"))
torch.cuda.synchronize()
# remote workers' RGB-D frames: upload + gather with misses, hits, a small evicting bank, 16-byte and scalar rows,
# strided destinations
import pickle as _pk
from soundspaces_b200 import frames as _fr
from soundspaces_b200.remote import FrameArray as _FA
_rng = np.random.default_rng(0)
for shape, dt in (((16, 16, 3), np.uint8), ((16, 16, 1), np.float32), ((5, 7, 3), np.uint8), ((3, 5, 1), np.float32)):
    pool = [(_rng.integers(0, 256, size=shape) if dt == np.uint8 else _rng.random(shape)).astype(dt) for _ in range(9)]
    row = int(np.prod(shape)) * np.dtype(dt).itemsize
    _fr.FrameStore.get("cuda:0", "san", dt, shape, max_bank_bytes=4 * row)
    for step in range(12):
        pick = _rng.integers(0, 9, size=3)
        refs = [_pk.loads(_pk.dumps(_FA(pool[i], (f"san{shape}", int(i), 0, "san")))) for i in pick]
        dst = torch.empty((3, int(np.prod(shape)) + 4), device="cuda")[:, : int(np.prod(shape))].view((3,) + shape)
        _fr.gather({"san": refs}, torch.device("cuda:0"), out={"san": dst})
torch.cuda.synchronize()
print("done")
