"""A/B of alternative builds of libssb200.so on the bench workload (C2: 128 envs x 44.1 kHz x 16384 taps).

    python scratch/ab_libs.py lib_a.so lib_b.so ...        # parent: one subprocess per library (SSB200_LIB)
    python scratch/ab_libs.py --child                      # child: measures the library named by SSB200_LIB
    python scratch/ab_libs.py --resnet lib_a.so lib_b.so   # bit-identity of the ResNet-18 entries (belief, SMTCNN)
    python scratch/ab_libs.py --policy-head lib_a.so lib_b.so   # bit-identity of the policy heads' accepted rows
    python scratch/ab_libs.py --smt lib_a.so lib_b.so      # bit-identity of ssb_smt_state_encoder_batch

Per library: ms/step (median of 5 x 200 steps, CUDA events) for 1..4 internal streams, the per-kernel event
sums with 2 streams, and a checksum of the spectrograms (all builds must agree to rounding)."""
import os, subprocess, sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def resnet_child():
    """SHA-256 of the outputs of ssb_resnet18_batch and ssb_smt_resnet18_batch on seeded inputs; symbols an older
    library lacks are dropped from the prototype table, so the parent commit's build loads too."""
    sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
    import ctypes, hashlib, torch
    from soundspaces_b200 import _lib
    lib = ctypes.CDLL(_lib.LIB_PATH)
    for name in [n for n in _lib.EXPORTS if not hasattr(lib, n)]:
        del _lib.EXPORTS[name]
    from belief_nets_models import make_net
    from soundspaces_b200.renderer import WaveformOps
    ops = WaveformOps.get("cuda:0")
    g = torch.Generator().manual_seed(3)
    h = hashlib.sha256()
    for B in (1, 16, 129):
        for kind, shape in (("tv21", (65, 26)), ("tv23", (65, 69)), ("smt2", (65, 26)), ("smt23", (65, 26))):
            x = torch.log1p(torch.rand((B,) + shape + (2,), generator=g) * 20.0).cuda()
            labels = torch.softmax(torch.randn(B, 21, generator=g) * 3.0, dim=1).cuda()
            net = make_net(kind, seed=B).cuda()
            out = (ops.resnet18(x, net) if kind.startswith("tv")
                   else ops.smt_resnet18(x, net, labels if kind == "smt23" else None))
            h.update(out.cpu().numpy().tobytes())
    print("AB-RESNET %-28s sha256=%s" % (os.path.basename(_lib.LIB_PATH), h.hexdigest()), flush=True)
    # ssb_smt_cnn_batch, hashed per group: depth at every shape; RGB where every bin is one pixel (no resize, 1 x 1,
    # 2 x 2, 64 x 1024); RGB resized with wider bins (the only group a change to how the product rounds may move)
    from smt_cnn_models import SMTCNN, observations, set_params
    groups = {"depth": [], "rgb-1px-bins": [], "rgb-wide-bins": []}
    for H, W, resize in ((64, 64, False), (1, 1, True), (2, 2, True), (64, 1024, True), (128, 128, True),
                         (48, 48, True), (100, 100, True), (480, 640, True), (1023, 1023, True)):
        model = set_params(SMTCNN({"rgb": 3, "depth": 1}, obs_transform="default" if resize else None), 5).cuda()
        obs = {k: v.cuda() for k, v in observations(16, H, W, seed=H + W).items()}
        groups["depth"].append(ops.smt_cnn(None, obs["depth"], None, model.depth_encoder, resize=resize))
        wide = resize and (H, W) not in ((1, 1), (2, 2), (64, 1024))
        groups["rgb-wide-bins" if wide else "rgb-1px-bins"].append(
            ops.smt_cnn(obs["rgb"], None, model.rgb_encoder, None, resize=resize))
    for name, outs in groups.items():
        h = hashlib.sha256(b"".join(o.cpu().numpy().tobytes() for o in outs)).hexdigest()
        print("AB-SMTCNN %-28s %-14s sha256=%s" % (os.path.basename(_lib.LIB_PATH), name, h), flush=True)
    # the train entries: outputs and all 62 gradients, a third of the rows with zero upstream gradient; torchvision's
    # also in eval mode, with the running statistics and num_batches_tracked after the forward
    if not hasattr(lib, "ssb_resnet18_train_forward_batch"):
        return
    from belief_nets_models import smt_net
    from audiogoal_train_models import set_params, tv_net
    from soundspaces_b200.belief_nets import (conv_norm_pairs, resnet18_buffers, resnet18_params,
                                              smt_resnet18_params)

    def upstream(B, n_out, seed):
        gr = torch.randn((B, n_out), generator=torch.Generator().manual_seed(seed))
        gr[::3] = 0.0
        return gr.cuda()

    def digest(ts):
        return hashlib.sha256(b"".join(t.detach().cpu().numpy().tobytes() for t in ts if t is not None)).hexdigest()

    for n_labels in (0, 21):
        for B in (1, 16, 129):
            net = smt_net(2 + n_labels, (65, 26), 2, B).cuda()
            x = torch.log1p(torch.rand((B, 65, 26, 2), generator=g) * 20.0).cuda()
            labels = (torch.softmax(torch.randn(B, n_labels, generator=g) * 3.0, dim=1).cuda() if n_labels else None)
            params = smt_resnet18_params(net)
            eps = tuple(float(n.eps) for _, n in conv_norm_pairs(net))
            out, ws = ops.smt_resnet18_train_forward(x, labels, params, eps)
            grads = ops.smt_resnet18_train_backward(x, labels, params, eps, ws, upstream(B, 2, B))
            print("AB-SMT-TRAIN %-28s ch=%-2d B=%-4d out=%s grads=%s" % (
                os.path.basename(_lib.LIB_PATH), 2 + n_labels, B, digest([out])[:16], digest(grads)[:16]), flush=True)
    for training in (True, False):
        for B, hw in ((2, (65, 26)), (16, (65, 69)), (129, (65, 26))):
            net = set_params(tv_net(23), 200 + B).cuda().train(training)
            x = torch.log1p(torch.rand((B,) + hw + (2,), generator=g) * 20.0).cuda()
            params, stats = resnet18_params(net), resnet18_buffers(net)
            eps = tuple(float(n.eps) for _, n in conv_norm_pairs(net))
            out, ws = ops.resnet18_train_forward(x, params, stats, eps, training, 0.1)
            grads = ops.resnet18_train_backward(x, params, stats, eps, training, ws, upstream(B, 23, B))
            print("AB-TV-TRAIN %-28s %-5s B=%-4d out=%s grads=%s stats=%s" % (
                os.path.basename(_lib.LIB_PATH), "train" if training else "eval", B, digest([out])[:16],
                digest(grads)[:16], digest(stats)[:16]), flush=True)


def policy_head_child():
    """SHA-256 of ssb_policy_head_batch's value, action, log_prob and probs on seeded accepted rows: every shape of
    tests/policy_head_domain_cases.py, all three heads, gains 0 to 300, the mode and Exp(1) draws, B = 129."""
    sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
    import ctypes, hashlib, torch
    from soundspaces_b200 import _lib
    lib = ctypes.CDLL(_lib.LIB_PATH)
    for name in [n for n in _lib.EXPORTS if not hasattr(lib, n)]:
        del _lib.EXPORTS[name]
    import policy_head_domain_cases as cases
    from soundspaces_b200.renderer import WaveformOps
    ops = WaveformOps.get("cuda:0")
    h, rows = hashlib.sha256(), 0
    for H, A in cases.ALL_SHAPES:
        x = cases.features(129, H, H + A).cuda()
        for head in cases.HEADS:
            for gain in cases.GAINS:
                aw, ab, cw, cb = cases.params(H, A, gain, H + A)
                actor, critic = torch.nn.Linear(H, A).cuda(), torch.nn.Linear(H, 1).cuda()
                with torch.no_grad():
                    for lin, w, b in ((actor, aw, ab), (critic, cw, cb)):
                        lin.weight.copy_(w); lin.bias.copy_(b)
                z64 = x.cpu().double() @ aw.double().t() + ab.double()
                mask = cases.make_mask("fraction", 129, A, H, z64).cuda() if head == "masked" else None
                q = torch.empty((129, A)).exponential_(1, generator=torch.Generator().manual_seed(A)).cuda()
                for qq in (None, q):
                    out = ops.policy_head(x, actor, critic, head != "logits", mask, qq, want_probs=True)
                    assert int(out[4].item()) == 0
                    for t in out[:4]:
                        h.update(t.cpu().numpy().tobytes())
                    rows += 129
    print("AB-POLICY-HEAD %-28s rows=%d sha256=%s" % (os.path.basename(_lib.LIB_PATH), rows, h.hexdigest()), flush=True)


def smt_child():
    """SHA-256 of ssb_smt_state_encoder_batch's outputs on seeded inputs: SAVi's shape with and without a goal at B 1,
    16 and 600 (300 slots, episode masks), pose encoding off, pretraining, and only the current token valid."""
    sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
    import ctypes, hashlib, torch
    from soundspaces_b200 import _lib
    lib = ctypes.CDLL(_lib.LIB_PATH)
    for name in [n for n in _lib.EXPORTS if not hasattr(lib, n)]:
        del _lib.EXPORTS[name]
    from smt_models import episode_masks, make_inputs, make_smt
    from soundspaces_b200.renderer import WaveformOps
    ops = WaveformOps.get("cuda:0")
    h, rows = hashlib.sha256(), 0
    cases = [(dict(), B, 300, goal, "episodes") for B in (1, 16, 600) for goal in (True, False)]
    cases += [(dict(D=40, pose_index=None, d_model=64, nhead=4), 33, 20, False, "episodes"),
              (dict(pretraining=True), 20, 50, False, "episodes"), (dict(), 20, 50, True, "none")]
    for i, (kw, B, M, goal, kind) in enumerate(cases):
        m = make_smt(seed=i, **kw).cuda()
        x, mem, _, g = make_inputs(B, M, D=kw.get("D", 276), d_model=kw.get("d_model", 256),
                                   pose_index=kw.get("pose_index", 272), seed=i, goal=goal)
        mk = episode_masks(B, M, 2 * M, 40, torch.Generator().manual_seed(i)) if kind == "episodes" else torch.zeros(B, M)
        out = ops.smt_state_encoder(m, x.cuda(), mem.cuda(), mk.cuda(), g.cuda() if g is not None else None)
        h.update(out.cpu().numpy().tobytes())
        rows += B
    print("AB-SMT %-28s rows=%d sha256=%s" % (os.path.basename(_lib.LIB_PATH), rows, h.hexdigest()), flush=True)


def child():
    sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
    import numpy as np, torch
    from synth import make_source
    from soundspaces_b200 import AudioRequest, BatchedAudioRenderer
    sr, L, B, NB = 44100, 16384, 128, 16
    g = torch.Generator(device="cuda").manual_seed(1)
    env = torch.exp(-torch.arange(L, device="cuda") / (L / 6.0))[None, :, None]
    bank = (torch.randn((NB * B, L, 2), device="cuda", generator=g) * env * 0.1).contiguous()
    r = BatchedAudioRenderer(sr, L)
    sid = r.add_source(make_source(7, sr))
    ids = r.set_dense_rir_bank(bank)
    sil = np.random.default_rng(99).random(B) < 0.05
    batches = [r.prepare([AudioRequest(rir=ids[k * B + i], source=sid, silent=bool(sil[i])) for i in range(B)])
               for k in range(NB)]
    out = torch.empty((B,) + r.spec_shape, device="cuda")
    res = {}
    cfgs = os.environ.get("AB_CONFIGS")
    if cfgs:                                   # "2x1,2x2,3x2": streams x chunks-per-stream
        out_s = []
        for c in cfgs.split(","):
            st, ch = (int(v) for v in c.split("x"))
            r.set_streams(st); r.set_chunks(ch)
            for i in range(30):
                r.execute(batches[i % NB], out=out)
            torch.cuda.synchronize()
            ts = []
            for rep in range(5):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for i in range(200):
                    r.execute(batches[i % NB], out=out)
                e1.record()
                torch.cuda.synchronize()
                ts.append(e0.elapsed_time(e1) / 200)
            out_s.append("%s=%.4f" % (c, sorted(ts)[2]))
        print("AB %-24s ms/step %s | chk=%.6f" % (os.path.basename(os.environ.get("SSB200_LIB", "default")), " ".join(out_s),
                                                  float(out.double().sum())), flush=True)
        return
    for streams in (2, 1, 3, 4):
        r.set_streams(streams)
        for i in range(30):
            r.execute(batches[i % NB], out=out)
        torch.cuda.synchronize()
        ts = []
        for rep in range(5):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for i in range(200):
                r.execute(batches[i % NB], out=out)
            e1.record()
            torch.cuda.synchronize()
            ts.append(e0.elapsed_time(e1) / 200)
        res[streams] = sorted(ts)[2]
    r.set_streams(2)
    r.execute(batches[0], out=out)
    torch.cuda.synchronize()
    chk = float(out.double().sum())
    r.ctx.set_kernel_timing(True)
    for i in range(100):
        r.execute(batches[i % NB], out=out)
    kt = r.ctx.get_kernel_timing()
    r.ctx.set_kernel_timing(False)
    ks = " ".join("%s=%.1f" % (k.replace("_kernel", ""), 1e3 * v[0] / 100) for k, v in kt.items() if v[1])
    print("AB %-28s ms/step s2=%.4f s1=%.4f s3=%.4f s4=%.4f | us: %s | chk=%.6f" % (
        os.path.basename(os.environ.get("SSB200_LIB", "default")), res[2], res[1], res[3], res[4], ks, chk), flush=True)


if __name__ == "__main__":
    mode = ("--resnet-child" if "--resnet" in sys.argv else
            "--policy-head-child" if "--policy-head" in sys.argv else
            "--smt-child" if "--smt" in sys.argv else "--child")
    if "--child" in sys.argv:
        child()
    elif "--resnet-child" in sys.argv:
        resnet_child()
    elif "--policy-head-child" in sys.argv:
        policy_head_child()
    elif "--smt-child" in sys.argv:
        smt_child()
    else:
        for lib in [a for a in sys.argv[1:] if not a.startswith("--")]:
            env = dict(os.environ, SSB200_LIB=os.path.abspath(lib))
            subprocess.call([sys.executable, os.path.abspath(__file__), mode], env=env)
