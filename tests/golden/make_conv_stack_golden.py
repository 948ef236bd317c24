"""Generate tests/golden/conv_stack_golden.npz by running the UNMODIFIED reference encoder classes of an upstream
sound-spaces checkout (path in ``SOUNDSPACES_REFERENCE``, as for the other oracle fixtures) in float64, forward and
backward: ``AudioCNN`` of ss_baselines/av_nav/models/audio_cnn.py at 16 kHz (65 x 26: 5/3/3 kernels) and 44.1 kHz
(65 x 69: 8/4/3), savi/models/audio_cnn.py with a distractor sound (21 category channels), ``VisualCNN`` of
av_nav/models/visual_cnn.py on RGB-D, depth and RGB, and ``MapCNN`` of av_wan/models/map_cnn.py on gm (200 x 200 x 2)
and am (20 x 20 x 1).

    SOUNDSPACES_REFERENCE=<sound-spaces checkout> python tests/golden/make_conv_stack_golden.py

Parameters come from ``set_params`` (tests/avnav_models.py), which leaves some ReLU units dead.  The inputs and the
upstream gradient come from seeds (``case_inputs`` in tests/conv_stack_models.py); the first input's last row holds a
NaN.  So only the configuration and the results are stored, per configuration ``<name>/<key>``: ``config`` (kind 0
audio / 1 visual / 2 map, N, hidden, param seed), ``out`` (the forward of every row, NaN in the last), and of the
gradients of the eight ``cnn`` parameters (conv1-3 weight and bias, Linear weight and bias) for sum(out[:-1] * dout)
over the finite rows, ``grad_summary``: ``g<j>`` whole for tensors of at most 512 elements, else ``g<j>_sample`` (256
seeded elements) and ``g<j>_proj`` (32 seeded Gaussian projections of every element).
"""
import importlib.util
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))

from avnav_models import set_params  # noqa: E402
from conv_stack_models import CASES, HIDDEN, N, case_inputs, grad_summary  # noqa: E402
from make_avnav_policy_golden import ObservationSpace, Space, _stub, load_reference  # noqa: E402
from make_map_cnn_golden import load_map_cnn  # noqa: E402


def load_audio():
    from oracle.ref_harness import REFERENCE_ROOT

    class Category:
        cls_uuid = "category"
    for pkg in ("soundspaces", "soundspaces.tasks"):
        _stub(pkg)
    _stub("soundspaces.tasks.nav", Category=Category)

    def load(modname, rel):
        spec = importlib.util.spec_from_file_location(modname, os.path.join(REFERENCE_ROOT, "ss_baselines", rel))
        mod = importlib.util.module_from_spec(spec)
        sys.modules[modname] = mod
        spec.loader.exec_module(mod)
        return mod
    return (load("ss_baselines.av_nav.models.audio_cnn", "av_nav/models/audio_cnn.py").AudioCNN,
            load("ss_baselines.savi.models.audio_cnn", "savi/models/audio_cnn.py").AudioCNN)


def main():
    visual_cls = load_reference()[0]
    map_cls = load_map_cnn()
    avnav_audio, savi_audio = load_audio()
    out = {}
    for i, (name, (kind, spec)) in enumerate(CASES.items()):
        pseed = 60 + i
        obs, dout = case_inputs(name)
        if kind.startswith("audio"):
            space = ObservationSpace({"audiogoal": Space(spec)})
            ref = (avnav_audio(space, HIDDEN, "audiogoal") if kind == "audio"
                   else savi_audio(space, HIDDEN, "audiogoal", has_distractor_sound=True))
            code = 0
        elif kind == "visual":
            n_rgb, n_depth, H, W = spec
            spaces = {}
            if n_rgb:
                spaces["rgb"] = Space((H, W, n_rgb))
            if n_depth:
                spaces["depth"] = Space((H, W, n_depth))
            ref = visual_cls(ObservationSpace(spaces), HIDDEN, extra_rgb=False)
            code = 1
        else:
            ref = map_cls(ObservationSpace({kind: Space(spec)}), HIDDEN, map_type=kind)
            code = 2
        set_params(ref, seed=pseed)
        ref = ref.double()
        with torch.no_grad():
            y_all = ref(obs)
        assert torch.isnan(y_all[-1]).all() and not torch.isnan(y_all[:-1]).any(), name
        acts = []
        hook = ref.cnn[1].register_forward_hook(lambda m, i, o: acts.append(o.detach().clone()))
        y = ref({k: v[:-1] for k, v in obs.items()})
        hook.remove()
        dead = (acts[0] == 0).double().mean().item()
        assert 0.02 < dead < 0.98, (name, dead)               # some conv1 ReLU outputs are dead, not all
        (y * dout).sum().backward()
        cnn = ref.cnn
        grads = [p.grad for c in (cnn[0], cnn[2], cnn[4], cnn[6]) for p in (c.weight, c.bias)]
        out[f"{name}/config"] = np.array([code, N, HIDDEN, pseed], np.int64)
        out[f"{name}/out"] = y_all.detach().numpy()
        for j, gr in enumerate(grads):
            for suffix, v in grad_summary(name, j, gr.numpy()).items():
                out[f"{name}/g{j}{suffix}"] = v
    dst = os.path.join(ROOT, "tests", "golden", "conv_stack_golden.npz")
    np.savez_compressed(dst, **out)
    print("wrote", dst, os.path.getsize(dst), "bytes")


if __name__ == "__main__":
    main()
