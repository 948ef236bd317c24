"""Generate tests/golden/avnav_policy_golden.npz by running the UNMODIFIED reference classes of an upstream
sound-spaces checkout (path in ``SOUNDSPACES_REFERENCE``, as for the other oracle fixtures) in float64:
``VisualCNN`` of ss_baselines/av_nav, av_wan and savi models/visual_cnn.py and ``RNNStateEncoder`` of
ss_baselines/av_nav/models/rnn_state_encoder.py.

    SOUNDSPACES_REFERENCE=<sound-spaces checkout> python tests/golden/make_avnav_policy_golden.py

The visual encoders run at 36 x 36, the smallest input with a non-empty conv3 at strides 4/2/2.  ``visual_cnn.py``
imports ``Flatten`` from ss_baselines.common.utils (whose other imports are habitat, moviepy, cv2 ...) and savi's
imports ``d3_40_colors_rgb`` from habitat_sim; both are stubbed here with their computation.  Parameters come from
``set_params`` (tests/avnav_models.py), so only inputs and outputs are stored, per configuration ``<name>/<key>``:
visual ``config`` (variant index, n_rgb, n_depth, H, W, hidden), ``rgb`` / ``depth`` and ``out``; GRU ``config``
(I, Hd, N), ``x``, ``h``, ``masks``, ``out`` and ``h_out``.
"""
import importlib.util
import os
import sys
import types

import numpy as np
import torch
import torch.nn as nn

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from avnav_models import gru_inputs, set_params, visual_obs  # noqa: E402
from oracle.ref_harness import REFERENCE_ROOT  # noqa: E402

VARIANT_INDEX = {"av_nav": 0, "av_wan": 1, "savi": 2}
# name: (variant, n_rgb, n_depth, H, W, hidden, N)
VISUAL = {
    "av_nav_rgbd": ("av_nav", 3, 1, 36, 36, 8, 2),
    "av_wan_depth": ("av_wan", 0, 1, 36, 44, 8, 2),
    "savi_rgb": ("savi", 3, 0, 44, 36, 8, 2),
}
# name: (I, Hd, N, masks)
GRU = {"gru_mixed": (10, 8, 5, "mixed"), "gru_zero": (7, 4, 3, 0.0), "gru_one": (9, 6, 3, 1.0)}


class Space:
    def __init__(self, shape):
        self.shape = shape


class ObservationSpace:
    def __init__(self, spaces):
        self.spaces = spaces


def _stub(name, **attrs):
    m = types.ModuleType(name)
    m.__dict__.update(attrs)
    m.__path__ = []
    sys.modules[name] = m
    return m


def load_reference():
    if not REFERENCE_ROOT:
        sys.exit("set SOUNDSPACES_REFERENCE to a sound-spaces checkout")

    class Flatten(nn.Module):
        def forward(self, x):
            return x.reshape(x.size(0), -1)

    for pkg in ("ss_baselines", "ss_baselines.av_nav", "ss_baselines.av_nav.models", "ss_baselines.av_wan",
                "ss_baselines.av_wan.models", "ss_baselines.savi", "ss_baselines.savi.models", "habitat_sim",
                "habitat_sim.utils"):
        _stub(pkg)
    Flatten.__module__ = "ss_baselines.common.utils"
    _stub("ss_baselines.common")
    _stub("ss_baselines.common.utils", Flatten=Flatten)
    _stub("habitat_sim.utils.common", d3_40_colors_rgb=np.zeros((40, 3), np.uint8))

    def load(modname, rel):
        spec = importlib.util.spec_from_file_location(modname, os.path.join(REFERENCE_ROOT, "ss_baselines", rel))
        mod = importlib.util.module_from_spec(spec)
        sys.modules[modname] = mod
        spec.loader.exec_module(mod)
        return mod

    av_nav = load("ss_baselines.av_nav.models.visual_cnn", "av_nav/models/visual_cnn.py")
    av_wan = load("ss_baselines.av_wan.models.visual_cnn", "av_wan/models/visual_cnn.py")
    savi = load("ss_baselines.savi.models.visual_cnn", "savi/models/visual_cnn.py")
    rnn = load("ss_baselines.av_nav.models.rnn_state_encoder", "av_nav/models/rnn_state_encoder.py")
    return av_nav.VisualCNN, av_wan.VisualCNN, savi.VisualCNN, rnn.RNNStateEncoder


def main():
    av_nav, av_wan, savi, rnn_cls = load_reference()
    out = {}
    for i, (name, (variant, n_rgb, n_depth, H, W, hidden, N)) in enumerate(VISUAL.items()):
        spaces = {}
        if n_rgb:
            spaces["rgb"] = Space((H, W, n_rgb))
        if n_depth:
            spaces["depth"] = Space((H, W, n_depth))
        space = ObservationSpace(spaces)
        if variant == "av_nav":
            ref = av_nav(space, hidden, extra_rgb=False)
        elif variant == "av_wan":
            ref = av_wan(space, hidden, encode_rgb=n_rgb > 0, encode_depth=n_depth > 0)
        else:
            ref = savi(space, hidden)
        set_params(ref, seed=10 + i)
        ref = ref.double().eval()
        obs = {k: v.double() for k, v in visual_obs(N, H, W, n_rgb, n_depth, seed=20 + i).items()}
        with torch.no_grad():
            y = ref(obs)
        out[f"{name}/config"] = np.array([VARIANT_INDEX[variant], n_rgb, n_depth, H, W, hidden], np.int64)
        for k, v in obs.items():
            out[f"{name}/{k}"] = v.numpy()
        out[f"{name}/out"] = y.numpy()
    for i, (name, (I, Hd, N, masks)) in enumerate(GRU.items()):
        ref = set_params(rnn_cls(I, Hd), seed=30 + i).double().eval()
        x, h, m = (t.double() for t in gru_inputs(N, I, Hd, seed=40 + i, masks=masks))
        with torch.no_grad():
            y, h_out = ref(x, h, m)
        out[f"{name}/config"] = np.array([I, Hd, N], np.int64)
        out[f"{name}/x"], out[f"{name}/h"], out[f"{name}/masks"] = x.numpy(), h.numpy(), m.numpy()
        out[f"{name}/out"], out[f"{name}/h_out"] = y.numpy(), h_out.numpy()
    dst = os.path.join(ROOT, "tests", "golden", "avnav_policy_golden.npz")
    np.savez_compressed(dst, **out)
    print("wrote", dst, os.path.getsize(dst), "bytes")


if __name__ == "__main__":
    main()
