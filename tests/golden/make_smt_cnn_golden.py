"""Generate tests/golden/smt_cnn_golden.npz by running the UNMODIFIED ``SMTCNN`` of an upstream sound-spaces checkout
(ss_baselines/savi/models/smt_cnn.py, with ``ResizeCenterCropper`` and ``custom_resnet18`` from
ss_baselines/common/utils.py and savi/models/smt_resnet.py; path in ``SOUNDSPACES_REFERENCE``) in float64:

    SOUNDSPACES_REFERENCE=<sound-spaces checkout> python tests/golden/make_smt_cnn_golden.py

``common/utils.py`` imports habitat, habitat_sim (``d3_40_colors_rgb``), gym, moviepy, cv2 and the tensorboard
writer at module level; they are stubbed here (none of them is used by the resize, the crop or the network).  The
observations (``smt_cnn_models.observations``) and the parameters (``smt_cnn_models.set_params``, seeded by module
name) are regenerated from seeds, so per shape ``<name>/<key>`` only stores ``config`` (B, H, W, seed), the sums of the
generated ``rgb`` / ``depth`` (to catch a drifting generator), the preprocessed 64 x 64 images ``rgb_img`` /
``depth_img`` (what ``obs_transform`` returns; the reference resizes in float32, so they are stored as float32) and
the RGB-D encoder's output ``out`` (B, 128).
"""
import importlib.util
import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from smt_cnn_models import observations, set_params  # noqa: E402
from oracle.ref_harness import REFERENCE_ROOT  # noqa: E402

# name: (B, H, W, seed): SAVi's 128 x 128 sensors, a 4:3 frame resized to 64 x 85, overlapping bins at 100 x 100,
# upsampling at 48 x 48, and 256 x 256
SHAPES = {"s128": (2, 128, 128, 1), "s96x128": (2, 96, 128, 2), "s100": (2, 100, 100, 3), "s48": (2, 48, 48, 4),
          "s256": (2, 256, 256, 5)}
PARAM_SEED = 7


class Box:
    def __init__(self, low=0.0, high=1.0, shape=None, dtype=np.float32):
        self.low, self.high, self.shape, self.dtype = low, high, tuple(shape), dtype


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
    anything = type("Anything", (), {"__call__": lambda self, *a, **k: self, "__getattr__": lambda self, n: self})()
    for pkg in ("ss_baselines", "ss_baselines.common", "ss_baselines.savi", "ss_baselines.savi.models", "habitat",
                "habitat.utils", "habitat.utils.visualizations", "habitat_sim", "habitat_sim.utils", "moviepy",
                "moviepy.audio", "gym"):
        _stub(pkg)
    sys.modules["habitat"].logger = anything
    _stub("habitat.utils.visualizations.utils", images_to_video=anything, draw_collision=anything)
    _stub("habitat.utils.visualizations.maps")
    sys.modules["habitat.utils.visualizations"].maps = sys.modules["habitat.utils.visualizations.maps"]
    _stub("habitat_sim.utils.common", d3_40_colors_rgb=np.zeros((40, 3), np.uint8))
    _stub("gym.spaces", Box=Box)
    _stub("moviepy.editor")
    _stub("moviepy.audio.AudioClip", CompositeAudioClip=anything, AudioArrayClip=anything)
    _stub("ss_baselines.common.tensorboard_utils", TensorboardWriter=anything)
    if "cv2" not in sys.modules:
        try:
            import cv2  # noqa: F401
        except Exception:
            _stub("cv2")

    def load(modname, rel):
        spec = importlib.util.spec_from_file_location(modname, os.path.join(REFERENCE_ROOT, "ss_baselines", rel))
        mod = importlib.util.module_from_spec(spec)
        sys.modules[modname] = mod
        spec.loader.exec_module(mod)
        return mod

    utils = load("ss_baselines.common.utils", "common/utils.py")
    load("ss_baselines.savi.models.smt_resnet", "savi/models/smt_resnet.py")
    smt_cnn = load("ss_baselines.savi.models.smt_cnn", "savi/models/smt_cnn.py")
    return smt_cnn.SMTCNN, utils.ResizeCenterCropper


def main():
    SMTCNN, _ = load_reference()
    out = {}
    for name, (B, H, W, seed) in SHAPES.items():
        space = ObservationSpace({"rgb": Box(0, 255, (H, W, 3)), "depth": Box(0.0, 1.0, (H, W, 1))})
        ref = set_params(SMTCNN(space), PARAM_SEED).double().eval()
        obs = observations(B, H, W, seed)
        obs64 = {k: v.double() for k, v in obs.items()}
        with torch.no_grad():
            y = ref(obs64)
            rgb_img = ref.obs_transform(obs64["rgb"].permute(0, 3, 1, 2) / 255.0)
            depth_img = ref.obs_transform(obs64["depth"].permute(0, 3, 1, 2))
        out[f"{name}/config"] = np.array([B, H, W, seed], np.int64)
        out[f"{name}/rgb_sum"] = np.array(obs["rgb"].double().sum().item())
        out[f"{name}/depth_sum"] = np.array(obs["depth"].double().sum().item())
        out[f"{name}/rgb_img"] = rgb_img.numpy().astype(np.float32)
        out[f"{name}/depth_img"] = depth_img.numpy().astype(np.float32)
        out[f"{name}/out"] = y.numpy()
    out["param_seed"] = np.array(PARAM_SEED)
    dst = os.path.join(ROOT, "tests", "golden", "smt_cnn_golden.npz")
    np.savez_compressed(dst, **out)
    print("wrote", dst, os.path.getsize(dst), "bytes")


if __name__ == "__main__":
    main()
