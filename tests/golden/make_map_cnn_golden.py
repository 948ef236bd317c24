"""Generate tests/golden/map_cnn_golden.npz by running the UNMODIFIED reference ``MapCNN`` of an upstream sound-spaces
checkout (path in ``SOUNDSPACES_REFERENCE``, as for the other oracle fixtures) in float64:
ss_baselines/av_wan/models/map_cnn.py on the 200 x 200 x 2 and 400 x 400 x 2 geometric maps and the 20 x 20 x 1
acoustic map, hidden = 8.

    SOUNDSPACES_REFERENCE=<sound-spaces checkout> python tests/golden/make_map_cnn_golden.py

``map_cnn.py`` imports ``Flatten`` from ss_baselines.common.utils (whose other imports are habitat, moviepy, cv2 ...)
and ``conv_output_dim`` / ``layer_init`` from ss_baselines/av_nav/models/visual_cnn.py; the first is stubbed with its
computation, the second is loaded unmodified.  Parameters come from ``set_params`` (tests/avnav_models.py) and maps
from ``map_obs`` (tests/map_cnn_models.py), both from seeds, so only the configuration and the outputs are stored, per
configuration ``<name>/<key>``: ``config`` (H, W, C, hidden, N, param seed, input seed) and ``out``.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))

from avnav_models import set_params  # noqa: E402
from make_avnav_policy_golden import ObservationSpace, Space, _stub, load_reference  # noqa: E402
from map_cnn_models import REFERENCE_SHAPES, map_obs  # noqa: E402

HIDDEN, N = 8, 2
# name: (param seed, input seed); the inputs are reference-like (map_obs kind = the map type)
SEEDS = {"gm200": (50, 60), "gm400": (51, 61), "am20": (52, 62)}


def load_map_cnn():
    import importlib.util
    from oracle.ref_harness import REFERENCE_ROOT
    load_reference()                    # stubs ss_baselines.common.utils and loads av_nav's visual_cnn
    _stub("ss_baselines.av_wan.models")
    spec = importlib.util.spec_from_file_location("ss_baselines.av_wan.models.map_cnn",
                                                  os.path.join(REFERENCE_ROOT, "ss_baselines", "av_wan", "models",
                                                               "map_cnn.py"))
    mod = importlib.util.module_from_spec(spec)
    sys.modules[spec.name] = mod
    spec.loader.exec_module(mod)
    return mod.MapCNN


def main():
    MapCNN = load_map_cnn()
    out = {}
    for name, (map_type, H, W, C) in REFERENCE_SHAPES.items():
        pseed, xseed = SEEDS[name]
        ref = MapCNN(ObservationSpace({map_type: Space((H, W, C))}), HIDDEN, map_type=map_type)
        set_params(ref, seed=pseed)
        ref = ref.double().eval()
        x = map_obs(N, H, W, C, seed=xseed, kind=map_type).double()
        with torch.no_grad():
            y = ref({map_type: x})
        assert (y.abs().amax(dim=1) > 0).all(), name
        out[f"{name}/config"] = np.array([H, W, C, HIDDEN, N, pseed, xseed], np.int64)
        out[f"{name}/out"] = y.numpy()
    dst = os.path.join(ROOT, "tests", "golden", "map_cnn_golden.npz")
    np.savez_compressed(dst, **out)
    print("wrote", dst, os.path.getsize(dst), "bytes")


if __name__ == "__main__":
    main()
