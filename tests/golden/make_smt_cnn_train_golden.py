"""Generate tests/golden/smt_cnn_train_golden.npz by running the UNMODIFIED ``SMTCNN`` of an upstream sound-spaces
checkout (ss_baselines/savi/models/smt_cnn.py, loaded with the stubs of make_smt_cnn_golden.py; path in
``SOUNDSPACES_REFERENCE``) in float64, forward and backward of sum(out * g) with a seeded g:

    SOUNDSPACES_REFERENCE=<sound-spaces checkout> python tests/golden/make_smt_cnn_train_golden.py

Observations, parameters and g come from seeds (tests/smt_cnn_train_models.py: 128 x 128 RGB-D, 96 x 128 RGB-D, RGB
only and depth only, 3-4 rows with an all-zero depth row and a row scaled by 1e-3), so per case ``<name>/<key>`` only
stores ``out`` and, of the 62 parameter gradients per encoder (RGB first; 20 conv weights, 20 GroupNorm weights, 20
biases, fc weight and bias), ``g<j>`` whole for tensors of at most 512 elements, else ``g<j>_sample`` and
``g<j>_proj`` (smt_resnet_train_models.grad_summary).
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from make_smt_cnn_golden import Box, ObservationSpace, load_reference  # noqa: E402
from smt_cnn_models import set_params  # noqa: E402
from smt_cnn_train_models import CASES, PARAM_SEED, case_grad, case_observations, forward_backward  # noqa: E402
from smt_resnet_train_models import grad_summary  # noqa: E402


def main():
    SMTCNN, _ = load_reference()
    out = {}
    for name, (B, H, W, mods, _) in CASES.items():
        spaces = {}
        if "rgb" in mods:
            spaces["rgb"] = Box(0, 255, (H, W, 3))
        if "depth" in mods:
            spaces["depth"] = Box(0.0, 1.0, (H, W, 1))
        ref = set_params(SMTCNN(ObservationSpace(spaces)), PARAM_SEED).double()
        obs = case_observations(name)
        y, grads = forward_backward(ref, obs, case_grad(name, 64 * len(mods)))
        out[f"{name}/out"] = y.numpy()
        for j, g in enumerate(grads):
            for k, v in grad_summary(name, j, g.numpy()).items():
                out[f"{name}/g{j}{k}"] = v
    dst = os.path.join(ROOT, "tests", "golden", "smt_cnn_train_golden.npz")
    np.savez_compressed(dst, **out)
    print("wrote", dst, os.path.getsize(dst), "bytes")


if __name__ == "__main__":
    main()
