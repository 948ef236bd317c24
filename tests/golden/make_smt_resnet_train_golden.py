"""Generate tests/golden/smt_resnet_train_golden.npz by running the UNMODIFIED reference ``custom_resnet18`` of an
upstream sound-spaces checkout (ss_baselines/savi/models/smt_resnet.py, path in ``SOUNDSPACES_REFERENCE``) in float64
with ``fc = Linear(4608, 2)``, as belief_predictor.py:65-71 builds the online location predictor, on 2 input channels
and on 23 (with the distractor sound's category channels, cnn_forward :123-134), forward and backward of
train_belief_predictor's masked MSE (ppo_trainer.py:375-381).

    SOUNDSPACES_REFERENCE=<sound-spaces checkout> python tests/golden/make_smt_resnet_train_golden.py

Parameters come from ``set_params`` and the inputs from seeds (``case_inputs`` in tests/smt_resnet_train_models.py:
4 rows of 65 x 26, row 1 silent, row 2 scaled by 1e-3), so only results are stored, per case ``<name>/<key>``:
``pred`` and, of the 62 parameter gradients (20 conv weights, 20 GroupNorm weights, 20 biases, fc weight and bias),
``g<j>`` whole for tensors of at most 512 elements, else ``g<j>_sample`` (48 seeded elements) and ``g<j>_proj`` (12
seeded Gaussian projections of every element).
"""
import importlib.util
import os
import sys

import numpy as np
import torch
import torch.nn as nn

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from smt_resnet_train_models import CASES, case_inputs, grad_summary, set_params, torch_grads  # noqa: E402


def load_custom_resnet18():
    from oracle.ref_harness import REFERENCE_ROOT
    path = os.path.join(REFERENCE_ROOT, "ss_baselines", "savi", "models", "smt_resnet.py")
    spec = importlib.util.spec_from_file_location("ss_baselines.savi.models.smt_resnet", path)
    mod = importlib.util.module_from_spec(spec)
    sys.modules[spec.name] = mod
    spec.loader.exec_module(mod)
    return mod.custom_resnet18


def main():
    custom_resnet18 = load_custom_resnet18()
    out = {}
    for name, n in CASES.items():
        net = custom_resnet18(num_input_channels=2 + n)
        net.fc = nn.Linear(4608, 2)
        set_params(net).double()
        x, labels, gts = case_inputs(name)
        pred, grads = torch_grads(net, x, labels, gts)
        out[f"{name}/pred"] = pred.numpy()
        for j, g in enumerate(grads):
            for suffix, v in grad_summary(name, j, g.numpy()).items():
                out[f"{name}/g{j}{suffix}"] = v
    dst = os.path.join(ROOT, "tests", "golden", "smt_resnet_train_golden.npz")
    np.savez_compressed(dst, **out)
    print("wrote", dst, os.path.getsize(dst), "bytes")


if __name__ == "__main__":
    main()
