"""Generate tests/golden/policy_head_train_golden.npz by running the UNMODIFIED reference ``Policy.evaluate_actions``
of an upstream sound-spaces checkout (path in ``SOUNDSPACES_REFERENCE``; loaded with ``CategoricalNet``,
``CategoricalNetWithMask``, ``CriticHead`` and ``CustomFixedCategorical`` as make_policy_head_golden.py loads them) in
float64 on the CPU, forward and backward of sum(gv value) + sum(glp log_probs) + ge entropy:

    SOUNDSPACES_REFERENCE=<sound-spaces checkout> python tests/golden/make_policy_head_train_golden.py

Cases, parameters and inputs come from seeds (tests/policy_head_train_models.py, ``CASES``); per case ``<name>/<key>``
stores the inputs ``features``, ``action_map`` (AV-WaN), ``actions``, ``gv``, ``glp`` and ``ge``, and the outputs
``value``, ``log_prob``, ``entropy`` (the mean) and the gradients ``dfeatures``, ``dactor_weight``, ``dactor_bias``,
``dcritic_weight`` and ``dcritic_bias``.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from make_policy_head_golden import load_reference  # noqa: E402
from policy_head_train_models import CASES, OUTPUTS, case_inputs, forward_backward, make_policy  # noqa: E402


def main():
    classes = load_reference()
    out = {}
    for name, (trainer, H, A, N, seed, gain, masking, special) in CASES.items():
        policy = make_policy(trainer, H, A, seed, gain, masking, special, classes=classes).double()
        features, amap, actions, gv, glp, ge = case_inputs(name)
        res = forward_backward(policy, trainer, features, amap, actions, gv, glp, ge)
        rec = {"features": features, "actions": actions, "gv": gv, "glp": glp, "ge": np.float64(ge)}
        if amap is not None:
            rec["action_map"] = amap
        rec.update(zip(OUTPUTS, res))
        for k, v in rec.items():
            out[f"{name}/{k}"] = v.numpy() if isinstance(v, torch.Tensor) else v
    dst = os.path.join(ROOT, "tests", "golden", "policy_head_train_golden.npz")
    np.savez_compressed(dst, **out)
    print("wrote", dst, os.path.getsize(dst), "bytes")


if __name__ == "__main__":
    main()
