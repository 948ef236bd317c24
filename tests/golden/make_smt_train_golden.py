"""Generate tests/golden/smt_train_golden.npz by running the UNMODIFIED ``SMTStateEncoder.single_forward`` of an
upstream sound-spaces checkout (ss_baselines/savi/models/smt_state_encoder.py, loaded as make_smt_golden.py loads it;
path in ``SOUNDSPACES_REFERENCE``) in float64, forward and backward of sum(out * g) with a seeded g, stored as float32:

    SOUNDSPACES_REFERENCE=<sound-spaces checkout> python tests/golden/make_smt_train_golden.py

Parameters, inputs and g come from seeds (tests/smt_train_models.py), so per case ``<name>/<key>`` only stores
``out``, ``dx``, ``dgoal`` (with a goal) and ``g<j>``, the gradient of the j-th tensor of
``soundspaces_b200.smt.smt_train_parameters`` (ssb_smt_params order).
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from make_smt_golden import load_reference_class  # noqa: E402
from smt_train_models import CASES, case_inputs, case_module, forward_backward  # noqa: E402


def main():
    cls = load_reference_class()
    out = {}
    for name in CASES:
        y, grads, dx, dgoal = forward_backward(case_module(cls, name), *case_inputs(name))
        out[f"{name}/out"] = y.float().numpy()
        out[f"{name}/dx"] = dx.float().numpy()
        if dgoal is not None:
            out[f"{name}/dgoal"] = dgoal.float().numpy()
        for j, g in enumerate(grads):
            out[f"{name}/g{j}"] = g.float().numpy()
    dst = os.path.join(ROOT, "tests", "golden", "smt_train_golden.npz")
    np.savez_compressed(dst, **out)
    print("wrote", dst, os.path.getsize(dst), "bytes")


if __name__ == "__main__":
    main()
