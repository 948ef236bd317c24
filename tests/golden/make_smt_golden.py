"""Generate tests/golden/smt_golden.npz by running the UNMODIFIED ``SMTStateEncoder.single_forward`` of an upstream
sound-spaces checkout (ss_baselines/savi/models/smt_state_encoder.py, which imports only torch) in float64:

    SOUNDSPACES_REFERENCE=<sound-spaces checkout> python tests/golden/make_smt_golden.py

Small seeded configurations cover pose encoding on and off, a goal and none, pretraining, only the current token
valid, wrapped ring masks and non-binary mask values.  Stored per configuration ``<name>/<key>``: ``config`` (D,
pose index or -1, d_model, nhead, pretraining, has goal), the parameters ``w/<state_dict key>``, the inputs ``x``,
``memory``, ``masks``, ``goal`` and the output ``out``.
"""
import importlib.util
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(ROOT, "tests"))

from smt_models import episode_masks, make_inputs, randomize  # noqa: E402

# name: (D, pose index or None, d_model, nhead, pretraining, goal, N, M, masks)
CONFIGS = {
    "pose_goal": (20, 16, 32, 4, False, True, 3, 9, "ring"),
    "pose_no_goal": (20, 16, 32, 4, False, False, 3, 9, "ring"),
    "no_pose_goal": (12, None, 16, 2, False, True, 2, 6, "ring"),
    "no_pose_no_goal": (12, None, 16, 1, False, False, 2, 6, "episodes"),
    "pretraining": (20, 16, 32, 8, True, False, 3, 9, "ring"),
    "current_only": (20, 16, 32, 4, False, True, 3, 9, "none"),
    "wrapped": (20, 16, 32, 4, False, False, 4, 12, "episodes"),
    "non_binary": (20, 16, 32, 4, False, True, 3, 9, "non_binary"),
}


def load_reference_class():
    root = os.environ.get("SOUNDSPACES_REFERENCE")
    if not root:
        sys.exit("set SOUNDSPACES_REFERENCE to a sound-spaces checkout")
    path = os.path.join(root, "ss_baselines", "savi", "models", "smt_state_encoder.py")
    spec = importlib.util.spec_from_file_location("reference_smt_state_encoder", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod.SMTStateEncoder


def main():
    cls = load_reference_class()
    out = {}
    for i, (name, (D, pi, d, nhead, pre, goal, N, M, kind)) in enumerate(CONFIGS.items()):
        torch.manual_seed(100 + i)
        ref = cls(D, nhead=nhead, dim_feedforward=d, dropout=0.0, pose_indices=None if pi is None else (pi, D),
                  pretraining=pre)
        randomize(ref, seed=200 + i)
        ref = ref.double().eval()
        x, memory, masks, g = make_inputs(N, M, D, d, pi, seed=300 + i, goal=goal)
        gen = torch.Generator().manual_seed(400 + i)
        if kind == "none":
            masks = torch.zeros(N, M)
        elif kind == "episodes":
            masks = episode_masks(N, M, 2 * M + 3, 5, gen)
        elif kind == "non_binary":
            masks = torch.tensor([0.0, 0.5, 1.0, 2.0, 0.999])[torch.randint(0, 5, (N, M), generator=gen)]
        with torch.no_grad():
            y = ref.single_forward(x.double(), memory.double(), masks.double(), None if g is None else g.double())
        out[f"{name}/config"] = np.array([D, -1 if pi is None else pi, d, nhead, int(pre), int(goal)], np.int64)
        for k, v in ref.state_dict().items():
            out[f"{name}/w/{k}"] = v.numpy()
        out[f"{name}/x"], out[f"{name}/memory"], out[f"{name}/masks"] = x.double().numpy(), memory.double().numpy(), masks.double().numpy()
        if g is not None:
            out[f"{name}/goal"] = g.double().numpy()
        out[f"{name}/out"] = y.numpy()
    dst = os.path.join(ROOT, "tests", "golden", "smt_golden.npz")
    np.savez_compressed(dst, **out)
    print("wrote", dst, os.path.getsize(dst), "bytes")


if __name__ == "__main__":
    main()
