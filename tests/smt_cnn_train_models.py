"""Cases of SAVi's visual encoder trained in the PPO update (ssb_smt_cnn_train_*) for
tests/golden/smt_cnn_train_golden.npz: seeded observations with an all-zero depth row and a row scaled by 1e-3, a
seeded upstream gradient g of the features, and the forward and backward of sum(out * g) through an ``SMTCNN`` in
its parameters' dtype.  Parameters come from ``smt_cnn_models.set_params``, keyed by module name, so the reference
class and the stand-in get equal values."""
import numpy as np
import torch

from smt_cnn_models import SMTCNN, observations, set_params

PARAM_SEED = 11
# name: (B, H, W, modalities, seed)
CASES = {"rgbd128": (4, 128, 128, ("rgb", "depth"), 21), "rgbd96x128": (3, 96, 128, ("rgb", "depth"), 22),
         "rgb128": (3, 128, 128, ("rgb",), 31), "depth128": (4, 128, 128, ("depth",), 24)}


def case_observations(name):
    """{modality: (B, H, W, C) float32}: row 1's depth all zero, row 2 scaled by 1e-3."""
    B, H, W, mods, seed = CASES[name]
    obs = observations(B, H, W, seed, rgb=3 if "rgb" in mods else 0, depth=1 if "depth" in mods else 0)
    if "depth" in obs:
        obs["depth"][1] = 0.0
    for m in obs:
        obs[m][2] *= 1e-3
    return obs


def case_grad(name, n_out):
    """The seeded upstream gradient (B, n_out) of the features."""
    B, _, _, _, seed = CASES[name]
    return torch.randn((B, n_out), generator=torch.Generator().manual_seed(1000 + seed), dtype=torch.float64)


def standin(name, dtype=torch.float64):
    """The stand-in ``SMTCNN`` of a case with the seeded parameters."""
    mods = CASES[name][3]
    return set_params(SMTCNN({m: 3 if m == "rgb" else 1 for m in mods}), PARAM_SEED).to(dtype)


def params(module):
    from soundspaces_b200.encoder import smt_cnn_params
    return smt_cnn_params(module)


def forward_backward(module, obs, g):
    """(out, the 62 n parameter gradients) of sum(module(obs) * g) in the parameters' dtype."""
    dt = next(module.parameters()).dtype
    module.zero_grad(set_to_none=True)
    out = module({m: v.to(dt) for m, v in obs.items()})
    (out * g.to(dt)).sum().backward()
    return out.detach(), [p.grad.detach().clone() for p in params(module)]
