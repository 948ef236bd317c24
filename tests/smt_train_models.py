"""Cases of SAVi's scene memory transformer trained in the PPO update (ssb_smt_state_encoder_train_*) for
tests/golden/smt_train_golden.npz: seeded modules and inputs (smt_models), a seeded upstream gradient g of the output,
and the forward and backward of sum(out * g) through an ``SMTStateEncoder`` in its parameters' dtype.  The cases cover
a goal and none, pose encoding and none, pretraining, rows with no valid memory, a memory token at the agent's exact
position, and wrapped ring masks."""
import torch

from smt_models import episode_masks, make_inputs, randomize, SMTStandIn as _StandIn


class SMTStandIn(_StandIn):
    """smt_models' stand-in with the distance as the reference computes it (``torch.norm``), whose backward is 0 at
    distance 0 where ``sqrt``'s is NaN: a memory token at the agent's exact position."""

    @staticmethod
    def _relative(agent, other):
        ha, hb = -agent[..., 2], -other[..., 2]
        dx, dy = other[..., 0] - agent[..., 0], other[..., 1] - agent[..., 1]
        r = torch.norm(agent[..., :2] - other[..., :2], dim=-1)
        phi = torch.atan2(dy, dx) - ha
        dh = hb - ha
        return torch.stack([r * torch.cos(phi), r * torch.sin(phi), -torch.atan2(torch.sin(dh), torch.cos(dh))], -1)

# name: (D, pose index or None, d_model, nhead, pretraining, goal, N, M, masks, seed)
CASES = {
    "pose_goal": (20, 16, 32, 4, False, True, 3, 9, "ring", 1),
    "pose_no_goal": (20, 16, 32, 4, False, False, 3, 9, "ring", 2),
    "no_pose_goal": (12, None, 16, 2, False, True, 2, 6, "ring", 3),
    "no_pose_no_goal": (12, None, 16, 1, False, False, 3, 6, "episodes", 4),
    "pretraining": (20, 16, 32, 8, True, False, 3, 9, "ring", 5),
    "current_only": (20, 16, 32, 4, False, True, 3, 9, "none", 6),
    "at_agent": (20, 16, 32, 4, False, False, 3, 9, "ring", 7),
    "wrapped": (20, 16, 32, 4, False, True, 4, 12, "episodes", 8),
}


def case_module(cls, name, dtype=torch.float64):
    """``cls`` (the reference ``SMTStateEncoder`` or smt_models.SMTStandIn) with the case's seeded parameters."""
    D, pi, d, nhead, pre, _, _, _, _, seed = CASES[name]
    if cls is SMTStandIn:
        m = SMTStandIn(D, nhead, d, 0.0, pi, pre)
    else:
        m = cls(D, nhead=nhead, dim_feedforward=d, dropout=0.0, pose_indices=None if pi is None else (pi, D),
                pretraining=pre)
    return randomize(m, seed=200 + seed).to(dtype).eval()


def case_inputs(name):
    """x (N, D), memory (M, N, D), masks (N, M), goal (N, d) or None, g (N, d), all float32.  ``current_only``:
    every row has no valid memory slot; ``at_agent``: a valid memory slot of each row lies at the agent's (x, y)."""
    D, pi, d, _, _, goal, N, M, kind, seed = CASES[name]
    x, memory, masks, gl = make_inputs(N, M, D, d, pi, seed=300 + seed, goal=goal)
    gen = torch.Generator().manual_seed(400 + seed)
    if kind == "none":
        masks = torch.zeros(N, M)
    elif kind == "episodes":
        masks = episode_masks(N, M, 2 * M + 3, 5, gen)
        masks[0] = 0.0
    if name == "at_agent":
        for n in range(N):
            j = int(torch.nonzero(masks[n])[0])
            memory[j, n, pi:pi + 2] = x[n, pi:pi + 2]
    g = torch.randn(N, d, generator=gen)
    return x, memory, masks, gl, g


def forward_backward(module, x, memory, masks, goal, g):
    """(out, [grads of smt_train_parameters(module)], dx, dgoal) of sum(single_forward(...) * g) in the module's
    dtype."""
    from soundspaces_b200.smt import smt_train_parameters
    dt = next(module.parameters()).dtype
    module.zero_grad(set_to_none=True)
    x = x.to(dt).clone().requires_grad_(True)
    goal = goal.to(dt).clone().requires_grad_(True) if goal is not None else None
    out = module.single_forward(x, memory.to(dt), masks.to(dt), goal)
    (out * g.to(dt)).sum().backward()
    grads = [p.grad.detach().clone() if p.grad is not None else torch.zeros_like(p)
             for p in smt_train_parameters(module)]
    return out.detach(), grads, x.grad.detach(), None if goal is None else goal.grad.detach()
