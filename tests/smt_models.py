"""A stand-in for SAVi's ``SMTStateEncoder`` (ss_baselines/savi/models/smt_state_encoder.py) written from its
documented computation, plus seeded weights and the inputs the tests feed it.  ``tests/golden/smt_golden.npz`` (made by
``tests/golden/make_smt_golden.py`` from the real class) pins it to the reference.

The computation: append an always-valid column for the current token to the (N, M) masks (zeros instead of the M
columns under pretraining); a token is padding iff ``1 - mask > 0``.  With pose encoding (``pi = pose_indices[0]``),
every token's pose (x, y, heading, time) at columns pi .. pi + 3 is taken relative to the agent's pose, formatted as
[x, y, cos h, sin h, exp(-t)] and replaced by ``pose_encoder`` (Linear(5, 16)).  ``fusion_encoder`` maps all M + 1
tokens to d_model; ``nn.Transformer`` (one encoder, one decoder layer, post-norm, ReLU) takes them as ``src`` and the
goal (or the fused current token) as ``tgt``, with the same padding mask for the source and the decoder's memory.
"""
import math

import torch
import torch.nn as nn


class SMTStandIn(nn.Module):
    def __init__(self, input_size, nhead=8, d_model=256, dropout=0.0, pose_index=None, pretraining=False):
        super().__init__()
        self._pose_indices = None if pose_index is None else (pose_index, input_size)
        self._use_pose_encoding = pose_index is not None
        self._pretraining = pretraining
        fused_in = input_size
        if self._use_pose_encoding:
            self.pose_encoder = nn.Linear(5, 16)
            fused_in = pose_index + 16
        self.fusion_encoder = nn.Sequential(nn.Linear(fused_in, d_model), nn.ReLU(), nn.Linear(d_model, d_model))
        self.transformer = nn.Transformer(d_model, nhead, 1, 1, d_model, dropout, "relu")

    @staticmethod
    def _relative(agent, other):
        """(x, y, heading) of ``other`` in ``agent``'s frame, heading measured from x towards -y."""
        ha, hb = -agent[..., 2], -other[..., 2]
        dx, dy = other[..., 0] - agent[..., 0], other[..., 1] - agent[..., 1]
        r = torch.sqrt(dx * dx + dy * dy)
        phi = torch.atan2(dy, dx) - ha
        dh = hb - ha
        return torch.stack([r * torch.cos(phi), r * torch.sin(phi), -torch.atan2(torch.sin(dh), torch.cos(dh))], -1)

    def _pose_tokens(self, feats, agent):
        pi = self._pose_indices[0]
        rel = self._relative(agent, feats[..., pi:pi + 3])
        t = feats[..., pi + 3]
        fmt = torch.stack([rel[..., 0], rel[..., 1], torch.cos(rel[..., 2]), torch.sin(rel[..., 2]), torch.exp(-t)], -1)
        return torch.cat([feats[..., :pi], self.pose_encoder(fmt)], -1)

    def single_forward(self, x, memory, memory_masks, goal=None):
        N, M = memory_masks.shape
        cols = torch.zeros_like(memory_masks) if self._pretraining else memory_masks
        masks = torch.cat([cols, memory_masks.new_ones(N, 1)], 1)
        padding = (1 - masks) > 0
        tokens = torch.cat([memory, x[None]], 0)                           # (M + 1, N, D)
        if self._use_pose_encoding:
            pi = self._pose_indices[0]
            tokens = self._pose_tokens(tokens, x[None, :, pi:pi + 3])
        fused = self.fusion_encoder(tokens)
        tgt = goal[None] if goal is not None else fused[-1:]
        return self.transformer(fused, tgt, src_key_padding_mask=padding, memory_key_padding_mask=padding)[-1]

    def forward(self, x, memory, *args, **kwargs):
        return self.single_forward(x, memory, *args, **kwargs)


def randomize(module, seed=0):
    """Seeded weights at a scale that keeps activations O(1); LayerNorm gamma / beta away from 1 / 0."""
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for name, p in module.named_parameters():
            if "norm" in name and name.endswith("weight"):
                p.copy_(1.0 + 0.3 * torch.randn(p.shape, generator=g))
            elif name.endswith("bias"):
                p.copy_(0.1 * torch.randn(p.shape, generator=g))
            else:
                p.copy_(torch.randn(p.shape, generator=g) / math.sqrt(p.shape[-1]))
    return module


def make_smt(D=276, pose_index=272, d_model=256, nhead=8, pretraining=False, seed=0, dropout=0.0):
    return randomize(SMTStandIn(D, nhead, d_model, dropout, pose_index, pretraining), seed)


def ring_masks(N, M, valid, start=0, gen=None):
    """Masks of a ring buffer of M slots holding ``valid[n]`` entries ending just before ``start[n]`` (wrapping)."""
    masks = torch.zeros(N, M)
    for n in range(N):
        v = valid[n] if hasattr(valid, "__len__") else valid
        s = start[n] if hasattr(start, "__len__") else start
        for i in range(v):
            masks[n, (s - 1 - i) % M] = 1.0
    return masks


def episode_masks(N, M, steps, dones_every, gen):
    """Masks after ``steps`` writes into slot ``t % M`` with episodes reset by dones (an env's slots are cleared when
    its episode ends, as the trainer's masks do)."""
    masks = torch.zeros(N, M)
    for t in range(steps):
        done = torch.rand(N, generator=gen) < 1.0 / dones_every
        masks[done] = 0.0
        masks[:, t % M] = 1.0
    return masks


def make_inputs(N, M, D=276, d_model=256, pose_index=272, seed=0, valid=None, goal=True, masks=None):
    """x (N, D), memory (M, N, D), masks (N, M), goal (N, d_model) or None; poses form trajectories (positions drift,
    headings wrap past pi, time counts steps)."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(N, D, generator=g)
    memory = torch.randn(M, N, D, generator=g)
    if pose_index is not None:
        T = M + 1
        steps = torch.randn(T, N, 2, generator=g).cumsum(0) * 0.5
        heading = (torch.randn(T, N, generator=g) * 0.4).cumsum(0)
        time = torch.arange(T, dtype=torch.float32)[:, None].expand(T, N) * 0.05
        pose = torch.stack([steps[..., 0], steps[..., 1], heading, time], -1)
        memory[..., pose_index:pose_index + 4] = pose[:M]
        x[:, pose_index:pose_index + 4] = pose[M]
    if masks is None:
        if valid is None:
            valid = [(M * (n + 1)) // (N + 1) for n in range(N)]
        masks = ring_masks(N, M, valid, start=[(7 * n) % max(M, 1) for n in range(N)]) if M else torch.zeros(N, 0)
    gl = torch.randn(N, d_model, generator=g) if goal else None
    return x, memory, masks, gl
