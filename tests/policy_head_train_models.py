"""Stand-ins for ``Policy.evaluate_actions`` of the reference's three trainers (ss_baselines/av_nav/ppo/policy.py:70-82,
savi/ppo/policy.py:73-93, av_wan/ppo/policy.py:68-80) on the heads of tests/policy_head_models.py, and the cases of
tests/golden/policy_head_train_golden.npz (tests/golden/make_policy_head_train_golden.py), which pins them to the
reference classes in float64.  ``FeatureNet`` stands in for ``self.net``: it hands back ``observations["features"]``
as the features, so a test chooses them bit for bit and they can be a leaf that collects dfeatures.
"""
import torch
import torch.nn as nn

import policy_head_models as phm

TRAINERS = ("av_nav", "savi", "av_wan")
# name: (trainer, H, A, N, seed, gain, masking, special); the five cases of make_policy_head_golden.py plus a head
# with a -Inf actor bias (every row has a -Inf logit beside finite ones) and masked-out actions taken
CASES = {
    "av_nav": ("av_nav", 16, 4, 6, 1, 3.0, 1, ""),
    "av_nav_flat": ("av_nav", 24, 4, 4, 2, 0.01, 1, ""),
    "savi": ("savi", 12, 4, 5, 3, 3.0, 1, ""),
    "av_wan_masked": ("av_wan", 16, 9, 6, 4, 3.0, 1, ""),
    "av_wan_unmasked": ("av_wan", 16, 9, 5, 5, 3.0, 0, ""),
    "av_nav_neg_inf": ("av_nav", 16, 4, 7, 6, 3.0, 1, "neg_inf"),
    "av_wan_masked_taken": ("av_wan", 16, 9, 8, 7, 3.0, 1, "masked_taken"),
}
NEG_INF_ACTION = 1          # the action whose bias is -Inf in "neg_inf" cases


class FeatureNet(nn.Module):
    def __init__(self, H, memory=False):
        super().__init__()
        self.output_size = H
        self.memory = memory

    def forward(self, observations, rnn_hidden_states, prev_actions, masks, *ext):
        features = observations["features"]
        return (features, rnn_hidden_states, features * 2) if self.memory else (features, rnn_hidden_states)


class AvNavPolicy(phm.AvNavPolicy):
    def evaluate_actions(self, observations, rnn_hidden_states, prev_actions, masks, action):
        features, rnn_hidden_states = self.net(observations, rnn_hidden_states, prev_actions, masks)
        distribution = self.action_distribution(features)
        value = self.critic(features)
        return value, distribution.log_probs(action), distribution.entropy().mean(), rnn_hidden_states


class SaviPolicy(phm.SaviPolicy):
    def evaluate_actions(self, observations, rnn_hidden_states, prev_actions, masks, action, ext_memory,
                         ext_memory_masks):
        features, rnn_hidden_states, ext_memory_feats = self.net(observations, rnn_hidden_states, prev_actions,
                                                                 masks, ext_memory, ext_memory_masks)
        distribution = self.action_distribution(features)
        value = self.critic(features)
        return (value, distribution.log_probs(action), distribution.entropy().mean(), rnn_hidden_states,
                ext_memory_feats)


class AvWanPolicy(phm.AvWanPolicy):
    def evaluate_actions(self, observations, rnn_hidden_states, prev_actions, masks, action):
        features, rnn_hidden_states = self.net(observations, rnn_hidden_states, prev_actions, masks)
        distribution = self.action_distribution(features, observations["action_map"])
        value = self.critic(features)
        return value, distribution.log_probs(action), distribution.entropy().mean(), rnn_hidden_states


POLICIES = {"av_nav": AvNavPolicy, "savi": SaviPolicy, "av_wan": AvWanPolicy}


def set_head_params(policy, seed, gain=1.0, special=""):
    """tests/policy_head_models.py's ``set_params`` for the two heads only; ``special`` "neg_inf" sets the actor's
    bias of ``NEG_INF_ACTION`` to -Inf."""
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for lin, scale in ((policy.action_distribution.linear, gain), (policy.critic.fc, 1.0)):
            lin.weight.copy_(torch.randn(lin.weight.shape, generator=g, dtype=torch.float32) * scale
                             / lin.in_features ** 0.5)
            lin.bias.copy_(torch.randn(lin.bias.shape, generator=g, dtype=torch.float32) * 0.1)
        if special == "neg_inf":
            policy.action_distribution.linear.bias[NEG_INF_ACTION] = float("-inf")
    return policy


def make_policy(trainer, H, A, seed=0, gain=1.0, masking=True, special="", classes=None):
    """A trainer's policy (the stand-ins, or ``classes`` such as the reference's) on a ``FeatureNet``."""
    net = FeatureNet(H, memory=trainer == "savi")
    cls = (classes or POLICIES)[trainer]
    policy = cls(net, A, bool(masking)) if trainer == "av_wan" else cls(net, A)
    return set_head_params(policy, seed, gain, special)


def case_inputs(name):
    """(features (N, H), action_map (N, A) or None, actions (N, 1) int64, g_value (N, 1), g_log_prob (N, 1),
    g_entropy scalar) of a case, from its seed, float32 values in float64 tensors."""
    trainer, H, A, N, seed, gain, masking, special = CASES[name]
    g = torch.Generator().manual_seed(200 + seed)
    features = torch.tanh(torch.randn((N, H), generator=g) * 2).double()
    amap = phm.action_map(N, A, seed).double() if trainer == "av_wan" else None
    actions = torch.randint(0, A, (N, 1), generator=g)
    if special == "neg_inf":
        actions[actions == NEG_INF_ACTION] = NEG_INF_ACTION + 1
    if special == "masked_taken":               # every other row takes a masked-out waypoint
        for n in range(0, N, 2):
            closed = torch.nonzero(amap[n] == 0).view(-1)
            if len(closed):
                actions[n, 0] = closed[0]
    gv, glp = (torch.randn((N, 1), generator=g).double() for _ in range(2))
    ge = float(torch.randn((), generator=g))
    return features, amap, actions, gv, glp, ge


def evaluate_args(trainer, observations, action):
    """Arguments of ``evaluate_actions`` for the trainer: (args, kwargs)."""
    N = action.shape[0]
    x = observations["features"]
    h = torch.zeros((1, N, 4), dtype=x.dtype, device=x.device)
    prev = torch.zeros((N, 1), dtype=torch.int64, device=x.device)
    masks = torch.ones((N, 1), dtype=x.dtype, device=x.device)
    args = [observations, h, prev, masks, action]
    if trainer == "savi":
        args += [torch.zeros((3, N, 4), dtype=x.dtype, device=x.device),
                 torch.ones((N, 3), dtype=x.dtype, device=x.device)]
    return args, {}


def forward_backward(policy, trainer, features, amap, actions, gv, glp, ge):
    """evaluate_actions on ``features`` (made a leaf) and the gradients of sum(gv value) + sum(glp log_probs) +
    ge entropy -> (value, log_probs, entropy, dfeatures, d actor weight, d actor bias, d critic weight,
    d critic bias)."""
    x = features.detach().clone().requires_grad_(True)
    obs = {"features": x}
    if amap is not None:
        obs["action_map"] = amap
    args, kw = evaluate_args(trainer, obs, actions)
    value, lp, ent = policy.evaluate_actions(*args, **kw)[:3]
    params = [policy.action_distribution.linear.weight, policy.action_distribution.linear.bias,
              policy.critic.fc.weight, policy.critic.fc.bias]
    loss = (gv * value).sum() + (glp * lp).sum() + ge * ent
    grads = torch.autograd.grad(loss, [x] + params)
    return (value.detach(), lp.detach(), ent.detach()) + tuple(grads)


OUTPUTS = ("value", "log_prob", "entropy", "dfeatures", "dactor_weight", "dactor_bias", "dcritic_weight",
           "dcritic_bias")
