"""Stand-ins for the policies' action and value heads, written from the reference's computation:
``CustomFixedCategorical``, ``CategoricalNet`` and ``CategoricalNetWithMask`` of ss_baselines/common/utils.py:41-87,
``CriticHead`` and ``Policy.act`` of ss_baselines/av_nav/ppo/policy.py:35-60, savi/ppo/policy.py:42-65 and
av_wan/ppo/policy.py:39-60.  tests/golden/policy_head_golden.npz pins them to the reference classes in float64
(tests/golden/make_policy_head_golden.py).  ``StubNet`` stands in for ``self.net``: a Linear and a tanh over
``observations["x"]``, passing the recurrent state through.
"""
import torch
import torch.nn as nn
from torch.distributions import Categorical

# trainer: (H, A) the trainers run: AudioNavBaselineNet's 512 hidden units and 4 actions, AV-WaN's 81 waypoints,
# SAVi's SMT output width (SCENE_MEMORY_TRANSFORMER.hidden_size 128)
SHAPES = {"av_nav": (512, 4), "av_wan": (512, 81), "savi": (128, 4)}


class CustomFixedCategorical(Categorical):
    """A categorical whose samples and modes are (N, 1) and whose ``log_probs`` take (N, 1) actions."""

    def sample(self, sample_shape=torch.Size()):
        return torch.unsqueeze(Categorical.sample(self, sample_shape), -1)

    def log_probs(self, actions):
        lp = Categorical.log_prob(self, actions[..., 0])
        return lp.reshape(actions.shape[0], -1).sum(dim=1, keepdim=True)

    def mode(self):
        return torch.argmax(self.probs, dim=-1).unsqueeze(-1)


class CategoricalNet(nn.Module):
    def __init__(self, H, A):
        super().__init__()
        self.linear = nn.Linear(H, A)

    def forward(self, x):
        return CustomFixedCategorical(logits=self.linear(x))


class CategoricalNetWithMask(nn.Module):
    def __init__(self, H, A, masking):
        super().__init__()
        self.masking = masking
        self.linear = nn.Linear(H, A)

    def forward(self, features, action_maps):
        p = torch.softmax(self.linear(features), dim=1)
        if self.masking:
            p = p * action_maps.reshape(action_maps.shape[0], -1).float()
        return CustomFixedCategorical(probs=p)


class CriticHead(nn.Module):
    def __init__(self, H):
        super().__init__()
        self.fc = nn.Linear(H, 1)

    def forward(self, x):
        return self.fc(x)


class StubNet(nn.Module):
    def __init__(self, n_in, H, memory=False):
        super().__init__()
        self.fc = nn.Linear(n_in, H)
        self.memory = memory
        self.output_size = H

    def forward(self, observations, rnn_hidden_states, prev_actions, masks, *ext):
        features = torch.tanh(self.fc(observations["x"]))
        return (features, rnn_hidden_states, features * 2) if self.memory else (features, rnn_hidden_states)


class _Policy(nn.Module):
    def __init__(self, net, A, masking=None):
        super().__init__()
        self.net = net
        H = net.output_size
        self.action_distribution = CategoricalNet(H, A) if masking is None else CategoricalNetWithMask(H, A, masking)
        self.critic = CriticHead(H)

    def _head(self, features, observations, deterministic):
        if isinstance(self.action_distribution, CategoricalNetWithMask):
            distribution = self.action_distribution(features, observations["action_map"])
        else:
            distribution = self.action_distribution(features)
        value = self.critic(features)
        action = distribution.mode() if deterministic else distribution.sample()
        return value, action, distribution.log_probs(action), distribution


class AvNavPolicy(_Policy):
    def act(self, observations, rnn_hidden_states, prev_actions, masks, deterministic=False):
        features, h = self.net(observations, rnn_hidden_states, prev_actions, masks)
        value, action, log_probs, _ = self._head(features, observations, deterministic)
        return value, action, log_probs, h


class SaviPolicy(_Policy):
    def act(self, observations, rnn_hidden_states, prev_actions, masks, ext_memory, ext_memory_masks,
            deterministic=False):
        features, h, ext_memory_feats = self.net(observations, rnn_hidden_states, prev_actions, masks, ext_memory,
                                                 ext_memory_masks)
        value, action, log_probs, _ = self._head(features, observations, deterministic)
        return value, action, log_probs, h, ext_memory_feats


class AvWanPolicy(_Policy):
    def __init__(self, net, A, masking=True):
        super().__init__(net, A, masking)

    def act(self, observations, rnn_hidden_states, prev_actions, masks, deterministic=False):
        features, h = self.net(observations, rnn_hidden_states, prev_actions, masks)
        value, action, log_probs, distribution = self._head(features, observations, deterministic)
        return value, action, log_probs, h, distribution


POLICIES = {"av_nav": AvNavPolicy, "savi": SaviPolicy, "av_wan": AvWanPolicy}


def set_params(policy, seed, gain=1.0):
    """Deterministic float32-valued parameters: the actor's weights N(0, gain^2 / H), the critic's and the stub net's
    N(0, 1 / fan_in), biases N(0, 0.1^2)."""
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for lin, scale in ((policy.action_distribution.linear, gain), (policy.critic.fc, 1.0),
                           (policy.net.fc, 1.0)):
            w = torch.randn(lin.weight.shape, generator=g, dtype=torch.float32) * scale / lin.in_features ** 0.5
            lin.weight.copy_(w)
            lin.bias.copy_(torch.randn(lin.bias.shape, generator=g, dtype=torch.float32) * 0.1)
    return policy


def make_policy(trainer, H, A, n_in=8, seed=0, gain=1.0, masking=True):
    net = StubNet(n_in, H, memory=trainer == "savi")
    cls = POLICIES[trainer]
    policy = cls(net, A, masking) if trainer == "av_wan" else cls(net, A)
    return set_params(policy, seed, gain)


def action_map(N, A, seed, p_open=0.6):
    """(N, A) 0 / 1 waypoint masks with at least one open waypoint per env."""
    g = torch.Generator().manual_seed(seed)
    m = (torch.rand((N, A), generator=g, dtype=torch.float32) < p_open).float()
    m[torch.arange(N), torch.randint(0, A, (N,), generator=g)] = 1.0
    return m


def act_args(trainer, observations, N, deterministic, positional=False):
    """Arguments of ``act`` for the trainer: (args, kwargs)."""
    h = torch.zeros((1, N, 4), dtype=observations["x"].dtype, device=observations["x"].device)
    prev = torch.zeros((N, 1), dtype=torch.int64, device=h.device)
    masks = torch.ones((N, 1), dtype=h.dtype, device=h.device)
    args = [observations, h, prev, masks]
    if trainer == "savi":
        args += [torch.zeros((3, N, 4), dtype=h.dtype, device=h.device), torch.ones((N, 3), dtype=h.dtype,
                                                                                    device=h.device)]
    if positional:
        return args + [deterministic], {}
    return args, {"deterministic": deterministic}
