"""The policy's action and value heads at rollout time: ``Policy.act`` of the reference's three trainers
(ss_baselines/av_nav/ppo/policy.py:35-60, savi/ppo/policy.py:42-65, av_wan/ppo/policy.py:39-60) with everything after
``self.net(...)`` -- the actor Linear of ``CategoricalNet`` / ``CategoricalNetWithMask``, ``CriticHead``,
``CustomFixedCategorical``'s ``sample()`` or ``mode()`` and ``log_probs()`` (common/utils.py:41-87) -- run by
``ssb_policy_head_batch`` in one launch.

    from soundspaces_b200.policy import patch_policy
    patch_policy(Policy)     # ss_baselines.{av_nav,savi,av_wan}.ppo.policy.Policy

Sampling draws the Exp(1) numbers ``q`` that ``torch.multinomial(p, 1, True)`` draws (ATen's single-sample path takes
``argmax(p / q)``) with the same call on the same generator, so a seeded rollout takes the reference's actions and
leaves the generator where the reference leaves it.  The reference validates its distribution on the host (at least
two syncs per step); the patched ``act`` reads one status word instead and raises ``ValueError`` naming the env rows
the reference would refuse.

``patch_policy(Policy, training=True)`` also replaces ``evaluate_actions`` (PPO's update; av_nav/ppo/policy.py:70-82,
savi/ppo/policy.py:73-93, av_wan/ppo/policy.py:68-80): after ``self.net`` the heads, ``log_probs(action)`` and the
per-row ``entropy()`` run through :class:`PolicyHeadFunction`, whose forward is ``ssb_policy_head_train_forward_batch``
(one launch, the rollout kernel's device code, so value and log-probabilities are bit-identical to what ``act``
returned for the same features and action and PPO's first ratio is exactly 1) and whose backward is
``ssb_policy_head_train_backward_batch`` (at most two launches, deterministic).  One status read per call replaces
the reference's two validation syncs.  ``get_value`` is untouched.
"""
from __future__ import annotations

import inspect
import sys

import torch
import torch.nn as nn
from torch.autograd.function import once_differentiable

from .rnn import _dense

MAX_ACTIONS = 256       # the kernel's limits (include/ssb200.h, ssb_policy_head_batch)
MAX_HIDDEN = 2048
MAX_ENVS = 65535
MAX_TRAIN_ROWS = 4096 * 256   # ssb_policy_head_train_*: the largest minibatch of the patched recurrent_generator


def policy_head_layout_error(policy) -> str:
    """Why ``policy``'s heads are not ``action_distribution.linear`` = ``nn.Linear(H, A)`` with bias and
    ``critic.fc`` = ``nn.Linear(H, 1)`` with bias, with A and H within the kernel's limits; ``""`` when they are.
    A ``masking`` attribute on ``action_distribution`` selects the masked head (CategoricalNetWithMask)."""
    actor = getattr(getattr(policy, "action_distribution", None), "linear", None)
    critic = getattr(getattr(policy, "critic", None), "fc", None)
    for name, lin in (("action_distribution.linear", actor), ("critic.fc", critic)):
        if type(lin) is not nn.Linear:
            return f"{name} is {type(lin).__name__}, not nn.Linear"
        if lin.bias is None:
            return f"{name} has no bias"
    if critic.out_features != 1:
        return f"critic.fc has {critic.out_features} outputs, expected 1"
    if critic.in_features != actor.in_features:
        return f"critic.fc takes {critic.in_features} features, action_distribution.linear {actor.in_features}"
    if actor.out_features > MAX_ACTIONS or actor.in_features > MAX_HIDDEN:
        return (f"{actor.out_features} actions of {actor.in_features} features, the kernel is built for at most "
                f"{MAX_ACTIONS} and {MAX_HIDDEN}")
    return ""


def _head_inputs(policy, features, observations, max_rows=MAX_ENVS):
    """(masked, mask or None) for the fused head on ``features``, or None when the call must run the reference's
    head: a parameter or ``features`` not contiguous CUDA float32 on one device, ``features`` not (N, H) with
    N <= ``max_rows``, or, with masking on, an ``action_map`` that does not hold A values per env on that device."""
    if not isinstance(features, torch.Tensor) or features.ndim != 2 or not _dense(features, features.device):
        return None
    actor, critic = policy.action_distribution.linear, policy.critic.fc
    dev = features.device
    if not all(_dense(p, dev) for p in (actor.weight, actor.bias, critic.weight, critic.bias)):
        return None
    N, H = features.shape
    if H != actor.in_features or N > max_rows:
        return None
    masked = hasattr(policy.action_distribution, "masking")
    if not (masked and policy.action_distribution.masking):
        return masked, None
    am = observations["action_map"]
    if not (isinstance(am, torch.Tensor) and am.device == dev and am.ndim >= 1 and am.shape[0] == N
            and am.numel() == N * actor.out_features):
        return None
    return masked, torch.reshape(am, (N, -1)).float().contiguous()


def _reference_head(policy, features, observations, deterministic):
    """The original's lines after ``self.net``, for calls the fused head does not take."""
    if hasattr(policy.action_distribution, "masking"):
        distribution = policy.action_distribution(features, observations["action_map"])
    else:
        distribution = policy.action_distribution(features)
    value = policy.critic(features)
    action = distribution.mode() if deterministic else distribution.sample()
    return value, action, distribution.log_probs(action), distribution


def fused_head(policy, features, observations, deterministic):
    """(value, action, log_probs, distribution) of ``policy``'s heads on ``features`` through the library, or None
    (the caller runs the reference's head) when the inputs do not qualify (:func:`_head_inputs`); the caller has
    checked that grad is off and the heads qualify (:func:`policy_head_layout_error`).  ``distribution`` is None for
    the logits head and ``CustomFixedCategorical(probs=probs, validate_args=False)`` for the masked head.  The one
    host sync is the status read; ``ValueError`` names the env rows the reference would refuse."""
    inputs = _head_inputs(policy, features, observations)
    if inputs is None:
        return None
    masked, mask = inputs
    N, A = features.shape[0], policy.action_distribution.linear.out_features
    q = None
    if not deterministic:       # what torch.multinomial(probs, 1, True) draws: empty_like(probs).exponential_(1)
        q = torch.empty((N, A), dtype=torch.float32, device=features.device).exponential_(1)
    from .renderer import WaveformOps
    value, action, log_prob, probs, status = WaveformOps.get(features.device).policy_head(
        features, policy.action_distribution.linear, policy.critic.fc, masked, mask, q, want_probs=masked)
    if status.item():
        rows = torch.nonzero(action.view(-1) < 0).view(-1).tolist()
        raise ValueError(f"the policy's action distribution is invalid at env rows {rows}: logits with a NaN, a +Inf "
                         "or no finite value, or a masked row that does not normalise to a probability vector")
    distribution = None
    if masked:
        cls = sys.modules[type(policy.action_distribution).__module__].CustomFixedCategorical
        distribution = cls(probs=probs, validate_args=False)
    return value, action, log_prob, distribution


_ACTION_DTYPES = (torch.int64, torch.int32, torch.int16, torch.int8, torch.uint8)


def _evaluate_inputs(policy, features, observations, action):
    """(masked, mask or None, action as contiguous int64) for :class:`PolicyHeadFunction`, or None when the call must
    run the reference's head lines: autocast on, :func:`_head_inputs` refusing with up to ``MAX_TRAIN_ROWS`` rows,
    an ``action_map`` that requires grad, or ``action`` not an integer (N, 1) tensor on the features' device."""
    if torch.is_autocast_enabled("cuda"):
        return None
    inputs = _head_inputs(policy, features, observations, MAX_TRAIN_ROWS)
    if inputs is None:
        return None
    masked, mask = inputs
    if mask is not None and observations["action_map"].requires_grad:
        return None
    if not (isinstance(action, torch.Tensor) and action.dtype in _ACTION_DTYPES and action.device == features.device
            and tuple(action.shape) == (features.shape[0], 1)):
        return None
    return masked, mask, action.long().contiguous()


def _reference_evaluate(policy, features, observations, action):
    """The original's lines after ``self.net`` in ``evaluate_actions``, with the per-row entropy."""
    if hasattr(policy.action_distribution, "masking"):
        distribution = policy.action_distribution(features, observations["action_map"])
    else:
        distribution = policy.action_distribution(features)
    value = policy.critic(features)
    return value, distribution.log_probs(action), distribution.entropy()


class PolicyHeadFunction(torch.autograd.Function):
    """(value (N, 1), log_probs (N, 1), per-row entropy (N,)) of ``policy``'s heads on ``features`` for ``action``
    through the library, differentiable in the features and the four head parameters (each an input, so that autograd
    and DDP see them), not in ``mask``.  The forward reads the refusal count once and raises ``ValueError`` naming
    the rows the reference would refuse.  The backward computes only the gradients autograd asks for and is not
    itself differentiable."""

    @staticmethod
    def forward(ctx, policy, masked, mask, action, features, actor_weight, actor_bias, critic_weight, critic_bias):
        from .renderer import WaveformOps
        ops = WaveformOps.get(features.device)
        value, log_prob, entropy, saved, status = ops.policy_head_train_forward(
            features, policy.action_distribution.linear, policy.critic.fc, masked, mask, action)
        if status.item():
            rows = torch.nonzero(torch.isnan(log_prob.view(-1))).view(-1).tolist()
            raise ValueError(f"the policy's action distribution is invalid at rows {rows}: logits with a NaN, a +Inf "
                             "or no finite value, a masked row that does not normalise to a probability vector, or "
                             "an action outside the support")
        ctx.masked = masked
        if any(ctx.needs_input_grad[4:]):
            ctx.save_for_backward(features, action, mask, saved, actor_weight, critic_weight)
        return value, log_prob, entropy

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_value, grad_log_prob, grad_entropy):
        from .renderer import WaveformOps
        features, action, mask, saved, actor_weight, critic_weight = ctx.saved_tensors
        grads = WaveformOps.get(features.device).policy_head_train_backward(
            features, actor_weight, critic_weight, ctx.masked, mask, action, saved, grad_value, grad_log_prob,
            grad_entropy, need=ctx.needs_input_grad[4:])
        return (None, None, None, None) + grads


def fused_evaluate(policy, features, observations, action):
    """(value, log_probs, per-row entropy) of ``policy``'s heads through :class:`PolicyHeadFunction`, or None (the
    caller runs the reference's head lines) when :func:`_evaluate_inputs` refuses the call; the caller has checked
    that the heads qualify (:func:`policy_head_layout_error`)."""
    inputs = _evaluate_inputs(policy, features, observations, action)
    if inputs is None:
        return None
    masked, mask, action = inputs
    actor, critic = policy.action_distribution.linear, policy.critic.fc
    return PolicyHeadFunction.apply(policy, masked, mask, action, features, actor.weight, actor.bias, critic.weight,
                                    critic.bias)


def _patch(cls, name, make):
    original = getattr(getattr(cls, name), "_ssb_original", getattr(cls, name))
    patched = make(original, inspect.signature(original))
    patched._ssb_original = original
    patched.__doc__ = original.__doc__
    setattr(cls, name, patched)


def _bind(signature, self, args, kwargs):
    """The original's arguments after ``self``, by name, in its order."""
    bound = signature.bind(self, *args, **kwargs)
    bound.apply_defaults()
    named = dict(bound.arguments)
    named.pop(next(iter(signature.parameters)))
    return named


def _make_act(original, signature):
    def act(self, *args, **kwargs):
        if torch.is_grad_enabled() or policy_head_layout_error(self):
            return original(self, *args, **kwargs)
        named = _bind(signature, self, args, kwargs)
        deterministic = named.pop("deterministic")
        observations = named["observations"]
        out = self.net(*named.values())
        features = out[0]
        head = fused_head(self, features, observations, deterministic)
        if head is None:
            head = _reference_head(self, features, observations, deterministic)
        value, action, log_prob, distribution = head
        result = (value, action, log_prob) + tuple(out[1:])
        return result + (distribution,) if hasattr(self.action_distribution, "masking") else result
    return act


def _make_evaluate_actions(original, signature):
    def evaluate_actions(self, *args, **kwargs):
        if policy_head_layout_error(self):
            return original(self, *args, **kwargs)
        named = _bind(signature, self, args, kwargs)
        action = named.pop("action")
        observations = named["observations"]
        out = self.net(*named.values())
        features = out[0]
        head = fused_evaluate(self, features, observations, action)
        if head is None:
            head = _reference_evaluate(self, features, observations, action)
        value, log_prob, entropy = head
        return (value, log_prob, entropy.mean()) + tuple(out[1:])
    return evaluate_actions


def patch_policy(cls, training: bool = False):
    """Replace ``cls.act`` of a reference ``Policy`` in place, and with ``training=True`` also
    ``cls.evaluate_actions``, nothing else; the originals stay reachable as ``._ssb_original`` and patching twice
    changes nothing.  Each patched method binds its arguments to the original's signature, runs ``self.net``
    unchanged and then the heads in the library, or the original's head lines when the inputs do not qualify, and
    returns the original's tuple.

    ``act``: the heads through :func:`fused_head`; ``(value, action, log_probs, rnn_hidden_states)`` plus SAVi's
    ``ext_memory_feats`` or AV-WaN's ``distribution``.  With grad enabled or heads that do not qualify
    (:func:`policy_head_layout_error`) it runs the original.

    ``evaluate_actions``: the heads through :func:`fused_evaluate` (:class:`PolicyHeadFunction`);
    ``(value, action_log_probs, distribution_entropy, rnn_hidden_states)`` plus SAVi's ``ext_memory_feats``, the
    entropy the mean of the per-row entropy as the reference takes it.  With heads that do not qualify it runs the
    original."""
    _patch(cls, "act", _make_act)
    if training:
        _patch(cls, "evaluate_actions", _make_evaluate_actions)
    return cls
