"""Generate tests/golden/policy_head_golden.npz by running the UNMODIFIED reference ``Policy.act`` of an upstream
sound-spaces checkout (path in ``SOUNDSPACES_REFERENCE``, as for the other oracle fixtures) in float64 on the CPU:
ss_baselines/av_nav/ppo/policy.py, savi/ppo/policy.py and av_wan/ppo/policy.py with ``CategoricalNet``,
``CategoricalNetWithMask`` and ``CustomFixedCategorical`` of ss_baselines/common/utils.py.

    SOUNDSPACES_REFERENCE=<sound-spaces checkout> python tests/golden/make_policy_head_golden.py

Only the heads run: ``self.net`` is tests/policy_head_models.py's ``StubNet``, and the imports the policy and utils
modules make for everything else (habitat, moviepy, cv2, gym, torchsummary, the encoders) are stubbed.  Parameters
come from ``set_params``, so per case ``<name>/<key>`` the file stores ``config`` (trainer index, H, A, N, n_in,
seed, gain, masking), the input ``x``, ``action_map`` (AV-WaN), ``value``, ``mode``, ``mode_log_prob``, ``actions``
with their ``log_probs``, and ``samples`` drawn after ``torch.manual_seed(sample_seeds[i])``.
"""
import importlib.util
import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from oracle.ref_harness import REFERENCE_ROOT  # noqa: E402
from policy_head_models import StubNet, action_map, set_params  # noqa: E402

TRAINERS = ("av_nav", "savi", "av_wan")
# name: (trainer, H, A, N, n_in, seed, gain, masking)
CASES = {
    "av_nav": ("av_nav", 16, 4, 6, 5, 1, 3.0, 1),
    "av_nav_flat": ("av_nav", 24, 4, 4, 3, 2, 0.01, 1),
    "savi": ("savi", 12, 4, 5, 4, 3, 3.0, 1),
    "av_wan_masked": ("av_wan", 16, 9, 6, 5, 4, 3.0, 1),
    "av_wan_unmasked": ("av_wan", 16, 9, 5, 5, 5, 3.0, 0),
}
SAMPLE_SEEDS = (11, 12, 13, 14)


class _Stub(types.ModuleType):
    """A module whose every attribute is a placeholder class: stands in for imports the heads never use."""

    def __getattr__(self, name):
        if name.startswith("__"):
            raise AttributeError(name)
        return type(name, (), {})


def _stub(name):
    m = _Stub(name)
    m.__path__ = []
    sys.modules[name] = m
    return m


def load_reference():
    if not REFERENCE_ROOT:
        sys.exit("set SOUNDSPACES_REFERENCE to a sound-spaces checkout")
    for name in ("cv2", "moviepy", "moviepy.editor", "moviepy.audio", "moviepy.audio.AudioClip", "gym",
                 "gym.spaces", "habitat", "habitat.utils", "habitat.utils.visualizations",
                 "habitat.utils.visualizations.utils", "habitat_sim", "habitat_sim.utils", "habitat_sim.utils.common",
                 "torchsummary", "soundspaces", "soundspaces.tasks", "soundspaces.tasks.nav", "ss_baselines",
                 "ss_baselines.common", "ss_baselines.common.tensorboard_utils", "ss_baselines.av_nav",
                 "ss_baselines.av_nav.models", "ss_baselines.av_nav.models.rnn_state_encoder",
                 "ss_baselines.av_nav.models.visual_cnn", "ss_baselines.av_nav.models.audio_cnn",
                 "ss_baselines.av_nav.ppo", "ss_baselines.savi", "ss_baselines.savi.models",
                 "ss_baselines.savi.models.visual_cnn", "ss_baselines.savi.models.audio_cnn",
                 "ss_baselines.savi.models.smt_state_encoder", "ss_baselines.savi.models.smt_cnn",
                 "ss_baselines.savi.ppo", "ss_baselines.av_wan", "ss_baselines.av_wan.models",
                 "ss_baselines.av_wan.models.visual_cnn", "ss_baselines.av_wan.models.map_cnn",
                 "ss_baselines.av_wan.models.audio_cnn", "ss_baselines.av_wan.ppo"):
        _stub(name)

    def load(modname, rel):
        spec = importlib.util.spec_from_file_location(modname, os.path.join(REFERENCE_ROOT, "ss_baselines", rel))
        mod = importlib.util.module_from_spec(spec)
        sys.modules[modname] = mod
        spec.loader.exec_module(mod)
        return mod

    load("ss_baselines.common.utils", "common/utils.py")
    return {t: load(f"ss_baselines.{t}.ppo.policy", f"{t}/ppo/policy.py").Policy for t in TRAINERS}


def main():
    policies = load_reference()
    torch.set_default_dtype(torch.float64)
    out = {"sample_seeds": np.array(SAMPLE_SEEDS, np.int64)}
    for name, (trainer, H, A, N, n_in, seed, gain, masking) in CASES.items():
        net = StubNet(n_in, H, memory=trainer == "savi")
        cls = policies[trainer]
        policy = cls(net, A, bool(masking)) if trainer == "av_wan" else cls(net, A)
        set_params(policy, seed, gain).double().eval()
        g = torch.Generator().manual_seed(100 + seed)
        obs = {"x": torch.randn((N, n_in), generator=g, dtype=torch.float64) * 2}
        if trainer == "av_wan":
            obs["action_map"] = action_map(N, A, seed).reshape(N, 3, 3) if A == 9 else action_map(N, A, seed)
        h = torch.zeros((1, N, 4))
        prev, masks = torch.zeros((N, 1), dtype=torch.int64), torch.ones((N, 1))
        ext = (torch.zeros((3, N, 4)), torch.ones((N, 3))) if trainer == "savi" else ()
        actions = torch.randint(0, A, (N, 1), generator=g)
        with torch.no_grad():
            res = policy.act(obs, h, prev, masks, *ext, deterministic=True)
            features = net(obs, h, prev, masks, *ext)[0]
            dist = (policy.action_distribution(features, obs["action_map"]) if trainer == "av_wan"
                    else policy.action_distribution(features))
            samples = []
            for s in SAMPLE_SEEDS:
                torch.manual_seed(s)
                samples.append(policy.act(obs, h, prev, masks, *ext, deterministic=False)[1][:, 0])
        rec = {"config": np.array([TRAINERS.index(trainer), H, A, N, n_in, seed, gain, masking], np.float64),
               "x": obs["x"], "value": res[0], "mode": res[1], "mode_log_prob": res[2], "actions": actions,
               "log_probs": dist.log_probs(actions), "samples": torch.stack(samples)}
        if trainer == "av_wan":
            rec["action_map"] = obs["action_map"]
        for k, v in rec.items():
            out[f"{name}/{k}"] = v.numpy() if isinstance(v, torch.Tensor) else v
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "policy_head_golden.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, len(out), "arrays")


if __name__ == "__main__":
    main()
