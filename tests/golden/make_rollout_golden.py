"""Generate tests/golden/rollout_golden.npz by running the UNMODIFIED reference rollout storage of an upstream
sound-spaces checkout (path in ``SOUNDSPACES_REFERENCE``, as for the other oracle fixtures) in float32 on the CPU:
ss_baselines/common/rollout_storage.py, ss_baselines/savi/models/rollout_storage.py (with its ``ExternalMemory``)
and ``PPO.get_advantages`` of ss_baselines/av_nav/ppo/ppo.py.  All three modules import only torch.

    SOUNDSPACES_REFERENCE=<sound-spaces checkout> python tests/golden/make_rollout_golden.py

The scripts are tests/rollout_models.py's ``SCRIPTS``: several rollouts with episodes ending at different steps per
env, SAVi's memory reaching capacity, sensors of several shapes and int64 actions, with ``use_gae`` on and off, and
1, 2 and 4 minibatches, each generator after ``torch.manual_seed``.  Keys are ``<script>/<gae|plain>/`` followed by
``run_script``'s keys.
"""
import importlib.util
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from oracle.ref_harness import REFERENCE_ROOT  # noqa: E402
import rollout_models as rm  # noqa: E402


def _load(rel, name):
    spec = importlib.util.spec_from_file_location(name, os.path.join(REFERENCE_ROOT, rel))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def main():
    if not os.path.isfile(os.path.join(REFERENCE_ROOT, "ss_baselines", "common", "rollout_storage.py")):
        raise SystemExit("set SOUNDSPACES_REFERENCE to an upstream sound-spaces checkout")
    common = _load("ss_baselines/common/rollout_storage.py", "ref_common_rollout_storage")
    savi = _load("ss_baselines/savi/models/rollout_storage.py", "ref_savi_rollout_storage")
    ppo = _load("ss_baselines/av_nav/ppo/ppo.py", "ref_av_nav_ppo")
    classes = dict(common=common.RolloutStorage, savi=savi.RolloutStorage)
    out = {}
    for name, script in rm.SCRIPTS.items():
        for use_gae in (True, False):
            res = rm.run_script(script, classes, ppo.PPO, use_gae)
            out.update({f"{rm.golden_key(name, use_gae)}/{k}": v for k, v in res.items()})
    path = os.path.join(ROOT, "tests", "golden", "rollout_golden.npz")
    np.savez_compressed(path, **out)
    print(f"wrote {path}: {len(out)} arrays")


if __name__ == "__main__":
    main()
