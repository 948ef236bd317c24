"""Generate tests/golden/belief_golden.npz by running the UNMODIFIED ``BeliefPredictor.update`` of an upstream
sound-spaces checkout (ss_baselines/savi/models/belief_predictor.py) on seeded rollouts:

    SOUNDSPACES_REFERENCE=<sound-spaces checkout> python tests/golden/make_belief_golden.py

``soundspaces/tasks/nav.py`` (the sensor uuids) comes in through ``oracle/ref_harness.py``.  The predictor is built
with ``object.__new__`` + ``nn.Module.__init__`` and its attributes are set directly: its ``__init__`` would build
torchvision ResNets with ``pretrained=True`` (a download) and load weights from disk.  ``cnn_forward`` and
``classifier`` are replaced by callables that return the seeded predictions of ``belief_oracle.make_sequence``, so the
recording holds only what ``update`` itself does.  Spectrograms come from ``belief_oracle.make_spectrograms`` (zero
rows for the silent steps).

Four configurations, 8 envs x 60 steps each: both beliefs with w = 0.5, both with current_pred_only, location only
(the pretrained 23-column head, w = 0.3) and label only (w = 0.3).  Stored per configuration ``<name>/<key>``: the
inputs (``silent``, ``dones``, ``pose``, ``loc_pred``, ``label_pred``), the rows ``update`` wrote (``loc_out``,
``cat_out``; zero where it wrote nothing) and the predictor's state after every step (``loc_valid`` / ``label_valid``:
the list entry is not None, ``last_pg`` / ``last_label``: its value, 0 when None).
"""
import importlib.util
import os
import sys
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import torch  # noqa: E402

from belief_oracle import make_sequence, make_spectrograms  # noqa: E402
from oracle import ref_harness as rh  # noqa: E402

T, B, SPEC_SHAPE = 60, 8, (65, 26, 2)
CONFIGS = {
    "both": dict(loc=True, label=True, w=0.5, cpo=False, loc_cols=2, seed=11),
    "current_pred_only": dict(loc=True, label=True, w=0.5, cpo=True, loc_cols=2, seed=12),
    "location_only": dict(loc=True, label=False, w=0.3, cpo=False, loc_cols=23, seed=13),
    "label_only": dict(loc=False, label=True, w=0.3, cpo=False, loc_cols=2, seed=14),
}


def load_belief_module():
    nav = rh.load_reference()["nav"]
    saved = dict(sys.modules)
    try:
        for name, rel in (("soundspaces", "soundspaces"), ("soundspaces.tasks", "soundspaces/tasks"),
                          ("ss_baselines", "ss_baselines"), ("ss_baselines.savi", "ss_baselines/savi"),
                          ("ss_baselines.savi.models", "ss_baselines/savi/models")):
            pkg = types.ModuleType(name)
            pkg.__path__ = [os.path.join(rh.REFERENCE_ROOT, rel)]
            sys.modules[name] = pkg
        sys.modules["soundspaces.tasks.nav"] = nav
        mods = {}
        for name, rel in (("ss_baselines.savi.models.smt_resnet", "ss_baselines/savi/models/smt_resnet.py"),
                          ("ss_baselines.savi.models.belief_predictor", "ss_baselines/savi/models/belief_predictor.py")):
            spec = importlib.util.spec_from_file_location(name, os.path.join(rh.REFERENCE_ROOT, rel))
            mods[name] = importlib.util.module_from_spec(spec)
            sys.modules[name] = mods[name]
            spec.loader.exec_module(mods[name])
        return mods["ss_baselines.savi.models.belief_predictor"]
    finally:
        for k in list(sys.modules):
            if k not in saved:
                del sys.modules[k]


def record(bp_mod, cfg):
    seq = make_sequence(cfg["seed"], T, B, loc_cols=cfg["loc_cols"])
    bp = object.__new__(bp_mod.BeliefPredictor)
    torch.nn.Module.__init__(bp)
    bp.config = rh.AttrDict(weighting_factor=cfg["w"], current_pred_only=cfg["cpo"], online_training=True,
                            use_location_belief=cfg["loc"], use_label_belief=cfg["label"])
    bp.device = torch.device("cpu")
    bp.predict_location, bp.predict_label, bp.has_distractor_sound = cfg["loc"], cfg["label"], False
    bp.last_pointgoal, bp.last_label = [None] * B, [None] * B
    out = {k: v for k, v in seq.items()}
    for k, shape in (("loc_out", (2,)), ("cat_out", (21,)), ("last_pg", (2,)), ("last_label", (21,)),
                     ("loc_valid", ()), ("label_valid", ())):
        out[k] = np.zeros((T, B) + shape, np.float32 if shape else bool)
    for t in range(T):
        spec = torch.from_numpy(make_spectrograms(seq["silent"][t], SPEC_SHAPE, seed=cfg["seed"] * 1000 + t))
        obs = {"spectrogram": spec, "pose": torch.from_numpy(seq["pose"][t].copy()),
               "location_belief": torch.zeros(B, 2), "category_belief": torch.zeros(B, 21)}
        bp.cnn_forward = lambda o, p=torch.from_numpy(seq["loc_pred"][t].copy()): p
        bp.classifier = lambda x, p=torch.from_numpy(seq["label_pred"][t].copy()): p
        bp.update(obs, [bool(d) for d in seq["dones"][t]])
        out["loc_out"][t], out["cat_out"][t] = obs["location_belief"].numpy(), obs["category_belief"].numpy()
        for i in range(B):
            if bp.last_pointgoal[i] is not None:
                out["loc_valid"][t, i], out["last_pg"][t, i] = True, bp.last_pointgoal[i]
            if bp.last_label[i] is not None:
                out["label_valid"][t, i], out["last_label"][t, i] = True, bp.last_label[i]
    return out


def main():
    if not rh.reference_available():
        raise SystemExit("set SOUNDSPACES_REFERENCE to an upstream sound-spaces checkout")
    bp_mod = load_belief_module()
    arrays = {}
    for name, cfg in CONFIGS.items():
        for k, v in record(bp_mod, cfg).items():
            arrays[f"{name}/{k}"] = v
        for k in ("loc", "label", "cpo"):
            arrays[f"{name}/{k}"] = np.array(cfg[k])
        arrays[f"{name}/w"] = np.array(cfg["w"])
    path = os.path.join(ROOT, "tests", "golden", "belief_golden.npz")
    np.savez_compressed(path, **arrays)
    print("wrote", path, sum(v.nbytes for v in arrays.values()), "bytes")


if __name__ == "__main__":
    main()
