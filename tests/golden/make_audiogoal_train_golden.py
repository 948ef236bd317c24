"""Generate tests/golden/audiogoal_train_golden.npz by running the UNMODIFIED reference ``AudioGoalPredictor`` of an
upstream sound-spaces checkout (ss_baselines/savi/pretraining/audiogoal_predictor.py, path in
``SOUNDSPACES_REFERENCE``, located through oracle/ref_harness.py) in float64: forward, running-statistics update and
the gradients of the pretraining loss (audiogoal_trainer.py:113-124, CrossEntropy + MSE).

    SOUNDSPACES_REFERENCE=<sound-spaces checkout> python tests/golden/make_audiogoal_train_golden.py

The class builds its network with ``torchvision.models.resnet18(pretrained=True)``; during construction only, that
call builds the same network without weights, so nothing is downloaded.  Parameters and running statistics come from
``set_params`` and the inputs from seeds (``CASES`` and ``case_inputs`` in tests/audiogoal_train_models.py: 65 x 26
and 65 x 69 inputs, 23, 21 and 2 outputs, B of 1, 7 and 64, a silent row and a row scaled by 1e-3, two consecutive
train-mode steps, one eval-mode case), so only results are stored, per case and step ``<name>/<step>/<key>``: ``pred``,
the 62 parameter gradients ``g<j>`` and the 40 running statistics after the step ``s<j>``, each whole up to 64
elements, else as 16 seeded elements (``_sample``) and 8 seeded Gaussian projections of every element (``_proj``).
"""
import contextlib
import importlib.util
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import torch  # noqa: E402
import torchvision  # noqa: E402

from audiogoal_train_models import CASES, case_inputs, record, reference_loss, set_params  # noqa: E402


def load_audiogoal_predictor():
    from oracle.ref_harness import REFERENCE_ROOT
    path = os.path.join(REFERENCE_ROOT, "ss_baselines", "savi", "pretraining", "audiogoal_predictor.py")
    spec = importlib.util.spec_from_file_location("ss_baselines.savi.pretraining.audiogoal_predictor", path)
    mod = importlib.util.module_from_spec(spec)
    sys.modules[spec.name] = mod
    spec.loader.exec_module(mod)
    return mod.AudioGoalPredictor


@contextlib.contextmanager
def no_pretrained_download():
    original = torchvision.models.resnet18

    def resnet18(pretrained=False, **kwargs):
        return original(weights=None, **kwargs)
    torchvision.models.resnet18 = resnet18
    try:
        yield
    finally:
        torchvision.models.resnet18 = original


def main():
    from soundspaces_b200.belief_nets import resnet18_buffers, resnet18_params
    AudioGoalPredictor = load_audiogoal_predictor()
    out = {}
    for name, (H, W, n_out, B, mode, steps) in CASES.items():
        with no_pretrained_download():
            model = AudioGoalPredictor(predict_label=n_out != 2, predict_location=n_out != 21)
        set_params(model.predictor).double()
        model.train(mode == "train")
        for step in range(steps):
            x, gts = case_inputs(name, step)
            model.zero_grad(set_to_none=True)
            pred = model({"spectrogram": x.double()})
            reference_loss(pred, gts.double()).backward()
            grads = [p.grad.detach() for p in resnet18_params(model.predictor)]
            stats = [t.detach() for t in resnet18_buffers(model.predictor)[:40]]
            assert all(int(t) == step + (mode == "train") for t in resnet18_buffers(model.predictor)[40:])
            out.update(record(name, step, pred.detach().numpy(), [g.numpy() for g in grads],
                              [s.numpy() for s in stats]))
    dst = os.path.join(ROOT, "tests", "golden", "audiogoal_train_golden.npz")
    np.savez_compressed(dst, **out)
    print("wrote", dst, os.path.getsize(dst), "bytes")


if __name__ == "__main__":
    main()
