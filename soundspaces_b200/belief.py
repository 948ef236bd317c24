"""SAVi's belief update at rollout time: ``BeliefPredictor.update`` (ss_baselines/savi/models/belief_predictor.py:136-202),
called once per rollout step by ppo_trainer.py:332-336, with its per-env loops run by ``ssb_belief_update_batch`` (one
launch) instead of Python loops that copy every env's spectrogram sum and pose to the host.

    from soundspaces_b200.belief import patch_belief_predictor
    patch_belief_predictor(BeliefPredictor)     # ss_baselines.savi.models.belief_predictor; BeliefPredictorDDP inherits it

The patched ``update`` makes the reference's network calls, in its order, under ``no_grad``
(``self.cnn_forward(observations)``, then ``self.classifier(spectrograms)``), then one launch that writes the
``location_belief`` / ``category_belief`` rows in place.  No ``.cpu()``, ``.item()`` or host copy.

    patch_belief_predictor(BeliefPredictor, networks=True)

also runs the two ResNet-18s in the library (``ssb_resnet18_batch``, ``ssb_smt_resnet18_batch``, see
:mod:`soundspaces_b200.belief_nets`) when they qualify; anything else runs the module as before.
"""
from __future__ import annotations

import torch

from .belief_nets import fused_forward

SPEC, POSE, LOC, CAT, CATEGORY = "spectrogram", "pose", "location_belief", "category_belief", "category"
N_LABELS = 21
MAX_ENVS = 1024       # BELIEF_MAX_ENVS of ssb200.cu: the dones bitmask of ssb_belief_update_batch holds 1024 envs


def _dense(t, device) -> bool:
    return isinstance(t, torch.Tensor) and t.is_cuda and t.device == device and t.dtype == torch.float32 and t.is_contiguous()


def _prediction(t, device, cols) -> bool:
    return (isinstance(t, torch.Tensor) and t.is_cuda and t.device == device and t.dtype == torch.float32 and t.ndim == 2
            and t.shape[1] >= cols and t.stride(1) == 1)


def _device_state(model, device):
    """(last_pointgoal list, last_label list, last_pg, loc_valid, last_label, label_valid) on ``device``, zeroed (no
    state) whenever code has replaced either list since the last call: that is how the reference starts over."""
    st = getattr(model, "_ssb_belief_state", None)
    if st is None or st[0] is not model.last_pointgoal or st[1] is not model.last_label or st[2].device != device:
        n_pg, n_label = len(model.last_pointgoal), len(model.last_label)
        st = (model.last_pointgoal, model.last_label,
              torch.zeros((n_pg, 2), dtype=torch.float32, device=device), torch.zeros(n_pg, dtype=torch.uint8, device=device),
              torch.zeros((n_label, N_LABELS), dtype=torch.float32, device=device),
              torch.zeros(n_label, dtype=torch.uint8, device=device))
        model._ssb_belief_state = st
    return st


def _location_prediction(model, observations):
    """``model.cnn_forward(observations)``, through the library when the predictor and its input qualify."""
    spec = observations[SPEC]
    labels = observations.get(CATEGORY) if getattr(model, "has_distractor_sound", False) else None
    if labels is None or isinstance(labels, torch.Tensor):
        out = fused_forward(model.predictor, spec, labels)
        if out is not None:
            return out
    return model.cnn_forward(observations)


def patch_belief_predictor(cls, networks: bool = False, training: bool = False):
    """Replace ``cls.update`` of SAVi's ``BeliefPredictor`` in place, nothing else; the original stays reachable as
    ``cls.update._ssb_original``.

    ``networks=True`` also runs the location predictor (in place of ``self.cnn_forward(observations)``) and the
    label classifier through the library when they have one of the two ResNet-18 topologies, with eval-mode
    BatchNorm and float32 parameters on the observation's device (:func:`soundspaces_b200.belief_nets.fused_forward`);
    the SMT predictor of a model with ``has_distractor_sound`` reads ``observations["category"]``.  Networks or inputs
    that do not qualify run as modules, as with ``networks=False``.  Each network in the library is a fixed number of
    launches (39 for a torchvision ResNet-18, 38 for the SMT network) whatever the batch.

    ``training=True`` also replaces ``cls.cnn_forward`` (the original stays reachable as
    ``cls.cnn_forward._ssb_original``): a grad-mode call that
    :func:`soundspaces_b200.belief_nets.smt_resnet18_train_error` allows runs the SMT location predictor through
    :class:`soundspaces_b200.belief_nets.SmtResNetFunction` (the online training of ``train_belief_predictor``, 38
    launches forward, 80 backward, 82 with the category channels); every other call runs the original.

    The device path runs when ``spectrogram`` (B, H, W, 2), ``pose`` and the belief rows the predictor writes are
    contiguous CUDA float32 tensors on one device, the batch holds at most ``MAX_ENVS`` (1024) envs, and the network
    outputs are CUDA float32 on that device.  Anything else (CPU tensors, other dtypes, views with row gaps, larger
    batches) runs the original ``update``, networks included; when only the network outputs disqualify, the original
    evaluates the networks a second time.  A batch larger than ``len(self.last_pointgoal)``
    (location) or ``len(self.last_label)`` (label) raises ``ValueError`` (the reference raises ``IndexError``).

    The beliefs' state lives in device memory, sized from ``len(self.last_pointgoal)`` and ``len(self.last_label)``
    and reset when code replaces those lists.  The lists themselves are no longer updated: nothing in the reference
    reads them outside ``update``.  The silence test is "any element != 0" rather than ``sum() != 0``; they differ
    only for finite values of both signs that cancel to exactly 0, which a spectrogram (>= 0) never holds."""
    original = getattr(cls.update, "_ssb_original", cls.update)

    def update(self, observations, dones):
        loc, label = bool(self.predict_location), bool(self.predict_label)
        spec = observations[SPEC]
        device = spec.device if isinstance(spec, torch.Tensor) else None
        rows = [SPEC] + ([POSE, LOC] if loc else []) + ([CAT] if label else [])
        if (not (loc or label) or not all(_dense(observations.get(k), device) for k in rows) or spec.ndim != 4
                or spec.shape[3] != 2):
            return original(self, observations, dones)
        B = spec.shape[0]
        if loc and B > len(self.last_pointgoal):
            raise ValueError(f"BeliefPredictor.update: {B} envs, last_pointgoal holds {len(self.last_pointgoal)}")
        if label and B > len(self.last_label):
            raise ValueError(f"BeliefPredictor.update: {B} envs, last_label holds {len(self.last_label)}")
        if B > MAX_ENVS:
            return original(self, observations, dones)
        with torch.no_grad():
            if networks:
                loc_pred = _location_prediction(self, observations) if loc else None
                label_pred = None
                if label:
                    label_pred = fused_forward(self.classifier, spec)
                    if label_pred is None:
                        label_pred = self.classifier(spec.permute(0, 3, 1, 2))
            else:
                loc_pred = self.cnn_forward(observations) if loc else None
                label_pred = self.classifier(spec.permute(0, 3, 1, 2)) if label else None
        if (loc and not _prediction(loc_pred, device, 2)) or (label and not _prediction(label_pred, device, N_LABELS)):
            return original(self, observations, dones)
        _, _, last_pg, loc_valid, last_label, label_valid = _device_state(self, device)
        from .renderer import WaveformOps
        WaveformOps.get(device).belief_update(
            spec, dones, self.config.weighting_factor, self.config.current_pred_only,
            pose=observations[POSE] if loc else None, loc_pred=loc_pred, last_pg=last_pg, loc_valid=loc_valid,
            loc_out=observations[LOC] if loc else None, label_pred=label_pred, last_label=last_label,
            label_valid=label_valid, cat_out=observations[CAT] if label else None)

    update._ssb_original = original
    update.__doc__ = original.__doc__
    cls.update = update
    if training:
        _patch_cnn_forward(cls)
    return cls


def _patch_cnn_forward(cls):
    from .belief_nets import smt_resnet18_train_error, smt_resnet18_train_forward
    original = getattr(cls.cnn_forward, "_ssb_original", cls.cnn_forward)

    def cnn_forward(self, observations):
        if not torch.is_grad_enabled() or smt_resnet18_train_error(self, observations):
            return original(self, observations)
        return smt_resnet18_train_forward(self, observations)

    cnn_forward._ssb_original = original
    cnn_forward.__doc__ = original.__doc__
    cls.cnn_forward = cnn_forward
