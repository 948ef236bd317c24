"""Batched GPU version of the SAVi pre-training dataset's audio path
(``ss_baselines/savi/pretraining/audiogoal_dataset.py:100-156``): random ``(rir, sound, index)`` triples ->
spectrogram batch, with the reference's quirk preserved: in the steady-state branch the 1-s slice starts
one sample EARLIER than the simulator's (``source[index*sr - L :]`` + ``mode='valid'`` + drop the last
sample  =>  ``y_full[index*sr - 1 : (index+1)*sr - 1]``).

:func:`patch_audiogoal_predictor` runs the network the pretraining trains, ``AudioGoalPredictor``
(``ss_baselines/savi/pretraining/audiogoal_predictor.py``), in the library's kernels."""
from __future__ import annotations

import logging
import random
from typing import Sequence

import torch

from .renderer import AudioRequest, BatchedAudioRenderer


def dataset_request(renderer: BatchedAudioRenderer, rir_id: int, source_id: int, index: int) -> AudioRequest:
    """The request equivalent to ``compute_audiogoal`` (audiogoal_dataset.py:114-140) for a given index."""
    sr = renderer.sr
    taps = renderer._rir_len[rir_id] if rir_id >= 0 else 0
    if taps == 0:
        taps = sr                                   # unreadable / empty file -> zeros((sr, 2)) (:118-123)
    if index * sr - taps < 0:
        return AudioRequest(rir=rir_id, source=source_id, offset=index * sr)
    return AudioRequest(rir=rir_id, source=source_id, offset=index * sr - 1)


class BatchedAudioGoalDataset:
    """``files``: sequence of ``(rir_id, source_id)``; clips are registered in the renderer."""

    def __init__(self, renderer: BatchedAudioRenderer, files: Sequence, rng: random.Random | None = None):
        self.r, self.files, self.rng = renderer, list(files), rng or random.Random()

    def __len__(self):
        return len(self.files)

    def audio_length(self, source_id: int) -> int:
        return self.r._sources[source_id].numel() // self.r.sr            # audiogoal_dataset.py:89-90

    def render(self, items: Sequence[int], indices: Sequence[int] | None = None, want_wave: bool = False):
        reqs = []
        for k, item in enumerate(items):
            rir_id, source_id = self.files[item]
            index = indices[k] if indices is not None else self.rng.randint(0, self.audio_length(source_id) - 2)
            reqs.append(dataset_request(self.r, rir_id, source_id, index))
        return self.r.render(reqs, want_wave=want_wave)


def patch_audiogoal_predictor(cls, training: bool = True):
    """Replace ``cls.forward`` of SAVi's ``AudioGoalPredictor`` (audiogoal_predictor.py:18-38) in place, nothing else;
    the original stays reachable as ``cls.forward._ssb_original`` and patching again replaces the patch.

    The replacement logs the input shape once, as the reference does, and runs a numpy spectrogram (the reference's
    single-observation branch) through the original.  A tensor call that
    :func:`soundspaces_b200.belief_nets.resnet18_train_error` allows runs ``predictor`` in the library, by the mode of
    its BatchNorms and grad mode:

    - ``eval()`` under ``torch.no_grad`` with B <= 1024: ``ssb_resnet18_batch`` (39 launches), as at rollout time;
    - with ``training=True``, ``train()`` with grad on or off (the trainer's train split): BatchNorm with batch
      statistics and the running statistics updated in place, through
      :class:`soundspaces_b200.belief_nets.ResNetFunction` (79 launches forward, 115 backward);
    - with ``training=True``, ``eval()`` with grad on (the trainer's val pass, which runs without ``no_grad``) or
      B > 1024: the same function with the running statistics, output bit-identical to ``ssb_resnet18_batch``
      (59 launches).

    Every other call runs the original.  The loss stays in torch."""
    from .belief_nets import MAX_ENVS, conv_norm_pairs, resnet18_train_error, resnet18_train_forward
    original = getattr(cls.forward, "_ssb_original", cls.forward)

    def forward(self, audio_feature):
        x = audio_feature["spectrogram"]
        if not torch.is_tensor(x):
            return original(self, audio_feature)
        if not getattr(self, "input_shape_printed", False):
            logging.info('Audiogoal predictor input audio feature shape: {}'.format(x.shape))
            self.input_shape_printed = True
        if resnet18_train_error(self, audio_feature):
            return original(self, audio_feature)
        bn_training = conv_norm_pairs(self.predictor)[0][1].training
        if not bn_training and not torch.is_grad_enabled() and x.shape[0] <= MAX_ENVS:
            from .renderer import WaveformOps
            return WaveformOps.get(x.device).resnet18(x, self.predictor)
        if not training:
            return original(self, audio_feature)
        return resnet18_train_forward(self, audio_feature)

    forward._ssb_original = original
    forward.__doc__ = original.__doc__
    cls.forward = forward
    return cls
