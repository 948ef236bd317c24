"""Stand-ins for the AV-Nav policy's visual encoder and state encoder, written from the reference's computation:
``VisualCNN`` of ss_baselines/av_nav/models/visual_cnn.py:53-161 (strides 4/2/2, conv3 64 channels),
av_wan/models/visual_cnn.py:17-118 (strides 4/2/1, conv3 32 channels) and savi/models/visual_cnn.py:17-188 (av_nav's
network plus 6 semantic channels, which the fused path does not run), and ``RNNStateEncoder`` of
ss_baselines/av_nav/models/rnn_state_encoder.py.  tests/golden/avnav_policy_golden.npz pins them to the reference
classes in float64 (tests/golden/make_avnav_policy_golden.py).  ``AudioNavBaselineNet`` mirrors the rollout-time
``Net.forward`` of ss_baselines/av_nav/ppo/policy.py:198-221 for the benchmark and the end-to-end test.
"""
import math

import torch
import torch.nn as nn

# name: (strides, conv3 channels)
VARIANTS = {"av_nav": ((4, 2, 2), 64), "av_wan": ((4, 2, 1), 32), "savi": ((4, 2, 2), 64)}
KERNELS = (8, 4, 3)


def conv_out(n, k, s):
    return (n - k) // s + 1


class VisualCNN(nn.Module):
    """``VisualCNN`` of the ``variant`` ('av_nav', 'av_wan' or 'savi') for n_rgb RGB and n_depth depth channels of an
    H x W observation.  n_semantic > 0 (savi only) adds the semantic channels; forward then needs the reference's
    semantic conversion and is not provided here."""

    def __init__(self, n_rgb, n_depth, H, W, output_size, variant="av_nav", n_semantic=0):
        super().__init__()
        strides, c3 = VARIANTS[variant]
        self._n_input_rgb, self._n_input_depth = n_rgb, n_depth
        if variant == "savi":
            self._n_input_semantic = n_semantic
        in_ch = n_rgb + n_depth + n_semantic
        if in_ch == 0:
            self.cnn = nn.Sequential()
            return
        h, w = H, W
        for k, s in zip(KERNELS, strides):
            h, w = conv_out(h, k, s), conv_out(w, k, s)
        self.cnn = nn.Sequential(
            nn.Conv2d(in_ch, 32, KERNELS[0], strides[0]), nn.ReLU(True),
            nn.Conv2d(32, 64, KERNELS[1], strides[1]), nn.ReLU(True),
            nn.Conv2d(64, c3, KERNELS[2], strides[2]),
            nn.Flatten(), nn.Linear(c3 * h * w, output_size), nn.ReLU(True))

    @property
    def is_blind(self):
        return self._n_input_rgb + self._n_input_depth + getattr(self, "_n_input_semantic", 0) == 0

    def forward(self, observations):
        cnn_input = []
        if self._n_input_rgb > 0:
            cnn_input.append(observations["rgb"].permute(0, 3, 1, 2) / 255.0)
        if self._n_input_depth > 0:
            cnn_input.append(observations["depth"].permute(0, 3, 1, 2))
        if getattr(self, "_n_input_semantic", 0) > 0:
            raise NotImplementedError("the stand-in has no semantic conversion")
        return self.cnn(torch.cat(cnn_input, dim=1))


class RNNStateEncoder(nn.Module):
    def __init__(self, input_size, hidden_size, num_layers=1, rnn_type="GRU"):
        super().__init__()
        self._num_recurrent_layers = num_layers
        self._rnn_type = rnn_type
        self.rnn = getattr(nn, rnn_type)(input_size=input_size, hidden_size=hidden_size, num_layers=num_layers)

    def _pack_hidden(self, h):
        return torch.cat([h[0], h[1]], dim=0) if "LSTM" in self._rnn_type else h

    def _unpack_hidden(self, h):
        if "LSTM" in self._rnn_type:
            return h[0:self._num_recurrent_layers], h[self._num_recurrent_layers:]
        return h

    def _mask_hidden(self, h, masks):
        return tuple(v * masks for v in h) if isinstance(h, tuple) else masks * h

    def single_forward(self, x, hidden_states, masks):
        hidden_states = self._unpack_hidden(hidden_states)
        x, hidden_states = self.rnn(x.unsqueeze(0), self._mask_hidden(hidden_states, masks.unsqueeze(0)))
        return x.squeeze(0), self._pack_hidden(hidden_states)

    def forward(self, x, hidden_states, masks):
        if x.size(0) == hidden_states.size(1):
            return self.single_forward(x, hidden_states, masks)
        raise NotImplementedError("the stand-in has no seq_forward")


def set_params(module, seed):
    """Deterministic parameters without a random generator: every tensor p gets
    ``sin(seed + 0.7310 k + 0.123 t) / sqrt(fan_in)`` for element k of the t-th tensor (fan_in = p.shape[-1] for a
    matrix, the product of the trailing dims for a conv weight, 1 for a bias)."""
    with torch.no_grad():
        for t, p in enumerate(module.parameters()):
            k = torch.arange(p.numel(), dtype=torch.float64)
            fan_in = math.prod(p.shape[1:]) if p.ndim > 1 else 4
            p.copy_((torch.sin(seed + 0.7310 * k + 0.123 * t) / math.sqrt(fan_in)).reshape(p.shape))
    return module


def visual_obs(N, H, W, n_rgb, n_depth, seed):
    """RGB in 0..255 (integers, as the sensor delivers them, as float) and depth in [0, 1)."""
    g = torch.Generator().manual_seed(seed)
    obs = {}
    if n_rgb:
        obs["rgb"] = torch.randint(0, 256, (N, H, W, n_rgb), generator=g).float()
    if n_depth:
        obs["depth"] = torch.rand((N, H, W, n_depth), generator=g)
    return obs


def gru_inputs(N, I, Hd, seed, masks="mixed"):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(N, I, generator=g)
    h = torch.randn(1, N, Hd, generator=g)
    if masks == "mixed":
        m = (torch.arange(N) % 3 != 0).float()[:, None]
    else:
        m = torch.full((N, 1), float(masks))
    return x, h, m


class AudioNavBaselineNet(nn.Module):
    """The rollout-time part of av_nav's ``AudioNavBaselineNet.forward`` (policy.py:198-221) with a depth or RGB-D
    visual encoder and the audio encoder: ``x = [audio(obs), visual(obs)]``, then the state encoder."""

    def __init__(self, audio_cnn, visual_cnn, hidden_size=512):
        super().__init__()
        self.audio_encoder = audio_cnn
        self.visual_encoder = visual_cnn
        self.state_encoder = RNNStateEncoder(2 * hidden_size, hidden_size)

    def forward(self, observations, rnn_hidden_states, masks):
        x = [self.audio_encoder(observations), self.visual_encoder(observations)]
        x1 = torch.cat(x, dim=1)
        return self.state_encoder(x1, rnn_hidden_states, masks)
