"""Stand-ins for AV-WaN's map encoder and policy network, written from the reference's computation: ``MapCNN`` of
ss_baselines/av_wan/models/map_cnn.py (``Conv2d(C -> 32) ReLU Conv2d(32 -> 64) ReLU Conv2d(64 -> 32) Flatten Linear
ReLU``, unpadded, on ``observations[map_type].permute(0, 3, 1, 2)``; kernel sizes and strides per map type and size)
and the rollout-time ``AudioNavBaselineNet.forward`` of ss_baselines/av_wan/ppo/policy.py:198-215.
tests/golden/map_cnn_golden.npz pins ``MapCNN`` to the reference class in float64
(tests/golden/make_map_cnn_golden.py).
"""
import torch
import torch.nn as nn

from avnav_models import RNNStateEncoder, conv_out

# (map type, MAP_SIZE): (kernel sizes, strides) of the three convolutions
GEOMETRY = {
    ("gm", 200): ((8, 4, 3), (4, 2, 1)),
    ("gm", 400): ((8, 4, 3), (5, 4, 2)),
    ("am", None): ((5, 3, 3), (2, 1, 1)),
}
# name: (map type, H, W, C) of the reference's three configurations
REFERENCE_SHAPES = {"gm200": ("gm", 200, 200, 2), "gm400": ("gm", 400, 400, 2), "am20": ("am", 20, 20, 1)}


def geometry(map_type, H):
    """The reference's choice: gm picks by the map's height (200, else 400), am has one geometry."""
    if map_type == "am":
        return GEOMETRY[("am", None)]
    return GEOMETRY[("gm", 200 if H == 200 else 400)]


class MapCNN(nn.Module):
    """``MapCNN`` for an (H, W, C) map of ``map_type`` ('gm' or 'am').  ``layers`` = (kernel sizes, strides)
    overrides the reference's geometry, for shapes the reference never builds."""

    def __init__(self, H, W, C, output_size, map_type="gm", layers=None):
        super().__init__()
        self._map_type = map_type
        self._n_input_gm = C
        kernels, strides = layers if layers is not None else geometry(map_type, H)
        h, w = H, W
        for k, s in zip(kernels, strides):
            h, w = conv_out(h, k, s), conv_out(w, k, s)
        self.cnn = nn.Sequential(
            nn.Conv2d(C, 32, kernels[0], strides[0]), nn.ReLU(True),
            nn.Conv2d(32, 64, kernels[1], strides[1]), nn.ReLU(True),
            nn.Conv2d(64, 32, kernels[2], strides[2]),
            nn.Flatten(), nn.Linear(32 * h * w, output_size), nn.ReLU(True))

    def forward(self, observations):
        return self.cnn(torch.cat([observations[self._map_type].permute(0, 3, 1, 2)], dim=1))


def map_obs(N, H, W, C, seed, kind):
    """A (N, H, W, C) float32 map on the CPU: 'gm' 0/1 occupancy values as the geometric map holds, 'am' sparse
    non-negative values as the acoustic map holds (about one pixel in eight set), 'dense' standard normal values."""
    g = torch.Generator().manual_seed(seed)
    if kind == "gm":
        return (torch.rand((N, H, W, C), generator=g) < 0.3).float()
    if kind == "am":
        v = torch.rand((N, H, W, C), generator=g) * 3
        return v * (torch.rand((N, H, W, C), generator=g) < 0.125).float()
    return torch.randn((N, H, W, C), generator=g)


class AudioNavBaselineNet(nn.Module):
    """The rollout-time part of av_wan's ``AudioNavBaselineNet.forward`` (policy.py:198-215) with a spectrogram goal,
    both maps and a visual encoder: ``x = [audio, gm, am, visual]``, then the state encoder.  The reference's
    ``isnan`` assert is left to the caller."""

    def __init__(self, audio_cnn, gm_cnn, am_cnn, visual_cnn, hidden_size=512):
        super().__init__()
        self.audio_encoder = audio_cnn
        self.gm_encoder = gm_cnn
        self.am_encoder = am_cnn
        self.visual_encoder = visual_cnn
        self.state_encoder = RNNStateEncoder(4 * hidden_size, hidden_size)

    def forward(self, observations, rnn_hidden_states, masks):
        x = [self.audio_encoder(observations), self.gm_encoder(observations), self.am_encoder(observations),
             self.visual_encoder(observations)]
        return self.state_encoder(torch.cat(x, dim=1), rnn_hidden_states, masks)
