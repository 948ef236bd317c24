"""Simulator factories the remote-mode tests start in worker processes (imported there by module name)."""
from types import SimpleNamespace

import numpy as np

from soundspaces_b200.simulator import B200ContinuousAudioMixin
from synth import make_rir


class ContinuousReplaySim(B200ContinuousAudioMixin):
    """The audio state of ``ContinuousSoundSpacesSim`` (continuous_simulator.py:384-387,413-456) stepped without
    habitat-sim: every step the previous RIR becomes ``_last_rir``, a new seeded RIR arrives in ``_prev_sim_obs`` and
    the sample window advances by ``int(sr * STEP_TIME)``, wrapping around the clip."""

    def __init__(self, sr, clip, seed, crossfade, deferred, duration=30, step_time=0.3):
        self.b200_deferred = deferred
        self.config = SimpleNamespace(STEP_TIME=step_time, AUDIO=SimpleNamespace(RIR_SAMPLING_RATE=sr,
                                                                                 CROSSFADE=crossfade))
        self._current_sound, self._source_sound_dict = "clip.wav", {"clip.wav": clip}
        self._episode_step_count, self._duration = 0, duration
        self._seed, self._n = seed, 0
        self._current_sample_index = (seed * 1700) % len(clip)
        self._last_rir = None
        self._prev_sim_obs = {"audio_sensor": self._rir()}
        self._is_episode_active = True

    def _rir(self):
        self._n += 1
        taps = 1500 + (97 * (self._seed + 3 * self._n)) % 6000
        return make_rir(1000 * self._seed + self._n, taps).T.astype(np.float64)

    @property
    def current_source_sound(self):
        return self._source_sound_dict[self._current_sound]

    def step(self, action):
        sr = self.config.AUDIO.RIR_SAMPLING_RATE
        self._last_rir = np.transpose(np.array(self._prev_sim_obs["audio_sensor"]))
        self._prev_sim_obs = {"audio_sensor": self._rir()}
        self._current_sample_index = (self._current_sample_index + int(sr * self.config.STEP_TIME)) % \
            len(self.current_source_sound)
        self._episode_step_count += 1


def continuous_sim(sr, clip, seed, crossfade, deferred="remote"):
    return ContinuousReplaySim(sr, clip, seed, crossfade, deferred)
