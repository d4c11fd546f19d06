"""BASELINE.json configs[4] ("audio-driven walk (examples/make_music_video.py), 30 fps x 10 s"): the interpolation
schedule T the walk follows, computed from the reference's own fixture tests/samples/choice.wav (22 050 Hz mono, 10 s;
tests/test_pipeline.py:53-68) with this package's librosa-free `get_timesteps_arr` restatement and the example's
arguments (fps 30, margin 1.0, smooth 0.2, offset 0, duration 10 — examples/make_music_video.py:43-55).

It also stores the first 2 s of choice.wav (int16 samples, choice_2s_i16.npy) and the schedule of that excerpt
(cfg5_choice_2s_T.npy, duration 2, 60 frames), so that the restatement is checked on the reference's own audio without
the reference checkout.  PARITY UNPINNED against librosa (not installable): the fixtures pin the restatement against
regressions.

    python tests/golden/make_cfg5_schedule.py <reference checkout>/tests/samples/choice.wav
"""
import importlib.util
import os
import sys

import numpy as np
from scipy.io import wavfile

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
EXCERPT_S = 2


def schedule(wav, duration=10):
    spec = importlib.util.spec_from_file_location("sdw_audio", os.path.join(ROOT, "stable-diffusion-videos_b200", "audio.py"))
    audio = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(audio)
    return audio.get_timesteps_arr(wav, offset=0, duration=duration, fps=30, margin=1.0, smooth=0.2)


if __name__ == "__main__":
    wav = sys.argv[1]
    T = schedule(wav)
    np.save(os.path.join(HERE, "cfg5_choice_T.npy"), T.astype(np.float64))
    print(T.shape, T[:5], T[-3:], "monotone:", bool(np.all(np.diff(T) >= 0)))
    sr, y = wavfile.read(wav)
    assert sr == 22050 and y.dtype == np.int16 and y.ndim == 1
    np.save(os.path.join(HERE, "choice_2s_i16.npy"), y[: EXCERPT_S * sr])
    np.save(os.path.join(HERE, "cfg5_choice_2s_T.npy"), schedule(wav, duration=EXCERPT_S).astype(np.float64))
