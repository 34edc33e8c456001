"""Encoder audio front-end (reference: models/encoder/audio.py:53-65), SURVEY.md §8f row N2.

``wav_to_mel_spectrogram(wav)``: 40-channel mel POWER spectrogram (25 ms window, 10 ms step, not log) as float32
[n_frames, 40], computed on the H100 (mb_melspec_*).  The reference calls librosa.feature.melspectrogram; librosa is
unpinned there, and its centered-frame padding changed from "reflect" (<= 0.9) to "constant" (>= 0.10):
``pad_mode`` selects which (default "reflect", the behaviour of the librosa releases contemporary with the reference).
Volume normalisation / VAD trimming (preprocess_wav, webrtcvad) are host-side preprocessing and out of scope."""
from __future__ import annotations

import numpy as np

from ..melspec import MelSpectrogram
from .params_data import mel_n_channels, mel_window_length, mel_window_step, sampling_rate

pad_mode = "reflect"
_front = {}


def wav_to_mel_spectrogram(wav):
    key = pad_mode
    if key not in _front:
        n_fft = int(sampling_rate * mel_window_length / 1000)
        _front[key] = MelSpectrogram(sampling_rate, n_fft, int(sampling_rate * mel_window_step / 1000), n_fft, mel_n_channels,
                                     0.0, sampling_rate / 2, pad_mode=key, power=2, transpose_out=True)
    return _front[key](np.asarray(wav, dtype=np.float32)).cpu().numpy()
