"""Encoder audio front-end (reference: models/encoder/audio.py:53-65), SURVEY.md §8f row N2.

``wav_to_mel_spectrogram(wav)``: 40-channel mel POWER spectrogram (25 ms window, 10 ms step, not log) as float32
[n_frames, 40], computed on the H100 (mb_melspec_*).  The reference calls librosa.feature.melspectrogram; librosa is
unpinned there, and its centered-frame padding changed from "reflect" (<= 0.9) to "constant" (>= 0.10):
``pad_mode`` selects which (default "reflect", the behaviour of the librosa releases contemporary with the reference).
Volume normalisation / VAD trimming (preprocess_wav, webrtcvad) are host-side preprocessing and out of scope."""
from __future__ import annotations

import numpy as np

from ..melspec import MelSpectrogram, as_wavs, check_wavs, min_signal_length
from .params_data import mel_n_channels, mel_window_length, mel_window_step, sampling_rate

pad_mode = "reflect"
_front = {}


N_FFT = int(sampling_rate * mel_window_length / 1000)


def mel_front(device=None) -> MelSpectrogram:
    """the front-end handle of the current pad_mode on `device` (default: the current CUDA device); its outputs live there"""
    import torch

    from .. import _lib

    dev = torch.device(device) if device is not None else _lib.require_cuda()
    key = (pad_mode, dev)
    if key not in _front:
        _front[key] = MelSpectrogram(sampling_rate, N_FFT, int(sampling_rate * mel_window_step / 1000), N_FFT, mel_n_channels,
                                     0.0, sampling_rate / 2, pad_mode=pad_mode, power=2, transpose_out=True, device=dev)
    return _front[key]


def check(wavs, signal_lengths=None):
    """check_wavs with the current pad_mode's shortest signal (host only: nothing is queued)"""
    check_wavs(wavs, min_signal_length(N_FFT, pad_mode), signal_lengths)


def wav_to_mel_spectrogram(wav):
    return mel_front()(np.asarray(wav, dtype=np.float32)).cpu().numpy()


def wav_to_mel_spectrograms(wavs):
    """wav_to_mel_spectrogram of many waveforms in one launch: a list of float32 [n_i, 40], entry i bitwise
    wav_to_mel_spectrogram(wavs[i]).  Every waveform is checked (1-D, not empty, long enough for the padding) before
    anything is queued; the ValueError names the first bad one."""
    wavs = as_wavs(wavs)
    check(wavs)
    return mel_front().many(wavs) if wavs else []
