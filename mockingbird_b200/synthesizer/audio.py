"""Synthesizer mel front-end (reference: models/synthesizer/audio.py:59-65), SURVEY.md §8f row N1.

``melspectrogram(wav, hparams)``: pre-emphasis -> STFT -> 80-band mel of the magnitudes -> dB - ref_level_db ->
symmetric normalisation to [-max_abs_value, max_abs_value]; float32 [num_mels, n_frames] like the reference, computed on
the H100 (mb_melspec_*).  ``pad_mode`` as in mockingbird_b200.encoder.audio."""
from __future__ import annotations

import numpy as np

from ..melspec import MelSpectrogram

pad_mode = "reflect"
_front = {}


def get_hop_size(hparams):
    hop_size = hparams.hop_size
    if hop_size is None:
        assert hparams.frame_shift_ms is not None
        hop_size = int(hparams.frame_shift_ms / 1000 * hparams.sample_rate)
    return hop_size


def melspectrogram(wav, hparams):
    if getattr(hparams, "use_lws", False):
        raise NotImplementedError("use_lws=True (lws STFT) is not built")
    if not getattr(hparams, "allow_clipping_in_normalization", True):
        raise NotImplementedError("allow_clipping_in_normalization=False is not built")
    key = (pad_mode, hparams.sample_rate, hparams.n_fft, get_hop_size(hparams), hparams.win_size, hparams.num_mels, hparams.fmin,
           hparams.fmax, hparams.preemphasis if hparams.preemphasize else 0.0, hparams.min_level_db, hparams.ref_level_db,
           bool(hparams.signal_normalization), hparams.max_abs_value, bool(hparams.symmetric_mels))
    if key not in _front:
        _front[key] = MelSpectrogram(hparams.sample_rate, hparams.n_fft, get_hop_size(hparams), hparams.win_size, hparams.num_mels,
                                     hparams.fmin, hparams.fmax, pad_mode=pad_mode,
                                     preemphasis=hparams.preemphasis if hparams.preemphasize else 0.0, power=1, to_db=True,
                                     min_level_db=hparams.min_level_db, ref_level_db=hparams.ref_level_db,
                                     normalize=bool(hparams.signal_normalization), max_abs_value=hparams.max_abs_value,
                                     symmetric=bool(hparams.symmetric_mels), transpose_out=False)
    return _front[key](np.asarray(wav, dtype=np.float32)).cpu().numpy()
