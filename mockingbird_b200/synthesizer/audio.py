"""Synthesizer mel front-end (reference: models/synthesizer/audio.py:59-65), SURVEY.md §8f row N1.

``melspectrogram(wav, hparams)``: pre-emphasis -> STFT -> 80-band mel of the magnitudes -> dB - ref_level_db ->
symmetric normalisation to [-max_abs_value, max_abs_value]; float32 [num_mels, n_frames] like the reference, computed on
the H100 (mb_melspec_*).  ``pad_mode`` as in mockingbird_b200.encoder.audio; it also sets the STFT padding of the
Griffin-Lim iterations.

``inv_mel_spectrogram(mel, hparams)`` / ``inv_mel_spectrograms(mels, hparams, seeds=None)``: the reference's Griffin-Lim
(audio.py:84-124) on the H100 (mb_griffinlim_*), float64 waveforms like the reference."""
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


def _mel_front(hparams):
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
    return _front[key]


def melspectrogram(wav, hparams):
    return _mel_front(hparams)(np.asarray(wav, dtype=np.float32)).cpu().numpy()


def melspectrograms(wavs, hparams):
    """melspectrogram of many waveforms in one launch: a list of float32 [num_mels, n_i], entry i bitwise
    melspectrogram(wavs[i], hparams).  Pre-emphasis starts afresh at each waveform's first sample.  Every waveform is
    checked (1-D, not empty, more than n_fft / 2 samples with reflect padding) before anything is queued; the ValueError
    names the first bad one."""
    from ..melspec import as_wavs, check_wavs, min_signal_length

    wavs = as_wavs(wavs)
    check_wavs(wavs, min_signal_length(hparams.n_fft, pad_mode))
    if not wavs:
        return []
    return _mel_front(hparams).many(wavs)


_inverse = {}


def _griffin_lim(hparams):
    from ..griffinlim import GriffinLim
    from .audio_host import mel_basis

    key = (pad_mode, hparams.sample_rate, hparams.n_fft, get_hop_size(hparams), hparams.win_size, hparams.num_mels, hparams.fmin,
           hparams.fmax, float(hparams.power), hparams.preemphasis if hparams.preemphasize else 0.0,
           bool(hparams.signal_normalization), bool(hparams.allow_clipping_in_normalization), bool(hparams.symmetric_mels),
           hparams.max_abs_value, hparams.min_level_db, hparams.ref_level_db)
    if key not in _inverse:
        # the reference's _mel_to_linear: np.linalg.pinv of the float32 librosa basis, in float32
        inv = np.linalg.pinv(mel_basis(hparams.sample_rate, hparams.n_fft, hparams.num_mels, hparams.fmin, hparams.fmax))
        _inverse[key] = GriffinLim(inv, hparams.n_fft, get_hop_size(hparams), hparams.win_size, pad_mode=pad_mode,
                                   power=hparams.power, preemphasis=hparams.preemphasis if hparams.preemphasize else 0.0,
                                   signal_normalization=hparams.signal_normalization,
                                   allow_clipping=hparams.allow_clipping_in_normalization, symmetric=hparams.symmetric_mels,
                                   max_abs_value=hparams.max_abs_value, min_level_db=hparams.min_level_db,
                                   ref_level_db=hparams.ref_level_db)
    return _inverse[key]


def inv_mel_spectrograms(mels, hparams, seeds=None):
    """Griffin-Lim (reference: models/synthesizer/audio.py:84-124) for a list of normalised dB mels [num_mels, T_b] in one
    sequence of launches on the H100 -> list of float64 waveforms of hop * (T_b - 1) samples.

    seeds=None: the initial phases are ``np.random.rand(n_fft // 2 + 1, T_b)`` drawn from numpy's global state for each mel
    in list order, so the phases and the final state of the generator are those of the same sequence of single reference
    calls.  seeds (one integer per mel): the phases are drawn on the device, keyed by (seed, bin, frame); numpy's state is
    not touched and a mel's result does not depend on the other mels."""
    if getattr(hparams, "use_lws", False):
        raise NotImplementedError("use_lws=True (lws STFT) is not built")
    mels = [np.asarray(m, dtype=np.float32) for m in mels]
    if not mels:
        return []
    gl = _griffin_lim(hparams)
    if seeds is None:
        uniforms = [np.random.rand(gl.n_bins, m.shape[1]) for m in mels]
        ys = gl(mels, hparams.griffin_lim_iters, uniforms=uniforms)
    else:
        if len(seeds) != len(mels):
            raise ValueError(f"{len(seeds)} seeds for {len(mels)} mels")
        ys = gl(mels, hparams.griffin_lim_iters, seeds=seeds)
    return [y.cpu().numpy().astype(np.float64) for y in ys]


def inv_mel_spectrogram(mel_spectrogram, hparams):
    """models/synthesizer/audio.py:84-99 on the H100 (see inv_mel_spectrograms): float64 waveform"""
    return inv_mel_spectrograms([mel_spectrogram], hparams)[0]
