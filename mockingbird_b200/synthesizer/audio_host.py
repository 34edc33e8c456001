"""Host-side audio utilities the reference's callers reach through ``Synthesizer`` / ``encoder.inference`` but that are NOT
on the accelerated path (SURVEY.md section 8: out of scope for kernels): file loading, volume normalisation, Griffin-Lim.
They exist so that the documented import switch (INTEGRATION.md) leaves no caller with an AttributeError.

  normalize_volume / preprocess_wav   models/encoder/audio.py:19-53, 108-117 (webrtcvad silence trimming only when the
                                      optional package is present, exactly like the reference's try/except import)
  load_wav                            librosa.load(sr=...) stand-in: scipy.io.wavfile + polyphase resampling
  inv_mel_spectrogram / griffin_lim   models/synthesizer/audio.py:84-124, 162-171 (librosa.stft/istft -> torch.stft/istft,
                                      Slaney mel basis restated in numpy)
librosa is not a dependency of this package; where the reference delegates to it the numerics differ at the 1e-6 level.
"""
from __future__ import annotations

from pathlib import Path
from typing import Optional, Union

import numpy as np

int16_max = (2 ** 15) - 1


def load_wav(path, sr: Optional[int]):
    """-> (float32 mono waveform in [-1, 1], sample rate); resampled to `sr` when given"""
    from scipy.io import wavfile
    from scipy.signal import resample_poly

    src_sr, data = wavfile.read(str(path))
    if data.dtype.kind == "i":
        data = data.astype(np.float32) / float(np.iinfo(data.dtype).max + 1)
    elif data.dtype.kind == "u":
        data = (data.astype(np.float32) - 128.0) / 128.0
    data = data.astype(np.float32)
    if data.ndim > 1:
        data = data.mean(axis=1)
    if sr is not None and src_sr != sr:
        g = np.gcd(int(src_sr), int(sr))
        data = resample_poly(data, sr // g, src_sr // g).astype(np.float32)
        src_sr = sr
    return data, src_sr


def normalize_volume(wav, target_dBFS, increase_only=False, decrease_only=False):
    """models/encoder/audio.py:108-117"""
    if increase_only and decrease_only:
        raise ValueError("Both increase only and decrease only are set")
    dBFS_change = target_dBFS - 10 * np.log10(np.mean(wav ** 2))
    if (dBFS_change < 0 and increase_only) or (dBFS_change > 0 and decrease_only):
        return wav
    return wav * (10 ** (dBFS_change / 20))


def trim_long_silences(wav, sampling_rate, vad_window_length=30, vad_moving_average_width=8, vad_max_silence_length=6):
    """models/encoder/audio.py:68-105; needs the optional webrtcvad package (returns wav unchanged without it)"""
    try:
        import webrtcvad
    except Exception:
        return wav
    import struct

    from scipy.ndimage import binary_dilation

    samples_per_window = (vad_window_length * sampling_rate) // 1000
    wav = wav[:len(wav) - (len(wav) % samples_per_window)]
    pcm_wave = struct.pack("%dh" % len(wav), *(np.round(wav * int16_max)).astype(np.int16))
    voice_flags = []
    vad = webrtcvad.Vad(mode=3)
    for window_start in range(0, len(wav), samples_per_window):
        window_end = window_start + samples_per_window
        voice_flags.append(vad.is_speech(pcm_wave[window_start * 2:window_end * 2], sample_rate=sampling_rate))
    voice_flags = np.array(voice_flags)

    def moving_average(array, width):
        array_padded = np.concatenate((np.zeros((width - 1) // 2), array, np.zeros(width // 2)))
        ret = np.cumsum(array_padded, dtype=float)
        ret[width:] = ret[width:] - ret[:-width]
        return ret[width - 1:] / width

    audio_mask = moving_average(voice_flags, vad_moving_average_width)
    audio_mask = np.round(audio_mask).astype(bool)
    audio_mask = binary_dilation(audio_mask, np.ones(vad_max_silence_length + 1))
    audio_mask = np.repeat(audio_mask, samples_per_window)
    return wav[audio_mask == True]  # noqa: E712


def preprocess_wav(fpath_or_wav: Union[str, Path, np.ndarray], source_sr: Optional[int] = None, normalize: Optional[bool] = True,
                   trim_silence: Optional[bool] = True, sampling_rate: int = 16000, audio_norm_target_dBFS: float = -30):
    """models/encoder/audio.py:19-53"""
    if isinstance(fpath_or_wav, (str, Path)):
        wav, source_sr = load_wav(fpath_or_wav, None)
    else:
        wav = fpath_or_wav
    if source_sr is not None and source_sr != sampling_rate:
        from scipy.signal import resample_poly

        g = np.gcd(int(source_sr), int(sampling_rate))
        wav = resample_poly(wav, sampling_rate // g, source_sr // g).astype(np.float32)
    if normalize:
        wav = normalize_volume(wav, audio_norm_target_dBFS, increase_only=True)
    if trim_silence:
        wav = trim_long_silences(wav, sampling_rate)
    return wav


# ---- Griffin-Lim (models/synthesizer/audio.py:84-124) ---------------------------------------------------------------
def _hz_to_mel(f):
    f = np.asarray(f, dtype=np.float64)
    lin = f / (200.0 / 3)
    logstep = np.log(6.4) / 27.0
    return np.where(f >= 1000.0, 15.0 + np.log(np.maximum(f, 1e-10) / 1000.0) / logstep, lin)


def _mel_to_hz(m):
    m = np.asarray(m, dtype=np.float64)
    logstep = np.log(6.4) / 27.0
    return np.where(m >= 15.0, 1000.0 * np.exp(logstep * (m - 15.0)), m * (200.0 / 3))


def mel_basis(sr: int, n_fft: int, n_mels: int, fmin: float, fmax: float) -> np.ndarray:
    """librosa.filters.mel (Slaney scale, slaney norm) restated"""
    fftfreqs = np.linspace(0, sr / 2.0, 1 + n_fft // 2)
    mel_f = _mel_to_hz(np.linspace(_hz_to_mel(fmin), _hz_to_mel(fmax), n_mels + 2))
    fdiff = np.diff(mel_f)
    ramps = mel_f[:, None] - fftfreqs[None, :]
    w = np.maximum(0, np.minimum(-ramps[:-2] / fdiff[:-1, None], ramps[2:] / fdiff[1:, None]))
    return (w * (2.0 / (mel_f[2:n_mels + 2] - mel_f[:n_mels]))[:, None]).astype(np.float32)


def ppg_melmat(sr: int, n_fft: int, n_mels: int, fmin: float, fmax: float, norm=1) -> np.ndarray:
    """``librosa.filters.mel(sr, n_fft, n_mels, fmin, fmax, norm=norm).T`` restated: [1 + n_fft // 2, n_mels], the
    ``frontend.logmel.melmat`` buffer of the PPG extractor (models/ppg_extractor/log_mel.py:47-49).  The reference pins no
    librosa version and ``norm=1`` changed meaning in librosa 0.8: before it, area ("slaney") normalisation; since, each
    filter divided by its L1 norm.  ``norm=1`` here is the current meaning, ``norm="slaney"`` the old one."""
    fftfreqs = np.linspace(0, sr / 2.0, 1 + n_fft // 2)
    mel_f = _mel_to_hz(np.linspace(_hz_to_mel(fmin), _hz_to_mel(fmax), n_mels + 2))
    fdiff = np.diff(mel_f)
    ramps = mel_f[:, None] - fftfreqs[None, :]
    w = np.maximum(0, np.minimum(-ramps[:-2] / fdiff[:-1, None], ramps[2:] / fdiff[1:, None])).astype(np.float32)
    if norm == "slaney":
        w = w * (2.0 / (mel_f[2:n_mels + 2] - mel_f[:n_mels]))[:, None].astype(np.float32)
    elif norm == 1:
        s = np.abs(w).astype(np.float64).sum(axis=1, keepdims=True)
        w = np.where(s > np.finfo(np.float32).tiny, w / np.maximum(s, np.finfo(np.float32).tiny), w)
    elif norm is not None:
        raise ValueError(f"unsupported mel norm {norm!r}")
    return np.ascontiguousarray(w.astype(np.float32).T)


_inv_basis = {}


def inv_mel_spectrogram(mel_spectrogram: np.ndarray, hp) -> np.ndarray:
    """normalised dB mel [80, T] -> waveform by Griffin-Lim"""
    import torch
    from scipy import signal

    if getattr(hp, "use_lws", False):
        raise NotImplementedError("use_lws=True is not supported (reference default is False)")
    D = mel_spectrogram
    if hp.signal_normalization:
        m, lo = hp.max_abs_value, hp.min_level_db
        if hp.symmetric_mels:
            D = ((np.clip(D, -m, m) + m) * -lo / (2 * m)) + lo if hp.allow_clipping_in_normalization else ((D + m) * -lo / (2 * m)) + lo
        else:
            D = (np.clip(D, 0, m) * -lo / m) + lo if hp.allow_clipping_in_normalization else (D * -lo / m) + lo
    key = (hp.sample_rate, hp.n_fft, hp.num_mels, hp.fmin, hp.fmax)
    if key not in _inv_basis:
        _inv_basis[key] = np.linalg.pinv(mel_basis(*key))
    S = np.maximum(1e-10, _inv_basis[key] @ np.power(10.0, (D + hp.ref_level_db) * 0.05)) ** hp.power
    hop = hp.hop_size if hp.hop_size is not None else int(hp.frame_shift_ms / 1000 * hp.sample_rate)
    win = torch.hann_window(hp.win_size, periodic=True, dtype=torch.float64)
    mag = torch.from_numpy(np.abs(S).astype(np.float64))

    def istft(c):
        return torch.istft(c, hp.n_fft, hop, hp.win_size, win, center=True)

    def stft(y):
        return torch.stft(y, hp.n_fft, hop, hp.win_size, win, center=True, pad_mode="reflect", return_complex=True)

    angles = torch.exp(2j * np.pi * torch.from_numpy(np.random.rand(*S.shape)))
    y = istft(mag * angles)
    for _ in range(hp.griffin_lim_iters):
        angles = torch.exp(1j * torch.angle(stft(y)))
        y = istft(mag * angles[:, : mag.shape[1]])
    y = y.numpy()
    if hp.preemphasize:
        y = signal.lfilter([1], [1, -hp.preemphasis], y)
    return y
