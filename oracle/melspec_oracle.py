"""TEST INFRASTRUCTURE ONLY - CPU restatement (numpy float64) of the two mel front-ends.  Only tests/,
__graft_entry__.smoke() and bench.py's cpu_baseline leg may import it.

PARITY UNPINNED: the reference computes these with librosa, which is neither vendored nor pinned
(/root/reference/requirements.txt:3 "librosa") and is absent from this image.  What is restated here is
librosa's published algorithm as the reference calls it:
  * models/encoder/audio.py:53-65      librosa.feature.melspectrogram(y, sr=16000, n_fft=400, hop_length=160, n_mels=40)
  * models/synthesizer/audio.py:59-65  _normalize(_amp_to_db(mel_basis @ |librosa.stft(preemphasis(wav))|) - ref_level_db)
    with :19-22 (preemphasis = lfilter([1, -k], [1])), :115-121 (librosa.stft(n_fft, hop_length, win_length)),
    :166-169 (librosa.filters.mel(sr, n_fft, n_mels, fmin, fmax)), :133-135, :156-172.
librosa.stft: center=True (pad n_fft//2; pad_mode "reflect" up to librosa 0.9, "constant" from 0.10 - a parameter
here), periodic Hann window of win_length centered in n_fft, rfft per frame; n_frames = 1 + len(y) // hop.
librosa.filters.mel: Slaney scale (htk=False), norm="slaney".  The STFT part is cross-checked against torch.stft in
tests/test_oracle_pinned.py, odd n_fft and odd window lengths included.
FFT-bin frequencies: librosa's fft_frequencies was np.linspace(0, sr / 2, 1 + n_fft // 2) before 0.10 and rfftfreq from it.
The two agree for even n_fft only, so, like pad_mode, the answer for odd n_fft depends on the librosa version.  No shipped
config uses an odd n_fft; mel_basis refuses one, as mb_melspec_create does.
"""
from __future__ import annotations

import numpy as np


def hz_to_mel(f):
    f = np.asanyarray(f, dtype=np.float64)
    f_sp = 200.0 / 3
    mels = f / f_sp
    min_log_hz = 1000.0
    min_log_mel = min_log_hz / f_sp
    logstep = np.log(6.4) / 27.0
    return np.where(f >= min_log_hz, min_log_mel + np.log(np.maximum(f, 1e-30) / min_log_hz) / logstep, mels)


def mel_to_hz(m):
    m = np.asanyarray(m, dtype=np.float64)
    f_sp = 200.0 / 3
    min_log_hz = 1000.0
    min_log_mel = min_log_hz / f_sp
    logstep = np.log(6.4) / 27.0
    return np.where(m >= min_log_mel, min_log_hz * np.exp(logstep * (m - min_log_mel)), f_sp * m)


def mel_basis(sr: int, n_fft: int, n_mels: int, fmin: float, fmax: float) -> np.ndarray:
    """librosa.filters.mel(sr, n_fft, n_mels, fmin, fmax) -> [n_mels, 1 + n_fft // 2] float32; n_fft even (module header)"""
    if n_fft % 2:
        raise ValueError(f"n_fft = {n_fft} is odd: librosa's FFT-bin frequencies for it depend on the librosa version")
    fftfreqs = np.linspace(0, sr / 2.0, 1 + n_fft // 2)
    mel_f = mel_to_hz(np.linspace(hz_to_mel(fmin), hz_to_mel(fmax), n_mels + 2))
    fdiff = np.diff(mel_f)
    ramps = mel_f[:, None] - fftfreqs[None, :]
    w = np.zeros((n_mels, 1 + n_fft // 2))
    for i in range(n_mels):
        lower = -ramps[i] / fdiff[i]
        upper = ramps[i + 2] / fdiff[i + 1]
        w[i] = np.maximum(0, np.minimum(lower, upper))
    enorm = 2.0 / (mel_f[2:n_mels + 2] - mel_f[:n_mels])
    return (w * enorm[:, None]).astype(np.float32)


def stft(y: np.ndarray, n_fft: int, hop: int, win: int, pad_mode: str = "reflect") -> np.ndarray:
    """librosa.stft(y, n_fft, hop_length, win_length) -> complex [1 + n_fft // 2, n_frames]"""
    y = np.asarray(y, dtype=np.float64)
    n = np.arange(win)
    w = 0.5 - 0.5 * np.cos(2 * np.pi * n / win)  # scipy.signal.get_window("hann", win, fftbins=True)
    lpad = (n_fft - win) // 2
    window = np.zeros(n_fft)
    window[lpad:lpad + win] = w
    yp = np.pad(y, n_fft // 2, mode=pad_mode)
    n_frames = 1 + (len(yp) - n_fft) // hop
    frames = np.stack([yp[i * hop:i * hop + n_fft] * window for i in range(n_frames)], axis=1)
    return np.fft.rfft(frames, axis=0)


def encoder_mel(wav: np.ndarray, pad_mode: str = "reflect") -> np.ndarray:
    """models/encoder/audio.py:53-65 -> float32 [n_frames, 40]"""
    S = np.abs(stft(wav, 400, 160, 400, pad_mode)) ** 2
    return (mel_basis(16000, 400, 40, 0.0, 8000.0).astype(np.float64) @ S).astype(np.float32).T


def synthesizer_mel(wav: np.ndarray, hp: dict, pad_mode: str = "reflect") -> np.ndarray:
    """models/synthesizer/audio.py:59-65 -> float32 [num_mels, n_frames].  Optional keys beyond the reference's hparams
    cover every mb_melspec_config: power (1: |D|, 2: |D|^2; default 1), to_db (default True), signal_normalization
    (default True, applied to the dB or linear values alike)."""
    from scipy.signal import lfilter

    y = lfilter([1, -hp["preemphasis"]], [1], np.asarray(wav, dtype=np.float64)) if hp.get("preemphasize", True) else wav
    D = stft(y, hp["n_fft"], hp["hop_size"], hp["win_size"], pad_mode)
    M = mel_basis(hp["sample_rate"], hp["n_fft"], hp["num_mels"], hp["fmin"], hp["fmax"]).astype(np.float64) @ \
        np.abs(D) ** hp.get("power", 1)
    S = M
    if hp.get("to_db", True):
        min_level = np.exp(hp["min_level_db"] / 20 * np.log(10))
        S = 20 * np.log10(np.maximum(min_level, M)) - hp["ref_level_db"]
    if not hp.get("signal_normalization", True):
        return S.astype(np.float32)
    A = hp["max_abs_value"]
    if hp.get("symmetric_mels", True):
        S = np.clip((2 * A) * ((S - hp["min_level_db"]) / (-hp["min_level_db"])) - A, -A, A)
    else:
        S = np.clip(A * ((S - hp["min_level_db"]) / (-hp["min_level_db"])), 0, A)
    return S.astype(np.float32)


SYNTH_HP = dict(sample_rate=16000, n_fft=1024, num_mels=80, hop_size=256, win_size=1024, fmin=55, fmax=7600,
                min_level_db=-100, ref_level_db=20, max_abs_value=4.0, preemphasis=0.97, preemphasize=True, symmetric_mels=True)
