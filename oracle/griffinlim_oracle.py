"""TEST INFRASTRUCTURE ONLY - CPU restatement (numpy) of the reference's Griffin-Lim inversion of a normalised dB mel
spectrogram.  Only tests/ and bench_griffinlim.py may import it.

PARITY UNPINNED, as melspec_oracle: the reference (models/synthesizer/audio.py:84-124, 162-166, 177-206) calls librosa,
which is neither vendored nor pinned and is absent here.  Restated is librosa's published algorithm:
  * librosa.stft: melspec_oracle.stft (centred frames, n_fft // 2 padding, periodic Hann of win_length centred in n_fft)
  * librosa.istft: irfft of each column (the imaginary parts of the DC and Nyquist bins ignored), times the window,
    overlap-add, divided by the window sum-square where that exceeds float32's smallest normal, trimmed by n_fft // 2 at
    both ends -> hop * (T - 1) samples
  * _griffin_lim: y = istft(S exp(2 pi i u)); n_iters times y = istft(S exp(i angle(stft(y))))
  * inv_preemphasis: scipy.signal.lfilter([1], [1, -k], y)
``dtype=np.float32`` runs the same algorithm in single precision (numpy's pocketfft computes float32 transforms in float32);
the tests use it to measure how far float32 arithmetic drifts from float64 on their inputs.
"""
from __future__ import annotations

import numpy as np

from melspec_oracle import mel_basis, stft


def _window(n_fft: int, win: int, dtype=np.float64) -> np.ndarray:
    w = np.zeros(n_fft)
    lpad = (n_fft - win) // 2
    w[lpad:lpad + win] = 0.5 - 0.5 * np.cos(2 * np.pi * np.arange(win) / win)
    return w.astype(dtype)


def inv_basis(hp) -> np.ndarray:
    """np.linalg.pinv of the float32 librosa basis, in float32 (audio.py:165)"""
    return np.linalg.pinv(mel_basis(hp.sample_rate, hp.n_fft, hp.num_mels, hp.fmin, hp.fmax))


def denormalize(D, hp) -> np.ndarray:
    """audio.py:194-206"""
    D = np.asarray(D, dtype=np.float64)
    A, lo = hp.max_abs_value, hp.min_level_db
    if hp.symmetric_mels:
        if hp.allow_clipping_in_normalization:
            D = np.clip(D, -A, A)
        return ((D + A) * -lo / (2 * A)) + lo
    if hp.allow_clipping_in_normalization:
        D = np.clip(D, 0, A)
    return (D * -lo / A) + lo


def magnitudes(mel, hp) -> np.ndarray:
    """S = max(1e-10, pinv @ 10^((D + ref_level_db) / 20)) ** power, float64 [n_fft // 2 + 1, T]"""
    D = denormalize(mel, hp) if hp.signal_normalization else np.asarray(mel, dtype=np.float64)
    amp = np.power(10.0, (D + hp.ref_level_db) * 0.05)
    return np.maximum(1e-10, inv_basis(hp).astype(np.float64) @ amp) ** hp.power


def _stft(y, n_fft, hop, win, pad_mode, dtype):
    if dtype == np.float64:
        return stft(y, n_fft, hop, win, pad_mode)
    window = _window(n_fft, win, dtype)
    yp = np.pad(np.asarray(y, dtype=dtype), n_fft // 2, mode=pad_mode)
    n_frames = 1 + (len(yp) - n_fft) // hop
    frames = np.stack([yp[i * hop:i * hop + n_fft] * window for i in range(n_frames)], axis=1)
    return np.fft.rfft(frames, axis=0)


def istft(C, n_fft: int, hop: int, win: int, dtype=np.float64) -> np.ndarray:
    """librosa.istft(C, hop_length=hop, win_length=win) for C [n_fft // 2 + 1, T] -> [hop * (T - 1)]"""
    T = C.shape[1]
    window = _window(n_fft, win, dtype)
    frames = np.fft.irfft(C, n=n_fft, axis=0).astype(dtype) * window[:, None]
    n = n_fft + hop * (T - 1)
    y = np.zeros(n, dtype=dtype)
    wss = np.zeros(n, dtype=dtype)
    for t in range(T):
        y[t * hop:t * hop + n_fft] += frames[:, t]
        wss[t * hop:t * hop + n_fft] += window * window
    nz = wss > np.finfo(np.float32).tiny
    y[nz] /= wss[nz]
    return y[n_fft // 2:n - n_fft // 2]


def phasors(u, dtype=np.float64) -> np.ndarray:
    """exp(2 pi i u), computed in float64 and rounded once"""
    p = np.exp(2j * np.pi * np.asarray(u, dtype=np.float64))
    return p.astype(np.complex64 if dtype == np.float32 else np.complex128)


def griffin_lim(S, u, n_iters: int, n_fft: int, hop: int, win: int, pad_mode: str = "reflect", dtype=np.float64):
    """audio.py:105-115 from the uniforms u [n_fft // 2 + 1, T] of np.random.rand(*S.shape)"""
    S = np.asarray(S).astype(dtype)
    y = istft(S * phasors(u, dtype), n_fft, hop, win, dtype)
    for _ in range(n_iters):
        y = iterate(S, y, n_fft, hop, win, pad_mode, dtype)
    return y


def iterate(S, y, n_fft: int, hop: int, win: int, pad_mode: str = "reflect", dtype=np.float64):
    """one Griffin-Lim step: istft(S exp(i angle(stft(y)))), with angle(0) = 0"""
    X = _stft(y, n_fft, hop, win, pad_mode, dtype)
    m = np.abs(X)
    P = np.where(m > 0, X / np.where(m > 0, m, 1), 1)
    return istft(np.asarray(S).astype(dtype) * P, n_fft, hop, win, dtype)


def inv_preemphasis(y, k):
    from scipy.signal import lfilter

    return lfilter([1], [1, -k], np.asarray(y, dtype=np.float64))


def inv_mel_spectrogram(mel, hp, u, pad_mode: str = "reflect", n_iters=None, dtype=np.float64):
    """audio.py:84-99 with the uniforms u given"""
    hop = hp.hop_size
    y = griffin_lim(magnitudes(mel, hp), u, hp.griffin_lim_iters if n_iters is None else n_iters, hp.n_fft, hop, hp.win_size,
                    pad_mode, dtype)
    return inv_preemphasis(y, hp.preemphasis) if hp.preemphasize else np.asarray(y, dtype=np.float64)


def spectral_convergence(S, y, n_fft: int, hop: int, win: int, pad_mode: str = "reflect") -> float:
    """|| S - |stft(y)| ||_F / || S ||_F"""
    M = np.abs(stft(y, n_fft, hop, win, pad_mode))
    return float(np.linalg.norm(S - M) / np.linalg.norm(S))
