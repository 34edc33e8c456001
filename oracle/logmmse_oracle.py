"""Float64 numpy restatement of the reference's log-MMSE denoiser (utils/logmmse.py) (TEST INFRASTRUCTURE).

Written from the algorithm, not from the reference's code: real FFTs (numpy rfft / irfft) of the half spectrum, the mirror
bins entering the VAD sum with weight 2, and E1 from scipy.special.exp1.  Besides the fp32 output it returns what the device
kernels produce along the way: each frame's VAD statistic and gain hw [nframes][n_fft / 2 + 1], and the final noise
estimate.  `denoise_loop` is the per-frame loop that bench_logmmse.py times as the CPU baseline."""
from __future__ import annotations

import math

import numpy as np
from scipy.special import exp1

EPS = np.finfo(np.float64).eps
AA = MU = 0.98
KSI_MIN = 10 ** (-25 / 10)


def params(sampling_rate, window_size=0):
    """-> (W, len1, len2, window, n_fft) as profile_noise picks them"""
    W = int(window_size) or int(math.floor(0.02 * sampling_rate))
    W += W % 2
    len1 = W // 2
    len2 = W - len1
    win = np.hanning(W)
    win = win * len2 / np.sum(win)
    return W, len1, len2, win, 2 * W


def profile_mu2(noise, win, n_fft):
    """noise_mu2 [n_fft]: the squared mean of |FFT| over the non-overlapping frames of the noise, in frame order"""
    W = len(win)
    x = np.asarray(noise, dtype=np.float64) + EPS
    n = len(x) // W
    acc = np.zeros(n_fft // 2 + 1)
    for j in range(n):
        acc = acc + np.abs(np.fft.rfft(win * x[j * W:(j + 1) * W], n_fft))
    half = (acc / n) ** 2
    return np.concatenate([half, half[1:n_fft // 2][::-1]])


def n_frames(L, W, len2):
    return L // len2 - W // len2


def denoise_loop(wav, win, n_fft, noise_mu2, eta=0.15):
    """-> (fp32 output [L], vad [nframes], hw [nframes][n_fft / 2 + 1], final noise_mu2 half spectrum)"""
    x = np.asarray(wav)
    if x.dtype != np.float32:
        raise ValueError(f"float32 input expected, got {x.dtype}")
    W = len(win)
    hop = W // 2
    L = len(x)
    if L < 2 * hop:
        raise ValueError(f"{L} samples: at least {2 * hop} are needed")
    x = x.astype(np.float64) + EPS
    nb = n_fft // 2 + 1
    weight = np.full(nb, 2.0)
    weight[0] = weight[-1] = 1.0
    nf = n_frames(L, W, hop)
    mu2 = np.array(noise_mu2[:nb], dtype=np.float64)
    xk = np.zeros(nb)
    prior = True
    y = np.zeros(nf * hop)
    tail = np.zeros(hop)
    vads = np.zeros(nf)
    hws = np.zeros((nf, nb))
    for f in range(nf):
        X = np.fft.rfft(win * x[f * hop:f * hop + W], n_fft)
        mag = np.abs(X)
        p = mag * mag
        g = np.minimum(p / mu2, 40.0)
        excess = np.maximum(g - 1.0, 0.0)
        if prior:
            ksi = AA + (1.0 - AA) * excess
        else:
            ksi = np.maximum(KSI_MIN, AA * xk / mu2 + (1.0 - AA) * excess)
        a = ksi / (1.0 + ksi)
        vads[f] = np.dot(weight, g * ksi / (1.0 + ksi) - np.log1p(ksi)) / W
        if vads[f] < eta:
            mu2 = MU * mu2 + (1.0 - MU) * p
        hw = a * np.exp(0.5 * exp1(np.maximum(a * g, 1e-8)))
        hws[f] = hw
        xk = (mag * hw) ** 2
        prior = bool(np.any(xk == 0))
        frame = np.fft.irfft(hw * X, n_fft)[:W]
        y[f * hop:(f + 1) * hop] = tail + frame[:hop]
        tail = frame[hop:]
    out = np.zeros(L, dtype=np.float32)
    out[:nf * hop] = y
    return out, vads, hws, mu2


def denoise(wav, win, n_fft, noise_mu2, eta=0.15):
    return denoise_loop(wav, win, n_fft, noise_mu2, eta)[0]


def load_preprocess(wav, sampling_rate=16000, rescaling_max=0.9):
    """the reference load_preprocess_wav after loading: rescale, then edge-profile + denoise for clips over 0.4 s"""
    wav = wav / np.abs(wav).max() * rescaling_max
    if len(wav) > sampling_rate * (0.3 + 0.1):
        edge = int(sampling_rate * 0.15)
        noise = np.concatenate([wav[:edge], wav[-edge:]])
        W, _, _, win, n_fft = params(sampling_rate)
        wav = denoise(wav, win, n_fft, profile_mu2(noise, win, n_fft))
    return wav


def speechlike(seed, n, sr=16000):
    """seeded fp32 test clip of n samples: harmonic bursts of a drifting pitch over background noise, peak 0.9"""
    rng = np.random.default_rng(seed)
    t = np.arange(n) / sr
    f0 = rng.uniform(90, 260) * (1 + 0.1 * np.sin(2 * np.pi * rng.uniform(0.2, 1.0) * t))
    phase = 2 * np.pi * np.cumsum(f0) / sr
    voiced = sum(np.sin(h * phase) / h for h in range(1, 6))
    env = np.clip(np.sin(2 * np.pi * rng.uniform(0.5, 2.0) * t + rng.uniform(0, 6)), 0, None) ** 2
    x = 0.3 * voiced * env + rng.uniform(0.005, 0.05) * rng.standard_normal(n)
    x = x.astype(np.float32)
    return x / np.abs(x).max() * np.float32(0.9)
