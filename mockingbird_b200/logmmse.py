"""Log-MMSE denoising on the device (mb_logmmse_*): a drop-in for the reference's ``utils/logmmse.py``.

``profile_noise(noise, sampling_rate, window_size=0)`` and ``denoise(wav, noise_profile, eta=0.15)`` have the reference's
signatures and results: a ``NoiseProfile`` with the same fields (host numpy arrays), and the denoised waveform as a float32
numpy array of the input's length.  ``profile_noise_many`` and ``denoise_many`` take lists of clips of any lengths and run
each list in one sequence of launches; every element equals its single call.

Input is float32, what every caller in the reference passes.  float64 is refused with ValueError, as the reference's
``denoise`` fails on it, and so are the integer formats, which no caller uses.  A clip shorter than two hops (320 samples
at 16 kHz) is refused with ValueError as in the reference; a noise signal shorter than one window, on which the reference
returns NaN, is refused too.  One device handle (FFT twiddles and a workspace that grows to the largest call) is kept per
window size."""
from __future__ import annotations

import ctypes as C
import math
from collections import namedtuple

import numpy as np
import torch

from . import _lib

NoiseProfile = namedtuple("NoiseProfile", "sampling_rate window_size len1 len2 win n_fft noise_mu2")


def _check_float32(x, what):
    x = np.asarray(x)
    if x.dtype == np.float64:
        raise ValueError(f"{what} is float64: utils/logmmse.denoise fails on float64 input; pass float32")
    if x.dtype != np.float32:
        raise ValueError(f"{what} has dtype {x.dtype}: only float32 waveforms are supported")
    if x.ndim != 1:
        raise ValueError(f"{what} must be one-dimensional, got shape {x.shape}")
    return x


def _params(sampling_rate, window_size):
    W = int(window_size) if window_size else int(math.floor(0.02 * sampling_rate))
    if W % 2 == 1:
        W += 1
    len1 = int(math.floor(W * 50 / 100))
    len2 = int(W - len1)
    win = np.hanning(W)
    win = win * len2 / np.sum(win)
    return W, len1, len2, win, 2 * W


class _Handle:
    def __init__(self, W, len1, len2, n_fft, device):
        cfg = _lib.LogMmseConfig()
        cfg.window_size, cfg.len1, cfg.len2, cfg.n_fft = W, len1, len2, n_fft
        self.W, self.len1, self.len2, self.n_fft = W, len1, len2, n_fft
        self._handle = C.c_void_p()
        _lib.check(_lib.lib().mb_logmmse_create(C.byref(cfg), C.byref(self._handle)))
        self.device = device
        self._arena = _lib.upload_weights("logmmse", self._handle, {}, device)
        self._workspace = None

    def workspace(self, lengths):
        L = _lib.lib()
        T = (C.c_int32 * len(lengths))(*lengths)
        need = int(L.mb_logmmse_workspace_bytes(self._handle, len(lengths), T))
        return T, _lib.workspace(need, self.device, self, "_workspace")

    def __del__(self):
        try:
            if getattr(self, "_handle", None) is not None and self._handle.value:
                _lib.lib().mb_logmmse_destroy(self._handle)
                self._handle = C.c_void_p()
        except Exception:
            pass


_handles: dict = {}


def _handle(W, len1, len2, n_fft) -> _Handle:
    key = (W, len1, len2, n_fft)
    h = _handles.get(key)
    if h is None:
        h = _handles[key] = _Handle(W, len1, len2, n_fft, _lib.require_cuda())
    return h


def _flat(clips, dev):
    if _resident(clips):
        return clips.data.to(dev)
    return torch.from_numpy(np.concatenate(clips) if len(clips) > 1 else clips[0]).to(dev)


def _resident(clips):
    from .resample import DeviceClips

    return isinstance(clips, DeviceClips)


def _lengths(clips):
    return list(clips.lengths) if _resident(clips) else [len(c) for c in clips]


def profile_noise_many(noises, sampling_rate, window_size=0):
    """profile_noise for every signal of `noises` in one launch -> list of NoiseProfile.  `noises` may be a
    resample.DeviceClips, read where it lies."""
    if not _resident(noises):
        noises = [_check_float32(n, f"noise {i}") for i, n in enumerate(noises)]
    W, len1, len2, win, n_fft = _params(sampling_rate, window_size)
    for i, n in enumerate(_lengths(noises)):
        if n < W:
            raise ValueError(f"noise {i} has {n} samples, fewer than one window of {W}")
    if not len(noises):
        return []
    h = _handle(W, len1, len2, n_fft)
    dev = h.device
    lengths = _lengths(noises)
    with torch.cuda.device(dev):
        T, ws = h.workspace(lengths)
        x = _flat(noises, dev)
        w = torch.from_numpy(win).to(dev)
        mu2 = torch.empty(len(noises), n_fft, dtype=torch.float64, device=dev)
        stream = torch.cuda.current_stream(dev).cuda_stream
        _lib.check(_lib.lib().mb_logmmse_profile(h._handle, C.c_void_p(x.data_ptr()), T, len(noises), C.c_void_p(w.data_ptr()),
                                                 C.c_void_p(mu2.data_ptr()), C.c_void_p(ws.data_ptr()), ws.numel(),
                                                 C.c_void_p(stream)))
        mu2 = mu2.cpu().numpy()
    return [NoiseProfile(sampling_rate, W, len1, len2, win, n_fft, m) for m in mu2]


def profile_noise(noise, sampling_rate, window_size=0) -> NoiseProfile:
    """utils/logmmse.py profile_noise: the noise estimate of a waveform that holds noise only"""
    return profile_noise_many([noise], sampling_rate, window_size)[0]


def denoise_many(wavs, noise_profiles, eta=0.15, vad_out=None):
    """denoise(wavs[i], noise_profiles[i], eta) for every i in one sequence of launches -> list of float32 arrays.  The
    profiles must share one window.  vad_out: a list that receives each clip's per-frame VAD statistics (float64).  `wavs`
    may be a resample.DeviceClips, read where it lies."""
    if not _resident(wavs):
        wavs = [_check_float32(w, f"wav {i}") for i, w in enumerate(wavs)]
    if len(noise_profiles) != len(wavs):
        raise ValueError(f"{len(noise_profiles)} noise profiles for {len(wavs)} waveforms")
    if not len(wavs):
        return []
    p0 = noise_profiles[0]
    for i, p in enumerate(noise_profiles):
        if (p.window_size, p.len1, p.len2, p.n_fft) != (p0.window_size, p0.len1, p0.len2, p0.n_fft) or \
                not np.array_equal(p.win, p0.win):
            raise ValueError(f"noise profile {i} has another window than profile 0: one call takes one window")
        if np.shape(p.noise_mu2) != (p0.n_fft,):
            raise ValueError(f"noise profile {i}: noise_mu2 must have n_fft = {p0.n_fft} entries, got {np.shape(p.noise_mu2)}")
    for i, n in enumerate(_lengths(wavs)):
        if n < 2 * p0.len2:
            raise ValueError(f"wav {i} has {n} samples; utils/logmmse.denoise needs at least 2 * len2 = {2 * p0.len2}")
    h = _handle(p0.window_size, p0.len1, p0.len2, p0.n_fft)
    dev = h.device
    lengths = _lengths(wavs)
    with torch.cuda.device(dev):
        T, ws = h.workspace(lengths)
        x = _flat(wavs, dev)
        win = torch.from_numpy(np.asarray(p0.win, dtype=np.float64)).to(dev)
        mu2 = torch.from_numpy(np.stack([np.asarray(p.noise_mu2, dtype=np.float64) for p in noise_profiles])).to(dev)
        out = torch.empty(sum(lengths), dtype=torch.float32, device=dev)
        frames = [n // p0.len2 - p0.window_size // p0.len2 for n in lengths]
        vad = torch.empty(max(1, sum(frames)), dtype=torch.float64, device=dev) if vad_out is not None else None
        stream = torch.cuda.current_stream(dev).cuda_stream
        _lib.check(_lib.lib().mb_logmmse_denoise(h._handle, C.c_void_p(x.data_ptr()), T, len(wavs), C.c_void_p(win.data_ptr()),
                                                 C.c_void_p(mu2.data_ptr()), float(eta), C.c_void_p(out.data_ptr()),
                                                 C.c_void_p(vad.data_ptr()) if vad is not None else None,
                                                 C.c_void_p(ws.data_ptr()), ws.numel(), C.c_void_p(stream)))
        out = out.cpu().numpy()
        if vad is not None:
            v = vad.cpu().numpy()
            vad_out.extend(np.split(v[:sum(frames)], np.cumsum(frames)[:-1]))
    return np.split(out, np.cumsum(lengths)[:-1])


def denoise(wav, noise_profile: NoiseProfile, eta=0.15):
    """utils/logmmse.py denoise: the clean waveform, float32, of the input's length"""
    return denoise_many([wav], [noise_profile], eta)[0]
