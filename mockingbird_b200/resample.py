"""Polyphase resampling and per-clip levelling on the device (mb_resample_*): DESIGN.md section 4k.

``resample_many(wavs, source_srs, target_sr)`` is ``scipy.signal.resample_poly`` (the ratio reduced by its gcd, the default
Kaiser window, zero padding) for a list of clips of any lengths and rates, in one launch: every result is bitwise the host
call on the same float32 samples, whatever it is batched with.  ``resample_device`` returns the same clips as a
``DeviceClips`` (one flat device tensor and the clip lengths), which the levelling steps below, the speaker encoder's
``embed_utterances``, the log-MMSE denoiser and the PPG extractor take without a host round trip.

Input is float32, or int16 PCM, which the device converts as x / 32768 (load_wav's conversion, exact).  Refused with a
ValueError naming the clip, before anything is queued: an empty or non-1-D clip, a non-integer or non-positive rate, and
float64 samples (the host computes those in float64; this path is float32 only) or any other dtype.

``normalize_volume_device`` is ``normalize_volume(wav, target_dBFS, increase_only=True)``: the mean square is summed on
the device in numpy's pairwise order, the gain is computed on the host with numpy's own scalar functions from the B mean
squares (one copy of B values), and the clips are scaled on the device.  ``rescale_device`` is
``wav / np.abs(wav).max() * peak``.  Both level float32 clips in float32 and float64 clips (the text-to-speech chain's
documents, gen_voice.py) in float64, each as numpy does for that dtype; resampling itself takes float32 only."""
from __future__ import annotations

import ctypes as C
import math
import numbers
from pathlib import Path

import numpy as np
import torch

from . import _lib


class DeviceClips:
    """Clips on the device: ``data`` holds clip i's ``lengths[i]`` samples (float32, or float64 for levelling only) after
    those of clips 0 .. i-1.  Indexing and iteration give 1-D views of ``data``; ``numpy()`` copies every clip to the host
    in one transfer."""

    def __init__(self, data: torch.Tensor, lengths, sample_rate: int):
        self.data = data
        self.lengths = [int(n) for n in lengths]
        self.sample_rate = int(sample_rate)
        self.offsets = np.concatenate([[0], np.cumsum(self.lengths, dtype=np.int64)]).tolist()
        if data.dim() != 1 or data.numel() != self.offsets[-1] or data.dtype not in (torch.float32, torch.float64):
            raise ValueError(f"DeviceClips: data must be 1-D float32 or float64 of {self.offsets[-1]} samples")

    def __len__(self):
        return len(self.lengths)

    def __getitem__(self, i):
        return self.data[self.offsets[i]:self.offsets[i + 1]]

    def __iter__(self):
        return (self[i] for i in range(len(self)))

    @property
    def device(self):
        return self.data.device

    def select(self, idx) -> "DeviceClips":
        """the clips idx, in that order, as a new DeviceClips (a device copy)"""
        idx = list(idx)
        data = torch.cat([self[i] for i in idx]) if idx else self.data[:0].clone()
        return DeviceClips(data, [self.lengths[i] for i in idx], self.sample_rate)

    def numpy(self):
        flat = self.data.cpu().numpy()
        return [flat[self.offsets[i]:self.offsets[i + 1]] for i in range(len(self))]


def design_filter(up: int, down: int) -> np.ndarray:
    """resample_poly's filter for a reduced ratio: firwin in float64, cast to float32, then multiplied by up in float32"""
    from scipy.signal import firwin

    max_rate = max(up, down)
    h = np.asarray(firwin(2 * 10 * max_rate + 1, 1.0 / max_rate, window=("kaiser", 5.0)), dtype=np.float32)
    h *= up
    return h


def ratio(source_sr: int, target_sr: int):
    """(up, down) reduced by their gcd, as resample_poly reduces them"""
    g = math.gcd(source_sr, target_sr)
    return target_sr // g, source_sr // g


def output_length(n: int, source_sr: int, target_sr: int) -> int:
    up, down = ratio(source_sr, target_sr)
    return n if up == down else -(-n * up // down)


def check_rate(sr, what) -> int:
    if isinstance(sr, bool) or not isinstance(sr, numbers.Real) or sr != int(sr) or int(sr) <= 0:
        raise ValueError(f"{what}: sample rate {sr!r} is not a positive integer")
    return int(sr)


def check_clip(x, what) -> np.ndarray:
    if torch.is_tensor(x):
        x = x.detach().cpu().numpy()
    x = np.asarray(x)
    if x.dtype == np.float64:
        raise ValueError(f"{what} is float64: the host path computes it in float64 and this path is float32; pass float32")
    if x.dtype not in (np.float32, np.int16):
        raise ValueError(f"{what} has dtype {x.dtype}: float32 samples or int16 PCM are supported")
    if x.ndim != 1:
        raise ValueError(f"{what} must be one-dimensional, got shape {x.shape}")
    if x.size == 0:
        raise ValueError(f"{what} is empty")
    return np.ascontiguousarray(x)


def read_native(path):
    """a WAV file at its own rate -> (int16 samples for mono 16-bit PCM, else load_wav's float32 mono, sample rate)"""
    from scipy.io import wavfile

    from .synthesizer import audio_host

    sr, data = wavfile.read(str(path))
    if data.dtype == np.int16 and data.ndim == 1:
        return data, int(sr)
    return audio_host.load_wav(path, None)


class _Resampler:
    def __init__(self, device, filter_smem_bytes=-1):
        self.device = device
        self._handle = C.c_void_p()
        _lib.check(_lib.lib().mb_resample_create(int(filter_smem_bytes), C.byref(self._handle)))
        self._index = {}
        self._arena = None
        self._ws = None

    def filter_index(self, up, down) -> int:
        """the handle's index of the ratio's filter, designing and uploading it on first use"""
        if up == down:
            return -1
        if (up, down) not in self._index:
            L = _lib.lib()
            h = design_filter(up, down)
            idx = C.c_int32()
            _lib.check(L.mb_resample_add_filter(self._handle, up, down, h.ctypes.data_as(C.c_void_p), h.size, C.byref(idx)))
            nbytes = int(L.mb_resample_arena_bytes(self._handle))
            with torch.cuda.device(self.device):
                self._arena = None
                self._arena = torch.empty(nbytes, dtype=torch.uint8, device=self.device)
                _lib.check(L.mb_resample_set_arena(self._handle, C.c_void_p(self._arena.data_ptr()), nbytes))
                _lib.check(L.mb_resample_finalize(self._handle, C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)))
            self._index[(up, down)] = idx.value
        return self._index[(up, down)]

    def in_smem(self, up, down) -> bool:
        return _lib.lib().mb_resample_filter_in_smem(self._handle, self.filter_index(up, down)) == 1

    def workspace(self, need):
        return _lib.workspace(need, self.device, self)

    def forward(self, clips, rates, target_sr) -> DeviceClips:
        L = _lib.lib()
        B = len(clips)
        pairs = [ratio(sr, target_sr) for sr in rates]
        fidx = [self.filter_index(u, d) for u, d in pairs]
        lengths = [c.size for c in clips]
        out_len = [n if u == d else -(-n * u // d) for n, (u, d) in zip(lengths, pairs)]
        dtype = 1 if all(c.dtype == np.int16 for c in clips) else 0
        if dtype == 0:  # a mixed list is uploaded as float32: int16 / 32768 is exact on the host as on the device
            clips = [c.astype(np.float32) / np.float32(32768.0) if c.dtype == np.int16 else c for c in clips]
        with torch.cuda.device(self.device):
            x = torch.from_numpy(np.concatenate(clips) if B > 1 else clips[0]).to(self.device)
            out = torch.empty(sum(out_len), dtype=torch.float32, device=self.device)
            need = int(L.mb_resample_workspace_bytes(self._handle, B))
            ws = self.workspace(need)
            stream = torch.cuda.current_stream(self.device).cuda_stream
            _lib.check(L.mb_resample_forward(self._handle, C.c_void_p(x.data_ptr()), dtype, (C.c_int32 * B)(*lengths),
                                             (C.c_int32 * B)(*fidx), B, C.c_void_p(out.data_ptr()), C.c_void_p(ws.data_ptr()),
                                             ws.numel(), C.c_void_p(stream)))
        return DeviceClips(out, out_len, target_sr)

    def __del__(self):
        try:
            if getattr(self, "_handle", None) is not None and self._handle.value:
                _lib.lib().mb_resample_destroy(self._handle)
                self._handle = C.c_void_p()
        except Exception:
            pass


_handles: dict = {}


def resampler(device=None, filter_smem_bytes=-1) -> _Resampler:
    """the handle of `device` (default: the current CUDA device); filter_smem_bytes >= 0 gives a separate handle whose
    filters above that size are read through L2 (the default handle stages filters up to 64 KB in shared memory)"""
    dev = torch.device(device) if device is not None else _lib.require_cuda()
    key = (dev, int(filter_smem_bytes))
    if key not in _handles:
        _handles[key] = _Resampler(dev, filter_smem_bytes)
    return _handles[key]


def _rates(source_srs, n):
    if isinstance(source_srs, (list, tuple, np.ndarray)):
        if len(source_srs) != n:
            raise ValueError(f"{len(source_srs)} source rates for {n} clips")
        return [check_rate(sr, f"clip {i}") for i, sr in enumerate(source_srs)]
    return [check_rate(source_srs, f"clip {i}") for i in range(n)]


def resample_device(wavs, source_srs, target_sr, device=None, filter_smem_bytes=-1) -> DeviceClips:
    """resample_poly of every clip from its source rate (one int, or one per clip) to target_sr in one launch, left on the
    device.  A clip already at target_sr is copied (int16: converted)."""
    target_sr = check_rate(target_sr, "target")
    clips = [check_clip(w, f"clip {i}") for i, w in enumerate(wavs)]
    rates = _rates(source_srs, len(clips))
    h = resampler(device, filter_smem_bytes)
    if not clips:
        return DeviceClips(torch.empty(0, dtype=torch.float32, device=h.device), [], target_sr)
    return h.forward(clips, rates, target_sr)


def resample_many(wavs, source_srs, target_sr, device=None, filter_smem_bytes=-1):
    """resample_device copied to the host: a list of float32 arrays, each bitwise resample_poly(x, up, down)"""
    return resample_device(wavs, source_srs, target_sr, device, filter_smem_bytes).numpy()


def _level_ws(clips: DeviceClips):
    B = len(clips)
    need = int(_lib.lib().mb_resample_level_workspace_bytes(B))
    return (C.c_int32 * B)(*clips.lengths), _lib.workspace(need, clips.device)


def _f64(clips: DeviceClips) -> bool:
    return clips.data.dtype == torch.float64


def mean_squares(clips: DeviceClips) -> np.ndarray:
    """np.mean(wav ** 2) of every clip, bitwise: sums of squares in numpy's pairwise order on the device, each divided by
    the length as np.mean does (float32 clips: in float64, rounded once to float32; float64 clips: in float64)"""
    f64 = _f64(clips)
    if len(clips) == 0:
        return np.zeros(0, np.float64 if f64 else np.float32)
    B = len(clips)
    T, ws = _level_ws(clips)
    with torch.cuda.device(clips.device):
        s = torch.empty(B, dtype=clips.data.dtype, device=clips.device)
        stream = torch.cuda.current_stream(clips.device).cuda_stream
        fn = _lib.lib().mb_resample_sumsq_f64 if f64 else _lib.lib().mb_resample_sumsq
        _lib.check(fn(C.c_void_p(clips.data.data_ptr()), T, B, C.c_void_p(s.data_ptr()), C.c_void_p(ws.data_ptr()), ws.numel(),
                      C.c_void_p(stream)))
        s = s.cpu().numpy()
    if f64:
        return np.array([np.float64(v) / n for v, n in zip(s, clips.lengths)], dtype=np.float64)
    return np.array([np.float32(np.float64(v) / n) for v, n in zip(s, clips.lengths)], dtype=np.float32)


def normalize_volume_device(clips: DeviceClips, target_dBFS, increase_only=False, decrease_only=False) -> DeviceClips:
    """normalize_volume (models/encoder/audio.py:108-117) of every clip -> a new DeviceClips, each clip bitwise the host call
    on an array of its dtype: the gain is numpy's scalar arithmetic on the mean square (float32 clips: in float32; float64
    clips: in float64), the scaling one rounded multiply of that dtype"""
    if increase_only and decrease_only:
        raise ValueError("Both increase only and decrease only are set")
    if len(clips) == 0:
        return clips
    f64 = _f64(clips)
    dt = np.float64 if f64 else np.float32
    gains = []
    # a silent clip: -inf dB, as on the host (which warns); float64 zeros then scale by inf, which gives NaN as numpy does
    with np.errstate(divide="ignore", over="ignore", invalid="ignore"):
        for m in mean_squares(clips):
            dBFS_change = target_dBFS - 10 * np.log10(m)
            if (dBFS_change < 0 and increase_only) or (dBFS_change > 0 and decrease_only):
                gains.append(dt(1.0))  # x * 1 is x
            else:
                gains.append(dt(10 ** (dBFS_change / 20)))
    B = len(clips)
    T, ws = _level_ws(clips)
    with torch.cuda.device(clips.device):
        g = torch.from_numpy(np.array(gains, dtype=dt)).to(clips.device)
        y = torch.empty_like(clips.data)
        stream = torch.cuda.current_stream(clips.device).cuda_stream
        fn = _lib.lib().mb_resample_scale_f64 if f64 else _lib.lib().mb_resample_scale
        _lib.check(fn(C.c_void_p(clips.data.data_ptr()), T, B, C.c_void_p(g.data_ptr()), C.c_void_p(y.data_ptr()),
                      C.c_void_p(ws.data_ptr()), ws.numel(), C.c_void_p(stream)))
    return DeviceClips(y, clips.lengths, clips.sample_rate)


def rescale_device(clips: DeviceClips, peak) -> DeviceClips:
    """wav / np.abs(wav).max() * peak of every clip -> a new DeviceClips.  float32 clips: peak rounded to float32 as numpy
    does; float64 clips: in float64, where a NaN sample makes the clip all NaN (np.max propagates it)"""
    if len(clips) == 0:
        return clips
    B = len(clips)
    T, ws = _level_ws(clips)
    with torch.cuda.device(clips.device):
        y = torch.empty_like(clips.data)
        stream = torch.cuda.current_stream(clips.device).cuda_stream
        if _f64(clips):
            fn, p = _lib.lib().mb_resample_rescale_f64, float(peak)
        else:
            fn, p = _lib.lib().mb_resample_rescale, float(np.float32(peak))
        _lib.check(fn(C.c_void_p(clips.data.data_ptr()), T, B, p, C.c_void_p(y.data_ptr()), C.c_void_p(ws.data_ptr()),
                      ws.numel(), C.c_void_p(stream)))
    return DeviceClips(y, clips.lengths, clips.sample_rate)


def load_clips(fpaths_or_wavs, source_srs, default_sr):
    """the clips of a mixed list of paths and arrays with their rates: a path is read at its own rate (read_native, its
    rate wins over source_srs), an array is at source_srs (one int, or one per clip, None entries allowed) or default_sr"""
    items = list(fpaths_or_wavs)
    srs = source_srs if isinstance(source_srs, (list, tuple, np.ndarray)) else [source_srs] * len(items)
    if len(srs) != len(items):
        raise ValueError(f"{len(srs)} source rates for {len(items)} clips")
    clips, rates = [], []
    for i, (x, sr) in enumerate(zip(items, srs)):
        if isinstance(x, (str, Path)):
            w, sr = read_native(x)
        else:
            w = check_clip(x, f"clip {i}")
            if w.dtype != np.float32:  # the host functions take arrays as samples, not as PCM
                raise ValueError(f"clip {i} has dtype {w.dtype}: arrays must hold float32 samples")
            sr = default_sr if sr is None else sr
        clips.append(check_clip(w, f"clip {i}"))
        rates.append(check_rate(sr, f"clip {i}"))
    return clips, rates
