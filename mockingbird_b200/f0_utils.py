"""F0 for voice conversion on the device (mb_f0_*): a drop-in for the reference's ``utils/f0_utils.py``.

``compute_f0(wav, sr=16000, frame_period=10.0)`` runs Harvest as restated in DESIGN §4n on the GPU and returns a float32
contour of ``1 + int(1000 * len / sr / frame_period)`` frames, 0 where unvoiced.  ``compute_f0_many`` takes a list of clips
of any lengths and runs it in one sequence of launches; every element is bitwise its single call.  The tracker settings are
the reference's (f0_floor = 80, f0_ceil = 600); 16 kHz and 10 ms, what every caller passes, are the only rates supported.

``f02lf0``, ``compute_mean_std``, ``convert_continuos_f0``, ``get_cont_lf0`` and ``get_converted_lf0uv`` work on the host
arrays as the reference's do, with its dtypes, its in-place edit of the argument of ``convert_continuos_f0``, its
all-unvoiced branch and its errors (interpolating from one voiced frame raises ValueError as ``interp1d`` does).
``get_converted_lf0uv_many`` computes the source clips' F0 in one ``compute_f0_many`` call.
"""
from __future__ import annotations

import ctypes as C
import logging

import numpy as np
import torch

from . import _lib

SAMPLE_RATE = 16000
FRAME_PERIOD = 10.0
F0_FLOOR = 80.0
F0_CEIL = 600.0
MAX_SAMPLES = 1 << 28


def _check_rate(sr, frame_period):
    if sr != SAMPLE_RATE or frame_period != FRAME_PERIOD:
        raise ValueError(f"compute_f0 supports sr = {SAMPLE_RATE} and frame_period = {FRAME_PERIOD} only "
                         f"(got sr = {sr}, frame_period = {frame_period})")


def num_frames(n, sr=SAMPLE_RATE, frame_period=FRAME_PERIOD):
    """frames of the contour of an n-sample clip: 1 + int(1000 n / sr / frame_period), as pyworld counts them"""
    return int(1000.0 * n / sr / frame_period) + 1


def _as_clip(w, i):
    w = np.asarray(w)
    if w.dtype not in (np.float32, np.float64):
        raise ValueError(f"wav {i} has dtype {w.dtype}: float32 or float64 waveforms are supported")
    if w.ndim != 1:
        raise ValueError(f"wav {i} must be one-dimensional, got shape {w.shape}")
    if len(w) == 0:
        raise ValueError(f"wav {i} is empty")
    if len(w) > MAX_SAMPLES:
        raise ValueError(f"wav {i} has {len(w)} samples, more than {MAX_SAMPLES}")
    return w.astype(np.float64)


class _Handle:
    def __init__(self, device):
        self._handle = C.c_void_p()
        _lib.check(_lib.lib().mb_f0_create(C.byref(self._handle)))
        self.device = device
        self._arena = _lib.upload_weights("f0", self._handle, {}, device)
        self._workspace = None

    def __del__(self):
        try:
            if getattr(self, "_handle", None) is not None and self._handle.value:
                _lib.lib().mb_f0_destroy(self._handle)
                self._handle = C.c_void_p()
        except Exception:
            pass


_handles: dict = {}


def _handle() -> _Handle:
    dev = _lib.require_cuda()
    h = _handles.get(dev)
    if h is None:
        h = _handles[dev] = _Handle(dev)
    return h


def harvest_many(wavs, debug=None):
    """float64 F0 contours (10 ms frames) of float64 16 kHz clips, in one sequence of launches.  debug: a dict that receives
    per-clip lists of the device's intermediate results ('raw_count', 'official_count', 'refined', 'scores' [T][91],
    'contour'), each per 1 ms frame."""
    clips = [_as_clip(w, i) for i, w in enumerate(wavs)]
    if not clips:
        return []
    h = _handle()
    dev = h.device
    lengths = [len(c) for c in clips]
    L = _lib.lib()
    Tn = (C.c_int32 * len(lengths))(*lengths)
    frames = [int(1000.0 * n / SAMPLE_RATE / 1.0) + 1 for n in lengths]
    outs = [num_frames(n) for n in lengths]
    with torch.cuda.device(dev):
        ws = _lib.workspace(int(L.mb_f0_workspace_bytes(h._handle, len(lengths), Tn)), dev, h, "_workspace")
        x = torch.from_numpy(np.concatenate(clips)).to(dev)
        f0 = torch.empty(sum(outs), dtype=torch.float64, device=dev)
        dbg = None
        if debug is not None:
            F = sum(frames)
            bufs = dict(raw_count=torch.empty(F, dtype=torch.int32, device=dev),
                        official_count=torch.empty(F, dtype=torch.int32, device=dev),
                        refined=torch.empty(F, 91, dtype=torch.float64, device=dev),
                        scores=torch.empty(F, 91, dtype=torch.float64, device=dev),
                        contour=torch.empty(F, dtype=torch.float64, device=dev))
            dbg = _lib.F0Debug(**{k: v.data_ptr() for k, v in bufs.items()})
        stream = torch.cuda.current_stream(dev).cuda_stream
        _lib.check(L.mb_f0_harvest(h._handle, C.c_void_p(x.data_ptr()), Tn, len(lengths), C.c_void_p(f0.data_ptr()),
                                   C.byref(dbg) if dbg is not None else None, C.c_void_p(ws.data_ptr()), ws.numel(),
                                   C.c_void_p(stream)))
        out = f0.cpu().numpy()
        if debug is not None:
            split = np.cumsum(frames)[:-1]
            for k, v in bufs.items():
                debug[k] = np.split(v.cpu().numpy(), split)
    return np.split(out, np.cumsum(outs)[:-1])


def compute_f0_many(wavs, sr=SAMPLE_RATE, frame_period=FRAME_PERIOD):
    """compute_f0 of every clip of `wavs` (a list of 1-D float32 or float64 arrays) in one sequence of launches"""
    _check_rate(sr, frame_period)
    return [f.astype(np.float32) for f in harvest_many(wavs)]


def compute_f0(wav, sr=SAMPLE_RATE, frame_period=FRAME_PERIOD):
    """utils/f0_utils.py compute_f0: Harvest F0 (f0_floor 80, f0_ceil 600) as float32, 0 on unvoiced frames"""
    return compute_f0_many([wav], sr, frame_period)[0]


def compute_mean_std(lf0):
    nonzero = np.nonzero(lf0)
    return np.mean(lf0[nonzero]), np.std(lf0[nonzero])


def f02lf0(f0):
    lf0 = f0.copy()
    nonzero = np.nonzero(f0)
    lf0[nonzero] = np.log(f0[nonzero])
    return lf0


def convert_continuos_f0(f0):
    """(uv, continuous f0): uv float32; f0 is edited in place (its ends are held at the first and last voiced values)"""
    uv = np.float32(f0 != 0)
    if (f0 == 0).all():
        logging.warning("all of the f0 values are 0.")
        return uv, f0
    voiced = f0[f0 != 0]
    start_f0, end_f0 = voiced[0], voiced[-1]
    start_idx = np.where(f0 == start_f0)[0][0]
    end_idx = np.where(f0 == end_f0)[0][-1]
    f0[:start_idx] = start_f0
    f0[end_idx:] = end_f0
    nz = np.where(f0 != 0)[0]
    if len(nz) < 2:
        raise ValueError("x and y arrays must have at least 2 entries")
    # scipy's interp1d(nz, f0[nz]) at every frame: np.interp for float64 values, its own two-weight formula otherwise
    t = np.arange(0, f0.shape[0]).astype(np.float64)
    y = f0[nz]
    if y.dtype == np.float64:
        return uv, np.interp(t, nz, y)
    k = np.clip(np.searchsorted(nz, t), 1, len(nz) - 1)
    x_lo, x_hi = nz[k - 1], nz[k]
    return uv, (t - x_lo) / (x_hi - x_lo) * y[k] + (x_hi - t) / (x_hi - x_lo) * y[k - 1]


def get_cont_lf0(f0, frame_period=10.0, lpf=False):
    if lpf:
        raise NotImplementedError("get_cont_lf0(lpf=True) (the low-pass-filtered contour) is not supported")
    uv, cont_f0 = convert_continuos_f0(f0)
    cont_lf0 = cont_f0.copy()
    cont_lf0[cont_f0 > 0] = np.log(cont_f0[cont_f0 > 0])
    return uv, cont_lf0


def _lf0uv(f0_src, lf0_mean_trg, lf0_std_trg, convert):
    if not convert:
        uv, cont_lf0 = get_cont_lf0(f0_src)
        return np.concatenate([cont_lf0[:, np.newaxis], uv[:, np.newaxis]], axis=1)
    lf0_src = f02lf0(f0_src)
    lf0_mean_src, lf0_std_src = compute_mean_std(lf0_src)
    lf0_vc = lf0_src.copy()
    v = lf0_src > 0.0
    lf0_vc[v] = (lf0_src[v] - lf0_mean_src) / lf0_std_src * lf0_std_trg + lf0_mean_trg
    f0_vc = lf0_vc.copy()
    f0_vc[v] = np.exp(lf0_vc[v])
    uv, cont_lf0_vc = get_cont_lf0(f0_vc)
    return np.concatenate([cont_lf0_vc[:, np.newaxis], uv[:, np.newaxis]], axis=1)


def get_converted_lf0uv(wav, lf0_mean_trg, lf0_std_trg, convert=True):
    """[frames, 2] (continuous log F0, voicing) of the source clip, its log F0 moved to the target's mean and std"""
    return _lf0uv(compute_f0(wav), lf0_mean_trg, lf0_std_trg, convert)


def get_converted_lf0uv_many(wavs, lf0_means, lf0_stds, convert=True):
    """get_converted_lf0uv(wavs[i], lf0_means[i], lf0_stds[i], convert) for every i; the F0 in one compute_f0_many call"""
    if len(lf0_means) != len(wavs) or len(lf0_stds) != len(wavs):
        raise ValueError(f"{len(wavs)} clips with {len(lf0_means)} means and {len(lf0_stds)} stds")
    return [_lf0uv(f, m, s, convert) for f, m, s in zip(compute_f0_many(wavs), lf0_means, lf0_stds)]
