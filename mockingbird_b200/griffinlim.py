"""Host wrapper of the Griffin-Lim kernels (mb_griffinlim_*): one object per parameter set and pseudo-inverse mel basis.

``GriffinLim(inv_mel_basis, n_fft, hop_length, win_length, ...)(mels, n_iters, uniforms=None, seeds=None)`` inverts a list
of normalised dB mel spectrograms [n_mels, T_b] in one sequence of launches and returns one fp32 device tensor of
hop * (T_b - 1) samples per utterance.  The initial phases come from ``uniforms`` (float64 [n_fft // 2 + 1, T_b] per
utterance, what ``np.random.rand(*S.shape)`` gives) or from ``seeds`` (one integer per utterance, drawn on the device).
The handle owns its arena (the pseudo-inverse, the window and the FFT twiddles) and a workspace that grows to the largest
batch seen."""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from . import _lib

PAD_MODES = {"reflect": 0, "constant": 1}


class GriffinLim:
    def __init__(self, inv_mel_basis, n_fft, hop_length, win_length, pad_mode="reflect", power=1.5, preemphasis=0.0,
                 signal_normalization=True, allow_clipping=True, symmetric=True, max_abs_value=4.0, min_level_db=-100.0,
                 ref_level_db=20.0, device=None):
        if pad_mode not in PAD_MODES:
            raise ValueError(f"pad_mode {pad_mode!r} is not one of {sorted(PAD_MODES)}")
        basis = torch.as_tensor(np.asarray(inv_mel_basis, dtype=np.float32))
        if basis.dim() != 2:
            raise ValueError(f"inv_mel_basis must be [n_fft // 2 + 1, n_mels], got {tuple(basis.shape)}")
        cfg = _lib.GriffinLimConfig()
        cfg.n_fft, cfg.hop_length, cfg.win_length, cfg.n_mels = n_fft, hop_length, win_length, basis.shape[1]
        cfg.pad_mode, cfg.power, cfg.preemphasis = PAD_MODES[pad_mode], float(power), float(preemphasis)
        cfg.signal_normalization, cfg.allow_clipping = int(bool(signal_normalization)), int(bool(allow_clipping))
        cfg.symmetric, cfg.max_abs_value = int(bool(symmetric)), float(max_abs_value)
        cfg.min_level_db, cfg.ref_level_db = float(min_level_db), float(ref_level_db)
        self._cfg = cfg
        self.n_fft, self.hop_length, self.n_mels, self.n_bins = n_fft, hop_length, int(basis.shape[1]), n_fft // 2 + 1
        self._basis = basis
        self._handle = C.c_void_p()
        _lib.check(_lib.lib().mb_griffinlim_create(C.byref(cfg), C.byref(self._handle)))
        self._device = torch.device(device) if device is not None else None
        self._arena = None
        self._workspace = None

    def workspace_bytes(self, frames) -> int:
        T = (C.c_int32 * len(frames))(*[int(t) for t in frames])
        return int(_lib.lib().mb_griffinlim_workspace_bytes(self._handle, len(frames), T))

    def _upload(self):
        if self._device is None:
            self._device = _lib.require_cuda()
        self._arena = _lib.upload_weights("griffinlim", self._handle, {"inv_mel_basis": self._basis}, self._device)

    def __call__(self, mels, n_iters, uniforms=None, seeds=None):
        """mels: list of [n_mels, T_b] arrays / tensors -> list of fp32 device tensors [hop * (T_b - 1)]"""
        if (uniforms is None) == (seeds is None):
            raise ValueError("pass exactly one of uniforms and seeds")
        if self._arena is None:
            self._upload()
        dev = self._device
        mels = [m if torch.is_tensor(m) else torch.from_numpy(np.asarray(m)) for m in mels]
        for i, m in enumerate(mels):
            if m.dim() != 2 or m.shape[0] != self.n_mels:
                raise ValueError(f"mel {i} must be [{self.n_mels}, T], got {tuple(m.shape)}")
        frames = [int(m.shape[1]) for m in mels]
        B = len(frames)
        flat = torch.cat([m.to(dev, torch.float32).reshape(-1) for m in mels])
        u_dev = None
        if uniforms is not None:
            if len(uniforms) != B:
                raise ValueError(f"{len(uniforms)} uniform blocks for {B} mels")
            for i, (u, t) in enumerate(zip(uniforms, frames)):
                if tuple(np.shape(u)) != (self.n_bins, t):
                    raise ValueError(f"uniforms {i} must be [{self.n_bins}, {t}], got {tuple(np.shape(u))}")
            u_dev = torch.from_numpy(np.concatenate([np.asarray(u, dtype=np.float64).reshape(-1) for u in uniforms])).to(dev)
        elif len(seeds) != B:
            raise ValueError(f"{len(seeds)} seeds for {B} mels")
        return self.forward_device(flat, frames, n_iters, u_dev, seeds)

    def forward_device(self, flat_mels, frames, n_iters, uniforms=None, seeds=None):
        """the launch sequence alone, on tensors already on the device: flat_mels fp32 (the [n_mels, T_b] blocks back to
        back), uniforms float64 (the [n_bins, T_b] blocks back to back) or seeds -> list of fp32 device tensors"""
        if self._arena is None:
            self._upload()
        dev = self._device
        B = len(frames)
        T = (C.c_int32 * B)(*frames)
        seeds_host = None if seeds is None else (C.c_uint64 * B)(*[int(s) & 0xFFFFFFFFFFFFFFFF for s in seeds])
        u_dev = uniforms
        flat = flat_mels
        lengths = [self.hop_length * (t - 1) for t in frames]
        L = _lib.lib()
        need = int(L.mb_griffinlim_workspace_bytes(self._handle, B, T))
        with torch.cuda.device(dev):
            _lib.workspace(need, dev, self, "_workspace")
            out = torch.empty(max(sum(lengths), 1), dtype=torch.float32, device=dev)
            stream = torch.cuda.current_stream(dev).cuda_stream
            _lib.check(L.mb_griffinlim_forward(self._handle, C.c_void_p(flat.data_ptr()), T, B,
                                               C.c_void_p(u_dev.data_ptr()) if u_dev is not None else None, seeds_host,
                                               int(n_iters), C.c_void_p(out.data_ptr()), C.c_void_p(self._workspace.data_ptr()),
                                               self._workspace.numel(), C.c_void_p(stream)))
        return list(torch.split(out[:sum(lengths)], lengths))

    def __del__(self):
        try:
            if getattr(self, "_handle", None) is not None and self._handle.value:
                _lib.lib().mb_griffinlim_destroy(self._handle)
                self._handle = C.c_void_p()
        except Exception:
            pass
