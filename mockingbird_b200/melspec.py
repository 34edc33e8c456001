"""Host wrapper of the mel-spectrogram front-end kernels (mb_melspec_*): one object per parameter set."""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from . import _lib


def as_wavs(wavs):
    """a list of waveforms as contiguous 1-D float32 host arrays; ValueError naming the first one that is not 1-D"""
    out = []
    for i, w in enumerate(wavs):
        a = np.ascontiguousarray(w.detach().cpu().numpy() if torch.is_tensor(w) else w, dtype=np.float32)
        if a.ndim != 1:
            raise ValueError(f"wav {i} has shape {a.shape}; a 1-D waveform is expected")
        out.append(a)
    return out


def min_signal_length(n_fft, pad_mode) -> int:
    """the shortest signal the centred framing takes: more than n_fft / 2 samples with reflect padding, else 1"""
    return int(n_fft) // 2 + 1 if pad_mode == "reflect" else 1


def check_wavs(wavs, min_signal, signal_lengths=None):
    """refuse, before anything is queued, an empty waveform or one whose signal is shorter than `min_signal` samples
    (reflect padding); the message names the utterance"""
    for i, w in enumerate(wavs):
        n = len(w)
        s = n if signal_lengths is None else int(signal_lengths[i])
        if n == 0:
            raise ValueError(f"wav {i} is empty")
        if s < n:
            raise ValueError(f"wav {i}: signal length {s} is shorter than its {n} samples")
        if s < min_signal:
            raise ValueError(f"wav {i} has {s} samples; reflect padding needs at least {min_signal}")


class MelSpectrogram:
    def __init__(self, sample_rate, n_fft, hop_length, win_length, n_mels, fmin, fmax, pad_mode="reflect", preemphasis=0.0,
                 power=2, to_db=False, min_level_db=-100.0, ref_level_db=20.0, normalize=False, max_abs_value=4.0,
                 symmetric=True, transpose_out=False, device=None):
        cfg = _lib.MelSpecConfig()
        cfg.sample_rate, cfg.n_fft, cfg.hop_length, cfg.win_length, cfg.n_mels = sample_rate, n_fft, hop_length, win_length, n_mels
        cfg.fmin, cfg.fmax = float(fmin), float(fmax)
        cfg.pad_mode = {"reflect": 0, "constant": 1}[pad_mode]
        cfg.preemphasis, cfg.power, cfg.to_db = float(preemphasis), int(power), int(bool(to_db))
        cfg.min_level_db, cfg.ref_level_db = float(min_level_db), float(ref_level_db)
        cfg.normalize, cfg.max_abs_value, cfg.symmetric = int(bool(normalize)), float(max_abs_value), int(bool(symmetric))
        cfg.transpose_out = int(bool(transpose_out))
        self._cfg = cfg
        self.n_mels, self.transpose_out = n_mels, bool(transpose_out)
        self._handle = C.c_void_p()
        L = _lib.lib()
        _lib.check(L.mb_melspec_create(C.byref(cfg), C.byref(self._handle)))
        self._device = torch.device(device) if device is not None else _lib.require_cuda()
        nbytes = int(L.mb_melspec_arena_bytes(self._handle))
        with torch.cuda.device(self._device):
            self._arena = torch.empty(nbytes, dtype=torch.uint8, device=self._device)
            stream = torch.cuda.current_stream(self._device).cuda_stream
            _lib.check(L.mb_melspec_set_arena(self._handle, C.c_void_p(self._arena.data_ptr()), nbytes, C.c_void_p(stream)))

    def __call__(self, wav) -> torch.Tensor:
        """wav: 1-D float array / tensor (host or device) -> device tensor [frames, n_mels] or [n_mels, frames]"""
        L = _lib.lib()
        x = torch.as_tensor(np.asarray(wav, dtype=np.float32) if not torch.is_tensor(wav) else wav, dtype=torch.float32)
        x = x.to(self._device).contiguous()
        n = int(x.numel())
        frames = int(L.mb_melspec_num_frames(self._handle, n))
        shape = (frames, self.n_mels) if self.transpose_out else (self.n_mels, frames)
        out = torch.empty(shape, dtype=torch.float32, device=self._device)
        with torch.cuda.device(self._device):
            stream = torch.cuda.current_stream(self._device).cuda_stream
            _lib.check(L.mb_melspec_forward(self._handle, C.c_void_p(x.data_ptr()), n, C.c_void_p(out.data_ptr()),
                                            C.c_void_p(stream)))
        return out

    def num_frames(self, n_samples: int) -> int:
        return 1 + int(n_samples) // int(self._cfg.hop_length)  # mb_melspec_num_frames (librosa center=True)

    def many_flat(self, wavs, signal_lengths=None):
        """The mels of many utterances in one launch (mb_melspec_forward_ragged).  wavs: 1-D float32 host arrays (the public
        wrappers run ``check_wavs`` on them first; the library refuses a bad one before its launch as well);
        signal_lengths[i] >= len(wavs[i]) frames utterance i as if zeros were appended to that length.
        Returns (device tensor holding utterance i's frames after those of 0 .. i-1, in the handle's layout, list of frame
        counts)."""
        with torch.cuda.device(self._device):
            x = torch.from_numpy(np.concatenate(wavs)).to(self._device)
        return self.many_flat_device(x, [len(w) for w in wavs], signal_lengths)

    def many_flat_device(self, x, lengths, signal_lengths=None):
        """``many_flat`` of utterances already on the device: x holds utterance i's lengths[i] float32 samples after those
        of 0 .. i-1 (a ``resample.DeviceClips``' data, for instance); moved to the handle's device if elsewhere"""
        sig = [int(n) for n in lengths] if signal_lengths is None else [int(n) for n in signal_lengths]
        L = _lib.lib()
        counts = [self.num_frames(n) for n in sig]
        B = len(lengths)
        if x.dtype != torch.float32 or x.dim() != 1 or x.numel() != sum(int(n) for n in lengths):
            raise ValueError(f"x must be 1-D float32 holding the {B} utterances back to back")
        lens = (C.c_int32 * B)(*[int(n) for n in lengths])
        sigs = (C.c_int32 * B)(*sig)
        with torch.cuda.device(self._device):
            x = x.to(self._device).contiguous()
            out = torch.empty(sum(counts) * self.n_mels, dtype=torch.float32, device=self._device)
            need = int(L.mb_melspec_ragged_workspace_bytes(self._handle, B))
            ws = _lib.workspace(need, self._device)
            stream = torch.cuda.current_stream(self._device).cuda_stream
            _lib.check(L.mb_melspec_forward_ragged(self._handle, C.c_void_p(x.data_ptr()), lens, sigs, B,
                                                   C.c_void_p(out.data_ptr()), C.c_void_p(ws.data_ptr()), ws.numel(),
                                                   C.c_void_p(stream)))
        return out, counts

    def many(self, wavs, signal_lengths=None):
        """``many_flat`` copied to the host and split: a list of float32 arrays [frames, n_mels] or [n_mels, frames]"""
        if len(wavs) == 0:
            return []
        out, counts = self.many_flat(wavs, signal_lengths)
        flat = out.cpu().numpy()
        res, o = [], 0
        for n in counts:
            blk = flat[o:o + n * self.n_mels]
            res.append(blk.reshape((n, self.n_mels) if self.transpose_out else (self.n_mels, n)))
            o += n * self.n_mels
        return res

    def __del__(self):
        try:
            if getattr(self, "_handle", None) is not None and self._handle.value:
                _lib.lib().mb_melspec_destroy(self._handle)
                self._handle = C.c_void_p()
        except Exception:
            pass
