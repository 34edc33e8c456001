"""DeepMind-style dual-softmax ``WaveRNN`` on the H100 path (reference: models/vocoder/wavernn/models/deepmind_version.py).

Same constructor and ``generate(seq_len) -> (output, coarse, fine)`` surface (``output = coarse * 256 + fine - 2**15``,
wavernn/audio.py:34-35).  The whole sample loop - R h, the coarse and the dependent fine gate / MLP / 256-way draw - runs in one
persistent cooperative kernel (csrc/deepmind.cu).  Sampling noise as in fatchord_version: ``rng="torch"`` (default) continues
the global torch CPU generator's MT19937 stream in the library (csrc/mt_stream.cu: per sample 256 coarse draws, then 256
fine draws, the order ``Categorical.sample()`` consumes them), so under ``torch.manual_seed`` the integer coarse / fine samples
equal the reference's CPU run; ``rng="device"`` uses the built-in counter-based generator.
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, Optional

import numpy as np
import torch

from .... import _lib
from .fatchord_version import set_torch_cpu_generator_position, torch_cpu_generator_position

CHUNK = 2000  # samples per kernel launch


def combine_signal(coarse, fine):
    """wavernn/audio.py:34-35"""
    return coarse * 256 + fine - 2 ** 15


class WaveRNN:
    def __init__(self, hidden_size=896, quantisation=256):
        self.hidden_size = hidden_size
        self.split_size = hidden_size // 2
        self.quantisation = quantisation
        self._handle = C.c_void_p()
        _lib.check(_lib.lib().mb_deepmind_create(hidden_size, quantisation, C.byref(self._handle)))
        self._state: Optional[Dict[str, torch.Tensor]] = None
        self._arena = None
        self._ws = None
        self._mt = None
        self._device = None
        self._ready = False
        self.rng = "torch"
        self.seed = 0

    def load_state_dict(self, sd, strict: bool = True):
        self._state = {k: v.detach() for k, v in sd.items()}
        self._ready = False
        return self

    def state_dict(self):
        return dict(self._state or {})

    def eval(self):
        return self

    def cuda(self):
        self._device = _lib.require_cuda()
        self._ready = False
        return self

    def to(self, device):
        device = torch.device(device)
        if device.type != "cuda":
            raise _lib.MbError("mockingbird_b200 WaveRNN runs on CUDA only (no CPU fallback)")
        self._device = device
        self._ready = False
        return self

    def _upload(self):
        if self._state is None:
            raise _lib.MbError("WaveRNN has no weights: call load_state_dict first")
        dev = self._device = self._device or _lib.require_cuda()
        self._arena = _lib.upload_weights("deepmind", self._handle, self.weights_for_upload(), dev)
        self._ws = torch.empty(int(_lib.lib().mb_deepmind_workspace_bytes(self._handle)) + 256, dtype=torch.uint8, device=dev)
        self._ready = True

    def weights_for_upload(self) -> Dict[str, torch.Tensor]:
        """every tensor of the checkpoint"""
        return dict(self._state)

    def generate(self, seq_len: int, noise: Optional[torch.Tensor] = None):
        """-> (output int64 [seq_len], coarse int64 [seq_len], fine int64 [seq_len]) numpy, like the reference (:75-162).
        ``noise`` (tests): Exp(1) draws [seq_len, 2, 256] used instead of the generator."""
        if not self._ready:
            self._upload()
        if self.rng not in ("torch", "device"):
            raise ValueError(f"rng must be 'torch' or 'device', got {self.rng!r}")
        L = _lib.lib()
        dev = self._device
        if seq_len <= 0:
            z = np.zeros(0, np.int64)
            return z, z, z
        per_step = 2 * self.quantisation
        use_mt = noise is None and self.rng == "torch"
        with torch.cuda.device(dev):
            stream = torch.cuda.current_stream(dev)
            coarse = torch.empty(seq_len, dtype=torch.int16, device=dev)
            fine = torch.empty(seq_len, dtype=torch.int16, device=dev)
            dbufs = [torch.empty(CHUNK * per_step, dtype=torch.float32, device=dev) for _ in range(2)] if (use_mt or noise is not None) else None
            raw = [torch.empty(CHUNK * per_step * 2, dtype=torch.int32, device=dev) for _ in range(2)] if use_mt else None
            if use_mt:
                if self._mt is None:
                    self._mt = C.c_void_p()
                    _lib.check(L.mb_mtstream_create(CHUNK * per_step * 2, 3, C.byref(self._mt)))
                g_state, g_left, g_next = torch_cpu_generator_position()
                _lib.check(L.mb_mtstream_begin(self._mt, g_state.ctypes.data, g_left, g_next, seq_len * per_step * 2, CHUNK * per_step * 2))
            step0, ci = 0, 0
            try:
                while step0 < seq_len:
                    n = min(CHUNK, seq_len - step0)
                    slot = ci & 1
                    nptr = None
                    if noise is not None:
                        dbufs[slot][: n * per_step].copy_(noise[step0:step0 + n].reshape(-1).to(torch.float32), non_blocking=True)
                        nptr = C.c_void_p(dbufs[slot].data_ptr())
                    elif use_mt:
                        _lib.check(L.mb_mtstream_next(self._mt, n * per_step, C.c_void_p(raw[slot].data_ptr()),
                                                      C.c_void_p(dbufs[slot].data_ptr()), C.c_void_p(stream.cuda_stream)))
                        nptr = C.c_void_p(dbufs[slot].data_ptr())
                    _lib.check(L.mb_deepmind_generate(self._handle, seq_len, step0, n, nptr, C.c_uint64(self.seed),
                                                      C.c_void_p(coarse.data_ptr()), C.c_void_p(fine.data_ptr()),
                                                      C.c_void_p(self._ws.data_ptr()), self._ws.numel(), C.c_void_p(stream.cuda_stream)))
                    if use_mt:
                        _lib.check(L.mb_mtstream_consumed(self._mt, C.c_void_p(stream.cuda_stream)))
                    step0 += n
                    ci += 1
            finally:
                if use_mt:
                    left_c, next_c = C.c_int32(), C.c_int32()
                    _lib.check(L.mb_mtstream_finish(self._mt, g_state.ctypes.data, C.byref(left_c), C.byref(next_c)))
                    set_torch_cpu_generator_position(g_state, left_c.value, next_c.value)
            c = coarse.cpu().numpy().astype(np.int64)
            f = fine.cpu().numpy().astype(np.int64)
        return combine_signal(c, f), c, f

    def __del__(self):
        try:
            if getattr(self, "_mt", None) is not None and self._mt.value:
                _lib.lib().mb_mtstream_destroy(self._mt)
                self._mt = None
            if getattr(self, "_handle", None) is not None and self._handle.value:
                _lib.lib().mb_deepmind_destroy(self._handle)
                self._handle = C.c_void_p()
        except Exception:
            pass
