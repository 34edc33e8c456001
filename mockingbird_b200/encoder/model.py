"""``SpeakerEncoder`` on the H100 path (reference: models/encoder/model.py:12-61).

Same constructor ``SpeakerEncoder(device, loss_device)`` and ``forward(utterances[B, n_frames, 40]) ->
embeds[B, 256]``; the 3-layer LSTM, the Linear+ReLU and the L2 normalisation run in the CUDA library
(mb_encoder_*).  Inference only: ``hidden_init`` other than None and the GE2E loss are not on the path.
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, Optional

import torch

from .. import _lib
from .params_data import mel_n_channels
from .params_model import model_embedding_size, model_hidden_size, model_num_layers

MAX_ROWS = 1024  # rows per library call (bounds the workspace: 160 frames -> ~0.9 GB)


class SpeakerEncoder:
    def __init__(self, device=None, loss_device=None):
        cfg = _lib.EncoderConfig()
        cfg.mel_n_channels, cfg.hidden_size = mel_n_channels, model_hidden_size
        cfg.num_layers, cfg.embedding_size = model_num_layers, model_embedding_size
        self._cfg = cfg
        self._handle = C.c_void_p()
        _lib.check(_lib.lib().mb_encoder_create(C.byref(cfg), C.byref(self._handle)))
        self._state: Optional[Dict[str, torch.Tensor]] = None
        self._arena = None
        self._ws = None
        self._device = torch.device(device) if device is not None and torch.device(device).type == "cuda" else None
        self._ready = False
        self.training = True

    def load_state_dict(self, sd, strict: bool = True):
        self._state = {k: v.detach() for k, v in sd.items()}
        self._ready = False
        return self

    def state_dict(self):
        return dict(self._state or {})

    def eval(self):
        self.training = False
        return self

    def to(self, device):
        device = torch.device(device)
        if device.type != "cuda":
            raise _lib.MbError("mockingbird_b200 SpeakerEncoder runs on CUDA only (no CPU fallback)")
        self._device = device
        self._ready = False
        return self

    def _upload(self):
        if self._state is None:
            raise _lib.MbError("SpeakerEncoder has no weights: call load_state_dict first")
        self._device = self._device or _lib.require_cuda()
        self._arena = _lib.upload_weights("encoder", self._handle, self.weights_for_upload(), self._device)
        self._ready = True

    def weights_for_upload(self) -> Dict[str, torch.Tensor]:
        """the LSTM and the Linear; similarity_weight / similarity_bias are loss only (model.py:27-28)"""
        return {k: v for k, v in self._state.items() if k.startswith("lstm.") or k.startswith("linear.")}

    def packed_arena(self) -> torch.Tensor:
        if not self._ready:
            self._upload()
        return self._arena

    def forward(self, utterances, hidden_init=None):
        if hidden_init is not None:
            raise NotImplementedError("hidden_init is not used on the inference path (inference.py:63)")
        if not self._ready:
            self._upload()
        dev = self._device
        L = _lib.lib()
        x = utterances.to(device=dev, dtype=torch.float32).contiguous()
        R, T, Cn = x.shape
        assert Cn == self._cfg.mel_n_channels
        out = torch.empty(R, self._cfg.embedding_size, dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            stream = torch.cuda.current_stream(dev).cuda_stream
            for r0 in range(0, R, MAX_ROWS):
                n = min(MAX_ROWS, R - r0)
                need = int(L.mb_encoder_workspace_bytes(self._handle, n, T)) + 256
                if self._ws is None or self._ws.numel() < need:
                    self._ws = torch.empty(need, dtype=torch.uint8, device=dev)
                _lib.check(L.mb_encoder_embed_frames(self._handle, C.c_void_p(x[r0:r0 + n].data_ptr()), n, T,
                                                     C.c_void_p(out[r0:r0 + n].data_ptr()),
                                                     C.c_void_p(self._ws.data_ptr()), self._ws.numel(), C.c_void_p(stream)))
        return out

    __call__ = forward

    def reduce_partials(self, partial_embeds: torch.Tensor, offsets) -> torch.Tensor:
        """L2(mean of the partial embeddings) per utterance (inference.py:164-166); offsets = CSR [U+1]"""
        dev = self._device
        off = torch.as_tensor(offsets, dtype=torch.int32).to(dev)
        U = off.numel() - 1
        out = torch.empty(U, self._cfg.embedding_size, dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            stream = torch.cuda.current_stream(dev).cuda_stream
            _lib.check(_lib.lib().mb_encoder_reduce_partials(self._handle, C.c_void_p(partial_embeds.data_ptr()),
                                                             C.c_void_p(off.data_ptr()), U, C.c_void_p(out.data_ptr()),
                                                             C.c_void_p(stream)))
        return out

    def __del__(self):
        try:
            if getattr(self, "_handle", None) is not None and self._handle.value:
                _lib.lib().mb_encoder_destroy(self._handle)
                self._handle = C.c_void_p()
        except Exception:
            pass
