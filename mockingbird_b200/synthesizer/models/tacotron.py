"""``Tacotron`` on the H100 path (reference: models/synthesizer/models/tacotron.py:140-298).

Same constructor arguments and ``generate(x, speaker_embedding, steps=2000, style_idx=0,
min_stop_token=5) -> (mel_outputs, linear, attn_scores)`` surface; ``r`` property backed by the loaded
``decoder.r`` buffer (base.py:16-22).  All layers run in the CUDA library (mb_tacotron_*).

The reference's PreNet dropout is always active (pre_net.py:23,26), so generate() is stochastic.
``dropout_masks=(enc, dec)`` injects keep-masks (uint8/bool, enc [2,B,Tc,256], dec [steps/r,2,B,256]) for
reproducible comparisons; otherwise they are drawn on the device from ``seed``.
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, Optional

import torch
import torch.nn.functional as F

from ... import _lib
from ..hparams import gst_hparams


class Tacotron:
    def __init__(self, embed_dims, num_chars, encoder_dims, decoder_dims, n_mels, fft_bins, postnet_dims, encoder_K,
                 lstm_dims, postnet_K, num_highways, dropout, stop_threshold, speaker_embedding_size):
        if fft_bins != n_mels:
            raise NotImplementedError("post_proj to fft_bins != n_mels is not part of the inference path")
        if abs(dropout - 0.5) > 1e-9:
            raise NotImplementedError("PreNet dropout p must be 0.5 (hparams.tts_dropout)")
        cfg = _lib.TacotronConfig()
        cfg.num_chars, cfg.embed_dims, cfg.encoder_dims, cfg.decoder_dims = num_chars, embed_dims, encoder_dims, decoder_dims
        cfg.n_mels, cfg.postnet_dims, cfg.encoder_K, cfg.lstm_dims = n_mels, postnet_dims, encoder_K, lstm_dims
        cfg.postnet_K, cfg.num_highways, cfg.speaker_embedding_size = postnet_K, num_highways, speaker_embedding_size
        cfg.gst_E, cfg.gst_tokens, cfg.gst_heads, cfg.max_r = gst_hparams.E, gst_hparams.token_num, gst_hparams.num_heads, 20
        self._cfg = cfg
        self.n_mels = n_mels
        self.encoder_dims, self.decoder_dims, self.lstm_dims = encoder_dims, decoder_dims, lstm_dims
        self.speaker_embedding_size = speaker_embedding_size
        self._handle = C.c_void_p()
        _lib.check(_lib.lib().mb_tacotron_create(C.byref(cfg), C.byref(self._handle)))
        self._state: Optional[Dict[str, torch.Tensor]] = None
        self._arena = None
        self._ws = None
        self._device = None
        self._ready = False
        self._r = 1
        self.step = torch.zeros(1, dtype=torch.long)
        self.stop_threshold = torch.tensor(stop_threshold, dtype=torch.float32)
        self.training = True
        self.seed = 0

    # -- Base (base.py) ---------------------------------------------------------------------------
    @property
    def r(self):
        return self._r

    @r.setter
    def r(self, value):
        self._r = int(value)

    def get_step(self):
        return self.step.data.item()

    def load(self, path, device=None, optimizer=None):
        checkpoint = torch.load(str(path), map_location="cpu")
        state = checkpoint["model_state"] if "model_state" in checkpoint else checkpoint["model"]
        self.load_state_dict(state, strict=False)

    def load_state_dict(self, sd, strict: bool = True):
        self._state = {k: v.detach() for k, v in sd.items()}
        if "decoder.r" in self._state:
            self._r = int(self._state["decoder.r"])
        if "step" in self._state:
            self.step = self._state["step"].clone()
        self._ready = False
        return self

    def state_dict(self):
        return dict(self._state or {})

    def eval(self):
        self.training = False
        return self

    def train(self, mode: bool = True):
        self.training = mode
        return self

    def to(self, device):
        device = torch.device(device)
        if device.type != "cuda":
            raise _lib.MbError("mockingbird_b200 Tacotron runs on CUDA only (no CPU fallback)")
        self._device = device
        self._ready = False
        return self

    def cuda(self):
        return self.to(_lib.require_cuda())

    # -- weights -----------------------------------------------------------------------------------
    def _gst_const_enc(self) -> torch.Tensor:
        """ReferenceEncoder(zeros) of tacotron.py:251 (global_style_token.py:56-72): the input is all
        zeros, so the result is a constant of the weights - folded here at load time (torch ops on
        the checkpoint tensors), like weight-norm folding in the GAN loaders."""
        sd = self._state
        out = torch.zeros(1, 1, 1, gst_hparams.n_mels)
        i = 0
        while f"gst.encoder.convs.{i}.weight" in sd:
            out = F.conv2d(out, sd[f"gst.encoder.convs.{i}.weight"].float(), sd[f"gst.encoder.convs.{i}.bias"].float(), 2, 1)
            p = f"gst.encoder.bns.{i}"
            out = F.batch_norm(out, sd[p + ".running_mean"].float(), sd[p + ".running_var"].float(), sd[p + ".weight"].float(),
                               sd[p + ".bias"].float(), False, 0.1, 1e-5)
            out = F.relu(out)
            i += 1
        x = out.transpose(1, 2).contiguous().view(1, -1)
        gi = F.linear(x, sd["gst.encoder.gru.weight_ih_l0"].float(), sd["gst.encoder.gru.bias_ih_l0"].float())
        gh = sd["gst.encoder.gru.bias_hh_l0"].float().unsqueeze(0)  # W_hh @ 0 + b_hh
        i_r, i_z, i_n = gi.chunk(3, 1)
        h_r, h_z, h_n = gh.chunk(3, 1)
        r = torch.sigmoid(h_r + i_r)
        z = torch.sigmoid(h_z + i_z)
        n = torch.tanh(i_n + h_n * r)
        return ((0.0 - n) * z + n).reshape(-1)

    def _upload(self):
        if self._state is None:
            raise _lib.MbError("Tacotron has no weights: call load_state_dict / load first")
        self._device = self._device or _lib.require_cuda()
        self._arena = _lib.upload_weights("tacotron", self._handle, self.weights_for_upload(), self._device)
        self._ready = True

    def weights_for_upload(self) -> Dict[str, torch.Tensor]:
        """the float tensors of the checkpoint without the GST reference encoder, which is folded into gst.const_enc"""
        tensors = {k: v for k, v in self._state.items()
                   if v.dtype.is_floating_point and not k.startswith("gst.encoder.") and k != "stop_threshold"}
        tensors["gst.const_enc"] = self._gst_const_enc()
        return tensors

    def packed_arena(self) -> torch.Tensor:
        if not self._ready:
            self._upload()
        return self._arena

    # -- generate ----------------------------------------------------------------------------------
    def generate(self, x, speaker_embedding, steps=2000, style_idx=0, min_stop_token=5, dropout_masks=None):
        self.eval()
        if not self._ready:
            self._upload()
        dev = self._device
        L = _lib.lib()
        chars = x.to(device=dev, dtype=torch.int32).contiguous()
        spk = speaker_embedding.to(device=dev, dtype=torch.float32).contiguous()
        B, Tc = chars.shape
        r = self._r
        nst = (steps + r - 1) // r
        M = nst * r
        mel = torch.empty(B * self.n_mels * M, dtype=torch.float32, device=dev)
        lin = torch.empty(B * self.n_mels * M, dtype=torch.float32, device=dev)
        attn = torch.empty(B * nst * Tc, dtype=torch.float32, device=dev)
        enc_p = dec_p = None
        if dropout_masks is not None:
            enc_m = dropout_masks[0].to(device=dev, dtype=torch.uint8).contiguous()
            dec_m = dropout_masks[1].to(device=dev, dtype=torch.uint8).contiguous()
            assert enc_m.numel() == 2 * B * Tc * self.encoder_dims and dec_m.numel() >= nst * 2 * B * 2 * self.decoder_dims
            enc_p, dec_p = C.c_void_p(enc_m.data_ptr()), C.c_void_p(dec_m.data_ptr())
        frames = C.c_int32(0)
        with torch.cuda.device(dev):
            need = int(L.mb_tacotron_workspace_bytes(self._handle, B, Tc, steps, r)) + 256
            if self._ws is None or self._ws.numel() < need:
                self._ws = torch.empty(need, dtype=torch.uint8, device=dev)
            stream = torch.cuda.current_stream(dev).cuda_stream
            _lib.check(L.mb_tacotron_generate(self._handle, C.c_void_p(chars.data_ptr()), C.c_void_p(spk.data_ptr()), B, Tc,
                                              int(steps), r, int(style_idx), C.c_float(float(min_stop_token)), enc_p, dec_p,
                                              C.c_uint64(self.seed), C.c_void_p(mel.data_ptr()), C.c_void_p(lin.data_ptr()),
                                              C.c_void_p(attn.data_ptr()), C.byref(frames), C.c_void_p(self._ws.data_ptr()),
                                              self._ws.numel(), C.c_void_p(stream)))
        f = frames.value
        mel = mel[: B * self.n_mels * f].view(B, self.n_mels, f)
        lin = lin[: B * self.n_mels * f].view(B, self.n_mels, f)
        attn = attn[: B * (f // r) * Tc].view(B, f // r, Tc)
        return mel, lin, attn

    def __del__(self):
        try:
            if getattr(self, "_handle", None) is not None and self._handle.value:
                _lib.lib().mb_tacotron_destroy(self._handle)
                self._handle = C.c_void_p()
        except Exception:
            pass
