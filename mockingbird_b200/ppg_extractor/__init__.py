"""The voice-conversion PPG extractor on the H100 path (reference: models/ppg_extractor/__init__.py).

Same surface as the reference module: ``build_model(args)``, ``load_model(model_file, device=None)`` (which sets the
module globals ``_model`` / ``_device``), ``PPGModel.forward(speech [B, L], speech_lengths [B]) -> [B, T, D]``,
``extract_from_wav(src_wav)``, ``load_state_dict`` / ``eval`` / ``to`` / ``cuda``.  Every layer runs in the CUDA
library (mb_ppgx_*); there is no CPU fallback.

Divergence from the reference's padded batch: the reference normalises and convolves a padded B > 1 batch across the
padding (after MVN the padded frames hold -mean / var^(1/4), which both Conv2d layers and the depthwise conv read), so
a row's output depends on the longest row.  Here every row is computed as its own B = 1 call, bitwise, which is what
``extract_from_wav`` (B = 1) computes in the reference.  ``extract_batch`` runs many utterances that way.

Positional table: the reference's PositionalEncoding is built with 5000 rows and only rebuilt when a longer input
arrives, so a relative position depends on the module instance's longest input so far.  ``PPGModel`` keeps that
high-water mark (``pe_len``) and builds the table with torch's own sin / cos for the library.

melmat (``frontend.logmel.melmat``) is an input weight: ``librosa.filters.mel(norm=1)`` meant area normalisation before
librosa 0.8 and per-filter L1 normalisation since, and the reference pins no version.  ``build_model`` fills it with the
current (L1) meaning; a ``melmat`` in a loaded state dict wins.
"""
from __future__ import annotations

import argparse
import ctypes as C
from pathlib import Path
from typing import Dict, List, Optional, Sequence

import numpy as np
import torch

from .. import _lib
from ..synthesizer.audio_host import ppg_melmat

MAX_ROWS = 128           # rows per library call
# rows x padded frames per extract_batch call.  The workspace is ~92 KB per padded frame at the stand-in config (D = 144,
# 80 mels: the conv.0 hi / lo planes 2 x 80 x 144 x 2 B plus embed.out.0's hi / lo operand tiles 2 x 11 520 x 2 B), so
# 8192 frames bound it at ~0.75 GB.  The model keeps the workspace for reuse; ``release_workspace()`` frees it.
MAX_BATCH_FRAMES = 8192
PE_MAX_LEN = 5000

# DefaultFrontend's own defaults (models/ppg_extractor/frontend.py:17-35; ``fs`` has none), and what the kernels implement
# of the options it accepts
_FRONTEND_DEFAULTS = dict(n_fft=1024, win_length=800, hop_length=160, center=True, pad_mode="reflect", normalized=False,
                          onesided=True, n_mels=80, fmin=None, fmax=None, htk=False, norm=1, frontend_conf=None,
                          kaldi_padding_mode=False, downsample_rate=1)
_FRONTEND_FIXED = dict(center=True, pad_mode="reflect", normalized=False, onesided=True, htk=False, frontend_conf=None)
_NORMALIZE_DEFAULTS = dict(norm_means=True, norm_vars=False, eps=1.0e-20)
_ENCODER_KEYS = {"attention_dim", "attention_heads", "linear_units", "num_blocks", "dropout_rate", "positional_dropout_rate",
                 "attention_dropout_rate", "input_layer", "normalize_before", "concat_after", "positionwise_layer_type",
                 "positionwise_conv_kernel_size", "macaron_style", "pos_enc_layer_type", "selfattention_layer_type",
                 "activation_type", "use_cnn_module", "cnn_module_kernel", "padding_idx", "no_subsample", "subsample_by_2"}
ENCODER_INPUT_SIZE = 80  # build_model passes ConformerEncoder(input_size=80) whatever n_mels is (__init__.py:69)

_model = None  # type: Optional[PPGModel]
_device = None

_INPUT = {"conv2d": 0, "linear": 1, "vgg2l": 2, "embed": 3}
_POS = {"abs_pos": 0, "scaled_abs_pos": 1, "rel_pos": 2}
_ATTN = {"selfattn": 0, "rel_selfattn": 1}
_FF = {"linear": 0, "conv1d": 1, "conv1d-linear": 2}
_ACT = {"swish": 0, "relu": 1}


def _code(table: dict, v, what: str) -> int:
    if v not in table:
        raise _lib.MbError(f"{what} {v!r} is not supported")
    return table[v]


def pos_table(d_model: int, pe_len: int, reverse: bool) -> torch.Tensor:
    """PositionalEncoding.extend_pe (embedding.py:56-77) for a pe_len-row table, built at full length with torch's own
    sin / cos so that every value matches the reference's bit for bit"""
    import math

    pe = torch.zeros(pe_len, d_model)
    if reverse:
        position = torch.arange(pe_len - 1, -1, -1.0, dtype=torch.float32).unsqueeze(1)
    else:
        position = torch.arange(0, pe_len, dtype=torch.float32).unsqueeze(1)
    div_term = torch.exp(torch.arange(0, d_model, 2, dtype=torch.float32) * -(math.log(10000.0) / d_model))
    pe[:, 0::2] = torch.sin(position * div_term)
    pe[:, 1::2] = torch.cos(position * div_term)
    return pe


def frontend_params(frontend_conf: dict) -> dict:
    """``frontend_conf`` resolved as DefaultFrontend resolves it (its defaults, ``win_length=None`` -> n_fft, fmax None ->
    fs / 2).  Raises MbError for keys it does not take and for options the kernels do not implement."""
    fe = dict(frontend_conf or {})
    unknown = set(fe) - set(_FRONTEND_DEFAULTS) - {"fs"}
    if unknown:
        raise _lib.MbError(f"frontend_conf: unexpected keys {sorted(unknown)} (DefaultFrontend does not take them)")
    if "fs" not in fe:
        raise _lib.MbError("frontend_conf: fs is required (DefaultFrontend has no default for it)")
    r = dict(_FRONTEND_DEFAULTS, **fe)
    for k, v in _FRONTEND_FIXED.items():
        if r[k] != v:
            raise _lib.MbError(f"frontend_conf: {k}={r[k]!r} is not supported (only {v!r})")
    if r["norm"] not in (1, "slaney", None):
        raise _lib.MbError(f"frontend_conf: norm={r['norm']!r} is not supported (1, 'slaney' or None)")
    if r["win_length"] is None:
        r["win_length"] = r["n_fft"]
    if r["fmin"] is None:
        r["fmin"] = 0.0
    if r["fmax"] is None:
        r["fmax"] = r["fs"] / 2
    if r["n_mels"] != ENCODER_INPUT_SIZE:
        raise _lib.MbError(f"frontend_conf: n_mels={r['n_mels']} is not supported: build_model builds the encoder for "
                           f"{ENCODER_INPUT_SIZE} mel bins")
    return r


class PPGModel:
    def __init__(self, frontend_conf: dict, normalize_conf: dict, encoder_conf: dict):
        fe = frontend_params(frontend_conf)
        nc, enc = dict(normalize_conf or {}), dict(encoder_conf)
        if set(nc) - set(_NORMALIZE_DEFAULTS):
            raise _lib.MbError(f"normalize_conf: unexpected keys {sorted(set(nc) - set(_NORMALIZE_DEFAULTS))}")
        nc = dict(_NORMALIZE_DEFAULTS, **nc)
        if nc["eps"] != 1.0e-20:
            raise _lib.MbError(f"normalize_conf: eps={nc['eps']!r} is not supported (only 1e-20)")
        if set(enc) - _ENCODER_KEYS:
            raise _lib.MbError(f"encoder_conf: unexpected keys {sorted(set(enc) - _ENCODER_KEYS)}")
        n_fft = int(fe["n_fft"])
        cfg = _lib.PpgxConfig()
        cfg.n_fft = n_fft
        cfg.win_length = int(fe["win_length"])
        cfg.hop_length = int(fe["hop_length"])
        cfg.n_mels = int(fe["n_mels"])
        cfg.kaldi_padding_mode = int(bool(fe["kaldi_padding_mode"]))
        cfg.downsample_rate = int(fe["downsample_rate"])
        cfg.norm_means = int(bool(nc["norm_means"]))
        cfg.norm_vars = int(bool(nc["norm_vars"]))
        cfg.attention_dim = int(enc.get("attention_dim", 256))
        cfg.attention_heads = int(enc.get("attention_heads", 4))
        cfg.linear_units = int(enc.get("linear_units", 2048))
        cfg.num_blocks = int(enc.get("num_blocks", 6))
        cfg.input_layer = _code(_INPUT, enc.get("input_layer", "conv2d"), "input_layer")
        cfg.no_subsample = int(bool(enc.get("no_subsample", False)))
        cfg.subsample_by_2 = int(bool(enc.get("subsample_by_2", False)))
        cfg.normalize_before = int(bool(enc.get("normalize_before", True)))
        cfg.concat_after = int(bool(enc.get("concat_after", False)))
        cfg.positionwise_layer_type = _code(_FF, enc.get("positionwise_layer_type", "linear"), "positionwise_layer_type")
        cfg.macaron_style = int(bool(enc.get("macaron_style", False)))
        cfg.pos_enc_layer_type = _code(_POS, enc.get("pos_enc_layer_type", "abs_pos"), "pos_enc_layer_type")
        cfg.selfattention_layer_type = _code(_ATTN, enc.get("selfattention_layer_type", "selfattn"), "selfattention_layer_type")
        cfg.activation_type = _code(_ACT, enc.get("activation_type", "swish"), "activation_type")
        cfg.use_cnn_module = int(bool(enc.get("use_cnn_module", False)))
        cfg.cnn_module_kernel = int(enc.get("cnn_module_kernel", 31))
        self._handle = C.c_void_p()
        _lib.check(_lib.lib().mb_ppgx_create(C.byref(cfg), C.byref(self._handle)))
        self.cfg = cfg
        self.d_model = cfg.attention_dim
        self.rel = cfg.pos_enc_layer_type == _POS["rel_pos"]
        self.pe_len = PE_MAX_LEN  # the instance's positional-table high-water mark (embedding.py:56-77)
        self._pe: Optional[torch.Tensor] = None
        self._pe_rows = 0
        self._default_melmat = torch.from_numpy(ppg_melmat(int(fe["fs"]), n_fft, cfg.n_mels, float(fe["fmin"]),
                                                           float(fe["fmax"]), norm=fe["norm"]))
        self._state: Optional[Dict[str, torch.Tensor]] = None
        self._arena = None
        self._ws = None
        self._device: Optional[torch.device] = None
        self._ready = False
        self.training = True

    # -- torch.nn.Module surface the callers use ----------------------------------------------------------------------
    def load_state_dict(self, sd, strict: bool = True):
        self._state = {k: v.detach() for k, v in sd.items()}
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
            raise _lib.MbError("mockingbird_b200 PPGModel runs on CUDA only (no CPU fallback)")
        if device.index is None:
            device = torch.device("cuda", torch.cuda.current_device())
        self._device = device
        self._ready = False
        self._pe = None
        return self

    def cuda(self):
        return self.to(_lib.require_cuda())

    def release_workspace(self):
        """free the cached per-call workspace (it is reallocated by the next call)"""
        self._ws = None

    def __call__(self, speech, speech_lengths):
        return self.forward(speech, speech_lengths)

    # -- weights -------------------------------------------------------------------------------------------------------
    def _upload(self):
        if self._state is None:
            raise _lib.MbError("PPGModel has no weights: call load_state_dict first")
        self._device = self._device or _lib.require_cuda()
        self._arena = _lib.upload_weights("ppgx", self._handle, self.weights_for_upload(), self._device, align=1024)
        self._ready = True

    def weights_for_upload(self) -> Dict[str, torch.Tensor]:
        """the float tensors of the checkpoint, with the default mel basis where the checkpoint has none"""
        state = {k: v for k, v in self._state.items() if v.dtype.is_floating_point}
        state.setdefault("frontend.logmel.melmat", self._default_melmat)
        return state

    def _prepare(self):
        self.eval()
        if self._device is None:
            self.cuda()
        if not self._ready:
            self._upload()

    def num_frames(self, n_samples: int) -> int:
        return int(_lib.lib().mb_ppgx_num_frames(self._handle, int(n_samples)))

    def _table(self, T: int) -> torch.Tensor:
        """rows [0, T) of the instance's positional table, after raising the high-water mark to T"""
        if T > self.pe_len:
            self.pe_len = T
            self._pe = None
        if self._pe is None or self._pe_rows < T:
            full = pos_table(self.d_model, self.pe_len, reverse=self.rel)
            self._pe = full.to(self._device).contiguous()
            self._pe_rows = self.pe_len
        return self._pe

    # -- inference -----------------------------------------------------------------------------------------------------
    def _run(self, wav: torch.Tensor, lengths: List[int], taps: bool = False):
        """one padded batch wav [B, n_max] (device) of <= MAX_ROWS rows -> (out [B, T_max, D], taps or None)"""
        dev = self._device
        Lb = _lib.lib()
        B, n_max = wav.shape
        T = self.num_frames(n_max)
        pe = self._table(T)
        D = self.d_model
        with torch.cuda.device(dev):
            out = torch.empty(B, T, D, device=dev)
            tp = torch.empty(self.cfg.num_blocks + 1, B, T, D, device=dev) if taps else None
            need = int(Lb.mb_ppgx_workspace_bytes(self._handle, B, n_max))
            if need == 0:
                raise ValueError(f"utterance of {n_max} samples is too short")
            _lib.workspace(need, dev, self)
            ns = (C.c_int32 * B)(*lengths)
            stream = torch.cuda.current_stream(dev).cuda_stream
            _lib.check(Lb.mb_ppgx_forward(
                self._handle, C.c_void_p(wav.data_ptr()), ns, B, n_max, self.pe_len, C.c_void_p(pe.data_ptr()),
                C.c_void_p(out.data_ptr()), C.c_void_p(tp.data_ptr()) if tp is not None else None,
                C.c_void_p(self._ws.data_ptr()), self._ws.numel(), C.c_void_p(stream)))
        return out, tp

    def forward(self, speech: torch.Tensor, speech_lengths: torch.Tensor, return_taps: bool = False):
        """speech [B, L], speech_lengths [B] -> [B, T, D] on the device (T = frames of max(speech_lengths); rows are
        zero past their own frames).  Each row is computed as its own B = 1 call.  ``return_taps=True`` also returns
        [num_blocks + 1, B, T, D]: the embed output and each block's output."""
        if speech.dim() != 2 or speech_lengths.dim() != 1 or speech_lengths.shape[0] != speech.shape[0]:
            raise ValueError("expected speech [B, L] and speech_lengths [B]")
        if speech.shape[0] > MAX_ROWS:
            raise ValueError(f"at most {MAX_ROWS} rows per call; use extract_batch for more")
        self._prepare()
        lengths = [int(v) for v in speech_lengths.tolist()]
        n_max = max(lengths)
        wav = speech[:, :n_max].to(device=self._device, dtype=torch.float32).contiguous()
        out, tp = self._run(wav, lengths, taps=return_taps)
        return (out, tp) if return_taps else out

    def extract_from_wav(self, src_wav):
        """__init__.py:60-63: one utterance (numpy or tensor [L]) -> [1, T, D]"""
        w = torch.as_tensor(np.asarray(src_wav, dtype=np.float32) if not torch.is_tensor(src_wav) else src_wav)
        return self.forward(w.reshape(1, -1), torch.LongTensor([w.numel()]))

    def extract_batch(self, wavs: Sequence) -> List[torch.Tensor]:
        """many utterances [L_i] -> a list of [T_i, D] device tensors.  Rows are length-sorted into padded calls of <= 128
        rows and <= MAX_BATCH_FRAMES padded frames, longest first; each result equals its own B = 1 call made in that
        order.  The order matters only past 5000 frames (50 s at a 10 ms hop): the positional table's high-water mark
        rises to the longest utterance before any shorter one runs, whereas B = 1 calls in the caller's order would
        see the mark each utterance's predecessors left.  `wavs` may be a resample.DeviceClips (clips resampled to the
        extractor's rate on the device), whose clips are read where they lie."""
        self._prepare()
        ws = [torch.as_tensor(np.asarray(w, dtype=np.float32) if not torch.is_tensor(w) else w).reshape(-1) for w in wavs]
        order = sorted(range(len(ws)), key=lambda i: -ws[i].numel())
        res: List[Optional[torch.Tensor]] = [None] * len(ws)
        pos = 0
        while pos < len(order):
            n_max = ws[order[pos]].numel()
            per = max(1, self.num_frames(n_max))
            take = max(1, min(MAX_ROWS, MAX_BATCH_FRAMES // per, len(order) - pos))
            idx = order[pos:pos + take]
            pos += take
            wav = torch.zeros(len(idx), n_max, device=self._device)
            for r, i in enumerate(idx):
                wav[r, :ws[i].numel()] = ws[i].to(self._device)
            lens = [ws[i].numel() for i in idx]
            out, _ = self._run(wav, lens)
            for r, i in enumerate(idx):
                res[i] = out[r, :self.num_frames(lens[r])]
        return res

    def __del__(self):
        try:
            if getattr(self, "_handle", None) is not None and self._handle.value:
                _lib.lib().mb_ppgx_destroy(self._handle)
                self._handle = C.c_void_p()
        except Exception:
            pass


def build_model(args):
    """__init__.py:66-72 (args: a namespace or dict with frontend_conf, normalize_conf, encoder_conf)"""
    a = vars(args) if isinstance(args, argparse.Namespace) else dict(args)
    return PPGModel(a.get("frontend_conf") or {}, a.get("normalize_conf") or {}, a["encoder_conf"])


def load_model(model_file, device=None):
    """__init__.py:75-102: the config is the first ``*.yaml`` under the checkpoint's directory; checkpoint keys that
    contain ``encoder`` replace the freshly built model's (whose melmat is the current librosa meaning)."""
    import yaml

    global _model, _device
    _device = torch.device(device) if device is not None else _lib.require_cuda()
    model_file = Path(model_file)
    configs = list(model_file.parent.rglob("*.yaml"))
    if not configs:
        raise FileNotFoundError(f"No model yaml config found for the PPG extractor under {model_file.parent}")
    with configs[0].open("r", encoding="utf-8") as f:
        args = yaml.safe_load(f)
    model = build_model(args)
    ckpt = torch.load(str(model_file), map_location="cpu")
    sd = {k: v for k, v in ckpt.items() if "encoder" in k}
    model.load_state_dict(sd)
    _model = model.eval().to(_device)
    return _model
