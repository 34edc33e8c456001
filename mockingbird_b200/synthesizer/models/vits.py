"""Host side of the VITS synthesizer over the mb_vits_* C ABI.

Mirrors the reference's ``Vits`` inference surface (models/synthesizer/models/vits.py:389-527): the constructor's
arguments, ``load_state_dict`` with the checkpoint's ``weight_g`` / ``weight_v`` keys, ``eval()``, ``to(device)``,
``remove_weight_norm()`` and ``infer``.  ``infer_many`` synthesizes many texts as independent rows.  All arithmetic runs
in the CUDA library; training (``forward``), the posterior encoder and the discriminators are not part of it.
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, List, Optional, Sequence

import numpy as np
import torch

from ... import _lib
from ...vocoder._gan import fold_weight_norm

EMO_DIM = 1024  # TextEncoder.emo_proj = nn.Linear(1024, hidden_channels) (vits.py:154)


def _ptr(t: Optional[torch.Tensor]):
    return C.c_void_p(t.data_ptr()) if t is not None else None


class Vits:
    """``Vits(...)`` of the reference, inference only.  ``precision`` picks the decoder's arithmetic (``MB_PREC_*``: "fp32",
    "f16x3" or "f16tc"); everything before the decoder is FP32."""

    MANY_BATCH = 16  # rows per infer_many batch

    def __init__(self, n_vocab, spec_channels, segment_size, inter_channels, hidden_channels, filter_channels, n_heads, n_layers,
                 kernel_size, p_dropout, resblock, resblock_kernel_sizes, resblock_dilation_sizes, upsample_rates,
                 upsample_initial_channel, upsample_kernel_sizes, n_speakers=0, gin_channels=0, use_sdp=True, precision="fp32",
                 **kwargs):
        if n_speakers == 1:
            raise ValueError("n_speakers == 1: Vits builds no speaker embedding for one speaker but infer indexes it")
        if n_speakers > 1 and gin_channels <= 0:
            raise ValueError(f"n_speakers = {n_speakers} needs gin_channels > 0")
        if n_speakers == 0 and gin_channels != 0:
            raise ValueError("gin_channels without speakers: Vits.infer conditions on no g")
        if precision not in _lib.PRECISIONS:
            raise ValueError(f"precision must be one of {sorted(_lib.PRECISIONS)}")
        rks = [int(k) for k in resblock_kernel_sizes]
        rds = [[int(d) for d in ds] for ds in resblock_dilation_sizes]
        if len({len(d) for d in rds}) != 1:
            raise ValueError("resblock_dilation_sizes must be rectangular")
        if len(rks) > 4 or len(rds[0]) > 4 or len(upsample_rates) > 8 or len(upsample_rates) != len(upsample_kernel_sizes):
            raise ValueError("at most 4 resblock kernels of 4 dilations and 8 upsampling stages, one kernel size per stage")
        self.n_vocab, self.inter_channels, self.hidden_channels = int(n_vocab), int(inter_channels), int(hidden_channels)
        self.n_speakers, self.gin_channels, self.use_sdp = int(n_speakers), int(gin_channels), bool(use_sdp)
        self.precision = precision
        cfg = _lib.VitsConfig()
        cfg.n_vocab, cfg.inter_channels, cfg.hidden_channels = self.n_vocab, self.inter_channels, self.hidden_channels
        cfg.filter_channels, cfg.n_heads, cfg.n_layers, cfg.kernel_size = int(filter_channels), int(n_heads), int(n_layers), int(kernel_size)
        cfg.resblock_type = 1 if str(resblock) == "1" else 2
        cfg.num_kernels = len(rks)
        cfg.num_dilations = len(rds[0])
        for j, (k, ds) in enumerate(zip(rks, rds)):
            cfg.resblock_kernel_sizes[j] = k
            for m, d in enumerate(ds):
                cfg.resblock_dilation_sizes[j][m] = d
        cfg.num_upsamples = len(upsample_rates)
        for i, (u, k) in enumerate(zip(upsample_rates, upsample_kernel_sizes)):
            cfg.upsample_rates[i], cfg.upsample_kernel_sizes[i] = int(u), int(k)
        cfg.upsample_initial_channel = int(upsample_initial_channel)
        cfg.n_speakers, cfg.gin_channels, cfg.use_sdp = self.n_speakers, self.gin_channels, int(self.use_sdp)
        cfg.precision = _lib.PRECISIONS[precision]
        self._cfg = cfg
        self._handle = C.c_void_p()
        _lib.check(_lib.lib().mb_vits_create(C.byref(cfg), C.byref(self._handle)))
        self.hop = int(_lib.lib().mb_vits_hop(self._handle))
        self._state: Optional[Dict[str, torch.Tensor]] = None
        self._arena: Optional[torch.Tensor] = None
        self._device: Optional[torch.device] = None
        self._ws_dur: Optional[torch.Tensor] = None  # the two calls' cached workspaces (_lib.workspace)
        self._ws_dec: Optional[torch.Tensor] = None
        self._ready = False
        self.training = True

    # -- nn.Module-like surface ------------------------------------------------------------------
    def load_state_dict(self, state_dict: Dict[str, torch.Tensor], strict: bool = True):
        self._state = {k: v.detach() for k, v in state_dict.items()}
        self._ready = False
        return self

    def eval(self):
        self.training = False
        return self

    def to(self, device):
        self._device = torch.device(device)
        if self._device.type != "cuda":
            raise _lib.MbError("mockingbird_b200 runs VITS on CUDA only (no CPU fallback)")
        self._ready = False
        return self

    def cuda(self):
        return self.to(_lib.require_cuda())

    def remove_weight_norm(self):
        """Fold weight norm (dec.ups / resblocks, the flow's WN layers) and upload the weights."""
        if self._state is None:
            raise _lib.MbError("load_state_dict must be called before remove_weight_norm")
        self._state = fold_weight_norm(self._state)
        self._upload()
        return self

    def _upload(self):
        if self._state is None:
            raise _lib.MbError("Vits has no weights: call load_state_dict first")
        self._device = self._device or _lib.require_cuda()
        self._arena = _lib.upload_weights("vits", self._handle, fold_weight_norm(self._state), self._device)
        self._ready = True

    def packed_arena(self) -> torch.Tensor:
        if not self._ready:
            self._upload()
        return self._arena

    # -- argument checks -------------------------------------------------------------------------
    def _check_sid(self, sid, B: int) -> Optional[torch.Tensor]:
        if self.n_speakers == 0:
            return None
        if sid is None:
            raise ValueError(f"a model with {self.n_speakers} speakers needs sid")
        s = torch.as_tensor(sid).reshape(-1).to(torch.int64)
        if s.numel() != B:
            raise ValueError(f"{s.numel()} speaker ids for a batch of {B}")
        if s.numel() and (int(s.min()) < 0 or int(s.max()) >= self.n_speakers):
            raise ValueError(f"speaker id out of range [0, {self.n_speakers})")
        return s.to(torch.int32)

    def _check_emo(self, emo, B: int) -> torch.Tensor:
        if emo is None:
            raise ValueError("emo is required: the text encoder adds emo_proj(emo) (a [B, 1024] emotion vector)")
        e = torch.as_tensor(emo).to(torch.float32).reshape(B, -1) if torch.as_tensor(emo).numel() == B * EMO_DIM else None
        if e is None:
            raise ValueError(f"emo must hold {B} x {EMO_DIM} values, got shape {tuple(torch.as_tensor(emo).shape)}")
        return e

    def _check_tokens(self, x: torch.Tensor, lengths: torch.Tensor) -> None:
        T = x.shape[1]
        if T > int(_lib.lib().mb_vits_max_tokens()):
            raise ValueError(f"{T} tokens, over the limit of {int(_lib.lib().mb_vits_max_tokens())}")
        if lengths.numel() and (int(lengths.min()) < 1 or int(lengths.max()) > T):
            raise ValueError(f"x_lengths must lie in [1, {T}]")
        if x.numel() and (int(x.min()) < 0 or int(x.max()) >= self.n_vocab):
            raise ValueError(f"token id out of range [0, {self.n_vocab})")

    # -- the two library calls -------------------------------------------------------------------
    def _durations(self, x, lengths, sid, emo, noise, noise_scale_w, length_scale):
        B, T = x.shape
        dev, I = self._device, self.inter_channels
        m_p = torch.empty(B, I, T, device=dev)
        logs_p = torch.empty(B, I, T, device=dev)
        w_ceil = torch.empty(B, T, dtype=torch.int32, device=dev)
        y_len = torch.empty(B, dtype=torch.int32, device=dev)
        L = _lib.lib()
        ws = _lib.workspace(int(L.mb_vits_durations_workspace_bytes(self._handle, B, T)), dev, self, "_ws_dur")
        st = torch.cuda.current_stream(dev).cuda_stream
        _lib.check(L.mb_vits_durations(self._handle, _ptr(x), _ptr(lengths), B, T, _ptr(sid), _ptr(emo), _ptr(noise),
                                       float(noise_scale_w), float(length_scale), _ptr(m_p), _ptr(logs_p), _ptr(w_ceil), _ptr(y_len),
                                       _ptr(ws), ws.numel(), C.c_void_p(st)))
        return m_p, logs_p, w_ceil, y_len

    def _decode(self, m_p, logs_p, w_ceil, lengths, sid, eps, noise_scale, t_dec, ragged, want_all):
        B, I, Tx = m_p.shape
        Ty = eps.shape[2]
        dev = self._device
        wav = torch.empty(B, 1, t_dec * self.hop, device=dev)
        extra = [torch.empty(B, 1, Ty, Tx, device=dev)] + [torch.empty(B, I, Ty, device=dev) for _ in range(4)] if want_all else [None] * 5
        L = _lib.lib()
        ws = _lib.workspace(int(L.mb_vits_decode_workspace_bytes(self._handle, B, Tx, Ty, t_dec)), dev, self, "_ws_dec")
        st = torch.cuda.current_stream(dev).cuda_stream
        attn, z_p, z, m_y, logs_y = extra
        _lib.check(L.mb_vits_decode(self._handle, _ptr(m_p), _ptr(logs_p), _ptr(w_ceil), _ptr(lengths), _ptr(sid), B, Tx, Ty, _ptr(eps),
                                    float(noise_scale), t_dec, int(ragged), _ptr(wav), _ptr(attn), _ptr(z_p), _ptr(z), _ptr(m_y),
                                    _ptr(logs_y), _ptr(ws), ws.numel(), C.c_void_p(st)))
        return wav, attn, z_p, z, m_y, logs_y

    # -- inference -------------------------------------------------------------------------------
    @torch.no_grad()
    def infer(self, x, x_lengths, sid=None, emo=None, noise_scale=1, length_scale=1, noise_scale_w=1., max_len=None):
        """``Vits.infer`` (vits.py:498-527) -> ``(o [B, 1, T*hop], attn [B, 1, T_y, T_x], y_mask [B, 1, T_y], (z, z_p, m_p,
        logs_p))`` as device tensors.  The SDP noise ``[B, 2, T_x]`` (use_sdp only) and the prior noise ``[B, inter, T_y]``
        are drawn from torch's global CPU generator in the reference's order, so a seeded padded batch reproduces the
        reference's padded batch."""
        x = torch.as_tensor(x)
        if x.dim() != 2:
            raise ValueError(f"x must be [B, T_x] token ids, got shape {tuple(x.shape)}")
        B, T = x.shape
        lengths = torch.as_tensor(x_lengths).reshape(-1).to(torch.int64)
        if lengths.numel() != B:
            raise ValueError(f"{lengths.numel()} lengths for a batch of {B}")
        self._check_tokens(x.to(torch.int64), lengths)
        emo_t = self._check_emo(emo, B)
        sid_t = self._check_sid(sid, B)
        if max_len is not None and int(max_len) < 1:
            raise ValueError("max_len must be at least 1")
        if not self._ready:
            self._upload()
        dev = self._device
        noise = torch.randn(B, 2, T) if self.use_sdp else None
        with torch.cuda.device(dev):
            xd = x.to(device=dev, dtype=torch.int32).contiguous()
            ld = lengths.to(device=dev, dtype=torch.int32)
            sd = sid_t.to(dev) if sid_t is not None else None
            m_p, logs_p, w_ceil, y_len = self._durations(xd, ld, sd, emo_t.to(dev), noise.to(dev) if noise is not None else None,
                                                         noise_scale_w, length_scale)
            y_len_h = y_len.cpu()
            Ty = int(y_len_h.max())
            # torch.randn_like(m_p) (vits.py:522) of the expanded m_p, a transposed matmul result: the same call on a tensor
            # with its strides draws the same numbers (torch fills a non-contiguous tensor element by element)
            eps = torch.randn_like(torch.empty(B, Ty, self.inter_channels).transpose(1, 2)).contiguous()
            t_dec = Ty if max_len is None else min(int(max_len), Ty)
            wav, attn, z_p, z, m_y, logs_y = self._decode(m_p, logs_p, w_ceil, ld, sd, eps.to(dev), noise_scale, t_dec, False, True)
            y_mask = (torch.arange(Ty, device=dev)[None, :] < y_len.to(torch.int64)[:, None]).to(torch.float32).unsqueeze(1)
        return wav, attn, y_mask, (z, z_p, m_y, logs_y)

    @staticmethod
    def many_plan(lengths: Sequence[int], batch_size: int) -> List[List[int]]:
        """infer_many's batches: indices sorted longest first (stable), cut into runs of at most batch_size"""
        order = sorted(range(len(lengths)), key=lambda i: -int(lengths[i]))
        return [order[s:s + batch_size] for s in range(0, len(order), batch_size)]

    @torch.no_grad()
    def infer_many(self, seqs, sids, emos, seeds, noise_scale=0.667, length_scale=1, noise_scale_w=0.8, batch_size=None):
        """Many texts, each computed as its own B = 1 ``infer_many`` call -> list of N float32 waveforms (numpy, y_i * hop
        samples each).  Utterance i draws its SDP noise [1, 2, T_i] and then its prior noise [1, inter, y_i] from
        ``torch.Generator().manual_seed(seeds[i])``, the latter over the same transposed storage ``infer`` draws it into.  Texts run in length-sorted ragged batches; a waveform is bitwise the
        same whatever texts share its batch."""
        N = len(seqs)
        if N == 0:
            return []
        rows = [torch.as_tensor(s).reshape(-1).to(torch.int64) for s in seqs]
        for i, r in enumerate(rows):
            if r.numel() == 0:
                raise ValueError(f"text {i} is empty")
        if len(seeds) != N:
            raise ValueError(f"{len(seeds)} seeds for {N} texts")
        emo_all = self._check_emo(emos, N)
        sid_all = self._check_sid(sids, N)
        for r in rows:
            self._check_tokens(r[None], torch.tensor([r.numel()]))
        if not self._ready:
            self._upload()
        dev, I = self._device, self.inter_channels
        out: List[Optional[np.ndarray]] = [None] * N
        for idx in self.many_plan([r.numel() for r in rows], int(batch_size or self.MANY_BATCH)):
            B = len(idx)
            T = max(rows[i].numel() for i in idx)
            x = torch.zeros(B, T, dtype=torch.int32)
            lens = torch.tensor([rows[i].numel() for i in idx], dtype=torch.int32)
            gens = [torch.Generator().manual_seed(int(seeds[i])) for i in idx]
            noise = torch.zeros(B, 2, T) if self.use_sdp else None
            for r, i in enumerate(idx):
                x[r, :rows[i].numel()] = rows[i].to(torch.int32)
                if noise is not None:
                    noise[r, :, :rows[i].numel()] = torch.randn(1, 2, rows[i].numel(), generator=gens[r])[0]
            with torch.cuda.device(dev):
                ld = lens.to(dev)
                sd = sid_all[idx].to(dev) if sid_all is not None else None
                m_p, logs_p, w_ceil, y_len = self._durations(x.to(dev), ld, sd, emo_all[idx].to(dev),
                                                             noise.to(dev) if noise is not None else None, noise_scale_w,
                                                             length_scale)
                y_h = y_len.cpu().tolist()
                Ty = max(y_h)
                eps = torch.zeros(B, I, Ty)
                for r in range(B):
                    eps[r, :, :y_h[r]] = torch.empty(1, y_h[r], I).transpose(1, 2).normal_(generator=gens[r])[0]
                wav = self._decode(m_p, logs_p, w_ceil, ld, sd, eps.to(dev), noise_scale, Ty, True, False)[0].cpu().numpy()
            for r, i in enumerate(idx):
                out[i] = wav[r, 0, :y_h[r] * self.hop].copy()
        return out  # type: ignore[return-value]

    def __del__(self):
        try:
            if getattr(self, "_handle", None) is not None and self._handle.value:
                _lib.lib().mb_vits_destroy(self._handle)
                self._handle = C.c_void_p()
        except Exception:
            pass
