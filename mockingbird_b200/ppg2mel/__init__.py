"""``MelDecoderMOLv2`` on the H100 path (reference: models/ppg2mel/__init__.py:20-209).

Same constructor keywords, ``load_state_dict`` / ``eval`` / ``to`` / ``cuda`` and
``inference(bottle_neck_features, logf0_uv=None, spembs=None) -> (mel [T,80], mel_postnet [T,80], alignments [n,T_enc])``
for one utterance (B = 1), exactly as the reference returns them.  All layers run in the CUDA library (mb_ppg2mel_*).

The reference's decoder PreNet dropout is always on (rnn_decoder_mol.py:20), so inference is stochastic.
``dropout_masks=(keep1, keep2)`` injects the keep masks (bool / uint8, keep1 [steps, 256], keep2 [steps, 128], at least
2 * (T // 4) steps) for reproducible comparisons; otherwise they are drawn on the device from ``seed``.
``inference_batch(..., seeds=[s_i])`` gives every utterance its own dropout stream: utterance i is bitwise
``inference(..., seed=s_i)`` whatever else is in the call (with ``seed=`` the draws of a row depend on its position).

The reference's ``inference`` with B > 1 calls ``Decoder.inference_batched``, which concatenates every row's frames
into one output and raises IndexError for a row whose stop token never fires, so no caller can depend on it; here B > 1
through ``inference`` is an error and ``inference_batch`` runs many utterances, each computed as its own B = 1 call.
"""
from __future__ import annotations

import ctypes as C
import numbers
from pathlib import Path
from typing import Dict, List, Optional, Sequence, Tuple

import torch

from .. import _lib

MAX_ROWS = 128  # rows per library call


class MelDecoderMOLv2:
    def __init__(self, num_speakers: int, spk_embed_dim: int, bottle_neck_feature_dim: int, encoder_dim: int = 256,
                 encoder_downsample_rates: Sequence[int] = (2, 2), attention_rnn_dim: int = 512,
                 decoder_rnn_dim: int = 512, num_decoder_rnn_layer: int = 1, concat_context_to_last: bool = True,
                 prenet_dims: Sequence[int] = (256, 128), num_mixtures: int = 5, frames_per_step: int = 2,
                 mask_padding: bool = True):
        rates, pdims = list(encoder_downsample_rates), list(prenet_dims)
        if len(rates) != 2 or len(pdims) != 2:
            raise _lib.MbError("encoder_downsample_rates and prenet_dims must have two entries")
        cfg = _lib.Ppg2MelConfig()
        cfg.bottle_neck_feature_dim, cfg.spk_embed_dim, cfg.encoder_dim = bottle_neck_feature_dim, spk_embed_dim, encoder_dim
        cfg.encoder_downsample_rates[0], cfg.encoder_downsample_rates[1] = rates
        cfg.attention_rnn_dim, cfg.decoder_rnn_dim = attention_rnn_dim, decoder_rnn_dim
        cfg.num_decoder_rnn_layer, cfg.concat_context_to_last = num_decoder_rnn_layer, int(bool(concat_context_to_last))
        cfg.prenet_dims[0], cfg.prenet_dims[1] = pdims
        cfg.num_mixtures, cfg.frames_per_step, cfg.num_mels = num_mixtures, frames_per_step, 80
        self._handle = C.c_void_p()
        _lib.check(_lib.lib().mb_ppg2mel_create(C.byref(cfg), C.byref(self._handle)))
        self.num_mels = 80
        self.bottle_neck_feature_dim = bottle_neck_feature_dim
        self.spk_embed_dim = spk_embed_dim
        self.frames_per_step = frames_per_step
        self.encoder_down_factor = rates[0] * rates[1]
        self._state: Optional[Dict[str, torch.Tensor]] = None
        self._arena = None
        self._ws = None
        self._device: Optional[torch.device] = None
        self._ready = False
        self.training = True
        self.seed = 0

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
            raise _lib.MbError("mockingbird_b200 MelDecoderMOLv2 runs on CUDA only (no CPU fallback)")
        if device.index is None:
            device = torch.device("cuda", torch.cuda.current_device())
        self._device = device
        self._ready = False
        return self

    def cuda(self):
        return self.to(_lib.require_cuda())

    # -- weights -------------------------------------------------------------------------------------------------------
    def _upload(self):
        if self._state is None:
            raise _lib.MbError("MelDecoderMOLv2 has no weights: call load_state_dict first")
        self._device = self._device or _lib.require_cuda()
        self._arena = _lib.upload_weights("ppg2mel", self._handle, self.weights_for_upload(), self._device)
        self._ready = True

    def weights_for_upload(self) -> Dict[str, torch.Tensor]:
        """the float tensors of the checkpoint (the library drops the ones inference never reads)"""
        return {k: v for k, v in self._state.items() if v.dtype.is_floating_point}

    # -- inference -----------------------------------------------------------------------------------------------------
    def _run(self, ppg: torch.Tensor, lf0_uv: torch.Tensor, spk: torch.Tensor, lengths: List[int], masks=None,
             seed: Optional[int] = None, return_stop: bool = False, row_seeds: Optional[torch.Tensor] = None):
        """one padded batch of <= MAX_ROWS rows -> per-row (mel, mel_postnet, alignments[, stop]); row_seeds (int64 [B]
        on the device, the seeds' 64 bits) selects per-row dropout streams (mb_ppg2mel_inference_rows)"""
        dev = self._device
        L = _lib.lib()
        B, T, _ = ppg.shape
        Te = T // 4
        S = 2 * Te
        with torch.cuda.device(dev):
            need = int(L.mb_ppg2mel_workspace_bytes(self._handle, B, T))
            if need == 0:
                raise ValueError(L.mb_last_error().decode())
            mel = torch.empty(B, 2 * S, self.num_mels, device=dev)
            post = torch.empty_like(mel)
            align = torch.empty(B, S, Te, device=dev)
            stop = torch.empty(B, S, device=dev)
            m1 = m2 = None
            if masks is not None:
                m1 = masks[0].to(device=dev, dtype=torch.uint8).contiguous()
                m2 = masks[1].to(device=dev, dtype=torch.uint8).contiguous()
                if tuple(m1.shape) != (S, B, 256) or tuple(m2.shape) != (S, B, 128):
                    raise ValueError(f"dropout masks must be [{S},{B},256] and [{S},{B},128]")
            _lib.workspace(need, dev, self)
            lens = (C.c_int32 * B)(*lengths)
            steps = (C.c_int32 * B)()
            stream = torch.cuda.current_stream(dev).cuda_stream
            io = (C.c_void_p(ppg.data_ptr()), C.c_void_p(lf0_uv.data_ptr()), C.c_void_p(spk.data_ptr()), lens, B, T)
            outs = (C.c_void_p(mel.data_ptr()), C.c_void_p(post.data_ptr()), C.c_void_p(align.data_ptr()),
                    C.c_void_p(stop.data_ptr()), steps, C.c_void_p(self._ws.data_ptr()), self._ws.numel(), C.c_void_p(stream))
            if row_seeds is not None:
                _lib.check(L.mb_ppg2mel_inference_rows(self._handle, *io, C.c_void_p(row_seeds.data_ptr()), *outs))
            else:
                _lib.check(L.mb_ppg2mel_inference(
                    self._handle, *io, C.c_void_p(m1.data_ptr()) if m1 is not None else None,
                    C.c_void_p(m2.data_ptr()) if m2 is not None else None, C.c_uint64(self.seed if seed is None else seed),
                    *outs))
        out = []
        for b in range(B):
            n, te = steps[b], lengths[b] // 4
            r = (mel[b, :2 * n], post[b, :2 * n], align[b, :n, :te])
            out.append(r + (stop[b, :n],) if return_stop else r)
        return out

    def _check_inputs(self, ppg: torch.Tensor, lf0_uv: torch.Tensor):
        if ppg.dim() != 2 or ppg.shape[1] != self.bottle_neck_feature_dim:
            raise ValueError(f"bottle_neck_features must be [T, {self.bottle_neck_feature_dim}], got {tuple(ppg.shape)}")
        if lf0_uv is None or lf0_uv.dim() != 2 or lf0_uv.shape[1] != 2:
            raise ValueError("logf0_uv must be [T, 2]")
        if lf0_uv.shape[0] != ppg.shape[0]:
            raise ValueError(f"bottle_neck_features has {ppg.shape[0]} frames but logf0_uv has {lf0_uv.shape[0]}")
        if ppg.shape[0] < 4:
            raise ValueError("need at least 4 PPG frames (one encoder frame after the 4x downsampling)")

    def _prepare(self):
        self.eval()
        if self._device is None:
            self.cuda()
        if not self._ready:
            self._upload()

    def inference(self, bottle_neck_features: torch.Tensor, logf0_uv: torch.Tensor = None, spembs: torch.Tensor = None,
                  dropout_masks=None, seed: Optional[int] = None):
        """bottle_neck_features [1, T, 144], logf0_uv [1, T, 2], spembs [1, 256] -> (mel [2n, 80], mel_postnet [2n, 80],
        alignments [n, T // 4]) on the device.  ``dropout_masks=(keep1 [S, 256], keep2 [S, 128])``, S >= 2 * (T // 4)."""
        if spembs is None:
            raise ValueError("spembs is required (the reference asserts it)")
        if bottle_neck_features.dim() != 3 or (logf0_uv is not None and logf0_uv.dim() != 3) or spembs.dim() != 2:
            raise ValueError("expected bottle_neck_features [1, T, D], logf0_uv [1, T, 2], spembs [1, E]")
        if bottle_neck_features.shape[0] != 1 or logf0_uv.shape[0] != 1 or spembs.shape[0] != 1:
            raise ValueError("MelDecoderMOLv2.inference takes one utterance (B = 1); use inference_batch for several")
        if spembs.shape[1] != self.spk_embed_dim:
            raise ValueError(f"spembs must be [1, {self.spk_embed_dim}]")
        ppg, lf0 = bottle_neck_features[0], logf0_uv[0]
        self._check_inputs(ppg, lf0)
        self._prepare()
        T = ppg.shape[0]
        masks = None
        if dropout_masks is not None:
            S = 2 * (T // 4)
            masks = (torch.as_tensor(dropout_masks[0])[:S].reshape(S, 1, 256),
                     torch.as_tensor(dropout_masks[1])[:S].reshape(S, 1, 128))
        dev = self._device
        args = [x.to(device=dev, dtype=torch.float32).contiguous() for x in (ppg[None], lf0[None], spembs)]
        return self._run(*args, [T], masks, seed)[0]

    def inference_batch(self, utterances: Sequence[Tuple[torch.Tensor, torch.Tensor]], spembs: torch.Tensor,
                        dropout_masks=None, seed: Optional[int] = None, return_stop: bool = False,
                        seeds: Optional[Sequence[int]] = None):
        """many utterances [(ppg [T_i, 144], lf0_uv [T_i, 2])] with spembs [N, 256] -> a list of per-utterance
        (mel, mel_postnet, alignments) as ``inference`` returns them.  Rows are length-sorted into padded batches of
        <= 128; each result equals the utterance's own B = 1 call with the same masks.
        ``dropout_masks``: a list of per-utterance (keep1 [S_i, 256], keep2 [S_i, 128]) pairs.
        ``seeds``: one dropout seed per utterance (integers in [0, 2**64)); utterance i is then bitwise
        ``inference(..., seed=seeds[i])``, whatever the other utterances are.  Not combined with ``seed`` or ``dropout_masks``."""
        n = len(utterances)
        if spembs.dim() != 2 or spembs.shape[0] != n or spembs.shape[1] != self.spk_embed_dim:
            raise ValueError(f"spembs must be [{n}, {self.spk_embed_dim}]")
        table = None
        if seeds is not None:
            if seed is not None or dropout_masks is not None:
                raise ValueError("pass seeds alone: not together with seed or dropout_masks")
            table = seed_table(seeds, n)
        for ppg, lf0 in utterances:
            self._check_inputs(ppg, lf0)
        self._prepare()
        dev = self._device
        order = sorted(range(n), key=lambda i: -utterances[i][0].shape[0])
        results: List = [None] * n
        for c0 in range(0, n, MAX_ROWS):
            idx = order[c0:c0 + MAX_ROWS]
            lens = [int(utterances[i][0].shape[0]) for i in idx]
            T = max(lens)
            B = len(idx)
            ppg = torch.zeros(B, T, self.bottle_neck_feature_dim, device=dev)
            lf0 = torch.zeros(B, T, 2, device=dev)
            for r, i in enumerate(idx):
                ppg[r, :lens[r]] = utterances[i][0].to(device=dev, dtype=torch.float32)
                lf0[r, :lens[r]] = utterances[i][1].to(device=dev, dtype=torch.float32)
            spk = spembs[idx].to(device=dev, dtype=torch.float32).contiguous()
            masks = None
            if dropout_masks is not None:
                S = 2 * (T // 4)
                m1 = torch.zeros(S, B, 256, dtype=torch.uint8)
                m2 = torch.zeros(S, B, 128, dtype=torch.uint8)
                for r, i in enumerate(idx):
                    s_i = 2 * (lens[r] // 4)
                    m1[:s_i, r] = torch.as_tensor(dropout_masks[i][0])[:s_i].to(torch.uint8)
                    m2[:s_i, r] = torch.as_tensor(dropout_masks[i][1])[:s_i].to(torch.uint8)
                masks = (m1, m2)
            rs = None
            if table is not None:
                rs = torch.tensor([table[i] for i in idx], dtype=torch.int64).to(dev)
            for r, res in zip(idx, self._run(ppg, lf0, spk, lens, masks, seed, return_stop, rs)):
                results[r] = res
        return results

    def __del__(self):
        try:
            if getattr(self, "_handle", None) is not None and self._handle.value:
                _lib.lib().mb_ppg2mel_destroy(self._handle)
                self._handle = C.c_void_p()
        except Exception:
            pass


def seed_table(seeds: Sequence[int], n: int) -> List[int]:
    """per-utterance dropout seeds as the int64 values whose 64 bits are the seeds (the library reads them as uint64)"""
    seeds = list(seeds)
    if len(seeds) != n:
        raise ValueError(f"{len(seeds)} seeds for {n} utterances")
    out = []
    for i, s in enumerate(seeds):
        if isinstance(s, bool) or not isinstance(s, numbers.Integral) or not 0 <= int(s) < 1 << 64:
            raise ValueError(f"seeds[{i}] = {s!r} is not an integer in [0, 2**64)")
        out.append(int(s) - (1 << 64) if int(s) >= 1 << 63 else int(s))
    return out


def load_model(model_file, device=None):
    """__init__.py:194-209: the model config is the first ``*.yaml`` under the checkpoint's directory (its ``model``
    section), the weights are ``ckpt["model"]``."""
    import yaml

    model_file = Path(model_file)
    configs = sorted(model_file.parent.rglob("*.yaml"))
    if not configs:
        raise FileNotFoundError(f"No model yaml config found for convertor under {model_file.parent}")
    with open(configs[0]) as f:
        cfg = yaml.safe_load(f)
    model = MelDecoderMOLv2(**cfg["model"])
    model.to(device if device is not None else _lib.require_cuda())
    ckpt = torch.load(str(model_file), map_location="cpu")
    model.load_state_dict(ckpt["model"])
    model.eval()
    return model
