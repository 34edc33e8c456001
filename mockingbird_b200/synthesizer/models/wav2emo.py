"""The wav2vec2 emotion model of extract_emo (models/synthesizer/models/wav2emo.py EmotionExtractorModel) on the GPU.

``EmotionExtractorModel(config)`` takes a dict or any object with the ``Wav2Vec2Config`` attributes it reads; transformers
is not imported.  Weights come from ``load_state_dict`` (either spelling of the positional conv's weight norm:
``weight_g`` / ``weight_v`` or transformers 5's ``parametrizations.weight.original0`` / ``original1``) or from
``from_pretrained(local_dir)`` on a downloaded snapshot.  ``model(input_values [B, L])`` returns
``(embedding [B, hidden], logits [B, num_labels])`` as the reference's forward does for equal-length rows, and
``run_clips`` takes a ragged list; every clip is computed as its own B = 1 call.
"""
from __future__ import annotations

import ctypes as C
import json
from pathlib import Path
from typing import Dict, List, Sequence, Tuple

import numpy as np
import torch

from ... import _lib
from ...vocoder._gan import fold_weight_norm

_POS = "wav2vec2.encoder.pos_conv_embed.conv."
_MAX_ROWS = 128
# samples of padded clips per device call.  The workspace grows with it (about 1.1 KB per sample with the stand-in shape,
# mostly the conv-0 rows and the conv-1 operand tiles: about 2.3 GB at this budget) and is kept by the model until
# release_workspace()
_SAMPLE_BUDGET = 2 << 20

DEFAULTS = dict(hidden_size=768, num_hidden_layers=12, num_attention_heads=12, intermediate_size=3072,
                conv_dim=(512,) * 7, conv_kernel=(10, 3, 3, 3, 3, 2, 2), conv_stride=(5, 2, 2, 2, 2, 2, 2), conv_bias=False,
                num_conv_pos_embeddings=128, num_conv_pos_embedding_groups=16, layer_norm_eps=1e-5,
                feat_extract_norm="group", do_stable_layer_norm=False, feat_extract_activation="gelu", hidden_act="gelu",
                add_adapter=False, num_labels=2)


def _get(config, key):
    if isinstance(config, dict):
        if key == "num_labels" and key not in config and "id2label" in config:
            return len(config["id2label"])
        return config.get(key, DEFAULTS[key])
    return getattr(config, key, DEFAULTS[key])


def make_config(config) -> _lib.EmoConfig:
    """the C config of a Wav2Vec2Config (dict or object); mb_emo_create refuses what the kernels do not run"""
    c = _lib.EmoConfig()
    for k in ("hidden_size", "num_hidden_layers", "num_attention_heads", "intermediate_size", "num_conv_pos_embeddings",
              "num_conv_pos_embedding_groups", "num_labels"):
        setattr(c, k, int(_get(config, k)))
    dims, ks, ss = list(_get(config, "conv_dim")), list(_get(config, "conv_kernel")), list(_get(config, "conv_stride"))
    if not (len(dims) == len(ks) == len(ss)) or not 1 <= len(dims) <= 8:
        raise _lib.MbError(f"conv_dim / conv_kernel / conv_stride must have one equal length in 1..8 ({dims}, {ks}, {ss})")
    c.num_conv_layers = len(dims)
    for i in range(len(dims)):
        c.conv_dim[i], c.conv_kernel[i], c.conv_stride[i] = int(dims[i]), int(ks[i]), int(ss[i])
    c.conv_bias = int(bool(_get(config, "conv_bias")))
    c.layer_norm_eps = float(_get(config, "layer_norm_eps"))
    c.feat_extract_norm = {"layer": 0, "group": 1}.get(_get(config, "feat_extract_norm"), -1)
    c.do_stable_layer_norm = int(bool(_get(config, "do_stable_layer_norm")))
    c.feat_extract_activation = 0 if _get(config, "feat_extract_activation") == "gelu" else 1
    c.hidden_act = 0 if _get(config, "hidden_act") == "gelu" else 1
    c.add_adapter = int(bool(_get(config, "add_adapter")))
    return c


def fold_pos_conv(sd: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
    """the positional conv's weight norm (dim=2, one norm per tap) folded into one weight, from either key spelling"""
    sd = dict(sd)
    for new, old in (("weight_g", "parametrizations.weight.original0"), ("weight_v", "parametrizations.weight.original1")):
        if _POS + old in sd:
            sd[_POS + new] = sd.pop(_POS + old)
    pos = {k: v for k, v in sd.items() if k.startswith(_POS + "weight_")}
    rest = {k: v for k, v in sd.items() if not k.startswith(_POS + "weight_")}
    rest.update(fold_weight_norm(pos, dim=2))
    return rest


class EmotionExtractorModel:
    def __init__(self, config):
        self.config = config
        self.hidden_size = int(_get(config, "hidden_size"))
        self.num_labels = int(_get(config, "num_labels"))
        cfg = make_config(config)
        self._handle = C.c_void_p()
        _lib.check(_lib.lib().mb_emo_create(C.byref(cfg), C.byref(self._handle)))
        self._weights = None
        self._arena = None
        self._device = None
        self._ws = None

    @classmethod
    def from_pretrained(cls, path, **_):
        """a downloaded snapshot: config.json plus pytorch_model.bin or model.safetensors"""
        d = Path(path)
        if not d.is_dir():
            raise _lib.MbError(f"from_pretrained needs a local directory holding config.json and the weights "
                               f"(pytorch_model.bin or model.safetensors); {str(path)!r} is not one. Download the "
                               "snapshot first (mockingbird_b200 does not fetch from the hub)")
        config = json.loads((d / "config.json").read_text())
        if (d / "model.safetensors").is_file():
            from safetensors.torch import load_file

            sd = load_file(str(d / "model.safetensors"))
        elif (d / "pytorch_model.bin").is_file():
            sd = torch.load(d / "pytorch_model.bin", map_location="cpu", weights_only=True)
        else:
            raise _lib.MbError(f"{d} has neither model.safetensors nor pytorch_model.bin")
        m = cls(config)
        m.load_state_dict(sd)
        return m

    def load_state_dict(self, sd, strict: bool = True):
        self._weights = {k: v.detach().float().cpu() for k, v in fold_pos_conv(sd).items()}
        self._arena = None
        return self

    def eval(self):
        return self

    def to(self, device):
        device = torch.device(device)
        if device.type != "cuda":
            raise _lib.MbError("mockingbird_b200 EmotionExtractorModel runs on CUDA only (no CPU fallback)")
        if device.index is None:
            device = torch.device("cuda", torch.cuda.current_device())
        if device != self._device:
            self._device, self._arena = device, None
        return self

    def cuda(self):
        return self.to(_lib.require_cuda())

    def num_frames(self, n_samples: int) -> int:
        return int(_lib.lib().mb_emo_num_frames(self._handle, int(n_samples)))

    def _prepare(self):
        if self._weights is None:
            raise _lib.MbError("EmotionExtractorModel has no weights: call load_state_dict first")
        self._device = self._device or _lib.require_cuda()
        if self._arena is None:
            self._arena = _lib.upload_weights("emo", self._handle, self._weights, self._device, align=1024)

    def _forward(self, wav: torch.Tensor, lengths: List[int], normalize: bool, normed: bool, hidden: bool):
        """one device call over clips concatenated in `wav` (float32 on the device)"""
        Lb = _lib.lib()
        B = len(lengths)
        ns = (C.c_int32 * B)(*lengths)
        need = int(Lb.mb_emo_workspace_bytes(self._handle, B, max(lengths)))
        dev = self._device
        emb = torch.empty(B, self.hidden_size, device=dev)
        logits = torch.empty(B, self.num_labels, device=dev)
        nrm = torch.empty_like(wav) if normed and normalize else None
        hid = torch.empty(B, self.num_frames(max(lengths)), self.hidden_size, device=dev) if hidden else None
        with torch.cuda.device(dev):
            ws = _lib.workspace(need, dev, self)
            stream = torch.cuda.current_stream(dev).cuda_stream
            ptr = lambda t: C.c_void_p(t.data_ptr()) if t is not None else None  # noqa: E731
            _lib.check(Lb.mb_emo_forward(self._handle, ptr(wav), ns, B, int(normalize), ptr(emb), ptr(logits), ptr(nrm), ptr(hid), ptr(ws),
                                         ws.numel(), C.c_void_p(stream)))
        return emb, logits, nrm, hid

    def run_clips(self, clips: Sequence, normalize: bool = True, normed: bool = False, hidden: bool = False):
        """ragged clips (1-D arrays or tensors) -> per clip (emb, logits[, normed][, hidden]) on the device.  normalize: the
        clips are raw samples and go through the feature extractor's normalisation first (normed returns its output);
        otherwise they are the model's input_values.  Clips are grouped by length into calls of at most 128 clips and a
        bounded sample count; each clip is its own B = 1 call."""
        self._prepare()
        xs = [torch.as_tensor(np.asarray(c, dtype=np.float32) if not torch.is_tensor(c) else c).float().reshape(-1)
              for c in clips]
        for i, x in enumerate(xs):
            if self.num_frames(x.numel()) < 1:
                raise ValueError(f"clip {i} has {x.numel()} samples: too short for one frame")
        order = sorted(range(len(xs)), key=lambda i: -xs[i].numel())
        out = [None] * len(xs)
        i = 0
        while i < len(order):
            n_max = xs[order[i]].numel()
            j = i + 1
            while j < len(order) and j - i < _MAX_ROWS and (j - i + 1) * n_max <= _SAMPLE_BUDGET:
                j += 1
            idx = order[i:j]
            wav = torch.cat([xs[k] for k in idx]).to(self._device, non_blocking=True)
            lens = [xs[k].numel() for k in idx]
            emb, logits, nrm, hid = self._forward(wav, lens, normalize, normed, hidden)
            offs = np.cumsum([0] + lens)
            for r, k in enumerate(idx):
                o = [emb[r], logits[r]]
                if normed and normalize:
                    o.append(nrm[offs[r]:offs[r + 1]])
                if hidden:
                    o.append(hid[r, :self.num_frames(lens[r])])
                out[k] = tuple(o)
            i = j
        return out

    def __call__(self, input_values) -> Tuple[torch.Tensor, torch.Tensor]:
        x = torch.as_tensor(input_values)
        if x.dim() != 2:
            raise ValueError(f"input_values must be [batch, samples], got shape {tuple(x.shape)}")
        rows = self.run_clips(list(x.float().cpu()), normalize=False)
        return torch.stack([r[0] for r in rows]), torch.stack([r[1] for r in rows])

    def release_workspace(self):
        self._ws = None

    def __del__(self):
        try:
            if getattr(self, "_handle", None) is not None and self._handle.value:
                _lib.lib().mb_emo_destroy(self._handle)
                self._handle = C.c_void_p()
        except Exception:
            pass
