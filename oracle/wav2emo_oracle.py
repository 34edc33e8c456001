"""Float64 restatement of the wav2vec2 emotion model (models/synthesizer/models/wav2emo.py EmotionExtractorModel on
transformers' Wav2Vec2Model with feat_extract_norm="layer", do_stable_layer_norm=True) and of the feature extractor's
normalisation (TEST INFRASTRUCTURE).  Written from the model's definition; imports neither transformers nor the reference.

forward(sd, cfg, x, dtype=torch.float64) runs one clip x (the normalised float32 samples, 1-D) and returns a dict:
  emb [D], logits [num_labels], and the taps features (after the conv stack, [T][C]), proj (after the feature projection),
  pos (after the positional conv is added), layer<i> (after encoder layer i), last (after the final LayerNorm).
"""
from __future__ import annotations

import math

import numpy as np
import torch
import torch.nn.functional as F


def normalize(x: np.ndarray) -> np.ndarray:
    """Wav2Vec2FeatureExtractor.zero_mean_unit_var_norm of one clip, in numpy float32 as the feature extractor runs it"""
    x = np.asarray(x, dtype=np.float32)
    return (x - x.mean()) / np.sqrt(x.var() + 1e-7)


def num_frames(cfg: dict, n: int) -> int:
    t = n
    for k, s in zip(cfg["conv_kernel"], cfg["conv_stride"]):
        if t < k:
            return 0
        t = (t - k) // s + 1
    return t


def pos_conv_weight(sd: dict, dtype=torch.float64) -> torch.Tensor:
    """the positional conv's weight norm (dim=2: one norm per tap over output and input channels), in either spelling"""
    p = "wav2vec2.encoder.pos_conv_embed.conv."
    if p + "weight" in sd:
        return sd[p + "weight"].to(dtype)
    g = sd.get(p + "parametrizations.weight.original0", sd.get(p + "weight_g")).to(dtype)
    v = sd.get(p + "parametrizations.weight.original1", sd.get(p + "weight_v")).to(dtype)
    return v * (g / v.pow(2).sum(dim=(0, 1), keepdim=True).sqrt())


def _ln(x, sd, name, eps):
    return F.layer_norm(x, x.shape[-1:], sd[name + ".weight"].to(x.dtype), sd[name + ".bias"].to(x.dtype), eps)


def _lin(x, sd, name):
    return x @ sd[name + ".weight"].to(x.dtype).T + sd[name + ".bias"].to(x.dtype)


def forward(sd: dict, cfg: dict, x, dtype=torch.float64) -> dict:
    """dtype: float64 for the tests; float32 gives the same graph as a host-thread baseline"""
    taps = {}
    h = torch.as_tensor(np.asarray(x, dtype=np.float32)).to(dtype)[None, None]  # [1, 1, n]
    for i, (k, s) in enumerate(zip(cfg["conv_kernel"], cfg["conv_stride"])):
        b = f"wav2vec2.feature_extractor.conv_layers.{i}."
        bias = sd[b + "conv.bias"].to(dtype) if cfg["conv_bias"] else None
        h = F.conv1d(h, sd[b + "conv.weight"].to(dtype), bias, stride=s)
        h = F.gelu(_ln(h.transpose(1, 2), sd, b + "layer_norm", 1e-5)).transpose(1, 2)
    h = h[0].T  # [T][C]
    taps["features"] = h
    eps = cfg["layer_norm_eps"]
    h = _lin(_ln(h, sd, "wav2vec2.feature_projection.layer_norm", eps), sd, "wav2vec2.feature_projection.projection")
    taps["proj"] = h
    k, G = cfg["num_conv_pos_embeddings"], cfg["num_conv_pos_embedding_groups"]
    pc = F.conv1d(h.T[None], pos_conv_weight(sd, dtype), sd["wav2vec2.encoder.pos_conv_embed.conv.bias"].to(dtype), padding=k // 2,
                  groups=G)
    if k % 2 == 0:
        pc = pc[:, :, :-1]
    h = h + F.gelu(pc[0].T)
    taps["pos"] = h
    D, H = cfg["hidden_size"], cfg["num_attention_heads"]
    dk = D // H
    T = h.shape[0]
    for i in range(cfg["num_hidden_layers"]):
        b = f"wav2vec2.encoder.layers.{i}."
        a = _ln(h, sd, b + "layer_norm", eps)
        q = _lin(a, sd, b + "attention.q_proj").reshape(T, H, dk).transpose(0, 1)
        kk = _lin(a, sd, b + "attention.k_proj").reshape(T, H, dk).transpose(0, 1)
        v = _lin(a, sd, b + "attention.v_proj").reshape(T, H, dk).transpose(0, 1)
        p = torch.softmax(q @ kk.transpose(1, 2) / math.sqrt(dk), dim=-1)
        ctx = (p @ v).transpose(0, 1).reshape(T, D)
        h = h + _lin(ctx, sd, b + "attention.out_proj")
        f = _ln(h, sd, b + "final_layer_norm", eps)
        f = _lin(F.gelu(_lin(f, sd, b + "feed_forward.intermediate_dense")), sd, b + "feed_forward.output_dense")
        h = h + f
        taps[f"layer{i}"] = h
    h = _ln(h, sd, "wav2vec2.encoder.layer_norm", eps)
    taps["last"] = h
    emb = h.mean(dim=0)
    logits = _lin(torch.tanh(_lin(emb, sd, "classifier.dense")), sd, "classifier.out_proj")
    taps["emb"] = emb
    taps["logits"] = logits
    return taps
