"""TEST INFRASTRUCTURE ONLY - CPU restatement of the speaker encoder (torch fp32 tensor ops, explicit
LSTM recurrence).  Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline leg may import it.

Follows models/encoder/model.py:41-61 (SpeakerEncoder.forward: nn.LSTM(40, 256, 3, batch_first) ->
hidden[-1] -> Linear -> ReLU -> x / (||x|| + 1e-5)) and models/encoder/inference.py:160-166 (utterance
embedding = L2 of the mean partial embedding).  LSTM cell equations: ATen lstm_cell, gates [i, f, g, o].
Pinned against the live reference by tests/golden/encoder_seed0.npz (oracle/make_golden_encoder.py).
"""
from __future__ import annotations

from typing import Dict

import numpy as np
import torch


def lstm_stack(x: torch.Tensor, sd: Dict[str, torch.Tensor], layers: int) -> torch.Tensor:
    """x [B, T, C] -> last hidden state of the top layer [B, H]"""
    B, T, _ = x.shape
    seq = x
    for l in range(layers):
        w_ih, w_hh = sd[f"lstm.weight_ih_l{l}"], sd[f"lstm.weight_hh_l{l}"]
        b_ih, b_hh = sd[f"lstm.bias_ih_l{l}"], sd[f"lstm.bias_hh_l{l}"]
        H = w_hh.shape[1]
        h = torch.zeros(B, H)
        c = torch.zeros(B, H)
        xp = seq @ w_ih.t() + b_ih
        outs = []
        for t in range(T):
            g = xp[:, t] + h @ w_hh.t() + b_hh
            i, f, gg, o = g.chunk(4, dim=1)
            c = torch.sigmoid(f) * c + torch.sigmoid(i) * torch.tanh(gg)
            h = torch.sigmoid(o) * torch.tanh(c)
            outs.append(h)
        seq = torch.stack(outs, dim=1)
    return seq[:, -1]


def embed_frames(sd: Dict[str, torch.Tensor], frames: torch.Tensor, layers: int = 3) -> torch.Tensor:
    """SpeakerEncoder.forward (model.py:41-61)"""
    with torch.no_grad():
        h = lstm_stack(frames.float(), sd, layers)
        raw = torch.relu(h @ sd["linear.weight"].t() + sd["linear.bias"])
        return raw / (torch.norm(raw, dim=1, keepdim=True) + 1e-5)


def embed_utterance_partials(sd: Dict[str, torch.Tensor], partial_frames: torch.Tensor) -> np.ndarray:
    """inference.py:160-166: partial_frames [P, n_frames, 40] -> utterance embedding [256] (numpy fp32)"""
    pe = embed_frames(sd, partial_frames).numpy()
    raw = np.mean(pe, axis=0)
    return raw / np.linalg.norm(raw, 2)


def reduce_partials(partial, offsets):
    """inference.py:164-166 per utterance u (partials offsets[u] .. offsets[u + 1]): e = mean of its partial embeddings, e / |e|,
    in float64, with the bound of an fp32 evaluation in any summation order (n partials, E features, u = 2^-24):
    mean: gamma(n + 2) sum |p| / n (n - 1 additions, the rounded 1 / n and the product); |e|^2: gamma(E + 6) |e|^2 plus the
    propagated 2 sum |e_j| d_j; 1 / sqrt: half the relative error of |e|^2 and 3 u (sqrt, reciprocal); the product one u."""
    p = np.asarray(partial, np.float64)
    off = np.asarray(offsets)
    U, E = len(off) - 1, p.shape[1]
    u24 = 2.0 ** -24

    def gamma(n):
        return n * u24 / (1 - n * u24)

    out, bound = np.zeros((U, E)), np.zeros((U, E))
    for i in range(U):
        blk = p[off[i]:off[i + 1]]
        n = blk.shape[0]
        mean = blk.mean(0)
        dm = gamma(n + 2) * np.abs(blk).sum(0) / n
        ss = float(mean @ mean)
        dss = gamma(E + 6) * ss + 2 * float(np.abs(mean) @ dm) + float(dm @ dm)
        inv = 1.0 / np.sqrt(ss)
        dinv = inv * (dss / ss / 2 * 1.01 + 3 * u24)
        out[i] = mean * inv
        bound[i] = dm * inv + np.abs(mean) * dinv + u24 * np.abs(out[i])
    return out, bound
