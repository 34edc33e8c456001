"""Plain-torch restatement of the PPG extractor's forward (models/ppg_extractor: PPGModel.forward with B = 1), pinned to
the live reference by tests/test_ppgx_cpu.py and runnable where the reference is absent (GPU tests, smoke, bench).

  frontend   stft.py:70-81      torch.stft without a window (rectangular, win_length ones centred in n_fft), center=True,
                                reflect padding; power re^2 + im^2 (frontend.py:98)
             log_mel.py:66-73   log(power @ melmat + 1e-20)
  normalize  utterance_mvn.py   mean over the utterance's frames; norm_vars divides by clamp(sqrt(var), 1e-20) ** 0.5
  embed      subsampling.py     conv -> ReLU -> conv -> ReLU over [1, 1, T, n_mels], (c, f) flattened c-major, Linear,
                                positional encoding (embedding.py): x * sqrt(D) (+ pe[:T] for abs_pos)
  blocks     encoder_layer.py   macaron FFN (1/2), MHSA, conv module, FFN (1/2), norm_final; LayerNorm eps 1e-12
  attention  attention.py       rel_pos: ((q + u) k^T + rel_shift((q + v) p^T)) / sqrt(d_k), legacy ESPnet rel_shift
"""
from __future__ import annotations

import math
from typing import Dict, List, Optional, Tuple

import torch
import torch.nn.functional as F

PE_MAX_LEN = 5000  # PositionalEncoding(max_len=5000): the table is built at construction and only ever grows


def stft_params(cfg: dict):
    """(n_fft, win_length, hop_length) with DefaultFrontend's defaults (frontend.py:17-35: 1024, 800, 160; a None
    win_length is n_fft, stft.py:24-27)"""
    fe = cfg["frontend_conf"]
    n_fft = fe.get("n_fft", 1024)
    win = fe.get("win_length", 800)
    return n_fft, n_fft if win is None else win, fe.get("hop_length", 160)


def pos_table(d_model: int, pe_len: int, reverse: bool) -> torch.Tensor:
    """PositionalEncoding.extend_pe (embedding.py:56-77) for a table of pe_len rows: [pe_len, d_model].  Built at full
    length exactly as the reference does, so every element comes out of the same torch sin / cos calls."""
    pe = torch.zeros(pe_len, d_model)
    if reverse:
        position = torch.arange(pe_len - 1, -1, -1.0, dtype=torch.float32).unsqueeze(1)
    else:
        position = torch.arange(0, pe_len, dtype=torch.float32).unsqueeze(1)
    div_term = torch.exp(torch.arange(0, d_model, 2, dtype=torch.float32) * -(math.log(10000.0) / d_model))
    pe[:, 0::2] = torch.sin(position * div_term)
    pe[:, 1::2] = torch.cos(position * div_term)
    return pe


def num_frames(cfg: dict, n_samples: int) -> int:
    t = 1 + n_samples // stft_params(cfg)[2]
    enc = cfg["encoder_conf"]
    if not enc.get("no_subsample", False):
        t //= 2
        if not enc.get("subsample_by_2", False):
            t //= 2
    return t


def features(sd: Dict[str, torch.Tensor], cfg: dict, wav: torch.Tensor) -> torch.Tensor:
    """wav [L] -> normalised log-mel [T_stft, n_mels]"""
    nc = cfg["normalize_conf"]
    n_fft, win, hop = stft_params(cfg)
    spec = torch.stft(wav[None].float(), n_fft=n_fft, win_length=win, hop_length=hop, center=True, pad_mode="reflect",
                      normalized=False, onesided=True, return_complex=True)
    power = (spec.real ** 2 + spec.imag ** 2).transpose(1, 2)  # [1, T, F]
    x = (torch.matmul(power, sd["frontend.logmel.melmat"].float()) + 1e-20).log()
    n = x.shape[1]
    mean = x.sum(dim=1, keepdim=True) / n
    if nc.get("norm_means", True):
        x = x - mean
        if nc.get("norm_vars", False):
            var = x.pow(2).sum(dim=1, keepdim=True) / n
            x = x / torch.clamp(var.sqrt(), min=1e-20).sqrt()
    elif nc.get("norm_vars", False):
        var = (x - mean).pow(2).sum(dim=1, keepdim=True) / n
        x = x / torch.clamp(var.sqrt(), min=1e-20)
    return x[0]


def conv_specs(cfg: dict) -> List[Tuple[int, int, int]]:
    """(kernel, stride, padding) of embed.conv.0 and embed.conv.2"""
    enc = cfg["encoder_conf"]
    if enc.get("no_subsample", False):
        return [(5, 1, 2), (5, 1, 2)]
    if enc.get("subsample_by_2", False):
        return [(5, 1, 2), (4, 2, 1)]
    return [(4, 2, 1), (4, 2, 1)]


def rel_shift(x: torch.Tensor) -> torch.Tensor:
    """the reference's legacy rel_shift (attention.py:124-140) of [..., T, T]"""
    zero_pad = torch.zeros((*x.size()[:-1], 1), dtype=x.dtype)
    x_padded = torch.cat([zero_pad, x], dim=-1)
    x_padded = x_padded.view(*x.size()[:-2], x.size(-1) + 1, x.size(-2))
    return x_padded[..., 1:, :].view_as(x)


def rel_shift_closed_form(bd: torch.Tensor) -> torch.Tensor:
    """element (i, j) of rel_shift(bd) for a square [T, T] bd: bd[i][T-1-i+j] for j <= i, 0 for j = i+1 and the NEXT
    query row's bd[i+1][j-i-2] for j > i+1 - what the attention kernel computes on the fly"""
    T = bd.shape[-1]
    out = torch.zeros_like(bd)
    for i in range(T):
        for j in range(T):
            if j <= i:
                out[..., i, j] = bd[..., i, T - 1 - i + j]
            elif j > i + 1:
                out[..., i, j] = bd[..., i + 1, j - i - 2]
    return out


def attention(q, kk, v, pp=None, pos_u=None, pos_v=None):
    """softmax(scores) . V of one utterance: q [1, T, H, dk], kk / v / pp [1, H, T, dk] (pp = linear_pos(pos_emb), rel_pos
    only), pos_u / pos_v [H, dk] -> [1, T, H dk].  rel_pos (pp given): ((q + u) k^T + rel_shift((q + v) p^T)) / sqrt(dk)"""
    dk = q.shape[-1]
    if pp is not None:
        qu = (q + pos_u).transpose(1, 2)
        qv = (q + pos_v).transpose(1, 2)
        scores = (torch.matmul(qu, kk.transpose(-2, -1)) + rel_shift(torch.matmul(qv, pp.transpose(-2, -1)))) / math.sqrt(dk)
    else:
        scores = torch.matmul(q.transpose(1, 2), kk.transpose(-2, -1)) / math.sqrt(dk)
    return torch.matmul(torch.softmax(scores, dim=-1), v).transpose(1, 2).contiguous().view(1, q.shape[1], -1)


def _ln(x, sd, name):
    return F.layer_norm(x, (x.shape[-1],), sd[name + ".weight"], sd[name + ".bias"], 1e-12)


def _lin(x, sd, name, bias=True):
    return F.linear(x, sd[name + ".weight"], sd[name + ".bias"] if bias else None)


def _act(x, kind):
    return x * torch.sigmoid(x) if kind == "swish" else torch.relu(x)


def forward(sd: Dict[str, torch.Tensor], cfg: dict, wav: torch.Tensor, pe_len: Optional[int] = None,
            taps: bool = False):
    """one utterance wav [L] -> PPG [T, D] (and, with taps=True, the list [embed output, block 0 .. n-1 outputs]).
    pe_len: rows of the positional table (default max(5000, T)), the module instance's high-water mark."""
    enc = cfg["encoder_conf"]
    D, H = enc["attention_dim"], enc["attention_heads"]
    dk = D // H
    act = enc.get("activation_type", "swish")
    rel = enc.get("pos_enc_layer_type", "abs_pos") == "rel_pos"
    sd = {k: v.float() for k, v in sd.items()}
    x = features(sd, cfg, wav)[None, None]  # [1, 1, T, F]
    for i, (k, s, p) in zip((0, 2), conv_specs(cfg)):
        x = torch.relu(F.conv2d(x, sd[f"encoder.embed.conv.{i}.weight"], sd[f"encoder.embed.conv.{i}.bias"], s, p))
    b, c, t, f = x.size()
    x = _lin(x.transpose(1, 2).contiguous().view(b, t, c * f), sd, "encoder.embed.out.0")
    T = x.shape[1]
    pe_len = max(PE_MAX_LEN, T) if pe_len is None else pe_len
    pe = pos_table(D, pe_len, reverse=rel)[None]
    x = x * math.sqrt(D)
    if rel:
        pos_emb = pe[:, :T]
    else:
        x = x + pe[:, :T]
    out_taps = [x[0].clone()]
    for blk in range(enc["num_blocks"]):
        pre = f"encoder.encoders.{blk}"
        macaron = f"{pre}.feed_forward_macaron.w_1.weight" in sd
        scale = 0.5 if macaron else 1.0
        if macaron:
            h = _ln(x, sd, pre + ".norm_ff_macaron")
            x = x + scale * _lin(_act(_lin(h, sd, pre + ".feed_forward_macaron.w_1"), act), sd,
                                 pre + ".feed_forward_macaron.w_2")
        h = _ln(x, sd, pre + ".norm_mha")
        q = _lin(h, sd, pre + ".self_attn.linear_q").view(1, T, H, dk)
        kk = _lin(h, sd, pre + ".self_attn.linear_k").view(1, T, H, dk).transpose(1, 2)
        v = _lin(h, sd, pre + ".self_attn.linear_v").view(1, T, H, dk).transpose(1, 2)
        pp = None
        if rel:
            pp = F.linear(pos_emb, sd[pre + ".self_attn.linear_pos.weight"]).view(1, -1, H, dk).transpose(1, 2)
        a = attention(q, kk, v, pp, sd.get(pre + ".self_attn.pos_bias_u"), sd.get(pre + ".self_attn.pos_bias_v"))
        x = x + _lin(a, sd, pre + ".self_attn.linear_out")
        if f"{pre}.conv_module.pointwise_conv1.weight" in sd:
            cm = pre + ".conv_module"
            h = _ln(x, sd, pre + ".norm_conv").transpose(1, 2)
            h = F.glu(F.conv1d(h, sd[cm + ".pointwise_conv1.weight"], sd[cm + ".pointwise_conv1.bias"]), dim=1)
            K = sd[cm + ".depthwise_conv.weight"].shape[-1]
            h = F.conv1d(h, sd[cm + ".depthwise_conv.weight"], sd[cm + ".depthwise_conv.bias"], padding=(K - 1) // 2, groups=D)
            h = F.batch_norm(h, sd[cm + ".norm.running_mean"], sd[cm + ".norm.running_var"], sd[cm + ".norm.weight"],
                             sd[cm + ".norm.bias"], False, 0.0, 1e-5)
            h = F.conv1d(_act(h, act), sd[cm + ".pointwise_conv2.weight"], sd[cm + ".pointwise_conv2.bias"])
            x = x + h.transpose(1, 2)
        h = _ln(x, sd, pre + ".norm_ff")
        x = x + scale * _lin(_act(_lin(h, sd, pre + ".feed_forward.w_1"), act), sd, pre + ".feed_forward.w_2")
        if f"{pre}.norm_final.weight" in sd:
            x = _ln(x, sd, pre + ".norm_final")
        out_taps.append(x[0].clone())
    x = _ln(x, sd, "encoder.after_norm")[0]
    return (x, out_taps) if taps else x
