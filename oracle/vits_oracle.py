"""Float64 restatement of VITS inference (models/synthesizer/models/vits.py:498-527 and the modules it calls).

Written from the equations, not from the reference source: each function below states one stage the way the CUDA kernels of
csrc/vits.cu compute it, in float64 torch, on a state dict with folded weight norm (synth_weights/ref_init.vits_state_dict).
tests/test_vits_cpu.py pins the whole chain to the goldens recorded from the live reference; tests/test_vits_kernels.py
checks each kernel stage against the matching function here.
"""
from __future__ import annotations

import math
from typing import Dict, Optional

import numpy as np
import torch
import torch.nn.functional as F

WINDOW = 4
BINS = 10
TAIL = 5.0
MIN_BIN = 1e-3
MIN_DERIV = 1e-3


def _d(t) -> torch.Tensor:
    return torch.as_tensor(np.asarray(t) if not torch.is_tensor(t) else t).to(torch.float64)


def mask_of(lengths, T: int) -> torch.Tensor:
    """[B, 1, T] float64, 1 for t < length"""
    lengths = torch.as_tensor(lengths).to(torch.int64)
    return (torch.arange(T)[None, :] < lengths[:, None]).to(torch.float64)[:, None, :]


def conv(sd, name, x, pad: Optional[int] = None, groups: int = 1, dilation: int = 1, bias: bool = True):
    w = _d(sd[name + ".weight"])
    k = w.shape[-1]
    p = (k - 1) * dilation // 2 if pad is None else pad
    b = _d(sd[name + ".bias"]) if bias and (name + ".bias") in sd else None
    return F.conv1d(x, w, b, padding=p, groups=groups, dilation=dilation)


def layer_norm(sd, name, x):
    """LayerNorm over channels of [B, C, T], eps 1e-5"""
    mu = x.mean(1, keepdim=True)
    var = ((x - mu) ** 2).mean(1, keepdim=True)
    return (x - mu) / torch.sqrt(var + 1e-5) * _d(sd[name + ".gamma"])[None, :, None] + _d(sd[name + ".beta"])[None, :, None]


def gelu(x):
    return 0.5 * x * (1 + torch.erf(x / math.sqrt(2)))


# ---- text encoder ---------------------------------------------------------------------------------------------------
def rel_attention(q, k, v, erk, erv, lengths, n_heads: int):
    """multi-head self-attention with shared relative embeddings erk / erv [1, 2W+1, dk] over |s - t| <= W; padded queries
    and keys score -1e4.  q, k, v [B, H, T] -> [B, H, T]"""
    B, H, T = q.shape
    dk = H // n_heads
    qh = q.view(B, n_heads, dk, T).transpose(2, 3) / math.sqrt(dk)  # [B, nh, T, dk]
    kh = k.view(B, n_heads, dk, T).transpose(2, 3)
    vh = v.view(B, n_heads, dk, T).transpose(2, 3)
    # the relative terms live on the 2W+1 diagonals s = t + r: scores[t, t + r] += q_t . erk[r], out_t += p[t, t + r] erv[r]
    t = torch.arange(T)
    band = [(r, t[(t + r >= 0) & (t + r < T)]) for r in range(-WINDOW, WINDOW + 1)]
    rl = qh @ _d(erk)[0].T  # [B, nh, T, 2W+1]
    scores = qh @ kh.transpose(2, 3)
    for r, tt in band:
        scores[:, :, tt, tt + r] += rl[:, :, tt, r + WINDOW]
    m = mask_of(lengths, T)[:, 0]
    valid = (m[:, None, :, None] * m[:, None, None, :]) > 0
    scores = torch.where(valid, scores, torch.full_like(scores, -1e4))
    p = torch.softmax(scores, -1)
    out = p @ vh
    rv = _d(erv)[0]
    for r, tt in band:
        out[:, :, tt] += p[:, :, tt, tt + r, None] * rv[r + WINDOW]
    return out.transpose(2, 3).reshape(B, H, T)


def text_encoder_layer(sd, cfg, l: int, h, lengths, last: bool):
    """encoder layer l on h [B, H, T]: LN_1(h + conv_o(attention)), then LN_2(h + FFN(h)); masked when it is the last"""
    m = mask_of(lengths, h.shape[2])
    K = cfg["kernel_size"]
    a = f"enc_p.encoder.attn_layers.{l}"
    y = rel_attention(conv(sd, a + ".conv_q", h), conv(sd, a + ".conv_k", h), conv(sd, a + ".conv_v", h), sd[a + ".emb_rel_k"],
                      sd[a + ".emb_rel_v"], lengths, cfg["n_heads"])
    h = layer_norm(sd, f"enc_p.encoder.norm_layers_1.{l}", h + conv(sd, a + ".conv_o", y))
    f = f"enc_p.encoder.ffn_layers.{l}"
    y = torch.relu(conv(sd, f + ".conv_1", h * m, pad=(K - 1) // 2))
    y = conv(sd, f + ".conv_2", y * m, pad=(K - 1) // 2) * m
    h = layer_norm(sd, f"enc_p.encoder.norm_layers_2.{l}", h + y)
    return h * m if last else h


def text_encoder(sd, cfg, x, lengths, emo):
    H = cfg["hidden_channels"]
    T = x.shape[1]
    m = mask_of(lengths, T)
    e = _d(emo) @ _d(sd["enc_p.emo_proj.weight"]).T + _d(sd["enc_p.emo_proj.bias"])
    h = (_d(sd["enc_p.emb.weight"])[torch.as_tensor(x).long()] * math.sqrt(H) + e[:, None, :]).transpose(1, 2) * m
    for i in range(cfg["n_layers"]):
        h = text_encoder_layer(sd, cfg, i, h, lengths, i == cfg["n_layers"] - 1)
    stats = conv(sd, "enc_p.proj", h) * m
    I = cfg["inter_channels"]
    return h, stats[:, :I], stats[:, I:]


# ---- duration predictors ----------------------------------------------------------------------------------------------
def ddsconv(sd, prefix, x, lengths):
    """DDSConv: three layers of depthwise conv (dilation 3^l) over x * mask, LN, GELU, 1x1, LN, GELU, residual; x * mask"""
    m = mask_of(lengths, x.shape[2])
    C = x.shape[1]
    for l in range(3):
        d = 3 ** l
        y = conv(sd, f"{prefix}convs_sep.{l}", x * m, pad=d, groups=C, dilation=d)
        y = gelu(layer_norm(sd, f"{prefix}norms_1.{l}", y))
        y = gelu(layer_norm(sd, f"{prefix}norms_2.{l}", conv(sd, f"{prefix}convs_1x1.{l}", y)))
        x = x + y
    return x * m


def spline_inverse(params, x):
    """inverse rational-quadratic spline with linear tails at +-TAIL; params [..., 3*BINS-1] (widths, heights / sqrt(C)
    already applied, then the BINS-1 inner derivatives), x [...]"""
    uw, uh, ud = params[..., :BINS], params[..., BINS:2 * BINS], params[..., 2 * BINS:]
    edge = math.log(math.expm1(1 - MIN_DERIV))
    ud = torch.cat([torch.full_like(ud[..., :1], edge), ud, torch.full_like(ud[..., :1], edge)], -1)

    def knots(u):
        w = MIN_BIN + (1 - MIN_BIN * BINS) * torch.softmax(u, -1)
        c = torch.cat([torch.zeros_like(w[..., :1]), torch.cumsum(w, -1)], -1) * 2 * TAIL - TAIL
        c[..., 0], c[..., -1] = -TAIL, TAIL
        return c

    cw, ch = knots(uw), knots(uh)
    der = MIN_DERIV + F.softplus(ud)
    edges = ch.clone()
    edges[..., -1] += 1e-6
    k = ((x[..., None] >= edges).sum(-1) - 1).clamp(0, BINS - 1)
    g = lambda t, j: t.gather(-1, j[..., None])[..., 0]  # noqa: E731
    x0, w_k = g(cw, k), g(cw, k + 1) - g(cw, k)
    y0, h_k = g(ch, k), g(ch, k + 1) - g(ch, k)
    s = h_k / w_k
    d0, d1 = g(der, k), g(der, k + 1)
    dy = x - y0
    a = dy * (d0 + d1 - 2 * s) + h_k * (s - d0)
    b = h_k * d0 - dy * (d0 + d1 - 2 * s)
    c = -s * dy
    theta = 2 * c / (-b - torch.sqrt(b * b - 4 * a * c))
    y = theta * w_k + x0
    inside = (x >= -TAIL) & (x <= TAIL)
    return torch.where(inside, y, x)


def convflow_spline(sd, index, h, z, lengths, c0: int, c1: int):
    """the spline half of ConvFlow `index` in reverse: proj(h) * mask parametrises channel c1 of z [B, 2, T]; returns z * mask"""
    C = h.shape[1]
    m = mask_of(lengths, h.shape[2])
    p = (conv(sd, f"dp.flows.{index}.proj", h) * m).transpose(1, 2)  # [B, T, 29]
    p = torch.cat([p[..., :2 * BINS] / math.sqrt(C), p[..., 2 * BINS:]], -1)
    out = z.clone()
    out[:, c1] = spline_inverse(p, z[:, c1])
    return out * m


def logw(sd, cfg, h, lengths, g, sdp_noise, noise_scale_w):
    """logw [B, 1, T] of either duration predictor on the encoder output h, conditioned on g [B, gin] when given"""
    m = mask_of(lengths, h.shape[2])
    gb = conv(sd, "dp.cond", g[:, :, None]) if g is not None else 0
    if cfg["use_sdp"]:
        x = ddsconv(sd, "dp.convs.", conv(sd, "dp.pre", h) + gb, lengths)
        x = conv(sd, "dp.proj", x) * m
        z = _d(sdp_noise) * noise_scale_w
        c0, c1 = 1, 0
        for f in (7, 5, 3):
            hh = ddsconv(sd, f"dp.flows.{f}.convs.", conv(sd, f"dp.flows.{f}.pre", z[:, c0:c0 + 1]) + x, lengths)
            z = convflow_spline(sd, f, hh, z, lengths, c0, c1)
            c0, c1 = c1, c0
        return (z[:, :1] - _d(sd["dp.flows.0.m"])[0, 0]) * torch.exp(-_d(sd["dp.flows.0.logs"])[0, 0]) * m
    x = h + gb
    x = layer_norm(sd, "dp.norm_1", torch.relu(conv(sd, "dp.conv_1", x * m)))
    x = layer_norm(sd, "dp.norm_2", torch.relu(conv(sd, "dp.conv_2", x * m)))
    return conv(sd, "dp.proj", x * m) * m


def durations(sd, cfg, h, lengths, g, sdp_noise, noise_scale_w, length_scale):
    """w = exp(logw) * mask * length_scale (float64)"""
    m = mask_of(lengths, h.shape[2])
    return torch.exp(logw(sd, cfg, h, lengths, g, sdp_noise, noise_scale_w)) * m * length_scale


# ---- prior expansion, flow, decoder -----------------------------------------------------------------------------------
def expand(m_p, logs_p, w_ceil, x_lengths, eps, noise_scale):
    """the monotonic path of integer durations and the expanded prior: attn [B, 1, T_y, T_x], z_p, m_p_y, logs_p_y with
    T_y = eps.shape[2]"""
    w = torch.as_tensor(w_ceil).to(torch.int64) * mask_of(x_lengths, m_p.shape[2])[:, 0].to(torch.int64)
    cum = torch.cumsum(w, 1)
    y_len = cum[:, -1].clamp_min(1)
    Ty = eps.shape[2]
    j = torch.arange(Ty)
    attn = ((j[None, :, None] < cum[:, None, :]) & (j[None, :, None] >= (cum - w)[:, None, :])
            & (j[None, :, None] < y_len[:, None, None])).to(torch.float64)
    m_y = attn @ m_p.transpose(1, 2)
    l_y = attn @ logs_p.transpose(1, 2)
    m_y, l_y = m_y.transpose(1, 2), l_y.transpose(1, 2)
    return attn[:, None], m_y + _d(eps) * torch.exp(l_y) * noise_scale, m_y, l_y, y_len


def wn_layer(sd, e, l, h, out, cond, lengths):
    """WN layer l of prefix e: returns (h, out) after the residual and skip updates; cond = cond_layer(g) [B, 2H*4] or None"""
    H = h.shape[1]
    m = mask_of(lengths, h.shape[2])
    xin = conv(sd, f"{e}in_layers.{l}", h)
    if cond is not None:
        xin = xin + cond[:, 2 * H * l:2 * H * (l + 1), None]
    acts = torch.tanh(xin[:, :H]) * torch.sigmoid(xin[:, H:])
    rs = conv(sd, f"{e}res_skip_layers.{l}", acts)
    if l < 3:
        return (h + rs[:, :H]) * m, (rs[:, H:] if out is None else out + rs[:, H:])
    return h, out + rs


def coupling_reverse(sd, f: int, z, y_len, g):
    """ResidualCouplingLayer flow.flows.(2f) in reverse on z [B, inter, T] (no flip), conditioned on g [B, gin] when given"""
    I = z.shape[1]
    m = mask_of(y_len, z.shape[2])
    n = f"flow.flows.{2 * f}"
    h = conv(sd, n + ".pre", z[:, :I // 2]) * m
    cond = conv(sd, n + ".enc.cond_layer", g[:, :, None])[:, :, 0] if g is not None else None
    out = None
    for l in range(4):
        h, out = wn_layer(sd, n + ".enc.", l, h, out, cond, y_len)
    stats = conv(sd, n + ".post", out * m) * m
    return torch.cat([z[:, :I // 2], (z[:, I // 2:] - stats) * m], 1)


def flow_reverse(sd, z, y_len, g):
    for f in (3, 2, 1, 0):
        z = coupling_reverse(sd, f, torch.flip(z, [1]), y_len, g)
    return z


def decoder(sd, cfg, z, g):
    lrelu = lambda v, s=0.1: F.leaky_relu(v, s)  # noqa: E731
    x = conv(sd, "dec.conv_pre", z)
    if g is not None:
        x = x + conv(sd, "dec.cond", g[:, :, None])
    nk = len(cfg["resblock_kernel_sizes"])
    for i, (u, k) in enumerate(zip(cfg["upsample_rates"], cfg["upsample_kernel_sizes"])):
        x = F.conv_transpose1d(lrelu(x), _d(sd[f"dec.ups.{i}.weight"]), _d(sd[f"dec.ups.{i}.bias"]), stride=u, padding=(k - u) // 2)
        acc = 0
        for j, (rk, ds) in enumerate(zip(cfg["resblock_kernel_sizes"], cfg["resblock_dilation_sizes"])):
            r = f"dec.resblocks.{i * nk + j}"
            y = x
            for mi, d in enumerate(ds):
                if str(cfg["resblock"]) == "1":
                    t = conv(sd, f"{r}.convs1.{mi}", lrelu(y), dilation=d)
                    y = y + conv(sd, f"{r}.convs2.{mi}", lrelu(t))
                else:
                    y = y + conv(sd, f"{r}.convs.{mi}", lrelu(y), dilation=d)
            acc = acc + y
        x = acc / nk
    return torch.tanh(conv(sd, "dec.conv_post", F.leaky_relu(x), bias=False))


def infer(sd: Dict[str, torch.Tensor], cfg: dict, x, x_lengths, sid, emo, sdp_noise, eps, noise_scale, noise_scale_w,
          length_scale, max_len=None) -> Dict[str, torch.Tensor]:
    """Vits.infer in float64 with the given noise tensors; durations are ceil'ed from the float64 w"""
    x_lengths = torch.as_tensor(x_lengths).to(torch.int64)
    h, m_p, logs_p = text_encoder(sd, cfg, x, x_lengths, emo)
    g = _d(sd["emb_g.weight"])[torch.as_tensor(sid).long()] if cfg["n_speakers"] > 1 else None
    w = durations(sd, cfg, h, x_lengths, g, sdp_noise, noise_scale_w, length_scale)
    w_ceil = torch.ceil(w)[:, 0].to(torch.int64)
    attn, z_p, m_y, l_y, y_len = expand(m_p, logs_p, w_ceil, x_lengths, eps, noise_scale)
    z = flow_reverse(sd, z_p, y_len, g)
    zin = (z * mask_of(y_len, z.shape[2]))[:, :, :max_len]
    o = decoder(sd, cfg, zin, g)
    return dict(w=w[:, 0], w_ceil=w_ceil, y_lengths=y_len, attn=attn, m_p=m_p, logs_p=logs_p, m_p_y=m_y, logs_p_y=l_y, z_p=z_p,
                z=z, o=o)
