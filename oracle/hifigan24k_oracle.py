"""CPU oracle for the 24 kHz HiFi-GAN generator (TEST INFRASTRUCTURE, not product code).

A plain torch-CPU fp32 restatement of the reference's ``Generator.forward`` (models/vocoder/hifigan/models.py:134-150) for
``h.sampling_rate == 24000``, where every upsampling layer is ``Sequential(InterpolationBlock(u), Conv1d(k, padding=(k-1)//2))``
(models.py:74-91, :107-118) instead of a ConvTranspose1d.  Shares the resblock / MRF / conv_post restatement with
``gan_oracle.hifigan_forward`` (which covers the other sampling rates); ``sd`` uses the checkpoint's keys (``ups.{i}.1.weight``)
and must be weight-norm folded.  Pinned against the live reference by tests/test_hifigan24k_cpu.py and the fixture
tests/golden/hifigan24k_seed0.npz (oracle/make_golden_hifigan24k.py).
"""
from __future__ import annotations

from typing import Dict

import torch
import torch.nn.functional as F

import gan_oracle as go


def interpolate_nearest(x: torch.Tensor, u: int) -> torch.Tensor:
    """InterpolationBlock(u).forward (models.py:82-91): nearest to size L*u, recompute_scale_factor=False"""
    return F.interpolate(x, size=x.shape[-1] * u, mode="nearest", align_corners=None, recompute_scale_factor=False)


def hifigan24k_forward(sd: Dict[str, torch.Tensor], cfg: dict, mel: torch.Tensor, quant: go.Quant = None) -> torch.Tensor:
    """mel [B,80,T] fp32 -> wav [B,1,T*prod(upsample_rates)]"""
    assert cfg.get("sampling_rate") == 24000, "the 24 kHz generator builds InterpolationBlock upsampling only at 24000 Hz"
    x = go._conv(mel, sd["conv_pre.weight"], sd["conv_pre.bias"], 1, 3, quant, "io")
    for i, (u, k) in enumerate(zip(cfg["upsample_rates"], cfg["upsample_kernel_sizes"])):
        x = F.leaky_relu(x, go.LRELU_SLOPE)
        x = interpolate_nearest(x, u)
        x = go._conv(x, sd[f"ups.{i}.1.weight"], sd[f"ups.{i}.1.bias"], 1, (k - 1) // 2, quant, "up")
        x = go._mrf(sd, cfg, i, x, quant)
    x = F.leaky_relu(x)  # default slope 0.01 (models.py:146)
    x = go._conv(x, sd["conv_post.weight"], sd["conv_post.bias"], 1, 3, quant, "io")
    return torch.tanh(x)


def fold_taps(u: int, k: int):
    """The polyphase lowering of nearest-upsample-by-u + Conv1d(k, padding=(k-1)//2), k odd: for each output phase r < u the list
    of (input offset d, first j, last j) in ascending d, where the kernel taps j = first .. last all read input row q + d."""
    p = (k - 1) // 2
    out = []
    for r in range(u):
        taps = {}
        for j in range(k):
            d = (r + j - p) // u
            lo, hi = taps.get(d, (j, j))
            taps[d] = (min(lo, j), max(hi, j))
        out.append([(d, lo, hi) for d, (lo, hi) in sorted(taps.items())])
    return out


def folded_forward(x: torch.Tensor, w: torch.Tensor, b: torch.Tensor, u: int, wround=None) -> torch.Tensor:
    """the folded layer evaluated directly: y[:, :, q*u + r] = b + sum_d V[r][d] x[:, :, q + d] (zero outside [0, L)); V summed
    in ascending j in w's dtype (then passed through ``wround``, if given) and applied in x's dtype.  Equal to
    conv1d(interpolate_nearest(x, u), w, b, padding=(k-1)//2) up to summation order."""
    B, _, L = x.shape
    k = w.shape[2]
    y = torch.zeros(B, w.shape[0], L * u, dtype=x.dtype, device=x.device)
    for r, taps in enumerate(fold_taps(u, k)):
        acc = b.to(x.dtype).view(1, -1, 1).expand(B, -1, L).clone()
        for d, lo, hi in taps:
            v = w[:, :, lo]
            for j in range(lo + 1, hi + 1):
                v = v + w[:, :, j]
            if wround is not None:
                v = wround(v)
            v = v.to(x.dtype)
            xs = torch.zeros_like(x)
            if d >= 0:
                xs[:, :, : max(L - d, 0)] = x[:, :, d:]
            else:
                xs[:, :, -d:] = x[:, :, : L + d]
            acc = acc + torch.einsum("oc,bcl->bol", v, xs)
        y[:, :, r::u] = acc
    return y
