"""Float64 references of one FP32 tap-conv launch (csrc/gan_fp32.cu) and of the fp16 planes its epilogue writes, for the
launch-level tests in tests/test_gan_fp32_layers.py (their CPU self-tests are in the same file).

A launch computes  v = op(act(x)) + bias (+ residual), then the accumulate mode, tanh, the output length mask, and optionally
a second destination y2 += v.  op is a Conv1d, a ConvTranspose1d (a polyphase bank) or nearest upsample + Conv1d (folded slabs).
The references evaluate op in float64 from the checkpoint tensors; the input activation is evaluated in fp32 as the kernel does
(tc_pair_oracle.act32), so the only differences left are the kernel's fp32 summation order and its fp32 fold of nearest slabs.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

import tc_pair_oracle as po


def op_forward(a: torch.Tensor, w: torch.Tensor, b: torch.Tensor, kind: str, *, dil: int = 1, stride: int = 1) -> torch.Tensor:
    """float64 op of an already activated input.  kind "conv": Conv1d weight [Cout, Cin, k], padding (k - 1) * dil / 2;
    "transposed": ConvTranspose1d weight [Cin, Cout, k], stride u, padding u/2 + u%2, output_padding u%2 (models.py:120-123);
    "nearest": nearest upsample by u, then Conv1d weight [Cout, Cin, k] (k odd), padding (k - 1) / 2"""
    a, w, b = a.double(), w.double(), b.double()
    k = w.shape[2]
    if kind == "transposed":
        u = stride
        return F.conv_transpose1d(a, w, b, u, u // 2 + u % 2, u % 2)
    if kind == "nearest":
        return F.conv1d(a.repeat_interleave(stride, dim=2), w, b, padding=(k - 1) // 2)
    return F.conv1d(a, w, b, padding=(k - 1) * dil // 2, dilation=dil)


def tapconv_reference(x, w, b, kind, *, dil=1, stride=1, slope_in=1.0, x_f16=False, res=None, mode="store", y0=None, div=1.0,
                      tanh=False, valid_in=None, valid_out=None, y2_0=None):
    """float64 result of one FP32 tap-conv launch and of its second destination (None without y2_0).
    x [B, Cin, L] not activated; valid_in / valid_out rows per utterance (None: all).  x_f16: the input is an fp16 plane written
    as fp16(lrelu_fp32(x)) (the kernel reads it without a further activation)."""
    B, _, L = x.shape
    a = po.act32(x, slope_in)
    if x_f16:
        a = po.q16(a)
    a = a * po.row_mask(B, L, valid_in, x.device)
    v = op_forward(a, w, b, kind, dil=dil, stride=stride)
    if res is not None:
        v = v + res.double()
    v = po.mode_apply(v, mode, y0, div)
    if tanh:
        v = torch.tanh(v)
    m = po.row_mask(B, v.shape[2], valid_out, x.device)
    y = v * m
    y2 = (y2_0.double() + y) * m if y2_0 is not None else None
    return y, y2


def tstore_planes(v: torch.Tensor, slope: float, hilo: bool):
    """the fp16 plane(s) the epilogue stores for the fp32 value v: hi = fp16_rn(lrelu(v)) and, for a hi/lo plane,
    lo = fp16_rn(lrelu(v) - hi), both evaluated in fp32 and returned as fp32 tensors"""
    a = v.float()
    a = torch.where(a > 0, a, a * slope) if slope != 1.0 else a
    hi = a.half()
    lo = (a - hi.float()).half().float() if hilo else None
    return hi.float(), lo


def fold_slabs(w: torch.Tensor, u: int):
    """the folded slabs of nearest upsample by u + Conv1d weight [Cout, Cin, k] (k odd): {(r, d): sum of the taps j with
    floor((r + j - p) / u) == d}, p = (k - 1) / 2, summed in float64"""
    k = w.shape[2]
    p = (k - 1) // 2
    out = {}
    for r in range(u):
        for j in range(k):
            d = (r + j - p) // u
            out[(r, d)] = out.get((r, d), 0) + w[:, :, j].double()
    return out


def folded_forward(a: torch.Tensor, w: torch.Tensor, b: torch.Tensor, u: int) -> torch.Tensor:
    """nearest upsample + Conv1d evaluated as the kernel evaluates it: output phase r of row q reads input row q + d through
    slab (r, d) (zero outside the input)"""
    B, _, L = a.shape
    a = a.double()
    y = torch.zeros(B, w.shape[0], L * u, dtype=torch.float64, device=a.device)
    for (r, d), s in fold_slabs(w, u).items():
        lo, hi = max(0, -d), min(L, L - d)
        if hi <= lo:
            continue
        y[:, :, r + u * lo:r + u * hi:u] += torch.einsum("oc,bcl->bol", s, a[:, :, lo + d:hi + d])
    return y + b.double().view(1, -1, 1)
