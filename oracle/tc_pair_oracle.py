"""Float64 references of the tensor-core tap conv's launches, rounded where the kernel rounds, and the elementwise checker
the fused-pair tests use (tests/test_gan_tc_pair.py; its sharpness is shown on CPU in tests/test_gan_tc_plan.py).

A fused resblock pair computes  y = c2(fp16(mask(lrelu(c1(a) + b1, slope_mid)))) + b2 + res  (then the accumulate mode and the
output length mask), with a = fp16(lrelu(x, slope_in)) and fp16 weights.  fp16 x fp16 products are exact in fp32, so the only
differences to a float64 evaluation are the kernel's fp32 summation order (far below 2e-5 of the output scale) and the one place
where that summation error can change a ROUNDED value: the fp16 intermediate "mid".  bound() accounts for both.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

MID_TIE_REL = 2.0 ** -20  # the kernel's fp32 c1 value is within this relative distance of the float64 one
ACC_REL = 2.0 ** -22      # fp32 accumulation error per unit of sum |terms| (K <= 11 * 64 terms, two fp32 ulps each)
TOL = 2e-5                # summation-order tolerance, relative to max |y|


def q16(t: torch.Tensor) -> torch.Tensor:
    """round to fp16 (nearest even), back in the tensor's dtype"""
    return t.half().to(t.dtype)


def act32(x: torch.Tensor, slope: float) -> torch.Tensor:
    """leaky-relu evaluated in fp32, as the conversion / epilogue kernels do, returned as float64"""
    x32 = x.float()
    return (F.leaky_relu(x32, slope) if slope != 1.0 else x32).double()


def lrelu(x: torch.Tensor, slope: float) -> torch.Tensor:
    return torch.where(x > 0, x, x * slope)


def row_mask(B: int, L: int, valid, device) -> torch.Tensor:
    """[B, 1, L] 1.0 for rows < valid[b] (valid None: all)"""
    rows = torch.arange(L, device=device).view(1, 1, L)
    if valid is None:
        return torch.ones(B, 1, L, dtype=torch.float64, device=device)
    v = torch.as_tensor(valid, device=device).view(B, 1, 1)
    return (rows < v).double()


def residual_value(res: torch.Tensor, kind, slope: float) -> torch.Tensor:
    """what the epilogue adds for a residual carried as fp32, as an activated fp16 plane, or as a hi/lo plane"""
    if kind is None:
        return torch.zeros_like(res, dtype=torch.float64)
    if kind == "f32":
        return res.double()
    a = act32(res, slope)
    if kind == "f16":
        v = q16(a)
    else:  # hi/lo: hi = fp16(a), lo = fp16(a - hi)
        hi = q16(a)
        v = hi + q16((a.float() - hi.float()).double())
    return torch.where(v >= 0, v, v / slope)


def tie_gap(m: torch.Tensor, slack: torch.Tensor) -> torch.Tensor:
    """fp16 rounding gap at elements whose value is within `slack` of a rounding midpoint (a computation that is off by at most
    slack may round them to the neighbouring fp16 value); 0 elsewhere"""
    lo, hi = q16(m - slack), q16(m + slack)
    return (hi - lo).abs()


def mode_apply(v: torch.Tensor, mode: str, S, div: float) -> torch.Tensor:
    if mode == "store":
        return v
    if mode == "add":
        return S.double() + v
    return (S.double() + v) / div


def pair_reference(x, w1, b1, w2, b2, dil, slope_in, slope_mid, *, res=None, res_kind=None, res_slope=1.0, mode="store",
                   S=None, div=1.0, valid=None):
    """two-stage rounded reference of a fused resblock pair (Conv1d weights [C, C, k]; valid = output rows per utterance).
    Returns (y, mid, gap): y float64 [B, C, L], the fp16 intermediate and its tie gap (see bound)."""
    B, C, L = x.shape
    k = w1.shape[2]
    h1, h2 = (k - 1) * dil // 2, (k - 1) // 2
    a = q16(act32(x, slope_in))
    qw1, qw2 = q16(w1.double()), q16(w2.double())
    m = F.conv1d(a, qw1, b1.double(), padding=h1, dilation=dil)
    # the fp32 c1 sum is off by at most ~ ACC_REL * sum |terms|; mid elements that close to a rounding midpoint may round either way
    slack = MID_TIE_REL * m.abs() + ACC_REL * (F.conv1d(a.abs(), qw1.abs(), b1.double().abs(), padding=h1, dilation=dil))
    mask = row_mask(B, L, valid, x.device)
    m = lrelu(m, slope_mid) * mask
    slack = slack * mask  # (leaky-relu scales the slack by at most 1)
    mid = q16(m)
    gap = tie_gap(m, slack)
    v = F.conv1d(mid, qw2, b2.double(), padding=h2) + residual_value(res, res_kind, res_slope) if res is not None else \
        F.conv1d(mid, qw2, b2.double(), padding=h2)
    y = mode_apply(v, mode, S, div) * mask
    return y, mid, gap


def pair_bound(y_ref: torch.Tensor, w2: torch.Tensor, gap: torch.Tensor, mode="store", div=1.0, valid=None) -> torch.Tensor:
    """elementwise bound on |y - y_ref|:  TOL * max|y_ref|  +  (|q(w2)| conv gap)  (divided by div for add_div; 0 past a length).

    Derivation: the kernel's y differs from the float64 y_ref in (1) its fp32 summation order, at most a few fp32 ulps of the sum of
    |terms| per output, which TOL * max|y| covers with room to spare; and (2) the fp16 rounding of mid: the kernel rounds its fp32
    c1 value, the reference its float64 value; they round to the same fp16 unless the value lies within the fp32 error (slack) of a
    rounding midpoint, in which case they may differ by exactly one fp16 gap.  Such a flipped mid element j changes output i by
    q(w2)[:, :, t] * gap[j] for the tap t that connects them, so |q(w2)| conv gap bounds the sum of all flips.  Rows past a length
    are exactly zero in the kernel, so the bound there is 0."""
    C, _, k = w2.shape
    h2 = (k - 1) // 2
    flip = F.conv1d(gap, q16(w2.double()).abs(), None, padding=h2)
    if mode == "add_div":
        flip = flip / div
    b = TOL * y_ref.abs().max() + flip
    B, _, L = y_ref.shape
    return b * row_mask(B, L, valid, y_ref.device)


def worst_ratio(y: torch.Tensor, y_ref: torch.Tensor, bound: torch.Tensor) -> float:
    """max |y - y_ref| / bound (elements with bound 0 count as inf unless they match exactly)"""
    d = (y.double() - y_ref).abs()
    r = torch.where(bound > 0, d / bound.clamp_min(1e-300), torch.where(d > 0, torch.full_like(d, float("inf")), torch.zeros_like(d)))
    return float(r.max()) if r.numel() else 0.0


def layer_reference(x, w, b, *, dil=1, stride=1, transposed=False, slope_in=1.0, rounded=True, res=None, res_kind=None,
                    res_slope=1.0, mode="store", S=None, div=1.0, valid=None):
    """float64 reference of one tap conv launch (Conv1d weight [Cout, Cin, k] or ConvTranspose1d weight [Cin, Cout, k]);
    rounded=False for the 3-term-split layers (FP32-equivalent operands)"""
    a = act32(x, slope_in)
    w = w.double()
    if rounded:
        a, w = q16(a), q16(w)
    k = w.shape[2]
    if transposed:
        u = stride
        v = F.conv_transpose1d(a, w, b.double(), u, u // 2 + u % 2, u % 2)
    else:
        v = F.conv1d(a, w, b.double(), padding=(k - 1) * dil // 2, dilation=dil)
    if res is not None:
        v = v + residual_value(res, res_kind, res_slope)
    B, _, L = v.shape
    return mode_apply(v, mode, S, div) * row_mask(B, L, valid, x.device)
