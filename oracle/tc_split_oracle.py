"""float64 references and error bounds for the 3-term-split tensor-core GEMMs of csrc/tacotron_tc.cu (tc_skinny, tc_gru,
tc_lstm_seq, tc_big) and their operand packers.

The kernels compute every product a*w as hi(a)hi(w) + lo(a)hi(w) + hi(a)lo(w), hi(v) = fp16(v), lo(v) = fp16(v - hi(v)), with the
weights pre-scaled by s = 2^(12 - e) (max |w| = f 2^e, f in [0.5, 1)) and the sum multiplied by 1 / s.  This module gives

  exact(...)       the float64 product of the unsplit fp32 operands;
  split_sum(...)   the *emulated split*: hi / lo from numpy float16 with the same scale rule, the three products summed in float64,
                   times 1 / s - what the kernel computes up to its FP32 accumulation;
  acc_bound(...)   |kernel - split_sum| allowed by FP32 accumulation (derivation below);
  rep_bound(...)   |split_sum - exact|, the representation error of the split, evaluated exactly per element;
  contract_bound   the closed-form per-product contract the documentation states (relative term + absolute floor);

and float64 epilogues (PLAIN, LSTM cell, GRU cell, big: ReLU -> BN -> residual), the im2col with per-sequence shifts, and CPU
unpackers of the swizzled operand tiles.

Accumulation bound (kernel vs split_sum).  fp16 x fp16 products are exact in fp32 (11 + 11 significand bits).  Each wgmma adds the
16 products of one k16 slice of one split term to the fp32 accumulator; the K loop issues, per k16 slice, hi*hi, lo*hi, hi*lo in
that order, so an output sees S = 3 * 4 * KB additions of block sums.  One such addition (block sum formed and added to the
accumulator, alignment / rounding or truncation to 24 significand bits) errs by at most 2^-23 of the magnitudes it combines; we
charge 2^-22 (two such roundings: the block sum and the accumulate) times (|P_s| + sum of |products| of the block), P_s the exact
running sum after step s.  Summed over the steps:
    |acc - P| <= 2^-22 * (sum_s |P_s| + sum_i |t_i|),
then x (1 / s) (exact, a power of two) and one fp32 rounding per epilogue addition (bias, pre): 2^-24 of each partial sum.

Representation bound (split_sum vs exact), per element: with a' = hi(a) + lo(a), r_a = a - a' (and w likewise, scaled),
    a w - split = lo(a) lo(w) + a' r_w + r_a w' + r_a r_w,
evaluated in float64 as the sum of absolute values.  In closed form (fp16: 11-bit significand, subnormal spacing 2^-24):
|r_a| <= 2^-22 |a| + 2^-25 and |lo(a)| <= 2^-11 |a| + 2^-25, so per product
    |a w - split| <= 2^-20 |a| |w| + 2^-24 (|w| + |a| / s)       for |a| < 65520 (hi(a) = inf beyond: the split is undefined).
The 2^-24 |w| term is the absolute floor: for |a| < 2^-3, lo(a) is an fp16 subnormal.

Cell epilogues: a pre-activation error d moves sigmoid by <= d / 4 and tanh by <= d; expf / tanhf / the division add a few ulps
(E_SIG = 8 * 2^-24, E_TANH = 4 * 2^-24 absolute, both functions bounded by 1), each fp32 multiply / add one 2^-24 relative rounding.
"""
from __future__ import annotations

import numpy as np

U24 = 2.0 ** -24
E_SIG = 8 * U24
E_TANH = 4 * U24
FP16_MAX_SPLIT = 65520.0  # fp16(v) = inf from here on


# ---- scale rule and split ------------------------------------------------------------------------------------------------
def pow2_scale(w) -> float:
    """tc_weight_scale: s = 2^(12 - e) with max |w| = f 2^e, f in [0.5, 1); zero / inf / NaN max -> 2^12"""
    mx = float(np.max(np.abs(np.asarray(w, np.float32)))) if np.size(w) else 0.0
    e = 0
    if 0.0 < mx < 3.0e38:
        _, e = np.frexp(np.float32(mx))
    return float(np.ldexp(np.float32(1.0), 12 - int(e)))


def split16(v):
    """(hi, lo) as float16 arrays, rounded like __float2half_rn: hi = fp16(v), lo = fp16(v - hi) with v - hi in fp32"""
    v = np.asarray(v, np.float32)
    with np.errstate(over="ignore", invalid="ignore"):
        hi = v.astype(np.float16)
        lo = (v - hi.astype(np.float32)).astype(np.float16)
    return hi, lo


def _f64(x):
    return np.asarray(x, np.float64)


def scaled_weight(W, scale):
    return (np.asarray(W, np.float32) * np.float32(scale)).astype(np.float32)


# ---- products -----------------------------------------------------------------------------------------------------------
def exact(A, W):
    """float64 A [M][K] . W [N][K]^T of the fp32 operands"""
    return _f64(A) @ _f64(W).T


def split_terms(A, W, scale):
    """the three split products (float64, still scaled by `scale`): hi*hi, lo*hi, hi*lo"""
    ah, al = split16(A)
    wh, wl = split16(scaled_weight(W, scale))
    ah, al, wh, wl = (_f64(t) for t in (ah, al, wh, wl))
    return ah, al, wh, wl


def split_sum(A, W, scale=None):
    """the emulated split: sum of the three products in float64, times 1 / scale"""
    if scale is None:
        scale = pow2_scale(W)
    ah, al, wh, wl = split_terms(A, W, scale)
    with np.errstate(invalid="ignore", over="ignore"):
        return (ah @ wh.T + al @ wh.T + ah @ wl.T) / scale


def acc_bound(A, W, scale=None, k_lo=0, k_hi=None):
    """FP32-accumulation bound of the kernel against split_sum over k in [k_lo, k_hi) (module docstring), after x 1 / scale"""
    if scale is None:
        scale = pow2_scale(W)
    ah, al, wh, wl = split_terms(A, W, scale)
    K = ah.shape[1]
    k_hi = K if k_hi is None else k_hi
    P = np.zeros((ah.shape[0], wh.shape[0]))
    run = np.zeros_like(P)
    for k0 in range(k_lo, k_hi, 16):
        sl = slice(k0, min(k0 + 16, k_hi))
        for a, w in ((ah, wh), (al, wh), (ah, wl)):
            t = a[:, sl] @ w[:, sl].T
            ta = np.abs(a[:, sl]) @ np.abs(w[:, sl]).T
            P += t
            run += np.abs(P) + ta
    return 2.0 ** -22 * run / scale


def rep_bound(A, W, scale=None):
    """|split_sum - exact| per element, bounded by the float64 sum of the absolute representation-error terms"""
    if scale is None:
        scale = pow2_scale(W)
    a = _f64(np.asarray(A, np.float32))
    w = _f64(scaled_weight(W, scale))
    ah, al, wh, wl = split_terms(A, W, scale)
    ap, wp = ah + al, wh + wl
    ra, rw = a - ap, w - wp
    b = np.abs(al) @ np.abs(wl).T + np.abs(ap) @ np.abs(rw).T + np.abs(ra) @ np.abs(wp).T + np.abs(ra) @ np.abs(rw).T
    return b * (1 + 2.0 ** -50) / scale


def contract_bound(A, W, scale=None):
    """the documented per-product contract summed over k: 2^-20 |a||w| + 2^-24 (|w| + |a| / s)"""
    if scale is None:
        scale = pow2_scale(W)
    a, w = np.abs(_f64(A)), np.abs(_f64(W))
    return 2.0 ** -20 * (a @ w.T) + U24 * (np.ones_like(a) @ w.T + a @ np.ones_like(w).T / scale)


# ---- epilogues (float64) ------------------------------------------------------------------------------------------------
def sigmoid(x):
    return 1.0 / (1.0 + np.exp(-_f64(x)))


def lstm_cell(g, c, H):
    """g [M][4H] pre-activations (i|f|g|o), c [M][H] -> (c', h')"""
    g = _f64(g)
    i, f, gg, o = sigmoid(g[:, :H]), sigmoid(g[:, H:2 * H]), np.tanh(g[:, 2 * H:3 * H]), sigmoid(g[:, 3 * H:])
    cn = f * _f64(c) + i * gg
    return cn, o * np.tanh(cn)


def lstm_cell_bound(g, c, H, dg, dc=0.0):
    """|kernel - lstm_cell| for pre-activation errors dg [M][4H] and a state error dc (module docstring)"""
    g = _f64(g)
    c = _f64(c)
    i, f, gg, o = sigmoid(g[:, :H]), sigmoid(g[:, H:2 * H]), np.tanh(g[:, 2 * H:3 * H]), sigmoid(g[:, 3 * H:])
    di, df = 0.25 * dg[:, :H] + E_SIG, 0.25 * dg[:, H:2 * H] + E_SIG
    dgg, do = dg[:, 2 * H:3 * H] + E_TANH, 0.25 * dg[:, 3 * H:] + E_SIG
    cn = f * c + i * gg
    dcn = np.abs(c) * df + np.abs(f) * dc + np.abs(gg) * di + np.abs(i) * dgg + 3 * U24 * (np.abs(f * c) + np.abs(i * gg))
    tc = np.tanh(cn)
    dh = np.abs(tc) * do + np.abs(o) * (dcn + E_TANH) + U24 * np.abs(o * tc)
    return dcn, dh


def gru_cell(gh, gi, h, H):
    """ATen gru_cell: gh = W_hh h + b_hh, gi = W_ih x + b_ih (r|z|n)"""
    gh, gi, h = _f64(gh), _f64(gi), _f64(h)
    r = sigmoid(gh[:, :H] + gi[:, :H])
    z = sigmoid(gh[:, H:2 * H] + gi[:, H:2 * H])
    n = np.tanh(gi[:, 2 * H:] + gh[:, 2 * H:] * r)
    return (h - n) * z + n


def gru_cell_bound(gh, gi, h, H, dgh, dh=0.0):
    gh, gi, h = _f64(gh), _f64(gi), _f64(h)
    pr, pz = gh[:, :H] + gi[:, :H], gh[:, H:2 * H] + gi[:, H:2 * H]
    r, z = sigmoid(pr), sigmoid(pz)
    dr = 0.25 * (dgh[:, :H] + U24 * np.abs(pr)) + E_SIG
    dz = 0.25 * (dgh[:, H:2 * H] + U24 * np.abs(pz)) + E_SIG
    vn = gh[:, 2 * H:]
    arg = gi[:, 2 * H:] + vn * r
    darg = np.abs(vn) * dr + np.abs(r) * dgh[:, 2 * H:] + 2 * U24 * (np.abs(vn * r) + np.abs(arg))
    n = np.tanh(arg)
    dn = darg + E_TANH
    hn = (h - n) * z + n
    return np.abs(h - n) * dz + np.abs(1 - z) * dn + np.abs(z) * dh + 3 * U24 * (np.abs(h) + np.abs(n) + np.abs(hn))


def big_epilogue(S, bias=None, act=0, bn_scale=None, bn_shift=None, res=None):
    t = _f64(S) + (0 if bias is None else _f64(bias)[None, :])
    if act == 1:
        t = np.maximum(t, 0.0)
    if bn_scale is not None:
        t = t * _f64(bn_scale)[None, :] + _f64(bn_shift)[None, :]
    if res is not None:
        t = t + _f64(res)
    return t


def big_epilogue_bound(S, dS, bias=None, act=0, bn_scale=None, bn_shift=None, res=None):
    """error of the kernel's epilogue given |dS| on the accumulator: each step Lipschitz 1 (ReLU) / |bn_scale|, one rounding each"""
    t = _f64(S) + (0 if bias is None else _f64(bias)[None, :])
    d = dS + U24 * np.abs(t)
    if act == 1:
        t = np.maximum(t, 0.0)
    if bn_scale is not None:
        t2 = t * _f64(bn_scale)[None, :] + _f64(bn_shift)[None, :]
        d = d * np.abs(_f64(bn_scale))[None, :] + U24 * (np.abs(t * _f64(bn_scale)[None, :]) + np.abs(t2))
        t = t2
    if res is not None:
        t = t + _f64(res)
        d = d + U24 * np.abs(t)
    return d


# ---- im2col and tile layouts ----------------------------------------------------------------------------------------------
def im2col(xs, shifts, K, M, T):
    """[M][nseg * K]: segment s of row m is xs[s][m + shift_s][:K] when m % T + shift_s stays inside [0, T) and m + shift_s < M
    (a last, partial sequence ends at row M), else zero"""
    out = np.zeros((M, len(xs) * K), np.float32)
    m = np.arange(M)
    for s, (x, sh) in enumerate(zip(xs, shifts)):
        t = m % T + sh
        ok = (t >= 0) & (t < T) & (m + sh < M)
        src = np.clip(m + sh, 0, None)
        out[ok, s * K:(s + 1) * K] = np.asarray(x, np.float32)[src[ok], :K]
    return out


def unpack_act_tiles(tiles, rows_pad, KB):
    """fp16 [KB][rows_pad][64] with 16-byte chunks at c8 ^ (m & 7) -> [rows_pad][KB * 64]"""
    t = np.asarray(tiles).reshape(KB, rows_pad, 8, 8)
    m = np.arange(rows_pad)
    out = np.empty((rows_pad, KB, 8, 8), t.dtype)
    for c8 in range(8):
        out[:, :, c8, :] = t[:, m, c8 ^ (m & 7), :].transpose(1, 0, 2)
    return out.reshape(rows_pad, KB * 64)


def unpack_weight_tiles(img, n_tiles, KB, rows):
    """weight image [tile][KB][hi|lo][rows][64] (rows = 32: tc_skinny_pack, 128: pack_big_w) -> (hi, lo) [n_tiles * rows][KB * 64]"""
    t = np.asarray(img).reshape(n_tiles, KB, 2, rows, 8, 8)
    n = np.arange(rows)
    out = np.empty((2, n_tiles, rows, KB, 8, 8), t.dtype)
    for c8 in range(8):
        out[:, :, :, :, c8, :] = t[:, :, :, n, c8 ^ (n & 7), :].transpose(2, 0, 3, 1, 4)
    out = out.reshape(2, n_tiles * rows, KB * 64)
    return out[0], out[1]


def gate_rows(H, gates):
    """source row of packed row j (gate-interleaved images): tile t holds the `gates` gates of hidden units [8t, 8t + 8)"""
    j = np.arange(H // 8 * 32)
    t, n = j // 32, j % 32
    return (n // 8) * H + 8 * t + (n % 8)
