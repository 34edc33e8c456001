"""float64 references and error bounds for the PPG extractor's kernels (csrc/ppg_extractor.cu, csrc/conv2d_tc.cu), one launch
at a time.  The 3-term split GEMM of conv2d_tc reuses tc_split_oracle; everything else runs in fp32 on the GPU and is bounded
here by the fp32 roundings the kernel performs (U24 = 2^-24 per rounding, gamma_n = n U24 for an n-term sequential sum).

Every reference takes a padded batch: row b has len[b] valid entries of T and the kernel must read nothing past them.

Operand tiles (the next GEMM's input) hold a value v as hi = fp16(v), lo = fp16(v - hi); hi + lo differs from v by at most
2^-22 |v| + 2^-25 (two fp16 roundings; 2^-25 is half the fp16 subnormal spacing): SPLIT_REL, SPLIT_ABS.
"""
from __future__ import annotations

import math

import numpy as np

import ppgx_oracle as po
import tc_split_oracle as so

U24 = so.U24
U53 = 2.0 ** -53
SPLIT_REL = 2.0 ** -22
SPLIT_ABS = 2.0 ** -25


def _f64(x):
    return np.asarray(x, np.float64)


def sigmoid(x):
    return 1.0 / (1.0 + np.exp(-_f64(x)))


def act(x, kind):
    """0 none, 1 ReLU, 2 swish"""
    x = _f64(x)
    return x if kind == 0 else np.maximum(x, 0.0) if kind == 1 else x * sigmoid(x)


def act_bound(x, dx, kind):
    """|kernel act - act| for an input error dx: Lipschitz 1 (none, ReLU), 1.1 (swish, |d/dx x sigmoid(x)| < 1.1) plus
    swish's own evaluation (expf, the add, the division and the product: 6 roundings of at most |x|)"""
    if kind == 2:
        return 1.1 * dx + 6 * U24 * np.abs(_f64(x))
    return dx


def conv_len(L, k, s, p):
    return (L + 2 * p - k) // s + 1


# ---- frontend ------------------------------------------------------------------------------------------------------------
def frames(wav, L, n_fft, win, hop):
    """[1 + L // hop][n_fft] float64 frames of wav[:L]: centre reflect padding by n_fft / 2, rectangular window of win samples
    centred in n_fft (zeros outside)"""
    x = _f64(wav[:L])
    xp = np.pad(x, n_fft // 2, mode="reflect")
    nf = 1 + L // hop
    idx = np.arange(nf)[:, None] * hop + np.arange(n_fft)[None, :]
    fr = xp[idx]
    left = (n_fft - win) // 2
    w = np.zeros(n_fft)
    w[left:left + win] = 1.0
    return fr * w


def log_mel(wav, L, n_fft, win, hop, melmat):
    """(log(power . melmat + 1e-20) [frames][n_mels], bound): power = |rfft(frame)|^2 in float64.

    The kernel sums re / im in double (|error| <= (win + 2) 2^-52 sum |frame| each, sin / cos tables included), rounds them
    to fp32 and squares and adds in fp32 (<= 3 U24 per square, U24 for the add: power relative 4.01 U24), sums power x melmat
    in double, rounds to fp32 (U24), adds 1e-20f (U24, and 1e-20f itself is 1e-20 to within U24) and takes logf (one ulp of
    the result plus its argument's relative error)."""
    fr = frames(wav, L, n_fft, win, hop)
    spec = np.fft.rfft(fr, axis=1)
    power = spec.real ** 2 + spec.imag ** 2
    mel = _f64(melmat)
    acc = power @ mel
    ref = np.log(acc + 1e-20)
    eps = (win + 2) * 2.0 ** -52 * np.abs(fr).sum(1, keepdims=True)
    dpow = 4.01 * U24 * power + 2 * eps * (np.abs(spec.real) + np.abs(spec.imag)) + 2 * eps ** 2
    rel = (dpow @ mel) / (acc + 1e-20) + 3.01 * U24
    return ref, rel * 1.01 + 2 * U24 * np.abs(ref)


def mvn(x, n, norm_means, norm_vars):
    """utterance_mvn of x[:n] [n][F] (float64, as ppgx_oracle.features) -> (y, bound).  The kernel: mean in double rounded to
    fp32, d = x - mean in fp32, var in double, sd = sqrtf((float) var) clamped at 1e-20, div = sqrtf(sd) with norm_means,
    then y = (x - mean) / div in fp32."""
    x = _f64(x[:n])
    mean = x.mean(0)
    if not norm_means and not norm_vars:
        return x, np.zeros_like(x)
    em = U24 * np.abs(mean) + n * U53 * np.abs(x).mean(0)  # the fp32 rounding of the mean (and the double sum)
    y1 = x - mean if norm_means else x
    dy1 = (em + U24 * np.abs(x - mean)) if norm_means else np.zeros_like(x)
    if not norm_vars:
        return y1, dy1
    d = x - mean
    var = (d ** 2).mean(0)
    sd = np.maximum(np.sqrt(var), 1e-20)
    div = np.sqrt(sd) if norm_means else sd
    rel_var = 3 * U24 + 2 * (em + U24 * np.abs(d).max(0)) * np.abs(d).mean(0) / np.maximum(var, 1e-300)
    rel_div = (0.25 if norm_means else 0.5) * rel_var + 3 * U24
    y = y1 / div
    return y, (np.abs(y) * (rel_div + U24) + dy1 / div) * 1.01


# ---- convolutions ----------------------------------------------------------------------------------------------------------
def im2col(X, lens, k, s, p):
    """channels-last X [B][T][F][C] -> ([B T_out F_out][k k C] with k = (dt k + df) C + c, T_out, F_out): zeros outside the
    plane and at t >= lens[b] (the row's own frames)"""
    X = np.asarray(X)
    B, T, F, C = X.shape
    To, Fo = conv_len(T, k, s, p), conv_len(F, k, s, p)
    A = np.zeros((B, To, Fo, k, k, C), X.dtype)
    for b in range(B):
        for dt in range(k):
            ti = np.arange(To) * s + dt - p
            tok = (ti >= 0) & (ti < lens[b])
            for df in range(k):
                fi = np.arange(Fo) * s + df - p
                fok = (fi >= 0) & (fi < F)
                vals = X[b][np.clip(ti, 0, T - 1)[:, None], np.clip(fi, 0, F - 1)[None, :]]  # [To][Fo][C]
                A[b, :, :, dt, df] = np.where((tok[:, None] & fok[None, :])[..., None], vals, 0)
    return A.reshape(B * To * Fo, k * k * C), To, Fo


def conv_weight_matrix(w):
    """w [N][C][k][k] -> [N][k k C] in im2col's k order"""
    w = np.asarray(w)
    N, C, kh, kw = w.shape
    return w.transpose(0, 2, 3, 1).reshape(N, kh * kw * C)


def conv2d_tc(X, lens, w, bias, k, s, p):
    """(ref of relu(bias + split product), bound, exact relu(bias + conv), exact bound, T_out, F_out) with rows (b, t, f):
    the split / accumulation bounds of tc_split_oracle (the kernel's 12 wgmmas per k-block of 64 are its hi.hi, lo.hi, hi.lo
    order per k16 step) and the fp32 bias add"""
    A, To, Fo = im2col(np.asarray(X, np.float32), lens, k, s, p)
    W = conv_weight_matrix(w)
    sc = so.pow2_scale(w)
    S = so.split_sum(A, W, sc)
    bias = _f64(bias)
    ref = so.big_epilogue(S, bias, act=1)
    bound = so.big_epilogue_bound(S, so.acc_bound(A, W, sc), bias, act=1)
    exact = so.big_epilogue(so.exact(A, W), bias, act=1)
    return ref, bound, exact, bound + so.rep_bound(A, W, sc), To, Fo


def conv0(x, lens, w, bias, k, s, p):
    """embed.conv.0 on [B][T][F] (1 channel) -> (relu(bias + conv) [B][T_out][F_out][N], bound): an FFMA chain of k^2 terms
    after the bias (gamma_{k^2 + 1} of the absolute terms)"""
    x = np.asarray(x)[..., None]
    A, To, Fo = im2col(x, lens, k, s, p)
    W = conv_weight_matrix(w)
    S = _f64(A) @ _f64(W).T + _f64(bias)
    mag = np.abs(_f64(A)) @ np.abs(_f64(W)).T + np.abs(_f64(bias))
    B = x.shape[0]
    N = W.shape[0]
    return np.maximum(S, 0).reshape(B, To, Fo, N), ((k * k + 1) * U24 * mag).reshape(B, To, Fo, N)


def depthwise(pw, lens, T, w, bias, bn_w, bn_b, bn_m, bn_v, act_kind):
    """conv module middle: GLU of pw [B T][2D] -> depthwise conv over each row's own frames (zeros outside [0, len)) -> eval
    BatchNorm (eps 1e-5) -> act, [B T][D] (rows t >= len zero), and the bound of the kernel's fp32 evaluation"""
    pw = _f64(pw)
    D = pw.shape[1] // 2
    B = len(lens)
    K = np.asarray(w).shape[-1]
    pad = (K - 1) // 2
    w = _f64(w).reshape(D, K)
    out = np.zeros((B * T, D))
    bound = np.zeros((B * T, D))
    for b in range(B):
        n = lens[b]
        r = pw[b * T:b * T + n]
        glu = r[:, :D] * sigmoid(r[:, D:])
        # the kernel's r * sigmoidf_(g): expf, add, divide, multiply (<= 5 U24 of |glu|)
        gp = np.zeros((n + 2 * pad, D))
        gp[pad:pad + n] = glu
        s = np.tile(_f64(bias), (n, 1))
        mag = np.tile(np.abs(_f64(bias)), (n, 1))
        for kk in range(K):
            s += gp[kk:kk + n] * w[:, kk]
            mag += np.abs(gp[kk:kk + n] * w[:, kk])
        es = (K + 1) * U24 * mag + 5 * U24 * mag
        sd = np.sqrt(_f64(bn_v) + 1e-5)
        z = (s - _f64(bn_m)) / sd
        y = z * _f64(bn_w) + _f64(bn_b)
        # s - m, sqrtf(v + eps) (2 roundings), the division, * w, + b
        ey = (es + U24 * np.abs(s - _f64(bn_m))) / sd * np.abs(_f64(bn_w)) + 6 * U24 * (np.abs(z * _f64(bn_w)) + np.abs(y))
        out[b * T:b * T + n] = act(y, act_kind)
        bound[b * T:b * T + n] = act_bound(y, ey, act_kind)
    return out, bound


# ---- LayerNorm ---------------------------------------------------------------------------------------------------------------
def layer_norm(x, g, be, eps=1e-12):
    """(LayerNorm of x [M][D] in float64, bound of the kernel's fp32 row_stats + affine): mean off by gamma_{D+1} of mean |x|,
    1 / sqrtf(var + eps) relatively by gamma_{D+8} plus the squared mean error over var, then three roundings"""
    x = _f64(x)
    D = x.shape[1]
    mean = x.mean(1, keepdims=True)
    var = ((x - mean) ** 2).mean(1, keepdims=True)
    rstd = 1.0 / np.sqrt(var + eps)
    z = (x - mean) * rstd
    y = z * _f64(g) + _f64(be)
    em = (D + 1) * U24 * np.abs(x).mean(1, keepdims=True)
    er = (D + 8) * U24 + em ** 2 / (var + eps)
    ey = np.abs(_f64(g)) * (em * rstd + np.abs(z) * (er + 3 * U24)) + 2 * U24 * (np.abs(y) + np.abs(_f64(be)))
    return y, ey * 1.01


# ---- attention -----------------------------------------------------------------------------------------------------------------
def attention(qkv, lens, T_max, H, dk, P=None, pu=None, pv=None):
    """one block's self-attention of a padded batch, qkv [B T_max][3 D] (q | k | v, head h at columns h dk), rel: P [>= T][H dk]
    rows of linear_pos(pos_emb), pos biases pu / pv [H][dk].  Scores built whole, with the LITERAL ppgx_oracle.rel_shift of
    the [T, T] bd matrix.  -> (ctx [B T_max][H dk] (zero past each row's T), bound).

    Bound: a score's fp32 error is at most (dk + 3) U24 (sum |qu||k| + sum |qv||p|) / sqrt(dk) + 3 U24 |s| (q + u, the two
    dk-term dot products, the division by sqrtf(dk)).  Scores off by at most Delta move every softmax weight by a factor in
    [e^-2Delta, e^2Delta], so the output moves by (e^2Delta - 1) sum_j w_j |v_j|.  The online softmax itself (expf, the
    rescaling by corr at every new maximum, T / 4 sequential adds per lane, the 4-lane merge, the final division) costs at most
    (2 T + 80) U24 sum_j w_j |v_j|."""
    import torch

    qkv = _f64(qkv)
    D = H * dk
    ld = qkv.shape[1] // 3
    B = len(lens)
    out = np.zeros((B * T_max, D))
    bound = np.zeros((B * T_max, D))
    for b in range(B):
        T = lens[b]
        rows = qkv[b * T_max:b * T_max + T]
        for h in range(H):
            c = slice(h * dk, (h + 1) * dk)
            q, k, v = rows[:, c], rows[:, ld:][:, c], rows[:, 2 * ld:][:, c]
            if P is not None:
                p = _f64(P)[:T, c]
                qu, qv = q + _f64(pu)[h], q + _f64(pv)[h]
                bd = po.rel_shift(torch.from_numpy(qv @ p.T)).numpy()
                bd_mag = po.rel_shift(torch.from_numpy(np.abs(qv) @ np.abs(p).T)).numpy()
                # rel_shift puts q_{i+1} + v above the diagonal: the magnitude matrix is shifted the same way
                s = (qu @ k.T + bd) / math.sqrt(dk)
                mag = (np.abs(qu) @ np.abs(k).T + bd_mag) / math.sqrt(dk)
            else:
                s = q @ k.T / math.sqrt(dk)
                mag = np.abs(q) @ np.abs(k).T / math.sqrt(dk)
            ds = (dk + 3) * U24 * mag + 3 * U24 * np.abs(s)
            w = np.exp(s - s.max(1, keepdims=True))
            w /= w.sum(1, keepdims=True)
            o = w @ v
            wv = w @ np.abs(v)
            delta = ds.max(1, keepdims=True)
            out[b * T_max:b * T_max + T, c] = o
            bound[b * T_max:b * T_max + T, c] = np.expm1(2 * delta) * wv + (2 * T + 80) * U24 * wv
    return out, bound * 1.01


# ---- operand tiles -------------------------------------------------------------------------------------------------------------
def tile_values(t_hi, t_lo, rows_total, cols):
    """fp16 operand tiles [ceil(cols / 64)][rows_total][64] (numpy float16) -> hi + lo as float64 [rows_total][KB 64]"""
    KB = (cols + 63) // 64
    hi = so.unpack_act_tiles(t_hi, rows_total, KB)
    lo = so.unpack_act_tiles(t_lo, rows_total, KB)
    return hi.astype(np.float64) + lo.astype(np.float64), hi, lo


def split_bound(v, dv):
    """the operand-tile value hi + lo of a kernel value within dv of v"""
    return dv + SPLIT_REL * (np.abs(v) + dv) + SPLIT_ABS
