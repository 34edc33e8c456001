"""float64 references and error bounds for the ppg2mel decoder's kernels (csrc/ppg2mel.cu), one launch at a time.

Every kernel runs in fp32 without FMA contraction (the library is built with -fmad=false), so each product and each add
rounds once: U24 = 2^-24 per rounding and gamma(n) = n U24 / (1 - n U24) for a sum whose terms pass through at most n
roundings.  expf and tanhf are charged 2 ulp, log1pf 1 ulp (the CUDA documented maxima); one ulp of x is at most
2 U24 |x|.  sqrtf and division are IEEE (one rounding).

Every reference takes a padded batch: row b has its own length and the kernel must read nothing past it.  Each returns
(ref, bound) in float64; an fp32 result r is correct when |r - ref| <= bound.
"""
from __future__ import annotations

import math

import numpy as np

U24 = 2.0 ** -24
TINY = 1e-38  # below fp32's normal range: saturated sigmoid / exp results are charged absolutely
E, H, NM, M, Q = 256, 512, 80, 5, 256
EPS_MOL = float(np.float32(1e-5))


def _f64(x):
    return np.asarray(x, np.float64)


def gamma(n):
    n = np.asarray(n, np.float64)
    return n * U24 / (1.0 - n * U24)


def ulp_rel(k):
    """k ulp of a result, relative to its magnitude"""
    return 2.0 * k * U24


def sigmoid(x):
    return 1.0 / (1.0 + np.exp(-_f64(x)))


def sigmoid_bound(x, dx):
    """|sigmoidf_(x~) - sigmoid(x)| for |x~ - x| <= dx: the slope's maximum over the interval times dx, plus the kernel's
    own 1 / (1 + expf(-x)) (expf 2 ulp, the add and the division: 6 U24 relative) and TINY for expf's overflow to inf"""
    x, dx = _f64(x), _f64(dx)
    near = np.maximum(np.abs(x) - dx, 0.0)
    s = sigmoid(near)
    return s * (1.0 - s) * dx + 6.0 * U24 * sigmoid(x + dx) + TINY


def tanh_bound(x, dx):
    x, dx = _f64(x), _f64(dx)
    near = np.maximum(np.abs(x) - dx, 0.0)
    return (1.0 - np.tanh(near) ** 2) * dx + ulp_rel(2) * np.abs(np.tanh(x)) + TINY


def lane_terms(widths):
    """terms one lane of dot_rows sums: float4 slices every 128 columns of each segment, the lane accumulator running on
    across segments"""
    return sum(4 * math.ceil(k / 128) for k in widths)


def dot_rows_gamma(widths):
    """dot_rows: each lane sums its terms in order, then a 5-level butterfly adds the 32 lane partials"""
    return gamma(lane_terms(widths) + 5)


# ---- conv_gemm ---------------------------------------------------------------------------------------------------------
def im2col(x, len_in, ks, stride, pad, T_out):
    """[B][T_out][Cin ks] with column c ks + tap = x[b, t stride - pad + tap, c], zero outside [0, len_in[b])"""
    x = _f64(x)
    B, T_in, Cin = x.shape
    A = np.zeros((B, T_out, Cin * ks))
    for b in range(B):
        for tap in range(ks):
            ti = np.arange(T_out) * stride - pad + tap
            ok = (ti >= 0) & (ti < len_in[b])
            A[b, ok, tap::ks] = x[b, ti[ok]]
    return A


def conv_gemm(x, len_in, w, ks, stride, pad, T_out, len_out, bias=None, bn=None, act=0, res=None, drop_k=0):
    """conv_gemm_kernel: y[b, t, n] = epilogue(sum_k w[n, k] A[b, t, k]) for t < len_out[b], exactly 0 past it.  Epilogue:
    + bias ([N] or per row [B][N]); eval BatchNorm folded as v alpha + (b - mean alpha), alpha = w / sqrtf(var + 1e-5f);
    act 1 LeakyReLU(0.1) / 2 tanh; + res.  The kernel accumulates k = c ks + tap in order in one fp32 accumulator.
    drop_k (self-tests only) leaves out the last drop_k columns of k."""
    A = im2col(x, len_in, ks, stride, pad, T_out)
    W = _f64(w)
    K = A.shape[2]
    if drop_k:
        A = A[..., :K - drop_k]
        W = W[:, :K - drop_k]
    v = A @ W.T
    e = gamma(K) * (np.abs(A) @ np.abs(W).T)
    if bias is not None:
        bb = _f64(bias)
        v = v + (bb[:, None, :] if bb.ndim == 2 else bb)
        e = e + U24 * np.abs(v)
    if bn is not None:
        mean, var, bw, bb = (_f64(a) for a in bn)
        alpha = bw / np.sqrt(var + 1e-5)
        beta = bb - mean * alpha
        # alpha: var + eps (and 1e-5f vs 1e-5), sqrtf, division: <= 4 U24 relative
        e1 = np.abs(alpha) * e * (1 + 5 * U24) + 5 * U24 * np.abs(v * alpha)
        e2 = 5 * U24 * np.abs(mean * alpha) + U24 * np.abs(beta)
        v = v * alpha + beta
        e = e1 + e2 + U24 * (np.abs(v) + e1 + e2)
    if act == 1:
        slope = np.where(np.abs(v) > e, np.where(v > 0, 1.0, 0.1), 1.0)
        v = np.where(v > 0, v, 0.1 * v)
        e = slope * e + 2 * U24 * np.abs(v)
    elif act == 2:
        e = tanh_bound(v, e)
        v = np.tanh(v)
    if res is not None:
        v = v + _f64(res)
        e = e + U24 * (np.abs(v) + e)
    t = np.arange(T_out)[None, :, None]
    live = t < np.asarray(len_out)[:, None, None]
    return np.where(live, v, 0.0), np.where(live, e * (1 + 1e-6) + TINY, 0.0)


# ---- instance_norm -----------------------------------------------------------------------------------------------------
def instance_norm(x, lens, add=None):
    """instance_norm_kernel on x [B][T][C]: statistics over t < len[b] in double; the mean is rounded to fp32, the variance
    taken in double about that rounded mean, inv = 1 / sqrtf((float) var + 1e-5f), then (x - mu) inv (+ add) in fp32;
    exactly 0 for t >= len[b]"""
    x = _f64(x)
    B, T, C = x.shape
    ref, bound = np.zeros_like(x), np.zeros_like(x)
    for b, L in enumerate(lens):
        xb = x[b, :L]
        mu = xb.mean(0)
        var = xb.var(0)
        inv = 1.0 / np.sqrt(var + 1e-5)
        d = xb - mu
        y = d * inv
        dmu = U24 * np.abs(mu) + L * 2.0 ** -52 * np.abs(xb).mean(0)  # fp32 mean; double sums
        # inv: (float) var, + 1e-5f (and its distance from 1e-5), sqrtf, the division; var grows by dmu^2
        dinv = inv * (4 * U24 + dmu ** 2 / (2 * (var + 1e-5)))
        e = (dmu + U24 * (np.abs(d) + dmu)) * inv * (1 + 5 * U24) + (np.abs(d) + dmu) * dinv + U24 * np.abs(y)
        if add is not None:
            y = y + _f64(add)[b, :L]
            e = e + U24 * (np.abs(y) + e)
        ref[b, :L], bound[b, :L] = y, e * (1 + 1e-6) + TINY
    return ref, bound


# ---- spk_bias ----------------------------------------------------------------------------------------------------------
def spk_bias(spk, W, bias):
    """spk_bias_kernel: bias + W[:, 256:256 + D] . F.normalize(spk) (eps 1e-12).  |spk|^2: 256 strided fp32 partial sums
    then an 8-level tree; den = max(sqrtf(.), 1e-12f); sn = spk / den; the dot runs over k in order."""
    s = _f64(spk)
    B, D = s.shape
    Wd = _f64(W)[:, E:E + D]
    norm = np.sqrt((s ** 2).sum(1))
    den = np.maximum(norm, 1e-12)
    clamped = norm <= 1e-12 * (1 + 1e-6)
    den_rel = np.where(clamped, U24, gamma(math.ceil(D / 256) + 8) / 2 + U24 + U24)
    sn = s / den[:, None]
    dsn = np.abs(sn) * (den_rel[:, None] + 2 * U24)
    acc = sn @ Wd.T
    e = dsn @ np.abs(Wd).T + gamma(D) * (np.abs(sn) @ np.abs(Wd).T)
    out = _f64(bias) + acc
    return out, e + U24 * (np.abs(out) + e) + TINY


# ---- prenet ------------------------------------------------------------------------------------------------------------
def prenet(frame, W1, W2, keep1, keep2):
    """prenet_kernel: relu(W1 x) * 2 keep1 -> relu(W2 h1) * 2 keep2 (each dot over k in order)"""
    x = _f64(frame)
    W1, W2 = _f64(W1), _f64(W2)
    a = x @ W1.T
    ea = gamma(NM) * (np.abs(x) @ np.abs(W1).T)
    k1, k2 = _f64(keep1), _f64(keep2)
    h1 = np.maximum(a, 0.0) * 2.0 * k1
    e1 = ea * 2.0 * k1
    c = h1 @ W2.T
    ec = e1 @ np.abs(W2).T + gamma(256) * (np.abs(h1) @ np.abs(W2).T)
    out = np.maximum(c, 0.0) * 2.0 * k2
    return out, ec * 2.0 * k2 * (1 + 1e-6) + TINY


# ---- the LSTM cell -----------------------------------------------------------------------------------------------------
def lstm(x, ctx, h, c, W_ih, W_hh, bias, swap_if=False):
    """lstm_kernel: gates = [x | ctx] . W_ih^T + h . W_hh^T + bias (dot_rows over segments x, ctx, h; gate order i, f, g, o),
    c' = sigmoid(f) c + sigmoid(i) tanh(g), h' = sigmoid(o) tanh(c').  swap_if (self-tests only) exchanges i and f."""
    xin = np.concatenate([_f64(x), _f64(ctx), _f64(h)], 1)
    Wf = np.concatenate([_f64(W_ih), _f64(W_hh)], 1)
    g = xin @ Wf.T + _f64(bias)
    eg = dot_rows_gamma([x.shape[1], E, H]) * (np.abs(xin) @ np.abs(Wf).T) + U24 * np.abs(g)
    gi, gf, gg, go = (g[:, i * H:(i + 1) * H] for i in range(4))
    ei, ef, eg_, eo = (eg[:, i * H:(i + 1) * H] for i in range(4))
    if swap_if:
        gi, gf, ei, ef = gf, gi, ef, ei
    si, sf, so = sigmoid(gi), sigmoid(gf), sigmoid(go)
    dsi, dsf, dso = sigmoid_bound(gi, ei), sigmoid_bound(gf, ef), sigmoid_bound(go, eo)
    tg, dtg = np.tanh(gg), tanh_bound(gg, eg_)
    c = _f64(c)
    p1, p2 = sf * c, si * tg
    cn = p1 + p2
    ec = dsf * np.abs(c) + U24 * np.abs(p1) + dsi * np.abs(tg) + (si + dsi) * dtg + U24 * np.abs(p2)
    ec = ec + U24 * (np.abs(cn) + ec)
    tc, dtc = np.tanh(cn), tanh_bound(cn, ec)
    hn = so * tc
    eh = dso * np.abs(tc) + (so + dso) * dtc
    eh = eh + U24 * (np.abs(hn) + eh)
    return (hn, cn), (eh * (1 + 1e-6) + TINY, ec * (1 + 1e-6) + TINY)


def query(ah, W, bias):
    """query_kernel: relu(W ah + b), dot_rows over one 512-wide segment"""
    a = _f64(ah)
    v = a @ _f64(W).T + _f64(bias)
    e = dot_rows_gamma([H]) * (np.abs(a) @ np.abs(_f64(W)).T) + U24 * np.abs(v)
    return np.maximum(v, 0.0), e * (1 + 1e-6) + TINY


# ---- MoL attention -----------------------------------------------------------------------------------------------------
def softplus(x):
    x = _f64(x)
    return np.where(x > 20, x, np.log1p(np.exp(np.minimum(x, 20.0))))


def softplus_bound(x, dx):
    """x > 20 ? x : log1pf(expf(x)): slope sigmoid(x) <= 1; expf 2 ulp moves log1p by <= 4 U24 sigmoid(x); log1pf 1 ulp; a
    threshold crossing moves the value by log1p(e^-20) < 2.1e-9"""
    x, dx = _f64(x), _f64(dx)
    sp = softplus(x)
    e = sigmoid(x + dx) * (dx + 4 * U24) + ulp_rel(1) * sp
    return e + np.where(np.abs(x - 20) <= dx + 20 * U24, 2.1e-9 + 40 * U24, 0.0)


def mol_params(q, W2, b2, mu_prev):
    """the 15 mixture parameters (dot_rows-like: 8 terms per lane, 5-level butterfly, + b2) -> w, sigma, mu with bounds"""
    q = _f64(q)
    W2 = _f64(W2)
    p = q @ W2.T + _f64(b2)
    dp = gamma(8 + 5) * (np.abs(q) @ np.abs(W2).T) + U24 * np.abs(p)
    pw, ps, pm = p[:, :M], p[:, M:2 * M], p[:, 2 * M:]
    dpw, dps, dpm = dp[:, :M], dp[:, M:2 * M], dp[:, 2 * M:]
    mx = pw.max(1, keepdims=True)
    ex = np.exp(pw - mx)
    sm = ex / ex.sum(1, keepdims=True)
    # softmax: input errors move w by <= w (|dp_m| + sum_k w_k |dp_k|) <= 2 w max dp; own: the subtraction
    # (U24 |p - max|), expf 2 ulp, the 5-term sum (gamma 4) and the division
    dmax = dpw.max(1, keepdims=True)
    dw = sm * (2 * dmax * (1 + 4 * dmax) + U24 * np.abs(pw - mx) + ulp_rel(2) + gamma(4) + U24)
    w = sm + 1e-5
    dw = dw + U24 * w + 1e-12
    sig = softplus(ps) + 1e-5
    dsig = softplus_bound(ps, dps) + U24 * sig + 1e-12
    mu = _f64(mu_prev) + softplus(pm)
    dmu = softplus_bound(pm, dpm) + U24 * np.abs(mu)
    return (w, sig, mu), (dw, dsig, dmu)


def mol_phi(params, dparams, Te):
    """phi at j = k + 0.5, k = 0..Te, summed over m in order as the kernel does -> (phi [B][Te + 1], absolute bound)"""
    (w, sig, mu), (dw, dsig, dmu) = params, dparams
    j = np.arange(Te + 1) + 0.5
    z = (mu[:, :, None] - j) / sig[:, :, None]
    dz = (dmu[:, :, None] + U24 * np.abs(mu[:, :, None] - j)) / sig[:, :, None] * (1 + 2 * U24) \
        + np.abs(z) * dsig[:, :, None] / sig[:, :, None] * (1 + 2 * dsig[:, :, None] / sig[:, :, None]) + U24 * np.abs(z)
    s = sigmoid(z)
    ds = sigmoid_bound(z, dz)
    r = 1.0 / (1.0 + s)
    dr = ds + 2 * U24 * r
    t = w[:, :, None] * r
    dt = dw[:, :, None] * (r + dr) + w[:, :, None] * dr + U24 * t
    phi = t.sum(1)
    dphi = dt.sum(1) + gamma(4) * t.sum(1)
    return phi, dphi


def mol_alpha(q, W2, b2, mu_prev, Te):
    """(alpha [B][Te] without the 1e-5 rule, its absolute bound, mu [B][5], mu bound)"""
    params, dparams = mol_params(q, W2, b2, mu_prev)
    phi, dphi = mol_phi(params, dparams, Te)
    a = phi[:, 1:] - phi[:, :-1]
    da = dphi[:, 1:] + dphi[:, :-1] + U24 * np.abs(a)
    return a, da * (1 + 1e-6) + TINY, params[2], dparams[2] * (1 + 1e-6) + TINY


def alpha_ok(got, ref, bound):
    """an alpha the kernel wrote is right when it is within the bound, or when it is exactly 1e-5f where the fp32 difference
    could have been 0 (|ref| <= bound); the kernel never returns an exact 0"""
    got = _f64(got)
    return (got != 0.0) & ((np.abs(got - ref) <= bound) | ((got == EPS_MOL) & (np.abs(ref) <= bound)))


def mol_context(alpha, dalpha, memory, got_alpha=None):
    """ctx = sum_j alpha_j memory_j (j in order).  Where the fp32 alpha could be 0 (|alpha| <= bound) the kernel may have
    substituted 1e-5: with the kernel's alphas (got_alpha) the reference takes 1e-5 exactly where the kernel did, without
    them it charges 1e-5 more at each such j."""
    a, da, mem = _f64(alpha), _f64(dalpha), _f64(memory)
    maybe = np.abs(a) <= da
    if got_alpha is not None:
        sub = maybe & (_f64(got_alpha) == EPS_MOL)
        a = np.where(sub, EPS_MOL, a)
        da = np.where(sub, 0.0, da)
    else:
        da = da + np.where(maybe, EPS_MOL, 0.0)
    ctx = a @ mem
    n = mem.shape[0]
    e = da @ np.abs(mem) + gamma(n) * ((np.abs(a) + da) @ np.abs(mem))
    return ctx, e * (1 + 1e-6) + TINY


# ---- projection and stop rule ------------------------------------------------------------------------------------------
def proj(dh, ctx, W, bias, wstop, bstop):
    """proj_kernel: mel = W [h | ctx] + b (160) and the stop logit, both dot_rows over segments 512 and 256"""
    x = np.concatenate([_f64(dh), _f64(ctx)], 1)
    g = dot_rows_gamma([H, E])
    mel = x @ _f64(W).T + _f64(bias)
    emel = g * (np.abs(x) @ np.abs(_f64(W)).T) + U24 * np.abs(mel)
    stop = x @ _f64(wstop) + float(bstop)
    estop = g * (np.abs(x) @ np.abs(_f64(wstop))) + U24 * np.abs(stop)
    return (mel, emel * (1 + 1e-6) + TINY), (stop, estop * (1 + 1e-6) + TINY)


def stop_decision(logit, bound, step, tenc):
    """the stop rule after step `step` (0-based) for a row of T_enc tenc: True / False, or None where the fp32 sigmoid could
    go either way (|logit| within its bound, plus a margin for the tiny logits whose expf(-v) rounds to 1 and sigmoid to
    0.5); a logit known to be exactly 0 is decided: no stop"""
    ns, mx = step + 1, 2 * tenc
    mn = mx - 5
    if ns >= mx:
        return True
    if ns < mn:
        return False
    if logit == 0 and bound <= 2 * TINY:
        return False  # an exact 0: expf(0) = 1, 1 / (1 + 1) = 0.5, not > 0.5
    if abs(logit) <= bound + 2.0 ** -22:
        return None
    return logit > 0


# ---- device-drawn PreNet keep flags -------------------------------------------------------------------------------------
def philox_keep(seed, step, row, units, layer):
    """Python restatement of the library's device-drawn keep flags (Philox-4x32-10, mb_wavernn_math.h)"""
    import torch

    Mk = 0xFFFFFFFF
    out = []
    for u in units:
        c = [u >> 2, row, step, (0x70326D00 + layer) & Mk]
        k0, k1 = seed & Mk, (seed >> 32) & Mk
        for _ in range(10):
            p0 = 0xD2511F53 * c[0]
            p1 = 0xCD9E8D57 * c[2]
            c = [((p1 >> 32) ^ c[1] ^ k0) & Mk, p1 & Mk, ((p0 >> 32) ^ c[3] ^ k1) & Mk, p0 & Mk]
            k0, k1 = (k0 + 0x9E3779B9) & Mk, (k1 + 0xBB67AE85) & Mk
        out.append((c[u & 3] >> 16) & 1)
    return torch.tensor(out, dtype=torch.bool)
