"""float64 references and error bounds for the FP32 kernels of the Tacotron path (csrc/tacotron_kernels.cu and the attention,
style-token, stop and mask kernels of csrc/tacotron.cu), one launch at a time.

Each function restates the operation in the reference's semantics (models/synthesizer/models/tacotron.py and sublayer/*) in
float64 and returns (ref, bound): the kernel's fp32 output must satisfy |out - ref| <= bound elementwise.  No bound depends on
the order in which the kernel sums, so the same bound accepts any fp32 evaluation of the operation:

  * a sum of n fp32 terms (every addition on the kernel's path counted: products, bias, shuffle / cross-warp / split partials)
    errs by at most gamma(n) * sum |terms|, gamma(n) = n u / (1 - n u), u = 2^-24;
  * each epilogue operation (add, multiply, fma) adds u |result|;
  * expf, tanhf and log10f add 2 ulp each (the library is built with -fmad=false and without fast math); sigmoid and tanh are
    bounded by 1, so their library errors are charged absolutely (E_SIG, E_TANH of tc_split_oracle);
  * an input error dx moves a sigmoid by <= dx / 4 and a tanh by <= dx;
  * the softmax and the context vector propagate the energy errors to first order (with a 1 % allowance for the second).

Epilogue order of launch_gemm (tacotron_kernels.cuh): bias, activation, eval-BatchNorm affine (after the ReLU,
common/batch_norm_conv.py:11-14), x2 dropout keep mask, residual.  The PreNet dropout keep flags are Philox4x32-10 bits
(fill_masks_kernel), restated exactly by `fill_masks`.
"""
from __future__ import annotations

import numpy as np

import tc_split_oracle as so

U24 = 2.0 ** -24
E_SIG, E_TANH = so.E_SIG, so.E_TANH
ACT_NONE, ACT_RELU, ACT_SIGMOID, ACT_TANH = 0, 1, 2, 3
ATT_K = 31  # location conv kernel, padding 15 (lsa.py)


def _f64(x):
    return np.asarray(x, np.float64)


def gamma(n):
    n = np.asarray(n, np.float64)
    return n * U24 / (1 - n * U24)


# ---- GEMM (launch_gemm: rowdot, gemm_skinny<1|4>, gemm<32|64>, gemm_big) ------------------------------------------------------
def gemm_operand(x, ld, K, M, T=1, shift=0, step=None, x_step=0, x_first=None):
    """[M][K] rows one segment of GemmArgs reads from the flat fp32 buffer `x`: row_j(m) = m + shift inside its length-T
    sequence (zero outside); in step mode segment 0 reads x + step * x_step, or the single row x_first at step 0"""
    x = np.asarray(x, np.float32).reshape(-1)
    out = np.zeros((M, K), np.float32)
    if step is not None and step == 0 and x_first is not None:
        out[:] = np.asarray(x_first, np.float32).reshape(-1)[:K][None, :]
        return out
    base = 0 if step is None else step * x_step
    for m in range(M):
        if shift:
            t = (m % T) + shift
            if t < 0 or t >= T:
                continue
        row = m + shift
        out[m] = x[base + row * ld: base + row * ld + K]
    return out


def gemm_weight(W, ldw, N, K, w_off=0, w_stride=1):
    """[N][K] weight block of one segment: W[n * ldw + w_off + k * w_stride] (Conv1d weights [co][ci][k] read in place)"""
    W = np.asarray(W, np.float32).reshape(-1)
    n = np.arange(N)[:, None]
    k = np.arange(K)[None, :]
    return W[n * ldw + w_off + k * w_stride]


def activation(v, act):
    if act == ACT_RELU:
        return np.maximum(v, 0.0)
    if act == ACT_SIGMOID:
        return 1.0 / (1.0 + np.exp(-v))
    if act == ACT_TANH:
        return np.tanh(v)
    return v


def activation_bound(v, dv, act):
    if act == ACT_SIGMOID:
        return dv / 4 + E_SIG
    if act == ACT_TANH:
        return dv + E_TANH
    return dv


def gemm(xs, ws, bias=None, act=ACT_NONE, bn_scale=None, bn_shift=None, keep=None, res=None, extra_adds=16):
    """xs / ws: per segment the [M][K_j] operand (gemm_operand) and [N][K_j] weights (gemm_weight).
    Y = res + keep * 2 * BN(act(sum_j x_j w_j^T + bias)).  `extra_adds` counts the additions beyond one per product (bias,
    cross-warp / shuffle reductions) charged to gamma."""
    S = sum(_f64(x) @ _f64(w).T for x, w in zip(xs, ws))
    A = sum(np.abs(_f64(x)) @ np.abs(_f64(w)).T for x, w in zip(xs, ws))
    n = sum(x.shape[1] for x in xs) + extra_adds
    if bias is not None:
        S = S + _f64(bias)[None, :]
        A = A + np.abs(_f64(bias))[None, :]
    d = gamma(n) * A
    t = activation(S, act)
    d = activation_bound(S, d, act)
    if bn_scale is not None:
        sc, sh = _f64(bn_scale)[None, :], _f64(bn_shift)[None, :]
        t = t * sc + sh
        d = d * np.abs(sc) + U24 * np.abs(t)
    if keep is not None:
        k = _f64(keep)
        t, d = t * 2 * k, d * 2 * k
    if res is not None:
        t = t + _f64(res)
        d = d + U24 * np.abs(t)
    return t, d


# ---- decoder PreNet (prenet_fused_kernel) -------------------------------------------------------------------------------
def prenet(x, W1, b1, W2, b2, keep1, keep2):
    """y = keep2 * 2 relu(W2 (keep1 * 2 relu(W1 x + b1)) + b2) (pre_net.py:11-27 with dropout always on)"""
    h, dh = gemm([x], [W1], b1, ACT_RELU, keep=keep1, extra_adds=6)
    hs, hA = h, np.abs(h)
    S = hs @ _f64(W2).T + _f64(b2)[None, :]
    A = hA @ np.abs(_f64(W2)).T + np.abs(_f64(b2))[None, :]
    d = gamma(W2.shape[1] + 6) * A + dh @ np.abs(_f64(W2)).T
    y = np.maximum(S, 0.0) * 2 * _f64(keep2)
    return y, d * 2 * _f64(keep2)


# ---- cells and elementwise kernels ---------------------------------------------------------------------------------------
def gru_cell(gi, gh, h, H):
    """ATen gru_cell (RNN.cpp): r = s(i_r + h_r), z = s(i_z + h_z), n = tanh(i_n + r (W_hn h + b_hn)), h' = (h - n) z + n"""
    ref = so.gru_cell(gh, gi, h, H)
    return ref, so.gru_cell_bound(gh, gi, h, H, np.zeros_like(_f64(gh)))


def lstm_cell(g, c, H, x=None):
    """ATen lstm_cell on pre-activations g (i|f|g|o): (c', h', x + h')"""
    cn, hn = so.lstm_cell(g, c, H)
    dc, dh = so.lstm_cell_bound(g, c, H, np.zeros_like(_f64(g)))
    if x is None:
        return cn, hn, None, dc, dh, None
    xn = _f64(x) + hn
    return cn, hn, xn, dc, dh, dh + U24 * np.abs(xn)


def highway(x12, y, C):
    """y' = g relu(x1) + (1 - g) y, g = sigmoid(x2) (highway_network.py:12-17)"""
    x1, x2, y = _f64(x12[:, :C]), _f64(x12[:, C:2 * C]), _f64(y)
    g = 1.0 / (1.0 + np.exp(-x2))
    r = np.maximum(x1, 0.0)
    out = g * r + (1 - g) * y
    d = np.abs(r - y) * E_SIG + 4 * U24 * (np.abs(g * r) + np.abs((1 - g) * y) + np.abs(out) + np.abs(y))
    return out, d


def maxpool2(x):
    """MaxPool1d(2, 1, 1)[:T] over time of [B][T][C]: out[t] = max(x[t - 1], x[t])"""
    x = _f64(x)
    out = x.copy()
    out[:, 1:] = np.maximum(x[:, 1:], x[:, :-1])
    return out


# ---- location-sensitive attention (lsa_step_kernel, lsa_ctx_kernel) ------------------------------------------------------
def loc_conv(cum, conv_w, conv_b):
    """conv1d(cumulative, k = 31, padding 15) + bias: [B][Tc] -> [B][Tc][32], with |terms| for the bound"""
    cum, w, b = _f64(cum), _f64(conv_w).reshape(32, ATT_K), _f64(conv_b)
    B, Tc = cum.shape
    pad = np.zeros((B, Tc + ATT_K - 1))
    pad[:, 15:15 + Tc] = cum
    win = np.stack([pad[:, j:j + Tc] for j in range(ATT_K)], -1)  # [B][Tc][31]: cum[t + j - 15]
    loc = win @ w.T + b
    A = np.abs(win) @ np.abs(w).T + np.abs(b)
    return loc, A


def softmax_bound(s, u, du, Tc):
    """first-order |ds| of s = softmax(u) over the last axis given |du|, plus exp / subtraction / sum / division roundings"""
    mx = np.max(u, -1, keepdims=True)
    e_rel = 4 * U24 + U24 * np.abs(u - mx)
    rel = du + np.sum(s * du, -1, keepdims=True) + e_rel + np.max(e_rel, -1, keepdims=True) + gamma(Tc + 8) + U24
    return 1.01 * s * rel


def lsa_step(pq, proj, seq, chars, cum, conv_w, conv_b, Lw, vw, q_in=None, Wq=None, bq=None, ctx=True):
    """one step of LSA (lsa.py:21-42): u = v . tanh(pq + proj + L loc(cum)), u *= (chars != 0) (padded positions score
    exp(0)), scores = softmax over all Tc, cum' = cum + scores, ctx = scores @ seq.  pq = Wq q + bq when q_in is given.
    Returns dict of (value, bound) for scores, cum, ctx."""
    proj, seq, Lw, vw = _f64(proj), _f64(seq), _f64(Lw), _f64(vw).reshape(-1)
    B, Tc, D = proj.shape
    if q_in is not None:
        q = _f64(q_in)
        pqv = q @ _f64(Wq).T + _f64(bq)
        dpq = gamma(D + 6) * (np.abs(q) @ np.abs(_f64(Wq)).T + np.abs(_f64(bq)))
    else:
        pqv, dpq = _f64(pq), np.zeros((B, D))
    loc, locA = loc_conv(cum, conv_w, conv_b)
    dloc = gamma(ATT_K + 1) * locA
    pl = loc @ Lw.T                                             # [B][Tc][D]
    dpl = gamma(32) * (np.abs(loc) @ np.abs(Lw).T) + dloc @ np.abs(Lw).T
    arg = pqv[:, None, :] + proj + pl
    darg = dpq[:, None, :] + dpl + 2 * U24 * (np.abs(pqv)[:, None, :] + np.abs(proj) + np.abs(pl) + np.abs(arg))
    th = np.tanh(arg)
    dth = darg + E_TANH
    u = th @ vw
    du = gamma(D + 4) * (np.abs(th) @ np.abs(vw)) + (dth + U24 * np.abs(th)) @ np.abs(vw)
    keep = np.asarray(chars) != 0
    u, du = np.where(keep, u, 0.0), np.where(keep, du, 0.0)
    e = np.exp(u - u.max(-1, keepdims=True))
    s = e / e.sum(-1, keepdims=True)
    ds = softmax_bound(s, u, du, Tc)
    cn = _f64(cum) + s
    out = {"scores": (s, ds), "cum": (cn, ds + U24 * np.abs(cn))}
    if ctx:
        out["ctx"] = context(s, seq, ds)
    return out


def context(s, seq, ds=None):
    """ctx[b] = scores[b] @ seq[b] (tacotron.py:104 via lsa.py:40)"""
    s, seq = _f64(s), _f64(seq)
    c = np.einsum("bt,btf->bf", s, seq)
    d = gamma(s.shape[1] + 4) * np.einsum("bt,btf->bf", np.abs(s), np.abs(seq))
    if ds is not None:
        d = d + np.einsum("bt,btf->bf", ds, np.abs(seq))
    return c, d


def lsa_step_rows(row_len, proj, seq, chars, cum, pq=None, q_in=None, ctx=True, **kw):
    """LSA step of a ragged batch in the reference's per-utterance semantics: row b is the B = 1 utterance of its first
    row_len[b] characters, unpadded (lsa_step on the row cut to its length, whose location conv pads with zeros past the end).
    Positions t >= row_len[b] are not part of the utterance: their score is exactly 0 (bound 0) and their cumulative
    attention is the input's (bound 0).  Same arguments and result as lsa_step."""
    B, Tc = np.asarray(chars).shape
    S = np.asarray(seq).shape[2]
    out = {"scores": (np.zeros((B, Tc)), np.zeros((B, Tc))), "cum": (_f64(cum).copy(), np.zeros((B, Tc)))}
    if ctx:
        out["ctx"] = (np.zeros((B, S)), np.zeros((B, S)))
    for b in range(B):
        n = int(row_len[b])
        one = lsa_step(pq=None if pq is None else pq[b:b + 1], proj=proj[b:b + 1, :n], seq=seq[b:b + 1, :n],
                       chars=np.asarray(chars)[b:b + 1, :n], cum=np.asarray(cum)[b:b + 1, :n],
                       q_in=None if q_in is None else q_in[b:b + 1], ctx=ctx, **kw)
        for k, (v, d) in one.items():
            if k == "ctx":
                out[k][0][b], out[k][1][b] = v[0], d[0]
            else:
                out[k][0][b, :n], out[k][1][b, :n] = v[0], d[0]
    return out


def context_rows(s, seq, row_len, ds=None):
    """context of a ragged batch: row b is context() of its first row_len[b] scores and encoder rows"""
    s = _f64(s)
    c, d = np.zeros((s.shape[0], np.asarray(seq).shape[2])), np.zeros((s.shape[0], np.asarray(seq).shape[2]))
    for b in range(s.shape[0]):
        n = int(row_len[b])
        cb, db = context(s[b:b + 1, :n], np.asarray(seq)[b:b + 1, :n], None if ds is None else ds[b:b + 1, :n])
        c[b], d[b] = cb[0], db[0]
    return c, d


# ---- global style token attention (gst_attention_kernel) -----------------------------------------------------------------
def gst_attention(q, keys, values, heads):
    """multi-head attention of global_style_token.py:110-145 for one query per row: scores = q_h k_h / sqrt(E / heads),
    softmax over the tokens, out_h = p_h v_h.  q [B][E], keys / values [ntok][E] -> [B][E]"""
    q, k, v = _f64(q), _f64(keys), _f64(values)
    B, E = q.shape
    hd = E // heads
    out, d = np.zeros((B, E)), np.zeros((B, E))
    scale = 1.0 / np.sqrt(hd)
    for h in range(heads):
        sl = slice(h * hd, (h + 1) * hd)
        a = q[:, sl] @ k[:, sl].T * scale
        da = (gamma(hd) * (np.abs(q[:, sl]) @ np.abs(k[:, sl]).T) * scale + 4 * U24 * np.abs(a))
        e = np.exp(a - a.max(-1, keepdims=True))
        p = e / e.sum(-1, keepdims=True)
        dp = softmax_bound(p, a, da, k.shape[0])
        out[:, sl] = p @ v[:, sl]
        d[:, sl] = gamma(k.shape[0]) * (p @ np.abs(v[:, sl])) + dp @ np.abs(v[:, sl])
    return out, d


# ---- stop projection and rule (stop_step_kernel, stop_flag_kernel) -------------------------------------------------------
def stop_value(xs, w, bias):
    """sigmoid(w . [x | ctx] + b) (tacotron.py:131-133) per row; xs: list of [M][K_j], w: [sum K_j]"""
    X = np.concatenate([_f64(x) for x in xs], 1)
    w, b = _f64(w).reshape(-1), float(np.asarray(bias).reshape(-1)[0])
    z = X @ w + b
    dz = gamma(X.shape[1] + 14) * (np.abs(X) @ np.abs(w) + abs(b))
    return 1.0 / (1.0 + np.exp(-z)), dz / 4 + E_SIG


def stop_flag(stopv, min_stop_token, step, r):
    """tacotron.py:275: stop when every row's stop * 10 > min_stop_token and the frame index step * r > 10"""
    return int(bool(np.all(np.asarray(stopv, np.float32) * np.float32(10) > np.float32(min_stop_token))) and step * r > 10)


def stop_rows(stopv, min_stop_token, r, caps):
    """per-row stop rule of a ragged batch, as the B = 1 decoder loop of tacotron.py:268-276 would break for each utterance:
    stopv [n_steps][B] stop values of decoder steps 0 ..; row b's loop runs si = 0 .. caps[b] - 1 (frame t = si * r, caps[b] =
    ceil(steps_b / r)) and breaks at the first si with stop * 10 > min_stop_token and t > 10.  Returns (done [B], flags
    [n_steps]): done[b] = the step the row's loop ends at (its last step, caps[b] - 1, without a break; -1 when it has not ended
    within n_steps), flags[si] = 1 when every row has ended by step si"""
    v = np.asarray(stopv, np.float32)
    n_steps, B = v.shape
    done = np.full(B, -1)
    for b in range(B):
        for si in range(min(int(caps[b]), n_steps)):
            if (v[si, b] * np.float32(10) > np.float32(min_stop_token) and si * r > 10) or si == int(caps[b]) - 1:
                done[b] = si
                break
    flags = np.array([int(np.all((done >= 0) & (done <= si))) for si in range(n_steps)])
    return done, flags


# ---- BN fold, layout kernels ---------------------------------------------------------------------------------------------
def bn_fold(g, b, mean, var):
    """eval BatchNorm as y = x scale + shift: scale = g / sqrt(var + 1e-5), shift = b - mean scale"""
    g, b, mean, var = (_f64(t) for t in (g, b, mean, var))
    s = g / np.sqrt(var + float(np.float32(1e-5)))
    sh = b - mean * s
    ds = 5 * U24 * np.abs(s)
    return (s, ds), (sh, np.abs(mean) * ds + 2 * U24 * (np.abs(mean * s) + np.abs(sh)))


def pack_melproj(W, n_mels, max_r, r):
    """rows of mel_proj [n_mels * max_r][K] regrouped frame-major: dst[j * n_mels + m] = W[m * max_r + j], j < r"""
    W = np.asarray(W)
    return np.concatenate([W[np.arange(n_mels) * max_r + j] for j in range(r)], 0)


def to_ncl(x, steps, B, C, frames):
    """[B][steps][C] (first `frames` rows) -> [B][C][frames]"""
    return np.asarray(x).reshape(B, steps, C)[:, :frames].transpose(0, 2, 1)


# ---- Philox4x32-10 dropout keep flags (fill_masks_kernel, fill_masks_steps_kernel) ---------------------------------------
M0, M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
W0, W1 = np.uint32(0x9E3779B9), np.uint32(0xBB67AE85)
MASK_TAG = 0x7461636F  # counter word 3 of the Tacotron dropout streams ("taco")


def philox4x32(c0, c1, c2, c3, k0, k1):
    """Philox4x32-10 (Salmon et al., SC'11) on uint32 arrays -> (o0, o1, o2, o3)"""
    c = [np.asarray(v, np.uint64) & np.uint64(0xFFFFFFFF) for v in (c0, c1, c2, c3)]
    c = [v.astype(np.uint32) for v in np.broadcast_arrays(*c)]
    k0, k1 = np.uint32(k0), np.uint32(k1)
    with np.errstate(over="ignore"):
        for _ in range(10):
            p0 = M0 * c[0].astype(np.uint64)
            p1 = M1 * c[2].astype(np.uint64)
            c = [((p1 >> np.uint64(32)).astype(np.uint32) ^ c[1] ^ k0), p1.astype(np.uint32),
                 ((p0 >> np.uint64(32)).astype(np.uint32) ^ c[3] ^ k1), p0.astype(np.uint32)]
            k0, k1 = np.uint32(k0 + W0), np.uint32(k1 + W1)
    return c


def fill_masks(n, seed, stream_id, first=0):
    """keep flags i in [first, first + n) of stream `stream_id`: bit 16 of word (i & 3) of Philox((i >> 2, i >> 34, stream_id,
    "taco"), (seed lo, seed hi))"""
    i = np.arange(first, first + n, dtype=np.uint64)
    o = philox4x32(i >> np.uint64(2), i >> np.uint64(34), np.uint32(stream_id), MASK_TAG, seed & 0xFFFFFFFF, seed >> 32)
    words = np.stack(o, 0)[(i & np.uint64(3)).astype(np.int64), np.arange(n)]
    return ((words >> np.uint32(16)) & np.uint32(1)).astype(np.uint8)


def fill_masks_steps(n_per_step, n_steps, seed):
    """fill_masks_steps_kernel: step s of all decoder steps uses stream_id = s"""
    return np.concatenate([fill_masks(n_per_step, seed, s) for s in range(n_steps)])


SEEDED_TAG = 0x72616767  # counter word 3 of the per-utterance dropout streams of ragged batches ("ragg")


def seeded_masks(seed, npos, units, dec):
    """one utterance's PreNet keep flags [2 layers][npos][units] drawn with its own seed (fill_masks_seeded_kernel): bit 16 of
    word (u & 3) of Philox((u >> 2, position, 2 dec + layer, "ragg"), (seed lo, seed hi)); position = character (dec 0, the
    encoder PreNet) or decoder step (dec 1).  Nothing depends on the row or the batch."""
    l, pos, u = np.meshgrid(np.arange(2), np.arange(npos), np.arange(units), indexing="ij")
    o = philox4x32(u >> 2, pos, 2 * dec + l, SEEDED_TAG, seed & 0xFFFFFFFF, seed >> 32)
    words = np.choose(u & 3, o)
    return ((words >> np.uint32(16)) & np.uint32(1)).astype(np.uint8)


def fill_masks_seeded(seeds, npos, units, dec):
    """the kernel's layouts of the per-utterance flags: dec 0 [2][B][npos][units], dec 1 [npos][2][B][units]"""
    m = np.stack([seeded_masks(int(s), npos, units, dec) for s in seeds], 1)  # [2][B][npos][units]
    return m if dec == 0 else np.ascontiguousarray(m.transpose(2, 0, 1, 3))
