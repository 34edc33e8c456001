"""CPU tests of oracle/tc_split_oracle.py: the bounds the tensor-core GEMM tests (test_taco_tc_gemm.py) use have teeth.

At the shapes of the GPU tests, a float32 emulation of the 3-term split in several summation orders (sequential, blocks of 16,
pairwise) stays inside acc_bound, and each of these kernel mistakes is rejected: a split term dropped, plain fp16 operands, one
k-block skipped, the split-K partial sum added twice, an im2col row read across a sequence boundary, and the bias of a
gate-interleaved image added in natural order."""
import numpy as np
import pytest

import tc_split_oracle as so

RNG = np.random.default_rng(7)


def _emulate(A, W, scale, order="seq", drop=None, fp16=False, skip_kb=None, k_lo=0, k_hi=None):
    """float32 accumulation of the split products in the kernel's term order, times 1 / scale"""
    ah, al = so.split16(A)
    wh, wl = so.split16(so.scaled_weight(W, scale))
    ah, al, wh, wl = (t.astype(np.float32) for t in (ah, al, wh, wl))
    K = A.shape[1]
    k_hi = K if k_hi is None else k_hi
    terms = [(ah, wh), (al, wh), (ah, wl)]
    if fp16:
        terms = terms[:1]
    if drop is not None:
        terms = [t for i, t in enumerate(terms) if i != drop]
    acc = np.zeros((A.shape[0], W.shape[0]), np.float32)
    blocks = [k for k in range(k_lo, k_hi, 16) if skip_kb is None or k // 64 != skip_kb]
    if order == "pairwise":
        prods = [a[:, k, None] * w[None, :, k] for k0 in blocks for a, w in terms for k in range(k0, min(k0 + 16, k_hi))]
        while len(prods) > 1:
            prods = [prods[i] + prods[i + 1] if i + 1 < len(prods) else prods[i] for i in range(0, len(prods), 2)]
        acc = prods[0].astype(np.float32)
    else:
        for k0 in blocks:
            for a, w in terms:
                if order == "block16":
                    blk = np.zeros_like(acc)
                    for k in range(k0, min(k0 + 16, k_hi)):
                        blk += a[:, k, None] * w[None, :, k]
                    acc += blk
                else:
                    for k in range(k0, min(k0 + 16, k_hi)):
                        acc += a[:, k, None] * w[None, :, k]
    return acc * np.float32(1.0 / scale)


def _ratio(got, ref, bound):
    return float(np.max(np.abs(np.asarray(got, np.float64) - ref) / bound))


def _case(M=100, N=160, K=170, wscale=0.05):
    A = RNG.standard_normal((M, K)).astype(np.float32)
    W = (RNG.standard_normal((N, K)) * wscale).astype(np.float32)
    return A, W, so.pow2_scale(W)


@pytest.mark.parametrize("order", ["seq", "block16", "pairwise"])
def test_bound_accepts_fp32_orders(order):
    A, W, s = _case()
    ref, b = so.split_sum(A, W, s), so.acc_bound(A, W, s)
    assert _ratio(_emulate(A, W, s, order), ref, b) <= 1.0


@pytest.mark.parametrize("mut", ["drop_lo_a_hi_w", "drop_hi_a_lo_w", "plain_fp16", "skip_kblock"])
def test_bound_rejects_product_mutations(mut):
    A, W, s = _case()
    ref, b = so.split_sum(A, W, s), so.acc_bound(A, W, s)
    kw = {"drop_lo_a_hi_w": {"drop": 1}, "drop_hi_a_lo_w": {"drop": 2}, "plain_fp16": {"fp16": True},
          "skip_kblock": {"skip_kb": 1}}[mut]
    assert _ratio(_emulate(A, W, s, **kw), ref, b) > 1.0


def test_bound_rejects_pre_added_twice():
    """split K: PLAIN over k-blocks [0, kb0), main launch over [kb0, KB) adding that partial sum (`pre`) once"""
    A, W, s = _case(M=65, N=160, K=256)
    kb0 = 1
    pre = _emulate(A, W, s, k_hi=64 * kb0)
    main = _emulate(A, W, s, k_lo=64 * kb0)
    ref = so.split_sum(A, W, s)
    b = so.acc_bound(A, W, s, k_hi=64 * kb0) + so.acc_bound(A, W, s, k_lo=64 * kb0) + so.U24 * (np.abs(ref) + np.abs(pre))
    assert _ratio(main + pre, ref, b) <= 1.0
    assert _ratio(main + 2 * pre, ref, b) > 1.0


def test_bound_rejects_im2col_row_across_sequence_boundary():
    M, T, K, N = 513, 48, 80, 132
    x = RNG.standard_normal((M, K)).astype(np.float32)
    shifts = [-2, 0, 2]
    W = (RNG.standard_normal((N, 3 * K)) * 0.05).astype(np.float32)
    s = so.pow2_scale(W)
    A = so.im2col([x] * 3, shifts, K, M, T)
    ref, b = so.split_sum(A, W, s), so.acc_bound(A, W, s)
    assert _ratio(_emulate(A, W, s, "block16"), ref, b) <= 1.0
    bad = A.copy()
    m = T - 1  # last row of the first sequence: tap +2 must read zeros, not the next sequence's row 1
    bad[m, 2 * K:] = x[m + 2]
    assert _ratio(_emulate(bad, W, s, "block16"), ref, b) > 1.0


def test_im2col_zero_outside_sequences():
    x = np.arange(1, 11, dtype=np.float32)[:, None]
    A = so.im2col([x, x], [-1, 1], 1, 10, 5)
    assert A[:, 0].tolist() == [0, 1, 2, 3, 4, 0, 6, 7, 8, 9]
    assert A[:, 1].tolist() == [2, 3, 4, 5, 0, 7, 8, 9, 10, 0]


def test_bound_rejects_bias_in_natural_order():
    """LSTM images are gate-interleaved (tile t holds i|f|g|o of units 8t..8t+7); so must the bias be"""
    M, H, K = 7, 64, 128
    A = RNG.standard_normal((M, K)).astype(np.float32)
    W = (RNG.standard_normal((4 * H, K)) * 0.05).astype(np.float32)
    bias = RNG.standard_normal(4 * H).astype(np.float32)
    c = RNG.standard_normal((M, H)).astype(np.float32)
    s = so.pow2_scale(W)
    G = so.split_sum(A, W, s) + bias
    dG = so.acc_bound(A, W, s) + so.U24 * np.abs(G)
    c_ref, h_ref = so.lstm_cell(G, c, H)
    dc, dh = so.lstm_cell_bound(G, c, H, dG)
    rows = so.gate_rows(H, 4)
    acc_tile = _emulate(A, W[rows], s)                   # accumulators in tile (packed) column order
    inv = np.argsort(rows)
    for bias_tile, ok in ((bias[rows], True), (bias, False)):
        g = (acc_tile + bias_tile)[:, inv]
        c1, h1 = so.lstm_cell(g, c, H)
        assert (_ratio(c1, c_ref, dc) <= 1.0 and _ratio(h1, h_ref, dh) <= 1.0) == ok


def test_rep_bound_within_contract_and_exact():
    """emulated split vs exact float64 over |a| log-uniform in [1e-8, 6e4]: inside rep_bound, which is inside the contract"""
    M, N, K = 64, 96, 40
    A = (np.exp(RNG.uniform(np.log(1e-8), np.log(6e4), (M, K))) * RNG.choice([-1, 1], (M, K))).astype(np.float32)
    W = (RNG.standard_normal((N, K)) * 0.05).astype(np.float32)
    W[0, :] *= 2.0 ** -20
    s = so.pow2_scale(W)
    ex, sp = so.exact(A, W), so.split_sum(A, W, s)
    rb, cb = so.rep_bound(A, W, s), so.contract_bound(A, W, s)
    assert np.all(np.abs(sp - ex) <= rb)
    assert np.all(rb <= cb)
    # plain fp16 operands break the contract
    ah = so.split16(A)[0].astype(np.float64)
    wh = so.split16(so.scaled_weight(W, s))[0].astype(np.float64)
    assert np.any(np.abs(ah @ wh.T / s - ex) > cb)


def test_split_of_fp16_overflow_is_not_finite():
    """|a| >= 65520 rounds hi(a) to inf: the contract's input range ends there"""
    hi, lo = so.split16(np.array([65519.0, 65520.0], np.float32))
    assert np.isfinite(hi[0]) and np.isinf(hi[1])


def test_pow2_scale_rule():
    assert so.pow2_scale(np.zeros(4)) == 4096.0
    for mx in (1.0, 0.75, 3e-5, 1234.5):
        s = so.pow2_scale(np.array([0.1 * mx, -mx], np.float32))
        assert 2048 <= mx * s < 4096


def test_unpackers_invert_the_swizzle():
    rows_pad, KB = 64, 2
    logical = RNG.standard_normal((rows_pad, KB * 64)).astype(np.float16)
    tiles = np.empty(KB * rows_pad * 64, np.float16)
    for m in range(rows_pad):
        for k in range(KB * 64):
            kb, c8, e = k // 64, (k % 64) // 8, k % 8
            tiles[((kb * rows_pad + m) * 8 + (c8 ^ (m & 7))) * 8 + e] = logical[m, k]
    assert np.array_equal(so.unpack_act_tiles(tiles, rows_pad, KB), logical)
    n_tiles, rows = 2, 32
    hi = RNG.standard_normal((n_tiles * rows, KB * 64)).astype(np.float16)
    lo = RNG.standard_normal((n_tiles * rows, KB * 64)).astype(np.float16)
    img = np.empty(n_tiles * KB * 2 * rows * 64, np.float16)
    for j in range(n_tiles):
        for kb in range(KB):
            for p, src in enumerate((hi, lo)):
                for n in range(rows):
                    for c8 in range(8):
                        o = ((((j * KB + kb) * 2 + p) * rows + n) * 8 + (c8 ^ (n & 7))) * 8
                        img[o:o + 8] = src[j * rows + n, kb * 64 + c8 * 8:kb * 64 + c8 * 8 + 8]
    h2, l2 = so.unpack_weight_tiles(img, n_tiles, KB, rows)
    assert np.array_equal(h2, hi) and np.array_equal(l2, lo)
