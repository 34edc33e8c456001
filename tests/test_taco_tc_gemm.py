"""GPU tests of the 3-term-split tensor-core GEMMs of csrc/tacotron_tc.cu, one launch at a time (mb_taco_tc_debug), against the
float64 references and bounds of oracle/tc_split_oracle.py.

Every case compares the kernel with the emulated split under the FP32-accumulation bound; a subset also compares with the exact
float64 product under accumulation + representation bound.  Outputs sit in NaN-filled buffers and nothing outside the region a
launch writes may change.  RAN records which kernel ran in which launch variant; the last test asserts every one was seen."""
import numpy as np
import pytest
import torch

import encoder_oracle as eo
import ref_init as ri
import tc_split_oracle as so

pytestmark = pytest.mark.gpu
RAN = set()
WORST = {}


def _dbg(*a, **k):
    from mockingbird_b200.synthesizer.tc_debug import parse_report, tc_debug

    rep = parse_report(tc_debug(*a, **k))
    kern = rep["kernel"]
    RAN.add((kern, "compact" if rep["compact"] == "1" else "noncompact"))
    RAN.add((kern, "cluster" + rep["cluster"]))
    for g in rep["mma_groups"].split(","):
        RAN.add((kern, "mma" + g))
    return rep


def _g(seed):
    return np.random.default_rng(seed)


def _cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _nan(*shape):
    return torch.full(shape, float("nan"), device="cuda")


def _check(name, got, ref, bound):
    got = np.asarray(got, np.float64)
    assert np.all(np.isfinite(got)), name
    r = float(np.max(np.abs(got - ref) / bound))
    WORST[name] = max(WORST.get(name, 0.0), r)
    assert r <= 1.0, (name, r)


# ---- tc_skinny PLAIN -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("M", [1, 7, 63, 64, 65, 100, 127, 128])
@pytest.mark.parametrize("N", [160, 1000])
@pytest.mark.parametrize("compact", [0, 1])
def test_skinny_plain(M, N, compact):
    if compact and M > 64:
        pytest.skip("the compact ring exists for <= 64 rows only")
    g = _g(M * 7 + N)
    K0, K1 = 100, 70  # partial last k-block (170 of 192), two segments
    A0 = g.standard_normal((M, K0)).astype(np.float32)
    A1 = g.standard_normal((M, K1)).astype(np.float32)
    W0 = (g.standard_normal((N, K0)) * 0.05).astype(np.float32)
    W1 = (g.standard_normal((N, K1)) * 0.05).astype(np.float32)
    b0, b1 = g.standard_normal(N).astype(np.float32), g.standard_normal(N).astype(np.float32)
    ldy = N + 8
    y = _nan(M + 1, ldy)
    rep = _dbg("plain", M=M, N=N, K0=K0, K1=K1, w=[_cuda(W0), _cuda(W1)], b=[_cuda(b0), _cuda(b1)],
               x=[_cuda(A0), _cuda(A1)], ldx=[K0, K1], y=y, ldy=ldy, compact=compact, cluster=1)
    assert rep["compact"] == str(compact) and rep["rows_pad"] == ("64" if M <= 64 else "128")
    assert rep["mma_groups"] == ("2,2" if M > 64 else "1,1")
    A, W = np.concatenate([A0, A1], 1), np.concatenate([W0, W1], 1)
    s = so.pow2_scale(W)
    assert abs(float(rep["inv_scale"]) * s - 1.0) < 1e-8
    bias = (b0.astype(np.float32) + b1).astype(np.float64)
    ref = so.split_sum(A, W, s) + bias
    bound = so.acc_bound(A, W, s) + so.U24 * (np.abs(ref) + np.abs(bias))
    out = y.cpu().numpy()
    _check("skinny_plain vs split", out[:M, :N], ref, bound)
    assert np.isnan(out[:M, N:]).all() and np.isnan(out[M:]).all()
    if M in (1, 65, 128):
        _check("skinny_plain vs exact", out[:M, :N], so.exact(A, W) + bias, bound + so.rep_bound(A, W, s))


@pytest.mark.parametrize("M", [64, 128])
@pytest.mark.parametrize("cluster", [2, 4, 8])
def test_skinny_cluster_multicast(M, cluster):
    """activation tiles multicast across clusters of 2 / 4 / 8 CTAs: bitwise equal to the unclustered launch"""
    g = _g(cluster + M)
    N, K = 256, 320
    A = g.standard_normal((M, K)).astype(np.float32)
    W = (g.standard_normal((N, K)) * 0.05).astype(np.float32)
    outs = []
    for cl in (1, cluster):
        y = _nan(M, N)
        rep = _dbg("plain", M=M, N=N, K0=K, w=[_cuda(W)], x=[_cuda(A)], ldx=[K], y=y, ldy=N, cluster=cl, compact=0)
        assert rep["cluster"] == str(cl)
        outs.append(y.cpu().numpy())
    s = so.pow2_scale(W)
    ref = so.split_sum(A, W, s)
    _check("skinny_cluster vs split", outs[1], ref, so.acc_bound(A, W, s) + so.U24 * np.abs(ref))
    assert np.array_equal(outs[0], outs[1])


def test_skinny_split_k_and_step_slab():
    """PLAIN over k-blocks [0, kb0) into `pre`, the main launch over [kb0, KB) adds it; written through the step pointer"""
    g = _g(3)
    M, N, K, kb0 = 70, 160, 256, 1
    A = g.standard_normal((M, K)).astype(np.float32)
    W = (g.standard_normal((N, K)) * 0.05).astype(np.float32)
    b = g.standard_normal(N).astype(np.float32)
    Ad, Wd = _cuda(A), _cuda(W)
    pre = _nan(M, N)
    _dbg("plain", M=M, N=N, K0=K, w=[Wd], x=[Ad], ldx=[K], y=pre, ldy=N, kb0=0, kb_count=kb0)
    step = torch.tensor([2], dtype=torch.int32, device="cuda")
    slabs = _nan(5, M, N)
    _dbg("plain", M=M, N=N, K0=K, w=[Wd], b=[_cuda(b)], x=[Ad], ldx=[K], y=slabs, ldy=N, kb0=kb0, kb_count=K // 64 - kb0,
         pre=pre, ldpre=N, step_ptr=step, step_j=1, y_step=M * N)
    full = _nan(M, N)
    _dbg("plain", M=M, N=N, K0=K, w=[Wd], b=[_cuda(b)], x=[Ad], ldx=[K], y=full, ldy=N)
    out = slabs.cpu().numpy()
    assert np.isnan(out[[0, 1, 2, 4]]).all()  # only slab 2 + 1 is written
    s = so.pow2_scale(W)
    ref = so.split_sum(A, W, s) + b
    bound = (so.acc_bound(A, W, s, k_hi=64 * kb0) + so.acc_bound(A, W, s, k_lo=64 * kb0)
             + so.U24 * (2 * np.abs(ref) + np.abs(pre.cpu().numpy()) + np.abs(b)))
    _check("skinny_splitk vs split", out[3], ref, bound)
    fb = so.acc_bound(A, W, s) + so.U24 * (np.abs(ref) + np.abs(b))
    _check("skinny_splitk vs full", out[3], full.cpu().numpy(), bound + fb)


def _unpack_fused(t, rows_pad, K):
    v = t.cpu().numpy().view(np.float16)
    return so.unpack_act_tiles(v, rows_pad, (K + 63) // 64)


def _assert_split_bits(tiles_hi, tiles_lo, rows_pad, Ktot, vals, k0, name):
    """the fused hi / lo chunks equal act_split of the same fp32 values, bit for bit"""
    hi, lo = so.split16(vals)
    M, n = vals.shape
    th, tl = _unpack_fused(tiles_hi, rows_pad, Ktot), _unpack_fused(tiles_lo, rows_pad, Ktot)
    assert np.array_equal(th[:M, k0:k0 + n].view(np.uint16), hi.view(np.uint16)), name
    assert np.array_equal(tl[:M, k0:k0 + n].view(np.uint16), lo.view(np.uint16)), name
    # nothing else of the tiles was touched (they were zero)
    mask = np.ones(th.shape, bool)
    mask[:M, k0:k0 + n] = False
    assert not th.view(np.uint16)[mask].any() and not tl.view(np.uint16)[mask].any(), name


def test_skinny_plain_fused_split_output():
    g = _g(11)
    M, N, K, s_k0 = 40, 160, 128, 64
    A = g.standard_normal((M, K)).astype(np.float32)
    W = (g.standard_normal((N, K)) * 0.05).astype(np.float32)
    Ktot = s_k0 + N + 32
    hi = torch.zeros(((Ktot + 63) // 64) * 64 * 64, dtype=torch.int16, device="cuda")
    lo = torch.zeros_like(hi)
    y = _nan(M, N)
    _dbg("plain", M=M, N=N, K0=K, w=[_cuda(W)], x=[_cuda(A)], ldx=[K], y=y, ldy=N, s_hi=[hi], s_lo=[lo], s_k0=[s_k0])
    _assert_split_bits(hi, lo, 64, Ktot, y.cpu().numpy(), s_k0, "plain slot 0")


# ---- tc_skinny LSTM ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("M", [5, 65, 128])
def test_skinny_lstm_steps(M):
    """LSTM cell with residual after one step and after 4 chained steps ([x | h] . [W_ih | W_hh]^T, the decoder's LSTMs)"""
    g = _g(M)
    H, K0 = 64, 96
    W0 = (g.standard_normal((4 * H, K0)) * 0.1).astype(np.float32)
    W1 = (g.standard_normal((4 * H, H)) * 0.1).astype(np.float32)
    b0, b1 = (g.standard_normal(4 * H) * 0.3).astype(np.float32), (g.standard_normal(4 * H) * 0.3).astype(np.float32)
    W = np.concatenate([W0, W1], 1)
    s = so.pow2_scale(W)
    bias = (b0 + b1).astype(np.float64)
    x = g.standard_normal((M, K0)).astype(np.float32)
    h = np.zeros((M, H), np.float32)
    c = (g.standard_normal((M, H)) * 0.5).astype(np.float32)
    xr = g.standard_normal((M, H)).astype(np.float32)
    c_ref, h_ref, xr_ref = c.astype(np.float64), h.astype(np.float64), xr.astype(np.float64)
    dc = dh = dx = 0.0
    rows_pad = 64 if M <= 64 else 128
    cd, xrd = _cuda(c), _cuda(xr)
    for step in range(4):
        hd = _nan(M, H)
        shi = [torch.zeros(2 * 64 * rows_pad, dtype=torch.int16, device="cuda") for _ in range(2)]
        slo = [torch.zeros_like(shi[0]) for _ in range(2)]
        _dbg("lstm", M=M, H=H, K0=K0, K1=H, w=[_cuda(W0), _cuda(W1)], b=[_cuda(b0), _cuda(b1)], x=[_cuda(x), _cuda(h)],
             ldx=[K0, H], c=cd, h=hd, xres=xrd, s_hi=shi, s_lo=slo, s_k0=[0, 64])
        A = np.concatenate([x, h], 1)
        # gate error: accumulation + representation at the kernel's own inputs + the propagated input error |W_hh| dh
        G_k = so.split_sum(A, W, s) + bias
        dG = so.acc_bound(A, W, s) + so.rep_bound(A, W, s) + so.U24 * np.abs(G_k) + np.broadcast_to(dh, (M, H)) @ np.abs(W1.astype(np.float64)).T
        G_ref = so.exact(np.concatenate([x.astype(np.float64), h_ref], 1), W) + bias
        dc_new, dh_new = so.lstm_cell_bound(G_ref, c_ref, H, dG, dc)
        c_ref, h_new = so.lstm_cell(G_ref, c_ref, H)
        xr_ref = xr_ref + h_new
        dx = dx + dh_new + so.U24 * np.abs(xr_ref)
        dc, dh, h_ref = dc_new, dh_new, h_new
        c_got, h_got, x_got = cd.cpu().numpy(), hd.cpu().numpy(), xrd.cpu().numpy()
        _check("skinny_lstm c", c_got, c_ref, dc)
        _check("skinny_lstm h", h_got, h_ref, dh)
        _check("skinny_lstm x", x_got, xr_ref, dx)
        _assert_split_bits(shi[0], slo[0], rows_pad, 128, x_got, 0, "lstm slot 0 (x')")
        _assert_split_bits(shi[1], slo[1], rows_pad, 128, h_got, 64, "lstm slot 1 (h')")
        h = h_got.astype(np.float32)


# ---- tc_gru ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("H", [64, 128, 256])
@pytest.mark.parametrize("ndir", [1, 2])
@pytest.mark.parametrize("M", [3, 64, 65, 128])
def test_gru_step(H, ndir, M):
    steps = 16 if (H, ndir, M) in ((128, 2, 65), (64, 1, 3)) else 1
    g = _g(H * 3 + ndir * 5 + M)
    Ws = [(g.standard_normal((3 * H, H)) * (0.5 / np.sqrt(H))).astype(np.float32) for _ in range(ndir)]
    bs = [(g.standard_normal(3 * H) * 0.2).astype(np.float32) for _ in range(ndir)]
    hs = [np.zeros((M, H), np.float32) for _ in range(ndir)]
    h_ref = [np.zeros((M, H)) for _ in range(ndir)]
    dh = [0.0] * ndir
    rows_pad = 64 if M <= 64 else 128
    for t in range(steps):
        gis = [g.standard_normal((M, 3 * H)).astype(np.float32) for _ in range(ndir)]
        hst = [_cuda(hs[d]) for d in range(ndir)]
        outs = [_nan(M, 2 * H) for _ in range(ndir)]
        nxt_hi = [torch.zeros(H * rows_pad, dtype=torch.int16, device="cuda") for _ in range(ndir)]
        nxt_lo = [torch.zeros_like(nxt_hi[0]) for _ in range(ndir)]
        s_hi = torch.zeros(((H + 64 + 63) // 64) * 64 * rows_pad, dtype=torch.int16, device="cuda")
        s_lo = torch.zeros_like(s_hi)
        _dbg("gru", M=M, H=H, K0=H, w=[_cuda(W) for W in Ws], b=[_cuda(b) for b in bs], x=[_cuda(h) for h in hs],
             ldx=[H] * ndir, gi=[_cuda(x) for x in gis], ldgi=3 * H, hst=hst, out=outs, ldout=2 * H, ndir=ndir,
             nxt_hi=nxt_hi, nxt_lo=nxt_lo, s_hi=[s_hi], s_lo=[s_lo], s_k0=[64])
        for d in range(ndir):
            W, b = Ws[d], bs[d].astype(np.float64)
            sc = so.pow2_scale(W)
            gh_k = so.split_sum(hs[d], W, sc) + b
            dgh = (so.acc_bound(hs[d], W, sc) + so.rep_bound(hs[d], W, sc) + so.U24 * np.abs(gh_k)
                   + np.broadcast_to(dh[d], (M, H)) @ np.abs(W.astype(np.float64)).T)
            gh_ref = so.exact(h_ref[d], W) + b
            dh[d] = so.gru_cell_bound(gh_ref, gis[d], h_ref[d], H, dgh, dh[d])
            h_ref[d] = so.gru_cell(gh_ref, gis[d], h_ref[d], H)
            got = hst[d].cpu().numpy()
            o = outs[d].cpu().numpy()
            _check("gru h (chained)" if steps > 1 else "gru h", got, h_ref[d], dh[d])
            assert np.array_equal(o[:, :H], got) and np.isnan(o[:, H:]).all()
            _assert_split_bits(nxt_hi[d], nxt_lo[d], rows_pad, H, got, 0, "gru nxt")
            if d == 0:
                _assert_split_bits(s_hi, s_lo, rows_pad, H + 64, got, 64, "gru s_hi")
            hs[d] = got


# ---- tc_lstm_seq -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("M", [1, 128, 129, 200, 1030])
def test_lstm_seq_step(M):
    """one encoder LSTM step over M rows, with the encoder's strided gi (row stride T * 4H) and out (T * H)"""
    g = _g(M + 1)
    H, T, t = 256, 3, 1
    W = (g.standard_normal((4 * H, H)) * (1 / np.sqrt(H))).astype(np.float32)
    h = (np.tanh(g.standard_normal((M, H)))).astype(np.float32)
    c = g.standard_normal((M, H)).astype(np.float32)
    gi_all = g.standard_normal((M, T, 4 * H)).astype(np.float32)
    out_all = _nan(M, T, H)
    cd = _cuda(c)
    gid = _cuda(gi_all)
    nh = torch.zeros(4 * ((M + 127) // 128 * 128) * 64, dtype=torch.int16, device="cuda")
    nl = torch.zeros_like(nh)
    rep = _dbg("lstm_seq", M=M, H=H, K0=H, w=[_cuda(W)], x=[_cuda(h)], ldx=[H], gi=[gid[:, t]], ldgi=T * 4 * H, c=cd,
               out=[out_all[:, t]], ldout=T * H, nxt_hi=[nh], nxt_lo=[nl])
    assert rep["grid"] == f"{H // 8},{(M + 127) // 128}"
    s = so.pow2_scale(W)
    G = so.split_sum(h, W, s) + gi_all[:, t]
    dG = so.acc_bound(h, W, s) + so.U24 * np.abs(G)
    c_ref, h_ref = so.lstm_cell(G, c, H)
    dc, dh = so.lstm_cell_bound(G, c, H, dG)
    _check("lstm_seq c", cd.cpu().numpy(), c_ref, dc)
    out = out_all.cpu().numpy()
    _check("lstm_seq h", out[:, t], h_ref, dh)
    assert np.isnan(out[:, [0, 2]]).all()
    _assert_split_bits(nh, nl, (M + 127) // 128 * 128, H, out[:, t], 0, "lstm_seq nxt")
    Gx = so.exact(h, W) + gi_all[:, t]
    dcx, dhx = so.lstm_cell_bound(Gx, c, H, dG + so.rep_bound(h, W, s))
    _check("lstm_seq h vs exact", out[:, t], so.lstm_cell(Gx, c, H)[1], dhx)


# ---- tc_big ----------------------------------------------------------------------------------------------------------------
BIG = [(512, 4, 40, 1, 1, 0), (513, 124, 80, 3, 48, 1), (640, 128, 256, 5, 3, 2), (1000, 132, 40, 2, 48, 3),
       (513, 260, 80, 4, 1, 1), (1000, 128, 256, 1, 48, 2), (640, 260, 40, 5, 48, 3), (512, 132, 80, 3, 3, 0)]


@pytest.mark.parametrize("M,N,K,nseg,T,epi", BIG)
def test_big(M, N, K, nseg, T, epi):
    """conv over time: nseg taps with shifts in -2..2 (zero outside each length-T sequence), epilogue 0: none,
    1: ReLU, 2: ReLU + BN, 3: BN + residual"""
    g = _g(M + N + K)
    shifts = [(-2, -1, 0, 1, 2)[(i * 3 + nseg) % 5] for i in range(nseg)]
    x = g.standard_normal((M, K)).astype(np.float32)
    Wc = (g.standard_normal((N, K, nseg)) * 0.05).astype(np.float32)  # Conv1d weight [co][ci][k], read with column stride k
    bias = g.standard_normal(N).astype(np.float32)
    act = 1 if epi in (1, 2) else 0
    bn_s = (g.uniform(0.5, 1.5, N)).astype(np.float32) if epi >= 2 else None
    bn_b = g.standard_normal(N).astype(np.float32) if epi >= 2 else None
    res = g.standard_normal((M, N)).astype(np.float32) if epi == 3 else None
    ldy = N + 4
    y = _nan(M + 3, ldy)
    xd = _cuda(x)
    rep = _dbg("big", M=M, N=N, K0=K, w=[_cuda(Wc)], ldw=K * nseg, b=[_cuda(bias)], x=[xd] * nseg, ldx=[K] * nseg,
               shift=shifts, w_off=list(range(nseg)), w_stride=[nseg] * nseg, nseg=nseg, T=T, y=y, ldy=ldy, act=act,
               bn_scale=None if bn_s is None else _cuda(bn_s), bn_shift=None if bn_b is None else _cuda(bn_b),
               res=None if res is None else _cuda(res), ldres=N)
    assert rep["grid"] == f"{(N + 127) // 128},{(M + 127) // 128}"
    A = so.im2col([x] * nseg, shifts, K, M, T)
    W = np.concatenate([Wc[:, :, j] for j in range(nseg)], 1)
    s = so.pow2_scale(Wc)
    S = so.split_sum(A, W, s)
    ref = so.big_epilogue(S, bias, act, bn_s, bn_b, res)
    bound = so.big_epilogue_bound(S, so.acc_bound(A, W, s), bias, act, bn_s, bn_b, res)
    out = y.cpu().numpy()
    _check("big vs split", out[:M, :N], ref, bound)
    assert np.isnan(out[:M, N:]).all() and np.isnan(out[M:]).all()
    if epi == 0:
        refx = so.big_epilogue(so.exact(A, W), bias)
        _check("big vs exact", out[:M, :N], refx, bound + so.rep_bound(A, W, s))


# ---- packers ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", ["max_last", "zero", "wide_range"])
def test_weight_pack(case):
    g = _g(5)
    M, N, K = 9, 64, 100
    W = (g.standard_normal((N, K)) * 0.05).astype(np.float32)
    if case == "max_last":
        W[-1, -1] = 0.75
    elif case == "zero":
        W[:] = 0
    else:
        W *= np.exp2(-20 * g.uniform(0, 1, (N, K))).astype(np.float32)
        W[3, 3] = 0.1
    A = g.standard_normal((M, K)).astype(np.float32)
    KB = (K + 63) // 64
    wt = torch.zeros(2 * 2 * KB * 32 * 64, dtype=torch.int16, device="cuda")
    at = torch.zeros(2 * KB * 64 * 64, dtype=torch.int16, device="cuda")
    y = _nan(M, N)
    rep = _dbg("plain", M=M, N=N, K0=K, w=[_cuda(W)], x=[_cuda(A)], ldx=[K], y=y, ldy=N, w_tiles=wt, a_tiles=at)
    s = so.pow2_scale(W)
    assert abs(float(rep["inv_scale"]) * s - 1.0) < 1e-8
    if case == "max_last":
        assert s == 4096.0  # 0.75 = 0.75 * 2^0 -> max |w| s in [2^11, 2^12)
    hi, lo = so.unpack_weight_tiles(wt.cpu().numpy().view(np.float16), 2, KB, 32)
    eh, el = so.split16(np.pad(so.scaled_weight(W, s), ((0, 0), (0, KB * 64 - K))))
    assert np.array_equal(hi.view(np.uint16), eh.view(np.uint16)) and np.array_equal(lo.view(np.uint16), el.view(np.uint16))
    av = at.cpu().numpy().view(np.float16)
    ah = so.unpack_act_tiles(av[:KB * 64 * 64], 64, KB)
    xh, _ = so.split16(np.pad(A, ((0, 64 - M), (0, KB * 64 - K))))
    assert np.array_equal(ah.view(np.uint16), xh.view(np.uint16))
    ref = so.split_sum(A, W, s)
    _check("pack vs exact", y.cpu().numpy(), so.exact(A, W), so.acc_bound(A, W, s) + so.rep_bound(A, W, s) + so.U24 * np.abs(ref) + 1e-300)


# ---- activation magnitudes ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["plain", "big"])
def test_activation_magnitude_sweep(kind):
    """|a| log-uniform in [1e-8, 6e4] (the contract's range, incl. the fp16-subnormal floor of lo(a) below 2^-3)"""
    g = _g(17)
    M, N, K = (100, 160, 40) if kind == "plain" else (640, 128, 40)
    A = (np.exp(g.uniform(np.log(1e-8), np.log(6e4), (M, K))) * g.choice([-1, 1], (M, K))).astype(np.float32)
    W = (g.standard_normal((N, K)) * 0.05).astype(np.float32)
    y = _nan(M, N)
    if kind == "plain":
        _dbg("plain", M=M, N=N, K0=K, w=[_cuda(W)], x=[_cuda(A)], ldx=[K], y=y, ldy=N)
    else:
        _dbg("big", M=M, N=N, K0=K, w=[_cuda(W)], ldw=K, x=[_cuda(A)], ldx=[K], shift=[0], w_off=[0], w_stride=[1], nseg=1,
             T=1, y=y, ldy=N)
    s = so.pow2_scale(W)
    out = y.cpu().numpy()
    acc = so.acc_bound(A, W, s) + so.U24 * np.abs(so.split_sum(A, W, s))
    _check(f"sweep {kind} vs split", out, so.split_sum(A, W, s), acc)
    _check(f"sweep {kind} vs contract", out, so.exact(A, W), acc + so.contract_bound(A, W, s))


# ---- speaker encoder on realistic frames --------------------------------------------------------------------------------
@pytest.mark.parametrize("rows", [4, 130])
def test_encoder_log_spread_mel_power(rows):
    """mel *power* frames spread over 1e-8 .. 10 (log-uniform per frame level), incl. all-zero frames and one all-quiet
    partial; 4 rows take tc_big for layer 0 (640 rows x frames), 130 rows two row blocks of tc_lstm_seq"""
    from mockingbird_b200.encoder import inference as enc_inf
    from mockingbird_b200.encoder.model import SpeakerEncoder

    m = SpeakerEncoder()
    sd = ri.encoder_state_dict(0)
    m.load_state_dict(sd)
    m.eval()
    enc_inf.set_model(m)
    g = _g(rows)
    level = np.exp(g.uniform(np.log(1e-8), np.log(10.0), (rows, 160, 1)))
    frames = (level * g.uniform(0, 1, (rows, 160, 40)) ** 4).astype(np.float32)
    frames[0, 40:60] = 0.0
    frames[1] = (frames[1] * 1e-6).astype(np.float32)
    got = enc_inf.embed_frames_batch(frames)
    idx = list(range(rows)) if rows <= 8 else [0, 1, 2, 64, 127, 128, 129]
    ref = eo.embed_frames(sd, torch.from_numpy(frames[idx])).numpy()
    err = float(np.abs(got[idx] - ref).max())
    WORST[f"encoder rows={rows} max_abs"] = err
    assert err < 1e-4, err


def test_every_variant_ran():
    need = {("tc_skinny_plain", v) for v in ("compact", "noncompact", "cluster1", "cluster2", "cluster4", "cluster8", "mma1", "mma2")}
    need |= {(k, v) for k in ("tc_gru", "tc_lstm_seq", "tc_big", "tc_skinny_lstm") for v in ("mma1", "mma2")}
    missing = sorted(need - RAN)
    print("worst |err| / bound:", {k: float(f"{v:.3g}") for k, v in sorted(WORST.items())})
    assert not missing, missing
