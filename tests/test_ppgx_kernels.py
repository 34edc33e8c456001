"""The PPG extractor's kernels one launch at a time (mb_ppgx_debug, and mb_taco_tc_debug for tc_big at the extractor's GEMM
shapes) against the float64 references and bounds of oracle/ppgx_kernel_oracle.py, at the tile widths, head sizes, row lengths
and edges the whole-model tests never reach; whole 2-block models at the unreached sizes against ppgx_oracle.forward; and CPU
self-tests of the references.

Outputs sit in NaN-filled buffers: nothing outside the region a launch owns may change, and the tile padding it owns (rows
past M, columns past K) must be zero.  Inputs past each row's length hold non-zero values, as the forward leaves them there.
RAN records which (kernel, instantiation) ran; the last GPU test asserts every one was seen."""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import gan_oracle as go
import ppgx_kernel_oracle as ko
import ppgx_oracle as po
import ref_init as ri
import tc_split_oracle as so

gpu = pytest.mark.gpu
RAN = set()
WORST = {}


def _dbg(kind, **kw):
    from mockingbird_b200.ppg_extractor.debug import parse_report, ppgx_debug

    rep = parse_report(ppgx_debug(kind, **kw))
    RAN.add((rep["kernel"],))
    return rep


def _g(seed):
    return np.random.default_rng(seed)


def _cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _i32(v):
    return torch.tensor(list(v), dtype=torch.int32, device="cuda")


def _nan(*shape):
    return torch.full(shape, float("nan"), device="cuda")


def _nan16(n):
    return torch.full((n,), float("nan"), dtype=torch.float16, device="cuda")


def _ceil128(m):
    return (m + 127) // 128 * 128


def _check(name, got, ref, bound):
    got = np.asarray(got, np.float64)
    assert np.all(np.isfinite(got)), name
    err = np.abs(got - ref)
    r = float(np.max(np.where(err == 0, 0.0, err / np.maximum(bound, 1e-300)), initial=0.0))
    WORST[name] = max(WORST.get(name, 0.0), r)
    assert r <= 1.0, (name, r)


def _tiles(yh, yl, rows_total, cols, M, name):
    """hi + lo of operand tiles [KB][rows_total][64] in NaN-filled buffers: the tail past the tiles untouched, no NaN inside,
    rows [M, rows_total) and columns [cols, KB 64) zero -> [M][cols] float64"""
    KB = (cols + 63) // 64
    n = KB * rows_total * 64
    th, tl = yh.cpu().numpy(), yl.cpu().numpy()
    assert np.isnan(th[n:]).all() and np.isnan(tl[n:]).all(), name
    val, hi, lo = ko.tile_values(th[:n], tl[:n], rows_total, cols)
    assert not np.isnan(val).any(), name
    for part in (hi, lo):
        assert not part[M:].view(np.uint16).any() and not part[:, cols:].view(np.uint16).any(), name
    return val[:M, :cols]


# ---- conv2d_tc (embed.conv.2) ----------------------------------------------------------------------------------------------
# N, C, k, stride, pad, B, T_in, F_in, len_in: NT 144 / 64 / 32 with one and several n-tiles; K = k^2 C with a partial last
# k-block in most; M < 128, = 128 and several CTAs with a partial last; odd and even inputs at stride 2
CONV = [
    (288, 8, 5, 1, 2, 3, 13, 11, [13, 7, 1]),
    (144, 144, 3, 1, 1, 1, 8, 16, [6]),
    (128, 32, 4, 2, 1, 2, 13, 20, [13, 8]),
    (64, 8, 4, 2, 1, 3, 12, 19, [11, 12, 4]),
    (96, 32, 5, 1, 2, 2, 9, 7, [9, 3]),
    (32, 144, 3, 1, 1, 2, 17, 5, [16, 9]),
    (288, 32, 4, 2, 1, 2, 23, 14, [21, 23]),
    (128, 144, 5, 1, 2, 1, 7, 9, [5]),
    (96, 8, 3, 1, 1, 1, 8, 16, [8]),
    (64, 32, 3, 1, 1, 4, 10, 20, [10, 1, 2, 7]),
]


@gpu
@pytest.mark.parametrize("N,C,k,s,p,B,T,Fi,lens", CONV)
def test_conv2d_tc(N, C, k, s, p, B, T, Fi, lens):
    g = _g(N + C + k + B + T)
    X = g.standard_normal((B, T, Fi, C)).astype(np.float32)  # non-zero past every row's len_in
    hi, lo = so.split16(X)
    w = (g.standard_normal((N, C, k, k)) / math.sqrt(C * k * k)).astype(np.float32)
    bias = (0.3 * g.standard_normal(N)).astype(np.float32)
    ref, bound, exact, xbound, To, Fo = ko.conv2d_tc(X, lens, w, bias, k, s, p)
    M = B * To * Fo
    rows_total, cols = _ceil128(B * To), N * Fo
    n = (cols + 63) // 64 * rows_total * 64
    yh, yl = _nan16(n + 512), _nan16(n + 512)
    rep = _dbg("conv2d_tc", B=B, T=T, F=Fi, C=C, N=N, k=k, stride=s, pad=p, rows_total=rows_total, len=_i32(lens),
               x_hi=_cuda(hi), x_lo=_cuda(lo), w=_cuda(w), bias=_cuda(bias), y_hi=yh, y_lo=yl)
    NT = 144 if N % 144 == 0 else 64 if N % 64 == 0 else 32
    assert rep["kernel"] == "conv2d_tc" and rep["inst"] == str(NT)
    assert rep["grid"] == f"{(M + 127) // 128},{N // NT},1"
    RAN.add(("conv2d_tc", NT, N // NT > 1))
    assert abs(float(rep["inv_scale"]) * so.pow2_scale(w) - 1.0) < 1e-8
    got = _tiles(yh, yl, rows_total, cols, B * To, f"conv2d_tc N={N}")

    def layout(a):  # rows (b, t, f) x n -> tile row b T_out + t, column n F_out + f
        return a.reshape(B, To, Fo, N).transpose(0, 1, 3, 2).reshape(B * To, N * Fo)

    _check("conv2d_tc vs split", got, layout(ref), ko.split_bound(layout(ref), layout(bound)))
    _check("conv2d_tc vs exact", got, layout(exact), ko.split_bound(layout(exact), layout(xbound)))


# ---- attention ----------------------------------------------------------------------------------------------------------------
ATTN_LENS = [301, 1, 2, 31, 32, 33, 63, 64, 65]


def _attention_dk(dk):
    return 16 if dk <= 16 else 32 if dk <= 32 else 40 if dk <= 40 else 64


@gpu
@pytest.mark.parametrize("dk", [8, 16, 20, 32, 36, 48, 64])
@pytest.mark.parametrize("rel", [0, 1])
def test_attn(dk, rel):
    g = _g(dk * 2 + rel)
    H = 3 if dk <= 20 else 2
    D = H * dk
    T_max = 320 if rel else 301
    lens = [int(v) for v in g.permutation(ATTN_LENS)]
    B = len(lens)
    qkv = g.standard_normal((B * T_max, 3 * D)).astype(np.float32)
    ldp = 2 * D + 8
    Pbuf = g.standard_normal((T_max, ldp)).astype(np.float32)
    pu = (0.5 * g.standard_normal((H, dk))).astype(np.float32)
    pv = (0.5 * g.standard_normal((H, dk))).astype(np.float32)
    Pd = _cuda(Pbuf)
    ctx = _nan(B * T_max + 3, D)
    rep = _dbg("attn", B=B, T=T_max, len=_i32(lens), H=H, dk=dk, D=D, ldp=ldp, rel=rel, x=_cuda(qkv),
               P=Pd[:, D:] if rel else None, pu=_cuda(pu) if rel else None, pv=_cuda(pv) if rel else None, y=ctx)
    DK = _attention_dk(dk)
    assert rep["kernel"] == "attn_kernel" and rep["inst"] == str(DK)
    assert rep["grid"] == f"{(T_max + 31) // 32},{H},{B}"
    RAN.add(("attn_kernel", DK, rel))
    if dk < DK:
        RAN.add(("attn_kernel", "dk<DK"))
    ref, bound = ko.attention(qkv, lens, T_max, H, dk, Pbuf[:, D:2 * D] if rel else None, pu, pv)
    out = ctx.cpu().numpy()
    assert np.isnan(out[B * T_max:]).all()
    for b, T in enumerate(lens):
        assert not out[b * T_max + T:(b + 1) * T_max].any(), (b, T)  # queries past the row's T: zeros
    _check(f"attn dk={dk} rel={rel}", out[:B * T_max], ref, bound)


# ---- depthwise conv module ------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("K", [1, 7, 15, 31])
@pytest.mark.parametrize("act", [0, 1, 2])
def test_dw(K, act):
    g = _g(K * 3 + act)
    D = 32 if K == 7 else 176 if K == 15 else 144
    T, lens = 40, [40, 1, 5, 23]
    B = len(lens)
    M = B * T
    rows_total = _ceil128(M)
    pw = g.standard_normal((M, 2 * D)).astype(np.float32)
    w = (0.4 * g.standard_normal((D, 1, K))).astype(np.float32)
    bias = (0.2 * g.standard_normal(D)).astype(np.float32)
    bn = [g.uniform(0.5, 1.5, D), 0.2 * g.standard_normal(D), 0.3 * g.standard_normal(D), g.uniform(0.25, 2.0, D)]
    bn = [v.astype(np.float32) for v in bn]
    n = (D + 63) // 64 * rows_total * 64
    yh, yl = _nan16(n + 256), _nan16(n + 256)
    _dbg("dw", B=B, T=T, len=_i32(lens), D=D, k=K, act=act, rows_total=rows_total, x=_cuda(pw), w=_cuda(w), bias=_cuda(bias),
         bn=[_cuda(v) for v in bn], y_hi=yh, y_lo=yl)
    got = _tiles(yh, yl, rows_total, D, M, f"dw K={K}")
    ref, bound = ko.depthwise(pw, lens, T, w, bias, *bn, act)
    for b, L in enumerate(lens):
        assert not got[b * T + L:(b + 1) * T].any(), (b, L)
    _check(f"dw K={K} act={act}", got, ref, ko.split_bound(ref, bound))


# ---- LayerNorm / activation operand tiles -----------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("D", [32, 144, 176])
def test_ln_tiles(D):
    g = _g(D)
    M = 300
    rows_total = _ceil128(M)
    x = (2.0 + 3.0 * g.standard_normal((M, D))).astype(np.float32)
    gam = g.uniform(0.5, 1.5, D).astype(np.float32)
    bet = (0.3 * g.standard_normal(D)).astype(np.float32)
    n = (D + 63) // 64 * rows_total * 64
    yh, yl = _nan16(n + 256), _nan16(n + 256)
    _dbg("ln_tiles", M=M, D=D, rows_total=rows_total, x=_cuda(x), w=_cuda(gam), bias=_cuda(bet), y_hi=yh, y_lo=yl)
    got = _tiles(yh, yl, rows_total, D, M, f"ln_tiles D={D}")
    ref, bound = ko.layer_norm(x, gam, bet)
    _check(f"ln_tiles D={D}", got, ref, ko.split_bound(ref, bound))


@gpu
@pytest.mark.parametrize("D", [32, 144, 176])
@pytest.mark.parametrize("act", [0, 1, 2])
def test_act_tiles(D, act):
    g = _g(D + act)
    M, ld = 130, D + 24
    rows_total = _ceil128(M)
    src = (2.0 * g.standard_normal((M, ld))).astype(np.float32)
    n = (D + 63) // 64 * rows_total * 64
    yh, yl = _nan16(n + 256), _nan16(n + 256)
    _dbg("act_tiles", M=M, D=D, ld=ld, act=act, rows_total=rows_total, x=_cuda(src), y_hi=yh, y_lo=yl)
    got = _tiles(yh, yl, rows_total, D, M, f"act_tiles D={D}")
    x = src[:, :D]
    if act < 2:  # exact in fp32: the tiles are the split of the value, bit for bit
        v = x if act == 0 else np.maximum(x, np.float32(0))
        hi, lo = so.split16(v)
        assert np.array_equal(got, hi.astype(np.float64) + lo.astype(np.float64))
        WORST.setdefault(f"act_tiles act={act} (bitwise)", 0.0)
    else:
        ref = ko.act(x, 2)
        _check(f"act_tiles swish D={D}", got, ref, ko.split_bound(ref, ko.act_bound(x, 0.0, 2)))


@gpu
@pytest.mark.parametrize("D", [32, 144, 176])
@pytest.mark.parametrize("zero_pad", [0, 1])
@pytest.mark.parametrize("inplace", [False, True])
def test_ln_rows(D, zero_pad, inplace):
    g = _g(D + zero_pad + 2 * inplace)
    T, lens = 50, [50, 17, 1]
    B = len(lens)
    M = B * T
    x = (1.0 + 2.0 * g.standard_normal((M + 2, D))).astype(np.float32)
    x[M:] = 7.0  # past the launch's rows: must survive
    gam = g.uniform(0.5, 1.5, D).astype(np.float32)
    bet = (0.3 * g.standard_normal(D)).astype(np.float32)
    xd = _cuda(x)
    y = xd if inplace else _nan(M + 2, D)
    _dbg("ln_rows", B=B, T=T, len=_i32(lens), D=D, flags=4 * zero_pad, x=xd, w=_cuda(gam), bias=_cuda(bet), y=y)
    out = y.cpu().numpy()
    assert (out[M:] == 7.0).all() if inplace else np.isnan(out[M:]).all()
    ref, bound = ko.layer_norm(x[:M], gam, bet)
    if zero_pad:
        for b, L in enumerate(lens):
            ref[b * T + L:(b + 1) * T] = 0.0
            bound[b * T + L:(b + 1) * T] = 0.0
    _check(f"ln_rows D={D}", out[:M], ref, bound)


# ---- frontend / MVN / conv0 ----------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("n_fft,win", [(400, 400), (512, 400), (512, 401), (1024, 800), (1024, 1023)])
def test_frontend(n_fft, win):
    g = _g(n_fft + win)
    hop, Fm = 160, 80
    # the shortest accepted input (both reflections in one frame), an exact multiple of hop, a row with a silent stretch
    lens = [n_fft // 2 + 1, 10 * hop, 6000, 2345]
    B, n_max = len(lens), 6037
    wav = (0.3 * g.standard_normal((B, n_max))).astype(np.float32)
    wav[2, 1500:4500] = 0.0
    for b, L in enumerate(lens):
        wav[b, L:] = 10.0 + g.standard_normal(n_max - L)  # never read
    melmat = g.uniform(0.0, 1.0, (n_fft // 2 + 1, Fm)).astype(np.float32)
    tf = [1 + L // hop for L in lens]
    Tf = 1 + n_max // hop
    out = _nan(B, Tf + 1, Fm)
    _dbg("frontend", B=B, T=Tf, len=_i32(lens), len2=_i32(tf), n_max=n_max, n_fft=n_fft, win_length=win, hop_length=hop, F=Fm,
         x=_cuda(wav), w=_cuda(melmat), y=out)
    o = out.cpu().numpy().reshape(-1, Fm)
    assert np.isnan(o[B * Tf:]).all()
    o = o[:B * Tf].reshape(B, Tf, Fm)
    silent = 0
    for b, L in enumerate(lens):
        ref, bound = ko.log_mel(wav[b], L, n_fft, win, hop, melmat)
        silent += int((ref < -46).sum())
        _check(f"frontend n_fft={n_fft}", o[b, :tf[b]], ref, bound)
        assert not o[b, tf[b]:].any()
    assert silent > 0  # power 0 -> log(1e-20) was reached


@gpu
@pytest.mark.parametrize("flags", [0, 1, 2, 3])
def test_mvn(flags):
    g = _g(flags)
    T, Fm, lens = 60, 80, [60, 23, 2]
    B = len(lens)
    x = (-5.0 + 3.0 * g.standard_normal((B, T, Fm))).astype(np.float32)
    for b, L in enumerate(lens):
        x[b, L:] = 1000.0 + g.standard_normal((T - L, Fm))  # past the row: neither read nor written
    y = _cuda(x)
    _dbg("mvn", B=B, T=T, len=_i32(lens), F=Fm, flags=flags, y=y)
    out = y.cpu().numpy()
    for b, L in enumerate(lens):
        assert np.array_equal(out[b, L:], x[b, L:])
        ref, bound = ko.mvn(x[b], L, flags & 1, flags >> 1)
        if flags == 0:
            assert np.array_equal(out[b, :L], x[b, :L])
        _check(f"mvn flags={flags}", out[b, :L], ref, bound)


@gpu
@pytest.mark.parametrize("k,s,p,T,Fm", [(5, 1, 2, 21, 80), (4, 2, 1, 21, 80), (4, 2, 1, 20, 79), (3, 1, 1, 9, 10)])
def test_conv0(k, s, p, T, Fm):
    g = _g(k + T + Fm)
    N, lens = 48, [T, T // 2, 1]
    B = len(lens)
    x = g.standard_normal((B, T, Fm)).astype(np.float32)
    w = (0.3 * g.standard_normal((N, 1, k, k))).astype(np.float32)
    bias = (0.3 * g.standard_normal(N)).astype(np.float32)
    To, Fo = ko.conv_len(T, k, s, p), ko.conv_len(Fm, k, s, p)
    n = B * To * Fo * N
    yh, yl = _nan16(n + 64), _nan16(n + 64)
    _dbg("conv0", B=B, T=T, len=_i32(lens), F=Fm, N=N, k=k, stride=s, pad=p, x=_cuda(x), w=_cuda(w), bias=_cuda(bias),
         y_hi=yh, y_lo=yl)
    th, tl = yh.cpu().numpy(), yl.cpu().numpy()
    assert np.isnan(th[n:]).all() and np.isnan(tl[n:]).all()
    got = th[:n].astype(np.float64) + tl[:n].astype(np.float64)
    ref, bound = ko.conv0(x, lens, w, bias, k, s, p)
    _check(f"conv0 k={k} s={s}", got.reshape(ref.shape), ref, ko.split_bound(ref, bound))


# ---- tc_big at the extractor's GEMM shapes (mb_taco_tc_debug) ---------------------------------------------------------------------
# (M, N, K, ldy, in-place residual): QKV (N = ldy = 3 D), w_2 / linear_out / pointwise_conv2 with res == y, embed.out.0 (K =
# D F2 = 11520, KB = 180), linear_pos of all 16 blocks (N = num_blocks D = 2304)
TC_BIG = [(301, 432, 144, 432, False), (301, 144, 576, 144, True), (301, 144, 11520, 144, False), (301, 2304, 144, 2304, False)]


@gpu
@pytest.mark.parametrize("M,N,K,ldy,inplace", TC_BIG)
def test_tc_big_extractor_shapes(M, N, K, ldy, inplace):
    from mockingbird_b200.synthesizer.tc_debug import parse_report, tc_debug

    g = _g(M + N + K)
    A = g.standard_normal((M, K)).astype(np.float32)
    W = (g.standard_normal((N, K)) / math.sqrt(K)).astype(np.float32)
    b = (0.3 * g.standard_normal(N)).astype(np.float32)
    res = g.standard_normal((M + 3, ldy)).astype(np.float32) if inplace else None
    y = _cuda(res) if inplace else _nan(M + 3, ldy)
    rep = parse_report(tc_debug("big", M=M, N=N, K0=K, w=[_cuda(W)], ldw=K, b=[_cuda(b)], x=[_cuda(A)], ldx=[K], shift=[0],
                                w_off=[0], w_stride=[1], nseg=1, T=1, y=y, ldy=ldy, res=y if inplace else None,
                                ldres=ldy if inplace else 0))
    assert rep["kernel"] == "tc_big"
    RAN.add(("tc_big", "inplace" if inplace else f"K={K}", N))
    s = so.pow2_scale(W)
    S = so.split_sum(A, W, s)
    r = res[:M, :N] if inplace else None
    ref = so.big_epilogue(S, b, res=r)
    bound = so.big_epilogue_bound(S, so.acc_bound(A, W, s), b, res=r)
    out = y.cpu().numpy()
    _check(f"tc_big N={N} K={K}" + (" res==y" if inplace else ""), out[:M, :N], ref, bound)
    if inplace:
        assert np.array_equal(out[M:], res[M:]) and np.array_equal(out[:, N:], res[:, N:])
    else:
        assert np.isnan(out[M:]).all() and np.isnan(out[:M, N:]).all()


# ---- whole 2-block models at the unreached sizes ---------------------------------------------------------------------------------------
WIDE = {
    "d64_h1": ri._ppgx_variant(ri.PPGX_CONFIG_SMALL, attention_dim=64, attention_heads=1, linear_units=128),   # dk 64, NT 64
    "d128_h4": ri._ppgx_variant(ri.PPGX_CONFIG_SMALL, attention_dim=128, attention_heads=4, linear_units=256),  # dk 32, NT 64 x 2
    "d288_h8": ri._ppgx_variant(ri.PPGX_CONFIG_SMALL, attention_dim=288, attention_heads=8, linear_units=576),  # dk 36, NT 144 x 2
}


@gpu
@pytest.mark.parametrize("name", list(WIDE))
def test_whole_model_wide_variants(name):
    from mockingbird_b200.ppg_extractor import build_model

    cfg = WIDE[name]
    sd = ri.ppg_extractor_state_dict(cfg, 0)
    m = build_model(cfg)
    m.load_state_dict(sd)
    m = m.cuda().eval()
    g = np.random.RandomState(5)
    wav = torch.from_numpy((0.3 * g.randn(8000)).astype(np.float32))
    out, taps = m.forward(wav[None], torch.LongTensor([wav.numel()]), return_taps=True)
    ref, ref_taps = po.forward(sd, cfg, wav, taps=True)
    e = go.rel_errors(out[0].cpu(), ref)
    WORST[f"model {name} max_rel"] = e["max_rel"]
    assert out.shape[1:] == ref.shape and e["max_rel"] <= 1e-3 and e["rms_rel"] <= 1e-3, e
    for i, r in enumerate(ref_taps):
        e = go.rel_errors(taps[i, 0].cpu(), r)
        assert e["max_rel"] <= 1e-3 and e["rms_rel"] <= 1e-3, (i, e)


@gpu
def test_every_instantiation_ran():
    need = {("conv2d_tc", NT, multi) for NT in (32, 64, 144) for multi in (False, True)}
    need |= {("attn_kernel", DK, rel) for DK in (16, 32, 40, 64) for rel in (0, 1)}
    need |= {(k,) for k in ("frontend_kernel", "mvn_kernel", "conv0_kernel", "ln_tiles_kernel", "act_tiles_kernel",
                            "ln_rows_kernel", "dw_kernel")}
    need |= {("attn_kernel", "dk<DK"), ("tc_big", "inplace", 144), ("tc_big", "K=11520", 144), ("tc_big", "K=144", 2304)}
    missing = sorted(need - RAN, key=str)
    print("worst |err| / bound:", {k: float(f"{v:.3g}") for k, v in sorted(WORST.items())})
    assert not missing, missing


# ---- CPU: the references themselves -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("k,s,p", [(5, 1, 2), (4, 2, 1), (3, 1, 1)])
def test_conv_reference_matches_torch(k, s, p):
    g = _g(k)
    B, T, Fm, C, N, lens = 3, 11, 13, 8, 5, [11, 6, 1]
    X = g.standard_normal((B, T, Fm, C))
    W = g.standard_normal((N, C, k, k))
    A, To, Fo = ko.im2col(X, lens, k, s, p)
    got = (A @ ko.conv_weight_matrix(W).T).reshape(B, To, Fo, N)
    Xm = X.copy()
    for b, L in enumerate(lens):
        Xm[b, L:] = 0.0
    ref = F.conv2d(torch.from_numpy(Xm).permute(0, 3, 1, 2), torch.from_numpy(W), stride=s, padding=p).permute(0, 2, 3, 1)
    assert np.allclose(got, ref.numpy(), rtol=1e-12, atol=1e-12)
    w1 = g.standard_normal((N, 1, k, k)).astype(np.float32)
    x1 = g.standard_normal((B, T, Fm)).astype(np.float32)
    b1 = g.standard_normal(N).astype(np.float32)
    r0, _ = ko.conv0(x1, lens, w1, b1, k, s, p)
    x1m = x1.astype(np.float64)
    for b, L in enumerate(lens):
        x1m[b, L:] = 0.0
    t0 = torch.relu(F.conv2d(torch.from_numpy(x1m)[:, None], torch.from_numpy(w1).double(), torch.from_numpy(b1).double(), s, p))
    assert np.allclose(r0, t0.permute(0, 2, 3, 1).numpy(), rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("act", [0, 1, 2])
def test_depthwise_reference_matches_torch(act):
    g = _g(act)
    D, K, T, lens = 6, 7, 12, [12, 4, 1]
    pw = g.standard_normal((len(lens) * T, 2 * D))
    w, bias = g.standard_normal((D, 1, K)), g.standard_normal(D)
    bn = [g.uniform(0.5, 1.5, D), g.standard_normal(D), g.standard_normal(D), g.uniform(0.5, 2.0, D)]
    got, _ = ko.depthwise(pw, lens, T, w, bias, *bn, act)
    for b, L in enumerate(lens):
        h = F.glu(torch.from_numpy(pw[b * T:b * T + L]).T[None], dim=1)
        h = F.conv1d(h, torch.from_numpy(w), torch.from_numpy(bias), padding=(K - 1) // 2, groups=D)
        t = [torch.from_numpy(v) for v in bn]
        h = F.batch_norm(h, t[2], t[3], t[0], t[1], False, 0.0, 1e-5)
        h = h if act == 0 else torch.relu(h) if act == 1 else h * torch.sigmoid(h)
        assert np.allclose(got[b * T:b * T + L], h[0].T.numpy(), rtol=1e-12, atol=1e-12)
        assert not got[b * T + L:(b + 1) * T].any()


@pytest.mark.parametrize("rel", [0, 1])
def test_attention_reference_matches_oracle(rel):
    g = _g(rel)
    H, dk, T_max, lens = 3, 5, 40, [37, 1, 40]
    D = H * dk
    qkv = g.standard_normal((len(lens) * T_max, 3 * D))
    P = g.standard_normal((T_max, D))
    pu, pv = g.standard_normal((H, dk)), g.standard_normal((H, dk))
    got, _ = ko.attention(qkv, lens, T_max, H, dk, P if rel else None, pu, pv)
    for b, T in enumerate(lens):
        r = torch.from_numpy(qkv[b * T_max:b * T_max + T])
        q = r[:, :D].reshape(1, T, H, dk)
        kk = r[:, D:2 * D].reshape(1, T, H, dk).transpose(1, 2)
        v = r[:, 2 * D:].reshape(1, T, H, dk).transpose(1, 2)
        pp = torch.from_numpy(P[:T]).reshape(1, T, H, dk).transpose(1, 2) if rel else None
        ref = po.attention(q, kk, v, pp, torch.from_numpy(pu), torch.from_numpy(pv))[0]
        assert np.allclose(got[b * T_max:b * T_max + T], ref.numpy(), rtol=1e-12, atol=1e-12)
        assert not got[b * T_max + T:(b + 1) * T_max].any()


@pytest.mark.parametrize("n_fft,win", [(400, 400), (512, 401), (1024, 800)])
def test_stft_reference_matches_torch(n_fft, win):
    g = _g(n_fft)
    for L in (n_fft // 2 + 1, 1600, 2345):
        wav = g.standard_normal(L)
        fr = ko.frames(wav, L, n_fft, win, 160)
        got = np.abs(np.fft.rfft(fr, axis=1)) ** 2
        spec = torch.stft(torch.from_numpy(wav)[None], n_fft=n_fft, win_length=win, hop_length=160, center=True,
                          pad_mode="reflect", normalized=False, onesided=True, return_complex=True)
        ref = (spec.real ** 2 + spec.imag ** 2)[0].T.numpy()
        assert got.shape == ref.shape and np.allclose(got, ref, rtol=1e-9, atol=1e-9)


@pytest.mark.parametrize("means,var", [(1, 1), (1, 0), (0, 1)])
def test_frontend_mvn_reference_matches_oracle(means, var):
    g = _g(means + 2 * var)
    n_fft, win, hop, Fm = 512, 400, 160, 20
    wav = (0.3 * g.standard_normal(3000)).astype(np.float32)
    melmat = g.uniform(0, 1, (n_fft // 2 + 1, Fm)).astype(np.float32)
    cfg = dict(frontend_conf=dict(n_fft=n_fft, win_length=win, hop_length=hop), normalize_conf=dict(norm_means=bool(means),
                                                                                                      norm_vars=bool(var)))
    ref = po.features({"frontend.logmel.melmat": torch.from_numpy(melmat)}, cfg, torch.from_numpy(wav)).numpy()
    lm, _ = ko.log_mel(wav, len(wav), n_fft, win, hop, melmat)
    got, _ = ko.mvn(lm, lm.shape[0], means, var)
    assert np.allclose(got, ref, rtol=1e-4, atol=1e-4)


def test_layer_norm_reference_matches_torch():
    g = _g(1)
    x, w, b = g.standard_normal((7, 33)) + 3, g.standard_normal(33), g.standard_normal(33)
    got, _ = ko.layer_norm(x, w, b)
    ref = F.layer_norm(torch.from_numpy(x), (33,), torch.from_numpy(w), torch.from_numpy(b), 1e-12)
    assert np.allclose(got, ref.numpy(), rtol=1e-12, atol=1e-12)


def test_rel_shift_closed_form_every_T():
    g = torch.Generator().manual_seed(1)
    for T in range(1, 71):
        bd = torch.randn(2, T, T, generator=g, dtype=torch.float64)
        assert torch.equal(po.rel_shift(bd), po.rel_shift_closed_form(bd)), T
