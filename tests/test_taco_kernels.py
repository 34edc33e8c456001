"""GPU tests of the FP32 kernels of the Tacotron path one launch at a time (mb_taco_debug), against the float64 references and
bounds of oracle/taco_kernel_oracle.py.

Outputs go into NaN-filled buffers with a row stride wider than the output where the kernel takes one; nothing outside the
written region may change.  Every check records its worst error / bound ratio (printed at the end); RAN records which kernel and
which launch_gemm route ran, and the last test asserts every one was seen."""
import numpy as np
import pytest
import torch

import ref_init as ri
import taco_kernel_oracle as ko
import tacotron_oracle as to
import tc_split_oracle as so

pytestmark = pytest.mark.gpu
RAN = set()
WORST = {}


def _dbg(kind, **k):
    from mockingbird_b200.synthesizer.taco_debug import parse_report, taco_debug

    rep = parse_report(taco_debug(kind, **k))
    RAN.add(rep["kernel"])
    return rep


def _g(seed):
    return np.random.default_rng(seed)


def _f32(a):
    return np.asarray(a, np.float32)


def _cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _nan(*shape):
    return torch.full(shape, float("nan"), device="cuda")


def _check(name, got, ref, bound):
    got = np.asarray(got, np.float64)
    assert np.all(np.isfinite(got)), name
    err = np.abs(got - ref)
    with np.errstate(divide="ignore", invalid="ignore"):
        r = float(np.max(np.where(err == 0, 0.0, err / bound), initial=0.0))
    WORST[name] = max(WORST.get(name, 0.0), r)
    assert r <= 1.0, (name, r)


def _written(buf, rows, cols):
    """buf [R][ld] NaN-filled: rows x cols written (finite), everything else untouched"""
    out = buf.cpu().numpy()
    assert np.isnan(out[rows:]).all() and np.isnan(out[:rows, cols:]).all()
    return out[:rows, :cols]


# ---- GEMM ------------------------------------------------------------------------------------------------------------------
def _route(M, N, shifted=False, epi=False):
    """launch_gemm's choice (tacotron_kernels.cu)"""
    if N == 1 and not shifted and not epi:
        return "rowdot"
    if M <= 64 and not shifted:
        return "gemm_skinny4" if N >= 2048 else "gemm_skinny1"
    if M >= 1024 and N >= 128:
        return "gemm_big"
    return "gemm32" if M <= 128 and N >= 512 else "gemm64"


def _gemm(g, M, N, K, *, ld=None, bias=False, act=0, bn=False, keep=False, res=False, seed_scale=0.1, name="gemm"):
    ld = ld or K
    x = _f32(g.standard_normal((M, ld)))
    W = _f32(g.standard_normal((N, K + 3)) * seed_scale)  # ldw = K + 3
    b = _f32(g.standard_normal(N)) if bias else None
    sc, sh = (_f32(g.uniform(0.5, 2, N)), _f32(g.standard_normal(N))) if bn else (None, None)
    kp = (g.random((M, N)) < 0.5).astype(np.uint8) if keep else None
    rs = _f32(g.standard_normal((M, N + 2))) if res else None
    ldy = N + 5
    y = _nan(M + 1, ldy)
    xd = _cuda(x)
    rep = _dbg("gemm", segs=[dict(x=xd, K=K, ld=ld)], W=_cuda(W), ldw=K + 3, bias=None if b is None else _cuda(b), M=M, N=N,
               act=act, bn_scale=None if sc is None else _cuda(sc), bn_shift=None if sh is None else _cuda(sh),
               mask=None if kp is None else _cuda(kp), res=None if rs is None else _cuda(rs), ldres=N + 2, y=y, ldy=ldy)
    ref, bound = ko.gemm([x[:, :K]], [W[:, :K]], b, act, sc, sh, kp, None if rs is None else rs[:, :N])
    _check(name, _written(y, M, N), ref, bound)
    return rep


@pytest.mark.parametrize("M", [1, 63, 64, 65, 127, 128, 129, 1023, 1024, 1025])
@pytest.mark.parametrize("N", [1, 2, 127, 128, 511, 512, 2047, 2048, 2049])
def test_gemm_routes(M, N):
    """K = 83 (not a multiple of 16, 8 or 4), ld = 90 != K, bias; the report names the route"""
    rep = _gemm(_g(M * 3 + N), M, N, 83, ld=90, bias=True, name="gemm routes")
    assert rep["kernel"] == _route(M, N), rep
    RAN.add("route:" + rep["kernel"])


@pytest.mark.parametrize("shape", [(3, 1), (1, 200), (64, 2048), (100, 600), (65, 130), (1024, 128)])
@pytest.mark.parametrize("act", [0, 1, 2, 3])
@pytest.mark.parametrize("epi", range(16))
def test_gemm_epilogues(shape, act, epi):
    """every combination of bias, activation, BN, keep mask and residual on every route"""
    M, N = shape
    bias, bn, keep, res = (bool(epi & 1), bool(epi & 2), bool(epi & 4), bool(epi & 8))
    rep = _gemm(_g(epi * 7 + act), M, N, 200, bias=bias, act=act, bn=bn, keep=keep, res=res, name="gemm epilogues")
    assert rep["kernel"] == _route(M, N, epi=bn or keep or res)
    RAN.add(f"epi:{rep['kernel']}:{epi}:{act}")


@pytest.mark.parametrize("M,N", [(5, 64), (40, 2048)])
def test_gemm_skinny_misaligned_segment(M, N):
    """segment pointer offset by one float (K and ld multiples of 4): gemm_skinny's scalar fallback"""
    g = _g(M)
    K = 64
    buf = _f32(g.standard_normal(M * K + 1))
    W = _f32(g.standard_normal((N, K)) * 0.1)
    bd = _cuda(buf)
    y = _nan(M, N + 3)
    rep = _dbg("gemm", segs=[dict(x=bd.data_ptr() + 4, K=K, ld=K)], W=_cuda(W), ldw=K, M=M, N=N, y=y, ldy=N + 3)
    assert rep["kernel"].startswith("gemm_skinny")
    ref, bound = ko.gemm([buf[1:].reshape(M, K)], [W])
    _check("gemm misaligned", _written(y, M, N), ref, bound)


@pytest.mark.parametrize("M,T,N", [(64, 16, 40), (128, 32, 512), (1024, 128, 128), (30, 10, 1)])
def test_gemm_conv_five_taps(M, T, N):
    """5 segments with shifts -2..2 reading a Conv1d weight [co][ci][5] in place (w_stride = 5), T dividing M"""
    g = _g(M + N)
    Ci, k = 37, 5
    x = _f32(g.standard_normal((M, Ci)))
    W = _f32(g.standard_normal((N, Ci, k)) * 0.1)
    b = _f32(g.standard_normal(N))
    xd = _cuda(x)
    segs = [dict(x=xd, K=Ci, ld=Ci, shift=j - 2, w_off=j, w_stride=k) for j in range(k)]
    y = _nan(M, N + 1)
    rep = _dbg("gemm", segs=segs, W=_cuda(W), ldw=Ci * k, bias=_cuda(b), M=M, N=N, T=T, act=1, y=y, ldy=N + 1)
    assert rep["kernel"] == _route(M, N, shifted=True)
    xs = [ko.gemm_operand(x, Ci, Ci, M, T, j - 2) for j in range(k)]
    ws = [ko.gemm_weight(W, Ci * k, N, Ci, j, k) for j in range(k)]
    ref, bound = ko.gemm(xs, ws, b, ko.ACT_RELU)
    _check("gemm conv taps", _written(y, M, N), ref, bound)
    RAN.add("conv:" + rep["kernel"])


@pytest.mark.parametrize("N", [1, 256, 2048])
@pytest.mark.parametrize("keep", [False, True])
@pytest.mark.parametrize("step", [0, 3])
def test_gemm_step_mode(N, keep, step):
    """segment 0 at x + step * x_step (x_first at step 0), mask + step * mask_step; step = *step_ptr + step_j.  N = 1 without a
    mask is the rowdot route, which read segment 0 at step 0 on every step before it honoured step mode"""
    g = _g(N + step)
    M, K, K1, nst = 3, 80, 24, 5
    xs_all = _f32(g.standard_normal(nst * 100 + M * 90))  # rows of stride 90, steps 100 floats apart
    first = _f32(g.standard_normal(K))
    x1 = _f32(g.standard_normal((M, K1)))
    W = _f32(g.standard_normal((N, K + K1)) * 0.1)
    b = _f32(g.standard_normal(N))
    kp = (g.random((nst, M, N)) < 0.5).astype(np.uint8) if keep else None
    if keep:
        kp[:, 0] = 1  # row 0 always kept, so a stale operand shows
    sp = torch.tensor([max(step - 1, 0)], dtype=torch.int32, device="cuda")
    y = _nan(M, N + 2)
    rep = _dbg("gemm", segs=[dict(x=_cuda(xs_all), K=K, ld=90), dict(x=_cuda(x1), K=K1, ld=K1, w_off=K)], W=_cuda(W), ldw=K + K1,
               bias=_cuda(b), M=M, N=N, mask=None if kp is None else _cuda(kp), y=y, ldy=N + 2, step_mode=1, step_ptr=sp,
               step_j=step - max(step - 1, 0), x_step=100, x_first=_cuda(first), mask_step=M * N)
    assert rep["kernel"] == _route(M, N, epi=keep)
    x0 = ko.gemm_operand(xs_all, 90, K, M, step=step, x_step=100, x_first=first)
    ref, bound = ko.gemm([x0, x1], [W[:, :K], W[:, K:]], b, keep=None if kp is None else kp[step])
    stale = ko.gemm([ko.gemm_operand(xs_all, 90, K, M), x1], [W[:, :K], W[:, K:]], b, keep=None if kp is None else kp[0])[0]
    assert np.any(np.abs(stale - ref) > 100 * bound + 1e-3), "the case must tell this step's rows from step 0's"
    _check("gemm step mode", _written(y, M, N), ref, bound)
    RAN.add(f"step:{rep['kernel']}:{step > 0}")


# ---- PreNet --------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B", [1, 3, 4, 5, 128, 130])
@pytest.mark.parametrize("K", [80, 128])
@pytest.mark.parametrize("H", [128, 256])
@pytest.mark.parametrize("step", [0, 2])
def test_prenet(B, K, H, step):
    g = _g(B * K + H + step)
    nst, x_ld, x_step = 4, 4 * K + 3, K + 1
    xs = _f32(g.standard_normal(B * x_ld + nst * x_step))
    first = np.zeros(K, np.float32)
    W1, b1 = _f32(g.standard_normal((H, K)) * 0.1), _f32(g.standard_normal(H) * 0.1)
    W2, b2 = _f32(g.standard_normal((H, H)) * 0.1), _f32(g.standard_normal(H) * 0.1)
    m = (g.random((nst, 2, B, H)) < 0.5).astype(np.uint8)
    ldy = H + 3
    y = _nan(B + 1, ldy)
    split = B <= 128
    rows_pad, k0 = (64 if B <= 64 else 128), 64
    KB = (k0 + H + 63) // 64
    hi = torch.zeros(KB * rows_pad * 64, dtype=torch.int16, device="cuda")
    lo = torch.zeros_like(hi)
    sp = torch.tensor([step], dtype=torch.int32, device="cuda")
    md = _cuda(m)
    _dbg("prenet", ins=[_cuda(xs), _cuda(first), _cuda(W1), _cuda(b1), _cuda(W2), _cuda(b2), md, md[0, 1]],
         outs=[y, hi if split else None, lo if split else None], n=[B, K, H, ldy, x_ld, x_step, 2 * B * H, k0, rows_pad],
         step_ptr=sp)
    x = np.stack([first if step == 0 else xs[b * x_ld + step * x_step: b * x_ld + step * x_step + K] for b in range(B)])
    ref, bound = ko.prenet(x, W1, b1, W2, b2, m[step, 0], m[step, 1])
    out = _written(y, B, H)
    _check("prenet", out, ref, bound)
    if split:
        th, tl = (so.unpack_act_tiles(t.cpu().numpy().view(np.float16), rows_pad, KB) for t in (hi, lo))
        h16, l16 = so.split16(out)
        assert np.array_equal(th[:B, k0:k0 + H].view(np.int16), h16.view(np.int16))
        assert np.array_equal(tl[:B, k0:k0 + H].view(np.int16), l16.view(np.int16))
        RAN.add("prenet:split")


# ---- cells and elementwise kernels ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("M,H", [(1, 128), (37, 128), (130, 256)])
def test_gru_cell(M, H):
    g = _g(M + H)
    ldgi, ldh, ldo = 3 * H + 5, H + 3, H + 7
    gi = _f32(g.standard_normal((M, ldgi)) * 2)
    gh = _f32(g.standard_normal((M, 3 * H)) * 2)
    h0 = _f32(g.standard_normal((M, ldh)))
    h = _cuda(h0)
    out2 = _nan(M + 1, ldo)
    _dbg("gru_cell", ins=[_cuda(gi), _cuda(gh)], outs=[h, out2], n=[M, H, ldgi, ldh, ldo])
    ref, bound = ko.gru_cell(gi[:, :3 * H], gh, h0[:, :H], H)
    hn = h.cpu().numpy()
    _check("gru_cell", hn[:, :H], ref, bound)
    assert np.array_equal(hn[:, H:], h0[:, H:])
    assert np.array_equal(_written(out2, M, H), hn[:, :H])


@pytest.mark.parametrize("M,H", [(1, 64), (37, 128), (130, 1024)])
@pytest.mark.parametrize("res", [False, True])
def test_lstm_cell(M, H, res):
    g = _g(M + H + res)
    gates = _f32(g.standard_normal((M, 4 * H)) * 2)
    c0, x0 = _f32(g.standard_normal((M, H))), _f32(g.standard_normal((M, H)))
    c, x = _cuda(c0), _cuda(x0)
    h = _nan(M, H)
    _dbg("lstm_cell", ins=[_cuda(gates)], outs=[c, h, x if res else None], n=[M, H])
    cn, hn, xn, dc, dh, dx = ko.lstm_cell(gates, c0, H, x0 if res else None)
    _check("lstm_cell c", c.cpu().numpy(), cn, dc)
    _check("lstm_cell h", h.cpu().numpy(), hn, dh)
    if res:
        _check("lstm_cell x", x.cpu().numpy(), xn, dx)
    else:
        assert np.array_equal(x.cpu().numpy(), x0)


@pytest.mark.parametrize("M,C", [(1, 128), (77, 128), (301, 80)])
def test_highway_maxpool_embedding_copy(M, C):
    g = _g(M + C)
    x12 = _f32(g.standard_normal((M, 2 * C)) * 3)
    y0 = _f32(g.standard_normal((M, C)))
    y = _cuda(y0)
    _dbg("highway", ins=[_cuda(x12)], outs=[y], n=[M, C])
    _check("highway", y.cpu().numpy(), *ko.highway(x12, y0, C))
    B, T = 3, max(M // 3, 1)
    x = _f32(g.standard_normal((B, T, C)))
    yp = _nan(B, T, C)
    _dbg("maxpool2", ins=[_cuda(x)], outs=[yp], n=[B, T, C])
    assert np.array_equal(yp.cpu().numpy(), ko.maxpool2(x))
    table = _f32(g.standard_normal((75, C)))
    ids = g.integers(0, 75, M).astype(np.int32)
    ye = _nan(M, C)
    _dbg("embedding", ins=[_cuda(ids), _cuda(table)], outs=[ye], n=[M, C])
    assert np.array_equal(ye.cpu().numpy(), table[ids])
    rps, off, n, ldd = 7, 5, C // 2, C + 9
    src = _f32(g.standard_normal(((M + rps - 1) // rps, C)))
    dst = _nan(M + 1, ldd)
    _dbg("copy_cols", ins=[_cuda(src)], outs=[dst], n=[M, n, C, rps, ldd, off])
    out = dst.cpu().numpy()
    assert np.array_equal(out[:M, off:off + n], src[np.arange(M) // rps, :n])
    assert np.isnan(out[:M, :off]).all() and np.isnan(out[:M, off + n:]).all() and np.isnan(out[M:]).all()


# ---- location-sensitive attention --------------------------------------------------------------------------------------------
def _max_chars():
    from mockingbird_b200 import _lib

    return int(_lib.lib().mb_tacotron_max_chars())


def _lsa_case(g, B, Tc, S=256):
    D = 128
    lens = np.maximum(1, (Tc * np.linspace(1, 0.3, B)).astype(int))
    chars = np.where(np.arange(Tc)[None, :] < lens[:, None], g.integers(1, 75, (B, Tc)), 0).astype(np.int32)
    if B >= 3:
        chars[B // 2] = 0  # a fully padded row
    return dict(pq=_f32(g.standard_normal((B, D)) * 0.5), proj=_f32(g.standard_normal((B, Tc, D)) * 0.5),
                seq=_f32(g.standard_normal((B, Tc, S))), chars=chars, cum=_f32(g.random((B, Tc)) * 2),
                conv_w=_f32(g.standard_normal((32, 1, 31)) * 0.3), conv_b=_f32(g.standard_normal(32) * 0.3),
                Lw=_f32(g.standard_normal((D, 32)) * 0.2), vw=_f32(g.standard_normal((1, D)) * 0.5),
                q=_f32(g.standard_normal((B, D))), Wq=_f32(g.standard_normal((D, D)) * 0.1), bq=_f32(g.standard_normal(D) * 0.1))


def _lsa_launch(a, cum_d, scores, scores_ld, ctx, threads, qpath, step_ptr=None, step_j=0, d=None):
    B, Tc, _ = a["proj"].shape
    S = a["seq"].shape[2]
    d = d or {k: _cuda(v) for k, v in a.items() if k != "cum"}
    rep = _dbg("lsa_step", ins=[None if qpath else d["pq"], d["proj"], d["seq"], d["chars"], d["conv_w"], d["conv_b"], d["Lw"],
                                d["vw"], d["q"] if qpath else None, d["Wq"], d["bq"]],
               outs=[cum_d, scores, ctx], n=[B, Tc, S, scores_ld, threads], step_ptr=step_ptr, step_j=step_j)
    assert rep["kernel"] == "lsa_step" and int(rep["smem"]) == 4 * (5438 + 38 * Tc) and rep["block"] == str(threads)
    return rep, d


def _lsa_ref(a, qpath, ctx=True):
    kw = {k: a[k] for k in ("proj", "seq", "chars", "cum", "conv_w", "conv_b", "Lw", "vw")}
    if qpath:
        return ko.lsa_step(pq=None, q_in=a["q"], Wq=a["Wq"], bq=a["bq"], ctx=ctx, **kw)
    return ko.lsa_step(pq=a["pq"], ctx=ctx, **kw)


LSA_TC = [1, 2, 15, 31, 33, 180, 181, 600, "limit"]


@pytest.mark.parametrize("Tc", LSA_TC)
@pytest.mark.parametrize("B", [1, 3, 70])
@pytest.mark.parametrize("threads,qpath,inctx", [(512, True, False), (256, False, True), (512, False, True), (256, True, False)])
def test_lsa_step(Tc, B, threads, qpath, inctx):
    """512 / 256 threads, query projected inside (q_in, Wq, bq) or given (pq), context in the kernel or by lsa_ctx_kernel"""
    Tc = _max_chars() if Tc == "limit" else Tc
    if B == 70 and (threads, qpath, inctx) != (512, True, False) and Tc not in (1, 181, _max_chars()):
        pytest.skip("the shipped variant covers every Tc at B = 70")
    g = _g(Tc * 5 + B + threads)
    a = _lsa_case(g, B, Tc, S=72 if inctx else 8)
    cum = _cuda(a["cum"])
    ld = Tc + 3
    scores = _nan(B + 1, ld)
    ctx = _nan(B, a["seq"].shape[2]) if inctx else None
    _lsa_launch(a, cum, scores, ld, ctx, threads, qpath)
    ref = _lsa_ref(a, qpath, ctx=inctx)
    _check("lsa_step scores", _written(scores, B, Tc), *ref["scores"])
    _check("lsa_step cum", cum.cpu().numpy(), *ref["cum"])
    if inctx:
        _check("lsa_step ctx", ctx.cpu().numpy(), *ref["ctx"])
    RAN.add(f"lsa:{threads}:{qpath}:{inctx}")
    if Tc == _max_chars():
        RAN.add("lsa:limit")
    if Tc * 38 * 4 + 5438 * 4 > 48 * 1024:
        RAN.add("lsa:smem_optin")


def test_lsa_chained_steps_and_ctx_split():
    """20 steps, each against the float64 step applied to the kernel's own previous cumulative state; alignment rows through
    the step pointer; lsa_ctx_kernel's context and its split outputs (bitwise split16 of the context)"""
    g = _g(20)
    B, Tc, S, nst = 3, 181, 512, 20
    a = _lsa_case(g, B, Tc, S)
    cum = _cuda(a["cum"])
    scores = _nan(B, nst * Tc)
    sp = torch.tensor([0], dtype=torch.int32, device="cuda")
    d = None
    rows_pad, KB = 64, S // 64
    for s in range(nst):
        prev = cum.cpu().numpy()
        sp.fill_(s - s % 2)
        _, d = _lsa_launch(dict(a, cum=prev), cum, scores, nst * Tc, None, 512, True, step_ptr=sp, step_j=s % 2, d=d)
        ref = _lsa_ref(dict(a, cum=prev), True, ctx=False)
        got = scores.cpu().numpy().reshape(B, nst, Tc)
        _check("lsa chained scores", got[:, s], *ref["scores"])
        _check("lsa chained cum", cum.cpu().numpy(), *ref["cum"])
        assert np.isnan(got[:, s + 1:]).all()
        ctx = _nan(B, S)
        tiles = [torch.zeros(KB * rows_pad * 64, dtype=torch.int16, device="cuda") for _ in range(4)]
        rep = _dbg("lsa_ctx", ins=[scores, d["seq"]], outs=[ctx] + tiles, n=[B, Tc, S, nst * Tc, rows_pad], step_ptr=sp,
                   step_j=s % 2)
        assert rep["kernel"] == "lsa_ctx" and rep["grid"] == f"{S // 256},{B}"
        c = ctx.cpu().numpy()
        _check("lsa_ctx", c, *ko.context(got[:, s], a["seq"]))
        h16, l16 = so.split16(c)
        for t, want in zip(tiles, (h16, l16, h16, l16)):
            u = so.unpack_act_tiles(t.cpu().numpy().view(np.float16), rows_pad, KB)[:B]
            assert np.array_equal(u.view(np.int16), want.view(np.int16))


# ---- GST, stop, masks, layouts ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("heads", range(1, 9))
@pytest.mark.parametrize("ntok", [1, 2, 7, 10, 16])
def test_gst_attention(heads, ntok):
    g = _g(heads * 20 + ntok)
    B, E = 3, 840  # divisible by 1..8
    q, k, v = _f32(g.standard_normal((B, E))), _f32(g.standard_normal((ntok, E))), _f32(g.standard_normal((ntok, E)))
    y = _nan(B, E)
    _dbg("gst_attention", ins=[_cuda(q), _cuda(k), _cuda(v)], outs=[y], n=[B, ntok, E, heads])
    _check("gst_attention", y.cpu().numpy(), *ko.gst_attention(q, k, v, heads))


@pytest.mark.parametrize("B", [1, 7, 128, 300])
def test_stop_step(B):
    """stop projection + rule in one launch: values within the bound and bitwise equal to the rowdot route (same summation
    order), two launches on one ticket (the last CTA resets it), and the step * r > 10 boundary"""
    g = _g(B)
    K0, K1, r = 1024, 576, 2
    x, c = _f32(g.standard_normal((B, K0))), _f32(g.standard_normal((B, K1)))
    w = _f32(g.standard_normal(K0 + K1) * 0.02)
    dx, dc, dw = _cuda(x), _cuda(c), _cuda(w)
    segs = [dict(x=dx, K=K0, ld=K0), dict(x=dc, K=K1, ld=K1, w_off=K0)]
    ticket = torch.zeros(1, dtype=torch.int32, device="cuda")
    flags = torch.full((8,), -1, dtype=torch.int32, device="cuda")
    sp = torch.tensor([4], dtype=torch.int32, device="cuda")
    for bias, step_j, mst in ((4.0, 1, 5.0), (4.0, 2, 5.0), (-40.0, 2, 5.0)):
        bd = _cuda(_f32([bias]))
        y = _nan(B, 3)
        _dbg("stop_step", segs=segs, W=dw, ldw=K0 + K1, bias=bd, M=B, N=1, y=y, ldy=3, step_ptr=sp, step_j=step_j,
             outs=[flags, ticket], n=[B, r], fval=mst)
        assert int(ticket.item()) == 0
        ref, bound = ko.stop_value([x, c], w, [bias])
        vals = _written(y, B, 1)[:, 0]
        _check("stop_step", vals, ref, bound)
        si = 4 + step_j
        want = ko.stop_flag(vals, mst, si, r)
        assert int(flags[si].item()) == want, (bias, si)
        assert want == (bias > 0 and si * r > 10)
        yr = _nan(B, 3)
        rep = _dbg("gemm", segs=segs, W=dw, ldw=K0 + K1, bias=bd, M=B, N=1, act=ko.ACT_SIGMOID, y=yr, ldy=3)
        assert rep["kernel"] == "rowdot"
        assert np.array_equal(_written(yr, B, 1)[:, 0], vals)


@pytest.mark.parametrize("B", [1, 5])
def test_stop_flag(B):
    sp = torch.tensor([3], dtype=torch.int32, device="cuda")
    for vals, mst, j in (([0.9] * B, 5.0, 3), ([0.9] * (B - 1) + [0.4], 5.0, 3), ([0.9] * B, 5.0, 2)):
        flags = torch.full((8,), -1, dtype=torch.int32, device="cuda")
        _dbg("stop_flag", ins=[_cuda(_f32(vals))], outs=[flags], n=[B, 2], fval=mst, step_ptr=sp, step_j=j)
        assert int(flags[3 + j].item()) == ko.stop_flag(vals, mst, 3 + j, 2)


@pytest.mark.parametrize("seed", [0, 7, 0x123456789ABCDEF0])
def test_fill_masks(seed):
    n = 2 * 3 * 41 * 256 + 5
    m = torch.full((n + 8,), 9, dtype=torch.uint8, device="cuda")
    _dbg("fill_masks", outs=[m], n=[n, 0xFFFFFFFF], seed=seed)
    out = m.cpu().numpy()
    assert np.array_equal(out[:n], ko.fill_masks(n, seed, 0xFFFFFFFF)) and (out[n:] == 9).all()
    sp = torch.tensor([5], dtype=torch.int32, device="cuda")
    _dbg("fill_masks", outs=[m], n=[1000, 32], seed=seed, step_ptr=sp)  # stream_id + *step_ptr
    assert np.array_equal(m.cpu().numpy()[:1000], ko.fill_masks(1000, seed, 37))
    per, steps = 2 * 3 * 512, 9
    ms = torch.full((per * steps + 4,), 9, dtype=torch.uint8, device="cuda")
    _dbg("fill_masks_steps", outs=[ms], n=[per, steps], seed=seed)
    got = ms.cpu().numpy()
    assert np.array_equal(got[:per * steps], ko.fill_masks_steps(per, steps, seed)) and (got[per * steps:] == 9).all()
    for s in (0, steps - 1):  # equal to fill_masks called per step
        one = torch.zeros(per, dtype=torch.uint8, device="cuda")
        _dbg("fill_masks", outs=[one], n=[per, s], seed=seed)
        assert np.array_equal(one.cpu().numpy(), got[s * per:(s + 1) * per])


def test_pack_melproj_to_ncl_bn_fold():
    g = _g(11)
    NM, max_r, K = 80, 20, 1024
    W = _f32(g.standard_normal((NM * max_r, K)))
    for r in (1, 2, 7):
        dst = _nan(r * NM + 1, K)
        _dbg("pack_melproj", ins=[_cuda(W)], outs=[dst], n=[NM, max_r, r, K])
        assert np.array_equal(_written(dst, r * NM, K), ko.pack_melproj(W, NM, max_r, r))
    B, steps, C, frames = 3, 12, 80, 9
    x = _f32(g.standard_normal((B, steps, C)))
    y = _nan(B * C * frames + 7)
    _dbg("to_ncl", ins=[_cuda(x)], outs=[y], n=[steps, B, C, frames])
    out = y.cpu().numpy()
    assert np.array_equal(out[:B * C * frames].reshape(B, C, frames), ko.to_ncl(x, steps, B, C, frames))
    assert np.isnan(out[B * C * frames:]).all()
    n = 300
    gam, bet, mean, var = _f32(g.standard_normal(n)), _f32(g.standard_normal(n)), _f32(g.standard_normal(n)), _f32(g.random(n) + 0.01)
    sc, sh = _nan(n), _nan(n)
    _dbg("bn_fold", ins=[_cuda(gam), _cuda(bet), _cuda(mean), _cuda(var)], outs=[sc, sh], n=[n])
    (rs, ds), (rsh, dsh) = ko.bn_fold(gam, bet, mean, var)
    _check("bn_fold scale", sc.cpu().numpy(), rs, ds)
    _check("bn_fold shift", sh.cpu().numpy(), rsh, dsh)


# ---- whole model: long inputs and the character limit ------------------------------------------------------------------------
@pytest.fixture(scope="module")
def sd():
    return ri.tacotron_state_dict(0, r=2, randomize_bn=True)


@pytest.fixture(scope="module")
def model(sd):
    from mockingbird_b200.synthesizer.inference import Synthesizer

    return Synthesizer("unused.pt", verbose=False).load_state(sd)


def _rel(a, b):
    return float((a - b).abs().max() / b.abs().max())


@pytest.mark.parametrize("Tc", [181, 600])
def test_long_inputs_vs_oracle(sd, model, Tc):
    """181 characters: the first length whose attention step needs more than 48 KB of shared memory; 600: well beyond"""
    g = torch.Generator().manual_seed(Tc)
    B, steps = 2, 8
    chars = torch.randint(2, 75, (B, Tc), generator=g)
    chars[1, Tc // 2:] = 0
    emb = torch.rand(B, 256, generator=g)
    emb = emb / emb.norm(dim=1, keepdim=True)
    nst = steps // 2
    enc = torch.rand(2, B, Tc, 256, generator=g) < 0.5
    dec = torch.rand(nst, 2, B, 256, generator=g) < 0.5
    masks = [enc[0], enc[1]] + [dec[i, j] for i in range(nst) for j in range(2)]
    mel_r, lin_r, attn_r = to.generate(sd, chars, emb, steps, -1, 10, masks, r=2)
    mel, lin, attn = model.generate(chars, emb, steps=steps, style_idx=-1, min_stop_token=10, dropout_masks=(enc, dec))
    assert mel.shape == mel_r.shape and attn.shape == attn_r.shape == (B, nst, Tc)
    for got, ref in ((mel, mel_r), (lin, lin_r), (attn, attn_r)):
        assert _rel(got.cpu(), ref) <= 2e-4, _rel(got.cpu(), ref)


def test_over_the_character_limit_refused(model):
    """more characters than the attention step's shared memory allows: refused before anything is queued (launch count
    unchanged, the limit named), by the C entry point as well as the Python surface; the handle still works afterwards"""
    import ctypes as C

    from mockingbird_b200 import _lib

    L = _lib.lib()
    limit = _max_chars()
    assert limit == (232448 // 4 - 5438) // 38 == 1386  # the H100's 227 KB opt-in: 4 * (5438 + 38 * Tc) bytes
    h = model._handle
    assert L.mb_tacotron_workspace_bytes(h, 2, limit + 1, 8, 2) == 0 and L.mb_tacotron_workspace_bytes(h, 2, limit, 8, 2) > 0
    chars = torch.ones(2, limit + 1, dtype=torch.int64)
    emb = torch.rand(2, 256)
    n0 = L.mb_launch_count()
    with pytest.raises(ValueError, match=str(limit)):
        model.generate(chars, emb, steps=8, style_idx=-1, min_stop_token=10)
    dummy = torch.zeros(1024, dtype=torch.uint8, device="cuda")
    p = C.c_void_p(dummy.data_ptr())
    frames = C.c_int32(0)
    rc = L.mb_tacotron_generate(h, p, p, 2, limit + 1, 8, 2, -1, C.c_float(10.0), None, None, C.c_uint64(0), p, p, p,
                                C.byref(frames), p, 1024, None)
    assert rc == 1 and str(limit).encode() in L.mb_last_error()  # MB_ERR_INVALID
    assert L.mb_launch_count() == n0, "nothing may be launched"
    mel, _, _ = model.generate(torch.randint(2, 75, (1, 12)), emb[:1], steps=4, style_idx=-1, min_stop_token=10)
    assert mel.shape == (1, 80, 4) and torch.isfinite(mel).all()


# ---- coverage -----------------------------------------------------------------------------------------------------------------
def test_every_kernel_route_and_variant_ran():
    for k, v in sorted(WORST.items()):
        print(f"worst error / bound  {k:24s} {v:.3g}")
    kernels = {"rowdot", "gemm_skinny1", "gemm_skinny4", "gemm32", "gemm64", "gemm_big", "prenet_fused", "gru_cell", "lstm_cell",
               "highway", "maxpool2", "embedding", "copy_cols", "lsa_step", "lsa_ctx", "gst_attention", "stop_step", "stop_flag",
               "fill_masks", "fill_masks_steps", "pack_melproj", "to_ncl", "bn_fold"}
    want = kernels | {f"route:{k}" for k in ("rowdot", "gemm_skinny1", "gemm_skinny4", "gemm32", "gemm64", "gemm_big")}
    want |= {f"epi:{k}:{e}:{a}" for k in ("gemm_skinny1", "gemm_skinny4", "gemm32", "gemm64", "gemm_big") for e in range(16)
             for a in range(4)}
    want |= {f"conv:{k}" for k in ("gemm64", "gemm32", "gemm_big")}
    want |= {f"step:{k}:{s}" for k in ("rowdot", "gemm_skinny1", "gemm_skinny4") for s in (False, True)}
    want |= {"prenet:split", "lsa:limit", "lsa:smem_optin"} | {f"lsa:{t}:{q}:{c}" for t, q, c in
                                                              ((512, True, False), (256, False, True), (512, False, True),
                                                               (256, True, False))}
    missing = sorted(want - RAN)
    assert not missing, missing
