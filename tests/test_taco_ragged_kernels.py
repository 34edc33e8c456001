"""GPU tests of the per-row arguments that ragged batches pass into the Tacotron and speaker-encoder kernels, one launch at a time
(mb_taco_debug, mb_taco_tc_debug, mb_encoder_reduce_partials), against float64 references that state each row as the B = 1
utterance of its own length (oracle/taco_kernel_oracle.py, oracle/tc_split_oracle.py, oracle/encoder_oracle.py).

Inputs past a row's end are NaN wherever the kernel must not let them reach the row, and outputs go into NaN-filled buffers, so a
stray read or a missing write shows.  Besides the float64 bounds, each row is compared bit for bit with a launch of that row
alone (or at another position, or in another batch size): the ragged paths promise that a row's bits do not depend on its batch.
RAN records which kernel and variant ran; the last test asserts every one was seen."""
import ctypes as C

import numpy as np
import pytest
import torch

import encoder_oracle as eo
import taco_kernel_oracle as ko
import tc_split_oracle as so

pytestmark = pytest.mark.gpu
RAN = set()
WORST = {}


def _dbg(kind, **k):
    from mockingbird_b200.synthesizer.taco_debug import parse_report, taco_debug

    rep = parse_report(taco_debug(kind, **k))
    RAN.add(rep["kernel"])
    return rep


def _tc(kind, **k):
    from mockingbird_b200.synthesizer.tc_debug import parse_report, tc_debug

    rep = parse_report(tc_debug(kind, **k))
    RAN.add(rep["kernel"])
    return rep


def _g(seed):
    return np.random.default_rng(seed)


def _f32(a):
    return np.asarray(a, np.float32)


def _cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _i32(a):
    return torch.tensor(np.asarray(a), dtype=torch.int32, device="cuda")


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


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


def _same(a, b, name):
    assert np.array_equal(_bits(np.asarray(a, np.float32)), _bits(np.asarray(b, np.float32))), name


def _max_chars():
    from mockingbird_b200 import _lib

    return int(_lib.lib().mb_tacotron_max_chars())


# ---- location-sensitive attention with row lengths ------------------------------------------------------------------------
def _lsa_rows(g, Tc, S, B_lens=None):
    """rows of lengths 1, 2, Tc - 1, Tc and one more of Tc with zero characters inside it; past each end the characters are 0
    (the pad id), the cumulative attention 0 (what the decoder keeps there) and proj / seq NaN"""
    lens = np.array(B_lens if B_lens is not None else sorted({n for n in (1, 2, Tc - 1, Tc) if 1 <= n <= Tc}) + [Tc])
    B, D = len(lens), 128
    inside = np.arange(Tc)[None, :] < lens[:, None]
    chars = np.where(inside, g.integers(1, 75, (B, Tc)), 0).astype(np.int32)
    chars[-1, ::3] = 0
    proj, seq = _f32(g.standard_normal((B, Tc, D)) * 0.5), _f32(g.standard_normal((B, Tc, S)))
    proj[~inside], seq[~inside] = np.nan, np.nan
    cum = np.where(inside, _f32(g.random((B, Tc)) * 2), 0).astype(np.float32)
    return lens, dict(pq=_f32(g.standard_normal((B, D)) * 0.5), proj=proj, seq=seq, chars=chars, cum=cum,
                      conv_w=_f32(g.standard_normal((32, 1, 31)) * 0.3), conv_b=_f32(g.standard_normal(32) * 0.3),
                      Lw=_f32(g.standard_normal((D, 32)) * 0.2), vw=_f32(g.standard_normal((1, D)) * 0.5),
                      q=_f32(g.standard_normal((B, D))), Wq=_f32(g.standard_normal((D, D)) * 0.1),
                      bq=_f32(g.standard_normal(D) * 0.1))


def _lsa_step(a, cum_d, scores, ld, ctx, threads, qpath, lens=None, step_ptr=None, step_j=0, d=None):
    B, Tc, _ = a["proj"].shape
    d = d or {k: _cuda(v) for k, v in a.items() if k != "cum"}
    rep = _dbg("lsa_step", ins=[None if qpath else d["pq"], d["proj"], d["seq"], d["chars"], d["conv_w"], d["conv_b"], d["Lw"],
                                d["vw"], d["q"] if qpath else None, d["Wq"], d["bq"]],
               outs=[cum_d, scores, ctx], n=[B, Tc, a["seq"].shape[2], ld, threads], step_ptr=step_ptr, step_j=step_j,
               row_len=lens)
    assert rep["kernel"] == "lsa_step" and rep["block"] == str(threads)
    return d


def _lsa_ctx(scores, ld, seq_d, B, Tc, S, lens=None, step_ptr=None, step_j=0):
    rows_pad, KB = (64 if B <= 64 else 128), S // 64
    ctx = _nan(B, S)
    tiles = [torch.zeros(KB * rows_pad * 64, dtype=torch.int16, device="cuda") for _ in range(4)]
    rep = _dbg("lsa_ctx", ins=[scores, seq_d], outs=[ctx] + tiles, n=[B, Tc, S, ld, rows_pad], step_ptr=step_ptr, step_j=step_j,
               row_len=lens)
    assert rep["kernel"] == "lsa_ctx"
    c = ctx.cpu().numpy()
    h16, l16 = so.split16(c)
    for t, want in zip(tiles, (h16, l16, h16, l16)):
        u = so.unpack_act_tiles(t.cpu().numpy().view(np.float16), rows_pad, KB)
        assert np.array_equal(u[:B].view(np.int16), want.view(np.int16)) and not u[B:].view(np.int16).any()
    return c


def _cut(a, b, n):
    """row b of an LSA case alone, cut to its n characters"""
    return {k: (v[b:b + 1, :n] if k in ("proj", "seq", "chars", "cum") else v[b:b + 1] if k in ("pq", "q") else v)
            for k, v in a.items()}


@pytest.mark.parametrize("Tc", [1, 2, 33, 181, 600, "limit"])
@pytest.mark.parametrize("threads,qpath,inctx", [(512, True, False), (256, False, True), (512, False, True), (256, True, False)])
def test_lsa_step_rows(Tc, threads, qpath, inctx):
    """scores and cum within the float64 bound of each row alone for t < len, exactly 0 / unchanged past it; each row bitwise a
    launch of that row alone (Tc = len, no lengths); the context in the kernel (seq_dim 72) or by lsa_ctx_kernel (256)"""
    Tc = _max_chars() if Tc == "limit" else Tc
    g = _g(Tc * 3 + threads + qpath)
    S = 72 if inctx else 256
    lens, a = _lsa_rows(g, Tc, S)
    B = len(lens)
    ld = Tc + 3
    cum, scores = _cuda(a["cum"]), _nan(B + 1, ld)
    ctx = _nan(B, S) if inctx else None
    d = _lsa_step(a, cum, scores, ld, ctx, threads, qpath, lens=_i32(lens))
    ref = ko.lsa_step_rows(lens, **{k: a[k] for k in ("proj", "seq", "chars", "cum", "conv_w", "conv_b", "Lw", "vw")},
                           pq=None if qpath else a["pq"], q_in=a["q"] if qpath else None, Wq=a["Wq"], bq=a["bq"], ctx=inctx)
    sc = scores.cpu().numpy()
    assert np.isnan(sc[B:]).all() and np.isnan(sc[:, Tc:]).all()
    s_got, c_got = sc[:B, :Tc], cum.cpu().numpy()
    past = np.arange(Tc)[None, :] >= lens[:, None]
    assert (s_got[past] == 0).all() and (c_got[past] == 0).all(), "past a row's end: score 0, cumulative attention untouched"
    _check("lsa rows scores", s_got, *ref["scores"])
    _check("lsa rows cum", c_got, *ref["cum"])
    if inctx:
        c_ctx = ctx.cpu().numpy()
        _check("lsa rows ctx (in kernel)", c_ctx, *ref["ctx"])
    else:
        c_ctx = _lsa_ctx(scores, ld, d["seq"], B, Tc, S, lens=_i32(lens))
        _check("lsa rows ctx (lsa_ctx)", c_ctx, *ko.context_rows(s_got, a["seq"], lens))
    for b, n in enumerate(lens):
        one = _cut(a, b, n)
        cum1, sc1 = _cuda(one["cum"]), _nan(1, n)
        ctx1 = _nan(1, S) if inctx else None
        d1 = _lsa_step(one, cum1, sc1, n, ctx1, threads, qpath)
        _same(sc1.cpu().numpy()[0], s_got[b, :n], "scores alone")
        _same(cum1.cpu().numpy()[0], c_got[b, :n], "cum alone")
        c1 = ctx1.cpu().numpy() if inctx else _lsa_ctx(sc1, n, d1["seq"], 1, n, S)
        _same(c1[0], c_ctx[b], "ctx alone")
    RAN.add(f"lsa rows:{threads}:{qpath}:{inctx}")
    if Tc == _max_chars():
        RAN.add("lsa rows:limit")


def test_lsa_rows_chained_steps():
    """20 steps through the step pointer, each against the float64 rows applied to the kernel's own previous cum: the cum past
    each row's end stays exactly 0 (the location conv of the next step reads it as the reference's zero padding); lsa_ctx with
    lengths and its split tiles at every step"""
    g = _g(21)
    Tc, S, nst = 181, 512, 20
    lens, a = _lsa_rows(g, Tc, S, B_lens=[181, 100, 2, 1])
    B = len(lens)
    ld_all = nst * Tc
    cum, scores = _cuda(a["cum"]), _nan(B, ld_all)
    sp = torch.tensor([0], dtype=torch.int32, device="cuda")
    ln = _i32(lens)
    past = np.arange(Tc)[None, :] >= lens[:, None]
    d = None
    kw = {k: a[k] for k in ("proj", "seq", "chars", "conv_w", "conv_b", "Lw", "vw", "Wq", "bq")}
    for s in range(nst):
        prev = cum.cpu().numpy()
        sp.fill_(s - s % 2)
        d = _lsa_step(dict(a, cum=prev), cum, scores, ld_all, None, 512, True, lens=ln, step_ptr=sp, step_j=s % 2, d=d)
        ref = ko.lsa_step_rows(lens, cum=prev, q_in=a["q"], ctx=False, **kw)
        got = scores.cpu().numpy().reshape(B, nst, Tc)
        c = cum.cpu().numpy()
        assert (c[past] == 0).all() and (got[:, s][past] == 0).all(), s
        _check("lsa rows chained scores", got[:, s], *ref["scores"])
        _check("lsa rows chained cum", c, *ref["cum"])
        assert np.isnan(got[:, s + 1:]).all()
        ctx = _lsa_ctx(scores, ld_all, d["seq"], B, Tc, S, lens=ln, step_ptr=sp, step_j=s % 2)
        _check("lsa_ctx rows", ctx, *ko.context_rows(got[:, s], a["seq"], lens))
    RAN.add("lsa rows:chained")


# ---- stop rule per row ------------------------------------------------------------------------------------------------------
# row kinds: (cap, passes at step si) -> the B = 1 loop ends at
#   0: cap 1                           -> step 0 (the cap)
#   1: passes from step 0, cap 20      -> step 6 (t = 12 > 10; t = 10 at step 5 is not)
#   2: passes up to step 5, cap 9      -> step 8 (passing while t <= 10 does not end it, and it fails afterwards)
#   3: passes from step 8, cap 20      -> step 8
#   4: already done (step 0) when the window starts, passes at every step: row_done must not move
#   5: never passes, cap 4 or 20       -> step 3, or not within the 10 steps
_NST, _R, _MST = 10, 2, 5.0


def _stop_plan(B, kind_of, cap5):
    kinds = np.array([kind_of(b) for b in range(B)])
    caps = np.array([{0: 1, 1: 20, 2: 9, 3: 20, 4: 20, 5: cap5}[k] for k in kinds])
    si = np.arange(_NST)[:, None]
    k = kinds[None, :]
    passes = (k == 1) | (k == 4) | ((k == 2) & (si <= 5)) | ((k == 3) & (si >= 8)) | (k == 0)
    preset = np.where(kinds == 4, 0, -1)
    return kinds, caps, passes, preset


def _stop_expected(vals, caps, preset):
    done, _ = ko.stop_rows(vals, _MST, _R, caps)
    done = np.where(preset >= 0, preset, done)
    return done, np.array([int(np.all((done >= 0) & (done <= si))) for si in range(_NST)])


@pytest.mark.parametrize("B", [1, 7, 128])
@pytest.mark.parametrize("cap5", [4, 20])
def test_stop_rule_rows(B, cap5):
    """both stop kernels over 10 decoder steps with row_done / row_caps: the done step of every row as its B = 1 loop breaks,
    rows done before the window left alone, flags[si] set exactly from the step the last row ends; the fused stop_step also
    within the float64 bound of its stop values, with its ticket reset after each launch"""
    g = _g(B + cap5)
    kind_runs = [lambda b, k=k: k for k in range(6)] if B == 1 else [lambda b: b % 6]
    K0, K1 = 1024, 576
    w = _f32(g.standard_normal(K0 + K1) * 0.02)
    dw = _cuda(w)
    ww = float(np.dot(w.astype(np.float64), w))
    for kind_of in kind_runs:
        kinds, caps, passes, preset = _stop_plan(B, kind_of, cap5)
        for kern in ("stop_step", "stop_flag"):
            done_d, caps_d = _i32(preset), _i32(caps)
            flags = torch.full((_NST + 2,), -1, dtype=torch.int32, device="cuda")
            ticket = torch.zeros(1, dtype=torch.int32, device="cuda")
            sp = torch.tensor([0], dtype=torch.int32, device="cuda")
            vals = np.zeros((_NST, B), np.float32)
            for si in range(_NST):
                sp.fill_(si - si % 2)
                if kern == "stop_flag":
                    vals[si] = np.where(passes[si], 0.9, 0.4)
                    _dbg("stop_flag", ins=[_cuda(vals[si])], outs=[flags], n=[B, _R], fval=_MST, step_ptr=sp, step_j=si % 2,
                         row_done=done_d, row_caps=caps_d)
                else:
                    c = np.where(passes[si], 6.0, -6.0) * (1 + 0.1 * g.random(B))
                    X = _f32(c[:, None] * w[None, :] / ww)
                    x, cx = np.ascontiguousarray(X[:, :K0]), np.ascontiguousarray(X[:, K0:])
                    y = _nan(B, 3)
                    _dbg("stop_step", segs=[dict(x=_cuda(x), K=K0, ld=K0), dict(x=_cuda(cx), K=K1, ld=K1, w_off=K0)], W=dw,
                         ldw=K0 + K1, bias=_cuda(_f32([0.0])), M=B, N=1, y=y, ldy=3, step_ptr=sp, step_j=si % 2,
                         outs=[flags, ticket], n=[B, _R], fval=_MST, row_done=done_d, row_caps=caps_d)
                    assert int(ticket.item()) == 0
                    yv = y.cpu().numpy()
                    assert np.isnan(yv[:, 1:]).all()
                    vals[si] = yv[:, 0]
                    _check("stop_step rows", vals[si], *ko.stop_value([x, cx], w, [0.0]))
                    assert np.array_equal(vals[si] * np.float32(10) > np.float32(_MST), passes[si]), "the case's pass pattern"
                done, want_flags = _stop_expected(vals[:si + 1], caps, preset)
                got_done = done_d.cpu().numpy()
                assert np.array_equal(got_done, np.where((done >= 0) & (done <= si), done, -1)), (kern, si, kinds)
                f = flags.cpu().numpy()
                assert f[si] == want_flags[si] and (f[si + 1:] == -1).all(), (kern, si)
            done, want_flags = _stop_expected(vals, caps, preset)
            assert np.array_equal(flags.cpu().numpy()[:_NST], want_flags)
            if B > 1:
                assert np.array_equal(done[kinds == 0], np.zeros((kinds == 0).sum())) and (done[kinds == 1] == 6).all()
                assert (done[kinds == 2] == 8).all() and (done[kinds == 3] == 8).all() and (done[kinds == 4] == 0).all()
                assert (done[kinds == 5] == (3 if cap5 == 4 else -1)).all()
                assert want_flags.any() == (cap5 == 4)
            RAN.add(f"stop rows:{kern}")


# ---- per-utterance dropout masks ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("seed", [0, 7, 0x123456789ABCDEF0])
@pytest.mark.parametrize("dec", [0, 1])
def test_fill_masks_seeded(seed, dec):
    """bitwise the numpy Philox of each utterance's own seed in both layouts; the utterance's flags are the same at any row, in
    any B and for any npos >= its own; nothing past the buffer's end is written"""
    seeds = [seed, 3, seed ^ 0xFFFF, 11]
    npos, units = 13, 256

    def run(sds, npos, units):
        n = 2 * len(sds) * npos * units
        m = torch.full((n + 16,), 9, dtype=torch.uint8, device="cuda")
        _dbg("fill_masks_seeded", outs=[m], n=[len(sds), npos, units, dec],
             row_seeds=torch.tensor(np.asarray(sds, np.uint64).view(np.int64), device="cuda"))
        out = m.cpu().numpy()
        assert (out[n:] == 9).all()
        return out[:n]

    for units_ in (units, 10):
        got = run(seeds, npos, units_)
        assert np.array_equal(got, ko.fill_masks_seeded(seeds, npos, units_, dec).reshape(-1)), units_
    own = ko.seeded_masks(seed, npos, units, dec)
    for sds, np_ in (([seed], npos), ([5, 6, 7, 8, seed], npos + 9), ([1] * 70 + [seed], npos + 1)):
        b, B = len(sds) - 1, len(sds)
        got = run(sds, np_, units)
        lay = got.reshape(2, B, np_, units)[:, b, :npos] if dec == 0 else got.reshape(np_, 2, B, units)[:npos, :, b].transpose(1, 0, 2)
        assert np.array_equal(lay, own), (B, np_)
    RAN.add(f"seeded:{dec}")


# ---- fma_chain GEMMs: one fmaf chain whatever M ----------------------------------------------------------------------------
FMA_KERNELS = ("gemm32", "gemm64", "gemm_big")


@pytest.mark.parametrize("M", [1, 63, 64, 65, 128, 129, 1025])
@pytest.mark.parametrize("N", [1, 256, 2048])
@pytest.mark.parametrize("use", ["prenet", "proj"])
def test_gemm_fma_chain(M, N, use):
    """the encoder PreNet layer (bias, ReLU, dropout keep mask) and the GST query / encoder_proj (bias only) with fma_chain: never
    rowdot or a skinny kernel; within the float64 bound; sampled rows bitwise equal to a 1-row launch of the same input"""
    g = _g(M * 7 + N + (use == "prenet"))
    K, ld = 200, 203
    x = _f32(g.standard_normal((M, ld)))
    W = _f32(g.standard_normal((N, K)) * 0.1)
    b = _f32(g.standard_normal(N))
    keep = (g.random((M, N)) < 0.5).astype(np.uint8) if use == "prenet" else None
    act = ko.ACT_RELU if use == "prenet" else ko.ACT_NONE
    xd, Wd, bd = _cuda(x), _cuda(W), _cuda(b)
    kd = None if keep is None else _cuda(keep)
    ldy = N + 3

    def launch(row0, rows):
        y = _nan(rows + 1, ldy)
        rep = _dbg("gemm", segs=[dict(x=xd[row0:], K=K, ld=ld)], W=Wd, ldw=K, bias=bd, M=rows, N=N, act=act,
                   mask=None if kd is None else kd[row0:], y=y, ldy=ldy, fma_chain=1)
        assert rep["kernel"] in FMA_KERNELS, rep
        RAN.add("fma:" + rep["kernel"])
        out = y.cpu().numpy()
        assert np.isnan(out[rows:]).all() and np.isnan(out[:rows, N:]).all()
        return out[:rows, :N]

    full = launch(0, M)
    ref, bound = ko.gemm([x[:, :K]], [W], b, act, keep=keep)
    _check("gemm fma_chain", full, ref, bound)
    for i in sorted({0, 1, M // 2, M - 1} & set(range(M))):
        _same(launch(i, 1)[0], full[i], f"fma_chain row {i} of {M}")


# ---- tc_big at small M and with sequence lengths ------------------------------------------------------------------------------
def _big(x, Wc, bias, shifts, K, M, T, N, lens=None, epi=0, bn=None, res=None):
    nseg = len(shifts)
    ldy = N + 4
    y = _nan(M + 3, ldy)
    xd = _cuda(x)
    act = 1 if epi in (1, 2) else 0
    rep = _tc("big", M=M, N=N, K0=K, w=[_cuda(Wc)], ldw=K * nseg, b=[_cuda(bias)], x=[xd] * nseg, ldx=[K] * nseg, shift=shifts,
              w_off=list(range(nseg)), w_stride=[nseg] * nseg, nseg=nseg, T=T, y=y, ldy=ldy, act=act,
              bn_scale=None if bn is None else _cuda(bn[0]), bn_shift=None if bn is None else _cuda(bn[1]),
              res=None if res is None else _cuda(res), ldres=N, len=None if lens is None else _i32(lens))
    assert rep["kernel"] == "tc_big" and rep["grid"] == f"{(N + 127) // 128},{(M + 127) // 128}"
    out = y.cpu().numpy()
    assert np.isnan(out[M:]).all() and np.isnan(out[:M, N:]).all()
    return out[:M, :N]


@pytest.mark.parametrize("M", [1, 2, 127, 128, 129, 160, 300])
def test_big_encoder_shape_small_m(M):
    """the speaker encoder's layer-0 input projection (nseg 1, K 40, T 1, N 4H = 1024) at the small M the row route now reaches:
    split and exact references; each row bitwise the same alone and at another position of a 128-row tile"""
    g = _g(M)
    K, N = 40, 1024
    x = _f32(g.standard_normal((M, K)))
    W = _f32(g.standard_normal((N, K, 1)) * 0.1)
    bias = _f32(g.standard_normal(N))
    out = _big(x, W, bias, [0], K, M, 1, N)
    A, Wm = x, W[:, :, 0]
    s = so.pow2_scale(W)
    S = so.split_sum(A, Wm, s)
    bound = so.big_epilogue_bound(S, so.acc_bound(A, Wm, s), bias)
    _check("big small M vs split", out, so.big_epilogue(S, bias), bound)
    _check("big small M vs exact", out, so.big_epilogue(so.exact(A, Wm), bias), bound + so.rep_bound(A, Wm, s))
    for i in sorted({0, M // 2, M - 1}):
        _same(_big(x[i:i + 1], W, bias, [0], K, 1, 1, N)[0], out[i], "row alone")
        shifted = np.concatenate([_f32(g.standard_normal((37, K))), x[i:i + 1]])
        _same(_big(shifted, W, bias, [0], K, 38, 1, N)[37], out[i], "row at position 37")
    RAN.add("big:small_m")


# (nseg = taps k of a bank conv or conv_project, T, M (T need not divide it), N, K, epilogue 0 none, 1 ReLU, 2 ReLU + BN, 3 BN + res)
BIG_ROWS = [(1, 7, 30, 128, 40, 0), (2, 5, 23, 128, 128, 1), (3, 9, 100, 256, 80, 2), (4, 6, 200, 128, 128, 3),
            (5, 11, 130, 128, 128, 1), (5, 13, 300, 132, 40, 2), (3, 4, 1, 128, 64, 3), (5, 8, 21, 256, 64, 0)]


@pytest.mark.parametrize("nseg,T,M,N,K,epi", BIG_ROWS)
def test_big_taps_with_lengths(nseg, T, M, N, K, epi):
    """CBHG tap convs with per-sequence lengths 1, T - 1, T (shifts -k/2 .. k - 1 - k/2, the input NaN past each end): every row
    of every utterance within the split / exact bounds of that utterance alone; the first and last utterance bitwise a launch of
    that utterance alone, and every row bitwise the same one 128-row tile position further on"""
    g = _g(nseg * 100 + T + M)
    shifts = [j - nseg // 2 for j in range(nseg)]
    nsq = (M + T - 1) // T
    lens = np.array([(1, T - 1, T)[j % 3] for j in range(nsq)]).clip(1)
    valid = np.zeros(M, bool)
    for j in range(nsq):
        valid[j * T:min(j * T + lens[j], M)] = True
    x = _f32(g.standard_normal((M, K)))
    x[~valid] = np.nan
    Wc = _f32(g.standard_normal((N, K, nseg)) * 0.05)
    bias = _f32(g.standard_normal(N))
    bn = (_f32(g.uniform(0.5, 1.5, N)), _f32(g.standard_normal(N))) if epi >= 2 else None
    res = _f32(g.standard_normal((M, N))) if epi == 3 else None
    out = _big(x, Wc, bias, shifts, K, M, T, N, lens, epi, bn, res)
    A = so.im2col_rows([x] * nseg, shifts, K, M, T, lens)[valid]
    W = np.concatenate([Wc[:, :, j] for j in range(nseg)], 1)
    s = so.pow2_scale(Wc)
    act = 1 if epi in (1, 2) else 0
    rv = None if res is None else res[valid]
    S = so.split_sum(A, W, s)
    ref = so.big_epilogue(S, bias, act, *(bn or (None, None)), rv)
    bound = so.big_epilogue_bound(S, so.acc_bound(A, W, s), bias, act, *(bn or (None, None)), rv)
    _check("big rows vs split", out[valid], ref, bound)
    if epi in (0, 3):
        refx = so.big_epilogue(so.exact(A, W), bias, act, *(bn or (None, None)), rv)
        repb = so.rep_bound(A, W, s) * (1 if bn is None else np.abs(bn[0])[None, :])
        _check("big rows vs exact", out[valid], refx, bound + repb)
    for j in sorted({0, nsq - 1}):
        r0, n = j * T, min(int(lens[j]), M - j * T)
        alone = _big(x[r0:r0 + n], Wc, bias, shifts, K, n, n, N, None, epi, bn, None if res is None else res[r0:r0 + n])
        _same(alone, out[r0:r0 + n], f"utterance {j} alone")
    pad = 128 // T * T  # whole sequences of length 1 in front: every row moves by `pad` rows inside the 128-row tiles
    pad -= T if pad == 128 else 0
    front = np.full((pad, K), np.nan, np.float32)
    front[::T] = 1.0
    xs = np.concatenate([front, x])
    lens2 = np.concatenate([np.ones(pad // T, int), lens])
    res2 = None if res is None else np.concatenate([np.zeros((pad, N), np.float32), res])
    moved = _big(xs, Wc, bias, shifts, K, M + pad, T, N, lens2, epi, bn, res2)[pad:]
    _same(moved[valid], out[valid], "rows moved inside the tiles")
    RAN.add(f"big:rows:{epi}")
    RAN.add(f"big:nseg{nseg}")


# ---- tc_gru: the backward direction starts at each row's own end --------------------------------------------------------------
def test_gru_rows_chained():
    """both directions stepped over T as run_cbhg steps them, lengths 1, 2, T, 3, T: direction 1 within the bound of the float64
    GRU started from h = 0 at each row's last step, and exact zeros in its state, out[1] and next-step tiles while t1 >= len
    (its gi is NaN there)"""
    g = _g(31)
    M, T, H = 5, 6, 128
    lens = np.array([1, 2, T, 3, T])
    Ws = [_f32(g.standard_normal((3 * H, H)) * (0.5 / np.sqrt(H))) for _ in range(2)]
    bs = [_f32(g.standard_normal(3 * H) * 0.2) for _ in range(2)]
    gi_f = _f32(g.standard_normal((M, T, 3 * H)))
    gi_b = _f32(g.standard_normal((M, T, 3 * H)))
    gi_b[np.arange(T)[None, :] >= lens[:, None]] = np.nan
    gfd, gbd = _cuda(gi_f), _cuda(gi_b)
    out_all = _nan(M, T, 2 * H)
    hst = [torch.zeros(M, H, device="cuda") for _ in range(2)]
    ln = _i32(lens)
    ref_seq = so.gru_reverse_rows(np.nan_to_num(gi_b), Ws[1], bs[1], lens)
    W, b = Ws[1], bs[1].astype(np.float64)
    sc = so.pow2_scale(W)
    h_k = np.zeros((M, H), np.float32)
    h_ref, dh = np.zeros((M, H)), np.zeros((M, H))
    for s in range(T):
        t_b = T - 1 - s
        nxt_hi = [torch.zeros(H * 64, dtype=torch.int16, device="cuda") for _ in range(2)]
        nxt_lo = [torch.zeros_like(nxt_hi[0]) for _ in range(2)]
        _tc("gru", M=M, H=H, K0=H, w=[_cuda(w) for w in Ws], b=[_cuda(v) for v in bs], x=[h.clone() for h in hst], ldx=[H, H],
            gi=[gfd[:, s], gbd[:, t_b]], ldgi=T * 3 * H, hst=hst, out=[out_all[:, s], out_all[:, t_b, H:]], ldout=T * 2 * H,
            ndir=2, nxt_hi=nxt_hi, nxt_lo=nxt_lo, len=ln, t1=t_b)
        active = t_b < lens
        got = hst[1].cpu().numpy()
        o = out_all.cpu().numpy()[:, t_b, H:]
        th = so.unpack_act_tiles(nxt_hi[1].cpu().numpy().view(np.float16), 64, H // 64)
        tl = so.unpack_act_tiles(nxt_lo[1].cpu().numpy().view(np.float16), 64, H // 64)
        assert not got[~active].any() and not o[~active].any(), t_b
        assert not th[:M][~active].view(np.int16).any() and not tl[:M][~active].view(np.int16).any(), t_b
        assert np.array_equal(o, got)
        gh_k = so.split_sum(h_k, W, sc) + b
        dgh = (so.acc_bound(h_k, W, sc) + so.rep_bound(h_k, W, sc) + so.U24 * np.abs(gh_k) + dh @ np.abs(W.astype(np.float64)).T)
        with np.errstate(invalid="ignore"):
            dh_new = so.gru_cell_bound(so.exact(h_ref, W) + b, gi_b[:, t_b], h_ref, H, dgh, dh)
        dh = np.where(active[:, None], dh_new, 0.0)
        h_ref = ref_seq[:, t_b]
        _check("gru rows backward", got[active], h_ref[active], dh[active])
        h_k = got
    assert np.isfinite(out_all.cpu().numpy()).all(), "every step wrote both directions"
    RAN.add("gru:rows")


def _gru_pool(g, n, H):
    W = [_f32(g.standard_normal((3 * H, H)) * (0.5 / np.sqrt(H))) for _ in range(2)]
    b = [_f32(g.standard_normal(3 * H) * 0.2) for _ in range(2)]
    h = [_f32(np.tanh(g.standard_normal((n, H)))) for _ in range(2)]
    gi = [_f32(g.standard_normal((n, 3 * H))) for _ in range(2)]
    return W, b, h, gi


@pytest.mark.parametrize("kind", ["gru", "lstm_seq"])
def test_recurrent_rows_independent_of_m(kind):
    """one step of tc_gru (both directions, lengths and t1 so that some rows hold h = 0) or tc_lstm_seq: the same rows at other
    positions of launches of M = 1, 64, 65, 128 (and 129, 300: row blocks of tc_lstm_seq) give bitwise the same results"""
    g = _g(41)
    H, P = 128, 128 if kind == "gru" else 300
    W, b, h, gi = _gru_pool(g, P, H)
    lens = g.integers(1, 9, P)
    t1 = 4
    Wl = _f32(g.standard_normal((4 * H, H)) * (1 / np.sqrt(H)))
    gl = _f32(g.standard_normal((P, 4 * H)))
    c0 = _f32(g.standard_normal((P, H)))

    def run(idx):
        m = len(idx)
        if kind == "gru":
            hst = [_cuda(h[d][idx]) for d in range(2)]
            outs = [_nan(m, H) for _ in range(2)]
            _tc("gru", M=m, H=H, K0=H, w=[_cuda(w) for w in W], b=[_cuda(v) for v in b], x=[_cuda(h[d][idx]) for d in range(2)],
                ldx=[H, H], gi=[_cuda(gi[d][idx]) for d in range(2)], ldgi=3 * H, hst=hst, out=outs, ldout=H, ndir=2,
                len=_i32(lens[idx]), t1=t1)
            return np.concatenate([o.cpu().numpy() for o in outs], 1)
        cd, out = _cuda(c0[idx]), _nan(m, H)
        _tc("lstm_seq", M=m, H=H, K0=H, w=[_cuda(Wl)], x=[_cuda(h[0][idx])], ldx=[H], gi=[_cuda(gl[idx])], ldgi=4 * H, c=cd,
            out=[out], ldout=H)
        return np.concatenate([out.cpu().numpy(), cd.cpu().numpy()], 1)

    base = run(np.arange(P))
    assert np.isfinite(base).all()
    if kind == "gru":
        assert not base[lens <= t1, H:].any() and base[lens > t1, H:].any()
    for m in (1, 64, 65, 128) + ((129, 300) if kind == "lstm_seq" else ()):
        idx = np.roll(np.arange(P), 3 * m + 1)[:m]
        _same(run(idx), base[idx], f"{kind} M = {m}")
    RAN.add(f"indep:{kind}")


# ---- speaker encoder: L2 of the mean of each utterance's partials ----------------------------------------------------------------
@pytest.mark.parametrize("E", [33, 100, 256])
def test_encoder_reduce_partials(E):
    """mb_encoder_reduce_partials over utterances of 1, 2, 600 and 5 partials (E not a multiple of 32 too) against float64"""
    from mockingbird_b200 import _lib

    L = _lib.lib()
    cfg = _lib.EncoderConfig(40, 64, 1, E)
    h = C.c_void_p()
    _lib.check(L.mb_encoder_create(C.byref(cfg), C.byref(h)))
    try:
        g = _g(E)
        counts = [1, 2, 600, 5]
        off = np.concatenate([[0], np.cumsum(counts)]).astype(np.int32)
        p = _f32(np.maximum(g.standard_normal((off[-1], E)), 0))
        p /= np.linalg.norm(p, axis=1, keepdims=True) + 1e-5
        pd, od = _cuda(p), _i32(off)
        out = _nan(len(counts) + 1, E)
        _lib.check(L.mb_encoder_reduce_partials(h, C.c_void_p(pd.data_ptr()), C.c_void_p(od.data_ptr()), len(counts),
                                                C.c_void_p(out.data_ptr()), C.c_void_p(torch.cuda.current_stream().cuda_stream)))
        torch.cuda.synchronize()
        got = out.cpu().numpy()
        assert np.isnan(got[len(counts):]).all()
        _check("reduce partials", got[:len(counts)], *eo.reduce_partials(p, off))
    finally:
        L.mb_encoder_destroy(h)
    RAN.add(f"reduce:{E}")


# ---- coverage -----------------------------------------------------------------------------------------------------------------
def test_every_ragged_variant_ran():
    for k, v in sorted(WORST.items()):
        print(f"worst error / bound  {k:28s} {v:.3g}")
    want = {"lsa_step", "lsa_ctx", "stop_step", "stop_flag", "fill_masks_seeded", "tc_big", "tc_gru", "tc_lstm_seq"}
    want |= {f"lsa rows:{t}:{q}:{c}" for t, q, c in ((512, True, False), (256, False, True), (512, False, True), (256, True, False))}
    want |= {"lsa rows:limit", "lsa rows:chained", "stop rows:stop_step", "stop rows:stop_flag", "seeded:0", "seeded:1"}
    want |= {f"fma:{k}" for k in FMA_KERNELS} | {"big:small_m", "gru:rows", "indep:gru", "indep:lstm_seq"}
    want |= {f"big:rows:{e}" for e in range(4)} | {f"big:nseg{n}" for n in range(1, 6)} | {f"reduce:{e}" for e in (33, 100, 256)}
    missing = sorted(want - RAN)
    assert not missing, missing
