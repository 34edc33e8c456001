"""CPU tests of oracle/taco_kernel_oracle.py: each float64 reference with its bound accepts fp32 torch arithmetic of the same
operation in another summation order (tacotron_oracle.py's functions or torch.nn.functional), and rejects the wrong variants
a kernel could plausibly compute.  The margins (worst |err| / bound) are printed, so a bound that is loose shows."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import taco_kernel_oracle as ko
import tacotron_oracle as to


def _ratio(got, ref, bound):
    err = np.abs(np.asarray(got, np.float64) - ref)
    with np.errstate(divide="ignore", invalid="ignore"):
        return float(np.max(np.where(err == 0, 0.0, err / bound)))  # dropped outputs are exact zeros with a zero bound


def _accept(name, got, ref, bound):
    r = _ratio(got, ref, bound)
    print(f"{name}: accepted at {r:.3g} of the bound")
    assert r <= 1.0, (name, r)


def _reject(name, got, ref, bound):
    r = _ratio(got, ref, bound)
    print(f"{name}: rejected at {r:.3g} x the bound")
    assert r > 1.0, (name, r)


def _g(seed):
    return np.random.default_rng(seed)


def _f32(a):
    return np.asarray(a, np.float32)


def _t(a):
    return torch.from_numpy(np.ascontiguousarray(a))


# ---- GEMM epilogue and conv taps ---------------------------------------------------------------------------------------------
def test_gemm_conv_taps_bn_mask_residual():
    """a CBHG BatchNormConv (k = 5 as shifted-row segments, ReLU -> BN) with a dropout mask and residual, vs torch fp32"""
    g = _g(1)
    B, T, Ci, Co, k = 3, 7, 24, 16, 5
    x = _f32(g.standard_normal((B * T, Ci)))
    W = _f32(g.standard_normal((Co, Ci, k)) * 0.2)
    bias = _f32(g.standard_normal(Co))
    sc, sh = _f32(g.uniform(0.5, 2, Co)), _f32(g.standard_normal(Co))
    keep = (g.random((B * T, Co)) < 0.5).astype(np.uint8)
    res = _f32(g.standard_normal((B * T, Co)))
    shifts = range(-2, 3)
    xs = [ko.gemm_operand(x, Ci, Ci, B * T, T, s) for s in shifts]
    ws = [ko.gemm_weight(W, Ci * k, Co, Ci, w_off=j, w_stride=k) for j in range(k)]
    ref, bound = ko.gemm(xs, ws, bias, ko.ACT_RELU, sc, sh, keep, res)
    conv = F.conv1d(_t(x).view(B, T, Ci).transpose(1, 2), _t(W), _t(bias), padding=2).transpose(1, 2).reshape(B * T, Co)
    y = F.relu(conv) * _t(sc) + _t(sh)
    got = (y * _t(keep).float() * 2 + _t(res)).numpy()
    _accept("gemm conv", got, ref, bound)
    # a tap shifted the wrong way at a sequence boundary: the shift crosses into the neighbouring utterance
    bad_xs = list(xs)
    m = np.arange(B * T)
    wrong = _f32(np.zeros_like(xs[0]))
    ok = m - 2 >= 0
    wrong[ok] = x[m[ok] - 2]
    bad_xs[0] = wrong
    _reject("tap across the sequence boundary", ko.gemm(bad_xs, ws, bias, ko.ACT_RELU, sc, sh, keep, res)[0], ref, bound)
    pre = sum(np.asarray(a, np.float64) @ np.asarray(w, np.float64).T for a, w in zip(xs, ws)) + bias
    bn_first = np.maximum(pre * sc + sh, 0) * 2 * keep + res
    _reject("BN before the ReLU", bn_first, ref, bound)
    mask_after = (np.maximum(pre, 0) * sc + sh + res) * 2 * keep
    _reject("mask after the residual", mask_after, ref, bound)


@pytest.mark.parametrize("act", [ko.ACT_SIGMOID, ko.ACT_TANH])
def test_gemm_activations(act):
    g = _g(act)
    x, W, b = _f32(g.standard_normal((9, 300))), _f32(g.standard_normal((5, 300)) * 0.05), _f32(g.standard_normal(5))
    ref, bound = ko.gemm([x], [W], b, act)
    f = torch.sigmoid if act == ko.ACT_SIGMOID else torch.tanh
    _accept(f"gemm act {act}", f(F.linear(_t(x), _t(W), _t(b))).numpy(), ref, bound)
    _reject(f"gemm act {act} without bias", ko.activation(np.asarray(x, np.float64) @ np.asarray(W, np.float64).T, act), ref, bound)


def test_gemm_step_mode_operand():
    """segment 0 in step mode: x + step * x_step, the x_first go row at step 0"""
    x = np.arange(60, dtype=np.float32)
    first = np.full(4, -1, np.float32)
    assert np.array_equal(ko.gemm_operand(x, 8, 4, 2, step=0, x_step=20, x_first=first), np.full((2, 4), -1))
    assert np.array_equal(ko.gemm_operand(x, 8, 4, 2, step=2, x_step=20, x_first=first), [[40, 41, 42, 43], [48, 49, 50, 51]])


# ---- PreNet ------------------------------------------------------------------------------------------------------------------
def test_prenet():
    g = _g(2)
    B, K, H = 5, 80, 256
    x = _f32(g.standard_normal((B, K)))
    W1, b1 = _f32(g.standard_normal((H, K)) * 0.1), _f32(g.standard_normal(H) * 0.1)
    W2, b2 = _f32(g.standard_normal((H, H)) * 0.1), _f32(g.standard_normal(H) * 0.1)
    k1, k2 = (g.random((B, H)) < 0.5), (g.random((B, H)) < 0.5)
    ref, bound = ko.prenet(x, W1, b1, W2, b2, k1, k2)
    sd = {"p.fc1.weight": _t(W1), "p.fc1.bias": _t(b1), "p.fc2.weight": _t(W2), "p.fc2.bias": _t(b2)}
    got = to._prenet(_t(x), sd, "p", [_t(k1), _t(k2)]).numpy()
    _accept("prenet", got, ref, bound)
    _reject("prenet masks swapped", ko.prenet(x, W1, b1, W2, b2, k2, k1)[0], ref, bound)


# ---- cells -------------------------------------------------------------------------------------------------------------------
def test_gru_cell():
    g = _g(3)
    M, H, Ki = 6, 64, 40
    x, h = _f32(g.standard_normal((M, Ki))), _f32(g.standard_normal((M, H)))
    Wi, Wh = _f32(g.standard_normal((3 * H, Ki)) * 0.2), _f32(g.standard_normal((3 * H, H)) * 0.2)
    bi, bh = _f32(g.standard_normal(3 * H)), _f32(g.standard_normal(3 * H))
    gi, gh = (_f32(F.linear(_t(x), _t(Wi), _t(bi)).numpy()), _f32(F.linear(_t(h), _t(Wh), _t(bh)).numpy()))
    ref, bound = ko.gru_cell(gi, gh, h, H)
    # tacotron_oracle._gru_dir's cell lines, one step from h
    r = torch.sigmoid(_t(gh[:, :H]) + _t(gi[:, :H]))
    z = torch.sigmoid(_t(gh[:, H:2 * H]) + _t(gi[:, H:2 * H]))
    n = torch.tanh(_t(gi[:, 2 * H:]) + _t(gh[:, 2 * H:]) * r)
    _accept("gru cell", ((_t(h) - n) * z + n).numpy(), ref, bound)
    # r multiplying W_hn h without b_hn
    ghn_nob = np.asarray(h, np.float64) @ np.asarray(Wh[2 * H:], np.float64).T
    rr = 1 / (1 + np.exp(-(np.float64(gh[:, :H]) + gi[:, :H])))
    zz = 1 / (1 + np.exp(-(np.float64(gh[:, H:2 * H]) + gi[:, H:2 * H])))
    nn = np.tanh(np.float64(gi[:, 2 * H:]) + bh[2 * H:] + rr * ghn_nob)
    _reject("GRU r without b_hn", (h - nn) * zz + nn, ref, bound)


def test_lstm_cell():
    g = _g(4)
    M, H = 5, 48
    gates, c, x = _f32(g.standard_normal((M, 4 * H)) * 2), _f32(g.standard_normal((M, H))), _f32(g.standard_normal((M, H)))
    cn, hn, xn, dc, dh, dx = ko.lstm_cell(gates, c, H, x)
    i, f, gg, o = _t(gates).chunk(4, 1)
    c_t = torch.sigmoid(f) * _t(c) + torch.sigmoid(i) * torch.tanh(gg)
    h_t = torch.sigmoid(o) * torch.tanh(c_t)
    _accept("lstm c", c_t.numpy(), cn, dc)
    _accept("lstm h", h_t.numpy(), hn, dh)
    _accept("lstm x + h", (_t(x) + h_t).numpy(), xn, dx)
    swapped = np.concatenate([gates[:, H:2 * H], gates[:, :H], gates[:, 2 * H:]], 1)
    _reject("LSTM gates i and f swapped", ko.lstm_cell(swapped, c, H)[0], cn, dc)


def test_highway_and_maxpool():
    g = _g(5)
    M, C = 11, 32
    x12, y = _f32(g.standard_normal((M, 2 * C)) * 3), _f32(g.standard_normal((M, C)))
    ref, bound = ko.highway(x12, y, C)
    gt = torch.sigmoid(_t(x12[:, C:]))
    _accept("highway", (gt * F.relu(_t(x12[:, :C])) + (1.0 - gt) * _t(y)).numpy(), ref, bound)
    g1 = 1 / (1 + np.exp(-np.float64(x12[:, :C])))
    _reject("highway gate from x1", g1 * np.maximum(x12[:, :C], 0) + (1 - g1) * y, ref, bound)
    x = _f32(g.standard_normal((3, 9, C)))
    ref = ko.maxpool2(x)
    got = F.max_pool1d(_t(x).transpose(1, 2), 2, 1, 1)[:, :, :9].transpose(1, 2).numpy()
    assert np.array_equal(got, ref)
    nxt = np.asarray(x, np.float64).copy()
    nxt[:, :-1] = np.maximum(x[:, :-1], x[:, 1:])
    assert not np.array_equal(nxt, ref), "the max pool looking at t + 1 must differ"


# ---- location-sensitive attention --------------------------------------------------------------------------------------------
def _lsa_inputs(seed, B=3, Tc=40, D=128, S=64):
    g = _g(seed)
    return dict(
        pq=_f32(g.standard_normal((B, D)) * 0.5), proj=_f32(g.standard_normal((B, Tc, D)) * 0.5),
        seq=_f32(g.standard_normal((B, Tc, S))), chars=np.where(np.arange(Tc)[None, :] < np.array([[Tc], [Tc - 9], [5]])[:B], 7, 0),
        cum=_f32(g.random((B, Tc)) * 2), conv_w=_f32(g.standard_normal((32, 1, 31)) * 0.3), conv_b=_f32(g.standard_normal(32) * 0.3),
        Lw=_f32(g.standard_normal((D, 32)) * 0.2), vw=_f32(g.standard_normal((1, D)) * 0.5))


def _lsa_torch(a, flip=False, mask="mul"):
    """tacotron_oracle.generate's LSA lines in torch fp32 (and wrong variants of them)"""
    cw = _t(a["conv_w"])
    if flip:
        cw = cw.flip(-1)
    loc = F.conv1d(_t(a["cum"]).unsqueeze(1), cw, _t(a["conv_b"]), 1, 15)
    ploc = F.linear(loc.transpose(1, 2), _t(a["Lw"]))
    u = F.linear(torch.tanh(_t(a["pq"]).unsqueeze(1) + _t(a["proj"]) + ploc), _t(a["vw"])).squeeze(-1)
    cm = _t((a["chars"] != 0).astype(np.float32))
    if mask == "mul":
        u = u * cm
    elif mask == "neginf":
        u = u.masked_fill(cm == 0, float("-inf"))
    s = F.softmax(u, dim=1)
    return s.numpy(), (_t(a["cum"]) + s).numpy(), torch.bmm(s.unsqueeze(1), _t(a["seq"])).squeeze(1).numpy()


def test_lsa_step():
    a = _lsa_inputs(6)
    ref = ko.lsa_step(**a)
    s, cum, ctx = _lsa_torch(a)
    for name, got in (("scores", s), ("cum", cum), ("ctx", ctx)):
        _accept(f"lsa {name}", got, *ref[name])
    _reject("char mask dropped", _lsa_torch(a, mask="none")[0], *ref["scores"])
    _reject("padded positions at -inf", _lsa_torch(a, mask="neginf")[0], *ref["scores"])
    _reject("location kernel flipped", _lsa_torch(a, flip=True)[0], *ref["scores"])


def test_lsa_query_inside():
    g = _g(7)
    a = _lsa_inputs(7, B=2, Tc=20)
    q, Wq, bq = _f32(g.standard_normal((2, 128))), _f32(g.standard_normal((128, 128)) * 0.1), _f32(g.standard_normal(128) * 0.1)
    a["pq"] = F.linear(_t(q), _t(Wq), _t(bq)).numpy()
    ref = ko.lsa_step(**dict(a, pq=None), q_in=q, Wq=Wq, bq=bq)
    _accept("lsa scores, query inside", _lsa_torch(a)[0], *ref["scores"])


# ---- GST -----------------------------------------------------------------------------------------------------------------------
def test_gst_attention():
    g = _g(8)
    B, E, heads, ntok = 3, 512, 8, 10
    q, k, v = _f32(g.standard_normal((B, E))), _f32(g.standard_normal((ntok, E))), _f32(g.standard_normal((ntok, E)))
    ref, bound = ko.gst_attention(q, k, v, heads)
    # tacotron_oracle._mha's head split, scores and softmax in torch fp32 (its values are projected keys: separate here)
    qh, kh, vh = (_t(t).view(-1, heads, E // heads) for t in (q, k, v))
    p = F.softmax(torch.einsum("bhd,khd->bhk", qh, kh) / (E // heads) ** 0.5, -1)
    _accept("gst", torch.einsum("bhk,khd->bhd", p, vh).reshape(B, E).numpy(), ref, bound)
    p_bad = torch.softmax(torch.einsum("bhd,khd->bhk", qh, kh) / E ** 0.5, -1)
    _reject("GST scale 1/sqrt(E)", torch.einsum("bhk,khd->bhd", p_bad, vh).reshape(B, E).numpy(), ref, bound)


# ---- stop, BN fold, layouts --------------------------------------------------------------------------------------------------
def test_stop_value_and_rule():
    g = _g(9)
    x, c, w, b = _f32(g.standard_normal((7, 1024))), _f32(g.standard_normal((7, 576))), _f32(g.standard_normal(1600) * 0.02), _f32([0.3])
    ref, bound = ko.stop_value([x, c], w, b)
    got = torch.sigmoid(F.linear(torch.cat([_t(x), _t(c)], 1), _t(w)[None], _t(b))).squeeze(1).numpy()
    _accept("stop", got, ref, bound)
    assert ko.stop_flag([0.9, 0.8], 5, 6, 2) == 1 and ko.stop_flag([0.9, 0.8], 5, 5, 2) == 0  # 12 > 10, 10 is not
    assert ko.stop_flag([0.9, 0.4], 5, 6, 2) == 0


def test_bn_fold_and_layouts():
    g = _g(10)
    n = 40
    gam, bet, mean, var = _f32(g.standard_normal(n)), _f32(g.standard_normal(n)), _f32(g.standard_normal(n)), _f32(g.random(n) + 0.1)
    (s, ds), (sh, dsh) = ko.bn_fold(gam, bet, mean, var)
    x = _f32(g.standard_normal((4, n, 3)))
    y = F.batch_norm(_t(x), _t(mean), _t(var), _t(gam), _t(bet), False, 0.1, 1e-5)
    fold = np.asarray(x, np.float64) * s[None, :, None] + sh[None, :, None]
    slack = np.abs(x) * ds[None, :, None] + dsh[None, :, None] + 4 * ko.U24 * (np.abs(fold) + np.abs(y.numpy()))
    _accept("bn fold vs F.batch_norm", y.numpy(), fold, slack)
    W = np.arange(6 * 5 * 3).reshape(6 * 5, 3)  # n_mels 6, max_r 5, K 3
    P = ko.pack_melproj(W, 6, 5, 2)
    assert np.array_equal(P[6 + 4], W[4 * 5 + 1])
    assert np.array_equal(torch.from_numpy(W).view(6, 5, 3)[:, :2].transpose(0, 1).reshape(12, 3).numpy(), P)
    x = np.arange(2 * 5 * 3).reshape(2, 5, 3)
    assert np.array_equal(ko.to_ncl(x, 5, 2, 3, 4), x[:, :4].transpose(0, 2, 1))


# ---- Philox ------------------------------------------------------------------------------------------------------------------
def test_philox_known_answers():
    """Random123's Philox4x32-10 known-answer vectors"""
    kat = [((0, 0, 0, 0, 0, 0), (0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8)),
           ((0xFFFFFFFF,) * 6, (0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD)),
           ((0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344, 0xA4093822, 0x299F31D0),
            (0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1))]
    for args, want in kat:
        assert tuple(int(v) for v in ko.philox4x32(*args)) == want


def test_fill_masks_known_bits():
    """keep flags 0..23 of fill_masks_kernel's streams (mb_philox4x32 of include/mb_wavernn_math.h evaluated on the host):
    a seed with the high 32 bits set, the encoder stream 0xffffffff and decoder step streams 0 and 37"""
    want = {(0x123456789ABCDEF0, 0xFFFFFFFF): "111010101111111110111111", (0x123456789ABCDEF0, 0): "100000011100100010011111",
            (0x123456789ABCDEF0, 37): "000010110100001100001010", (7, 0xFFFFFFFF): "100000100100000110001000",
            (7, 0): "100010110100010000101011", (7, 37): "100100111010101001011001"}
    for (seed, sid), bits in want.items():
        assert "".join(map(str, ko.fill_masks(24, seed, sid))) == bits, (hex(seed), sid)
    steps = ko.fill_masks_steps(10, 38, 7)
    assert "".join(map(str, steps[370:380])) == "".join(map(str, ko.fill_masks(10, 7, 37)))
    # the high counter word: index 2^34 + i is counter (i >> 2, 1)
    hi = ko.fill_masks(8, 7, 0, first=1 << 34)
    o = ko.philox4x32(np.arange(2), 1, 0, ko.MASK_TAG, 7, 0)
    assert [int((o[i & 3][i >> 2] >> 16) & 1) for i in range(8)] == hi.tolist()


# ---- ragged batches: each row is the B = 1 utterance of its own length -----------------------------------------------------
def test_lsa_step_rows_is_each_row_alone():
    """the ragged LSA step of a row is torch's LSA step on that row alone, cut to its length; past the end the score is 0 and
    the cumulative attention untouched.  The padded-batch row (positions past the end scored as chars == 0) is rejected."""
    a = _lsa_inputs(11, B=3, Tc=40)
    lens = np.array([40, 23, 1])
    a["chars"] = np.where(np.arange(40)[None, :] < lens[:, None], 9, 0)
    a["chars"][0, 5] = 0  # a zero character inside the row: scored as exp(0), as in the reference
    a["cum"][np.arange(40)[None, :] >= lens[:, None]] = 0
    ref = ko.lsa_step_rows(lens, **a)
    for b, n in enumerate(lens):
        one = {k: (v[b:b + 1, :n] if k in ("proj", "seq", "chars", "cum") else v[b:b + 1] if k == "pq" else v) for k, v in a.items()}
        s, cum, ctx = _lsa_torch(one)
        _accept("lsa rows scores", s, ref["scores"][0][b:b + 1, :n], ref["scores"][1][b:b + 1, :n])
        _accept("lsa rows cum", cum, ref["cum"][0][b:b + 1, :n], ref["cum"][1][b:b + 1, :n])
        _accept("lsa rows ctx", ctx, ref["ctx"][0][b:b + 1], ref["ctx"][1][b:b + 1])
        assert not ref["scores"][0][b, n:].any() and not ref["scores"][1][b, n:].any()
        assert np.array_equal(ref["cum"][0][b, n:], a["cum"][b, n:]) and not ref["cum"][1][b, n:].any()
    padded = ko.lsa_step(**a)
    _reject("padded-batch row scores", padded["scores"][0][1:2], ref["scores"][0][1:2], ref["scores"][1][1:2])
    cs, cd = ko.context_rows(ref["scores"][0], a["seq"], lens, ref["scores"][1])
    assert np.array_equal(cs, ref["ctx"][0]) and np.array_equal(cd, ref["ctx"][1])


def test_stop_rows():
    """the per-row stop rule as the B = 1 loop breaks: at the first step with stop * 10 > min_stop and t = si r > 10, else at the
    cap; a row that passed at t <= 10 and fails later does not end; flags once every row has ended"""
    r, mst = 2, 5.0
    v = np.full((10, 5), 0.4, np.float32)
    v[:, 1] = 0.9  # passes from the start: ends at si = 6 (t = 12), not 5 (t = 10)
    v[:6, 2] = 0.9  # passes while t <= 10, fails after: runs to its cap
    v[8:, 3] = 0.9
    caps = np.array([1, 20, 9, 20, 20])
    done, flags = ko.stop_rows(v, mst, r, caps)
    assert done.tolist() == [0, 6, 8, 8, -1]
    assert flags.tolist() == [0] * 10
    done, flags = ko.stop_rows(v[:, :4], mst, r, caps[:4])
    assert flags.tolist() == [0] * 8 + [1, 1]
    # B = 1 rows agree with the padded rule's flag at the step they end (stop_flag), and a batch of one row is its own loop
    for b in range(4):
        d, f = ko.stop_rows(v[:, b:b + 1], mst, r, caps[b:b + 1])
        assert d[0] == done[b] and f[d[0]] == 1 and not f[:d[0]].any()
        if d[0] < caps[b] - 1:
            assert ko.stop_flag(v[d[0], b:b + 1], mst, d[0], r) == 1


def test_seeded_masks_bits_and_independence():
    """fill_masks_seeded: bit 16 of word (u & 3) of Philox((u >> 2, position, 2 dec + layer, "ragg"), seed); an utterance's flags
    do not depend on its row, the batch or npos, and differ from the padded path's "taco" streams and from a swapped counter"""
    seed = 0x123456789ABCDEF0
    m = ko.seeded_masks(seed, 7, 12, 1)
    o = ko.philox4x32(5 >> 2, 3, 2 * 1 + 1, ko.SEEDED_TAG, seed & 0xFFFFFFFF, seed >> 32)
    assert m[1, 3, 5] == (int(o[5 & 3]) >> 16) & 1
    seeds = [7, seed, 0]
    for dec in (0, 1):
        lay = ko.fill_masks_seeded(seeds, 9, 16, dec)
        wide = ko.fill_masks_seeded([3] + seeds, 11, 16, dec)
        for b, s in enumerate(seeds):
            own = ko.seeded_masks(s, 9, 16, dec)
            got = lay[:, b] if dec == 0 else lay[:, :, b].transpose(1, 0, 2)
            got_w = wide[:, b + 1, :9] if dec == 0 else wide[:9, :, b + 1].transpose(1, 0, 2)
            assert np.array_equal(got, own) and np.array_equal(got_w, own)
    l, pos, u = np.meshgrid(np.arange(2), np.arange(9), np.arange(16), indexing="ij")
    sw = ko.philox4x32(pos >> 2, u, l, ko.SEEDED_TAG, 7, 0)
    swapped = ((np.choose(u & 3, sw) >> np.uint32(16)) & np.uint32(1)).astype(np.uint8)
    assert not np.array_equal(swapped, ko.seeded_masks(7, 9, 16, 0))
    assert 0.4 < ko.seeded_masks(7, 64, 256, 0).mean() < 0.6


def test_im2col_rows_is_each_utterance_alone():
    """im2col with per-sequence lengths @ the tap weights = torch's zero-padded Conv1d of each utterance alone; the padded
    batch's im2col (taps reading the rows past the end) is rejected"""
    import tc_split_oracle as so

    g = _g(12)
    T, Ci, Co, k = 9, 6, 5, 4
    lens = [9, 1, 5, 2]
    M = T * 3 + 2  # a last, partial sequence of 2 rows
    x = _f32(g.standard_normal((M, Ci)))
    W = _f32(g.standard_normal((Co, Ci, k)))
    shifts = [j - k // 2 for j in range(k)]
    A = so.im2col_rows([x] * k, shifts, Ci, M, T, lens)
    Wc = np.concatenate([W[:, :, j] for j in range(k)], 1)
    got = np.asarray(A, np.float64) @ np.asarray(Wc, np.float64).T
    for j, n in enumerate(lens):
        r0 = j * T
        xc = _t(x[r0:r0 + n]).T[None]
        ref = F.conv1d(F.pad(xc, (k // 2, k - 1 - k // 2)), _t(W))[0].T.numpy()
        bound = np.abs(np.asarray(A[r0:r0 + n], np.float64)) @ np.abs(np.asarray(Wc, np.float64)).T * ko.gamma(Ci * k)
        _accept("im2col rows", ref, got[r0:r0 + n], bound + 1e-300)
        assert np.isnan(A[r0 + n:(j + 1) * T]).all()
    padded = np.asarray(so.im2col([x] * k, shifts, Ci, M, T), np.float64) @ np.asarray(Wc, np.float64).T
    _reject("padded im2col", padded[T:T + 1], got[T:T + 1], np.abs(got[T:T + 1]) * 1e-6)


def test_gru_reverse_rows_is_each_row_alone():
    """the backward GRU of a ragged batch = torch's GRU run over each row's own steps reversed, from h = 0"""
    import tc_split_oracle as so

    g = _g(13)
    M, T, H, Ki = 4, 7, 8, 5
    lens = [7, 1, 2, 4]
    x = _f32(g.standard_normal((M, T, Ki)))
    gru = torch.nn.GRU(Ki, H, batch_first=True)
    with torch.no_grad():
        for p in gru.parameters():
            p.copy_(_t(_f32(g.standard_normal(tuple(p.shape)) * 0.5)))
    gi = F.linear(_t(x), gru.weight_ih_l0, gru.bias_ih_l0).detach().numpy()
    ref = so.gru_reverse_rows(gi, gru.weight_hh_l0.detach().numpy(), gru.bias_hh_l0.detach().numpy(), lens)
    for m, n in enumerate(lens):
        with torch.no_grad():
            y, _ = gru(_t(x[m:m + 1, :n]).flip(1))
        _accept("gru reverse rows", y.flip(1)[0].numpy(), ref[m, :n], 1e-5 * (1 + np.abs(ref[m, :n])))
        assert not ref[m, n:].any()
    padded, _ = gru(_t(x[1:2]).flip(1))
    _reject("backward GRU from the padded end", padded.flip(1)[0, :1].detach().numpy(), ref[1, :1], 1e-5 * np.ones((1, H)))


def test_reduce_partials():
    """L2(mean of the partials) per utterance: the bound accepts a float32 numpy evaluation and rejects the unnormalised mean"""
    import encoder_oracle as eo

    g = _g(14)
    E = 100
    counts = [1, 2, 600, 3]
    off = np.concatenate([[0], np.cumsum(counts)])
    p = _f32(np.abs(g.standard_normal((off[-1], E))))
    p /= np.linalg.norm(p, axis=1, keepdims=True)
    ref, bound = eo.reduce_partials(p, off)
    for u in range(len(counts)):
        raw = np.mean(p[off[u]:off[u + 1]], axis=0, dtype=np.float32)
        _accept("reduce partials", raw / np.linalg.norm(raw, 2), ref[u:u + 1], bound[u:u + 1])
    raw = np.mean(p[off[2]:off[3]], axis=0)
    _reject("mean without the norm", raw[None], ref[2:3], bound[2:3])
