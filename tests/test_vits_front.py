"""The FP32 front end of VITS (everything in csrc/vits.cu before the decoder) launch by launch and stage by stage, against
float64 references at the lengths real sentences reach: up to the 1024-token limit and thousands of frames.

Single-kernel stages (conv1d_kernel, layernorm_kernel, rel_attn_kernel) are held to per-element bounds derived from their
roundings: u = 2^-24 per float32 operation, and a float32 sum of n terms errs by at most n u sum|terms|.  Composite stages
(an encoder layer, the whole text encoder, logw, a coupling layer, the whole flow) are held to 1e-5 of each row's largest
valid magnitude.  Rows past each length hold large garbage and outputs start as NaN, so a read past a length or an unwritten
output shows.  Three configurations: the full SDP model, "odd" (widths that are not tile multiples, K = 7, the 256-wide
DurationPredictor) and "wide" (one 256-wide head)."""
from __future__ import annotations

import ctypes as C
import math
import sys
from pathlib import Path

import numpy as np
import pytest
import torch
import torch.nn.functional as F

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "synth_weights"))
sys.path.insert(0, str(ROOT / "oracle"))
import ref_init as ri  # noqa: E402
import vits_oracle as vo  # noqa: E402

from mockingbird_b200 import _lib  # noqa: E402
from mockingbird_b200.synthesizer.models.vits import Vits  # noqa: E402

pytestmark = pytest.mark.gpu
U = 2.0 ** -24
GARBAGE = 1e3
COMPOSITE = 1e-5
MB_ERR_INVALID = 1
CFGS = {
    "full": ri.VITS_CONFIG,
    # Cin 9 (coupling pre) and 40, Cout 40, K = 7, head width 8, DurationPredictor(24, 256)
    "odd": dict(ri.VITS_TOY, hidden_channels=24, n_heads=3, filter_channels=40, kernel_size=7, inter_channels=18, use_sdp=False),
    "wide": dict(ri.VITS_CONFIG, hidden_channels=256, n_heads=1),  # head width kMaxHead = 256
}
_models = {}


def model(name):
    if name not in _models:
        cfg = CFGS[name]
        sd = ri.vits_state_dict(cfg, 21)
        m = Vits(**cfg)
        m.load_state_dict(sd)
        m.cuda()
        m.remove_weight_norm()
        _models[name] = (m, cfg, sd)
    return _models[name]


def debug(m, kind, B, T, **fields):
    """one mb_vits_debug call; tensors are passed by pointer, everything else as the field's value.  Returns the status."""
    s = _lib.VitsDebugSpec()
    s.kind, s.batch, s.frames = _lib.MB_VITS_DBG[kind], B, T
    for k, v in fields.items():
        if v is not None:
            setattr(s, k, v.data_ptr() if torch.is_tensor(v) else v)
    L = _lib.lib()
    ws = torch.empty(max(1, int(L.mb_vits_debug_workspace_bytes(m._handle, C.byref(s)))), dtype=torch.uint8, device="cuda")
    rc = L.mb_vits_debug(m._handle, C.byref(s), C.c_void_p(ws.data_ptr()), ws.numel(),
                         C.c_void_p(torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    return rc


def ragged(gen, B, Cc, T, lens, scale=1.0):
    """[B, C, T] float32: N(0, scale) up to each length, uniform +-GARBAGE after it"""
    x = (torch.rand(B, Cc, T, generator=gen, dtype=torch.float64) * 2 - 1) * GARBAGE
    for b, L in enumerate(lens):
        x[b, :, :L] = torch.randn(Cc, L, generator=gen, dtype=torch.float64) * scale
    return x.float()


def lens_of(T, B=3):
    return [T, T // 2 + 1, 1][:B]


def mask(lens, T):
    return vo.mask_of(torch.tensor(lens), T)  # [B, 1, T] float64


def nan(*shape):
    return torch.full(shape, float("nan"), device="cuda")


def worst(got, ref, bound):
    """max err / bound; fails on NaN"""
    got = got.detach().cpu().double()
    assert not torch.isnan(got).any()
    return float(((got - ref).abs() / (bound + 1e-30)).max())


def row_rel(got, ref, lens):
    """max over rows of max |err| / max |ref| over the row's valid frames (the last axis)"""
    got = got.detach().cpu().double()
    r = 0.0
    for b, L in enumerate(lens):
        g, e = got[b, ..., :L], ref[b, ..., :L]
        assert not torch.isnan(g).any()
        r = max(r, float((g - e).abs().max() / e.abs().max().clamp_min(1e-30)))
    return r


def padded_zero(got, lens):
    got = got.detach().cpu()
    return all(bool((got[b, ..., L:] == 0).all()) for b, L in enumerate(lens))


# ---- conv1d_kernel -----------------------------------------------------------------------------------------------------
CONV_RAN = {k: set() for k in ("K", "dil", "cin", "cout", "T", "mode", "flags")}
# name: cin, cout, K, dil, T, mode (0 store, 1 acc, 2 sub), relu, in_mask, out_mask, bbias
CONV_CASES = {
    "enc_1x1_wide": (1024, 768, 1, 1, 1000, 0, 0, 0, 1, 0),
    "ffn_k3": (17, 33, 3, 1, 65, 1, 1, 1, 1, 1),
    "k5_d2": (16, 32, 5, 2, 64, 2, 0, 1, 0, 0),
    "odd_ffn_1": (24, 40, 7, 1, 63, 0, 1, 1, 0, 0),
    "odd_ffn_2_k7_d2": (40, 24, 7, 2, 1000, 0, 0, 1, 1, 0),
    "halo_14": (192, 29, 3, 7, 129, 1, 1, 0, 1, 1),
    "t1": (1, 1, 5, 3, 1, 0, 1, 1, 1, 1),
    "dp_k3_d3": (256, 256, 3, 3, 300, 2, 1, 1, 1, 1),
    "cin9_k7": (9, 33, 7, 1, 65, 1, 0, 0, 0, 1),
    "cin1024_k3": (1024, 32, 3, 1, 64, 0, 1, 1, 1, 0),
}


def conv_reference(x, w, bias, bb, y0, lens, K, dil, pad, mode, relu, in_mask, out_mask):
    """float64 value and derived bound of one conv1d_kernel launch; x [B, cin, T] (already the slice read), y0 the output
    slice before the launch"""
    B, cin, T = x.shape
    halo = (K - 1) * dil
    m = mask(lens, T)
    xin = x.double() * m if in_mask else x.double()
    xp = torch.zeros(B, cin, pad + T + halo, dtype=torch.float64)
    xp[..., pad:pad + T] = xin
    wd = w.double()
    v = F.conv1d(xp, wd, dilation=dil)[..., :T]
    mag = F.conv1d(xp.abs(), wd.abs(), dilation=dil)[..., :T]
    if bias is not None:
        v, mag = v + bias.double()[None, :, None], mag + bias.double().abs()[None, :, None]
    if bb is not None:
        v, mag = v + bb.double()[:, :, None], mag + bb.double().abs()[:, :, None]
    if relu:
        v = torch.relu(v)
    if mode == 1:
        v = y0.double() + v
    elif mode == 2:
        v = y0.double() - v
    # the cin K products and two bias adds in float32, then one rounding of the epilogue's add
    bound = (cin * K + 2) * U * mag * 1.01 + (U * v.abs() if mode else 0)
    if out_mask:
        v, bound = v * m, bound * m
    return v, bound


def run_conv(m, gen, cin, cout, K, dil, T, mode, relu, in_mask, out_mask, bbias, pad=None, lens=None, x_ch=None, y_ch=None):
    """one CONV launch reading channels [x_off, x_off + cin) of a [B, xC, T] buffer and writing channels [y_off, y_off +
    cout) of a [B, yC, T] buffer, with x garbage past each length; returns (got slice, reference, bound, lengths)"""
    B = 3
    lens = lens or lens_of(T)
    pad = (K - 1) * dil // 2 if pad is None else pad
    xC, x_off = x_ch or (cin, 0)
    yC, y_off = y_ch or (cout, 0)
    x = ragged(gen, B, xC, T, lens)
    w = torch.randn(cout, cin, K, generator=gen) / math.sqrt(cin * K)
    bias = torch.randn(cout, generator=gen) * 0.1
    bbs = cout + 3
    bb = torch.randn(B, bbs, generator=gen) * 0.1 if bbias else None
    y = torch.full((B, yC, T), float("nan"))
    if mode:
        y[:, y_off:y_off + cout] = torch.randn(B, cout, T, generator=gen)
    y0 = y[:, y_off:y_off + cout].clone()
    yd = y.cuda()
    xd, wd, bd = x.cuda(), w.cuda(), bias.cuda()
    bbd = bb.cuda() if bbias else None
    args = dict(lengths=torch.tensor(lens, dtype=torch.int32).cuda(), x=xd[:, x_off:], w=wd, bias=bd, bbias=bbd, bbs=bbs,
                y=yd[:, y_off:], xbs=xC * T, ybs=yC * T, cin=cin, cout=cout, k=K, dil=dil, pad=pad, in_mask=in_mask,
                out_mask=out_mask, relu=relu, mode=mode)
    # x=xd[:, x_off:] is a view: its data_ptr is the slice's first element, the batch stride comes from xbs
    assert debug(m, "conv", B, T, **args) == 0
    ref, bound = conv_reference(x[:, x_off:x_off + cin], w, bias, bb[:, :cout] if bbias else None, y0, lens, K, dil, pad, mode,
                                relu, in_mask, out_mask)
    for k, v in (("K", K), ("dil", dil), ("cin", cin), ("cout", cout), ("T", T), ("mode", mode)):
        CONV_RAN[k].add(v)
    CONV_RAN["flags"].update(f for f, on in (("relu", relu), ("in_mask", in_mask), ("out_mask", out_mask), ("bbias", bbias)) if on)
    got = yd.cpu()
    # channels outside the written slice keep their NaN
    others = torch.cat([got[:, :y_off], got[:, y_off + cout:]], 1)
    assert torch.isnan(others).all()
    return got[:, y_off:y_off + cout], ref, bound, lens


@pytest.mark.parametrize("case", list(CONV_CASES))
def test_conv(case):
    m, _, _ = model("odd")
    cin, cout, K, dil, T, mode, relu, in_mask, out_mask, bbias = CONV_CASES[case]
    got, ref, bound, lens = run_conv(m, torch.Generator().manual_seed(len(case) * 7 + cin), cin, cout, K, dil, T, mode, relu,
                                     in_mask, out_mask, bbias)
    r = worst(got, ref, bound)
    print(case, "worst err / bound", r)
    assert r <= 1, (case, r)
    if out_mask:
        assert padded_zero(got, lens)


def test_conv_strided_slices():
    """ConvFlow pre reads one channel of z [B, 2, T] (x batch stride 2T, Cin 1); the coupling post subtracts into the x1
    half of z [B, inter, T] (y batch stride inter T); emo_proj is a T = 1 call over [B, 1024] rows"""
    m, _, _ = model("odd")
    gen = torch.Generator().manual_seed(11)
    for name, kw in (("convflow_pre", dict(cin=1, cout=192, K=1, dil=1, T=1000, mode=0, relu=0, in_mask=0, out_mask=0, bbias=0,
                                           x_ch=(2, 1))),
                     ("coupling_post", dict(cin=24, cout=9, K=1, dil=1, T=65, mode=2, relu=0, in_mask=1, out_mask=1, bbias=0,
                                            y_ch=(18, 9))),
                     ("emo_proj", dict(cin=1024, cout=192, K=1, dil=1, T=1, mode=0, relu=0, in_mask=0, out_mask=0, bbias=0))):
        got, ref, bound, lens = run_conv(m, gen, **kw)
        r = worst(got, ref, bound)
        print(name, "worst err / bound", r)
        assert r <= 1, (name, r)
        CONV_RAN["flags"].add(name)


@pytest.mark.parametrize("K,dil", [(3, 8), (9, 1), (7, 3), (5, 4)])
def test_conv_refuses_what_the_tile_cannot_hold(K, dil):
    """K > 7 or a halo (K - 1) dil > 14 (the shared-memory row width) is refused before any launch"""
    m, _, _ = model("odd")
    T, cin, cout = 65, 4, 4
    x, w = torch.randn(1, cin, T).cuda(), torch.randn(cout, cin, K).cuda()
    y = nan(1, cout, T)
    rc = debug(m, "conv", 1, T, x=x, w=w, y=y, xbs=cin * T, ybs=cout * T, cin=cin, cout=cout, k=K, dil=dil, pad=0)
    assert rc == MB_ERR_INVALID and b"unsupported" in _lib.lib().mb_last_error()
    assert torch.isnan(y).all()
    CONV_RAN["flags"].add("refused")


def test_conv_bounds_are_sharp():
    """the conv bound rejects a reference whose mask is one frame off, one with a tap shifted, one with a channel's bias
    dropped"""
    m, _, _ = model("odd")
    gen = torch.Generator().manual_seed(5)
    cin, cout, K, dil, T = 24, 40, 7, 1, 129
    lens = [129, 70, 1]
    x = ragged(gen, 3, cin, T, lens)
    w = torch.randn(cout, cin, K, generator=gen) / math.sqrt(cin * K)
    bias = torch.randn(cout, generator=gen) * 0.1
    y = nan(3, cout, T)
    assert debug(m, "conv", 3, T, lengths=torch.tensor(lens, dtype=torch.int32).cuda(), x=x.cuda(), w=w.cuda(), bias=bias.cuda(),
                 y=y, xbs=cin * T, ybs=cout * T, cin=cin, cout=cout, k=K, dil=dil, pad=3, in_mask=1, out_mask=1) == 0
    y0 = torch.zeros(3, cout, T)

    def ref(lens_r=lens, w_r=w, b_r=bias):
        return conv_reference(x, w_r, b_r, None, y0, lens_r, K, dil, 3, 0, 0, 1, 1)

    assert worst(y, *ref()) <= 1
    off_by_one = [lens[0], lens[1] + 1, lens[2]]
    shifted = w.clone()
    shifted[:, :, 2], shifted[:, :, 3] = w[:, :, 3], w[:, :, 2]
    dropped = bias.clone()
    dropped[17] = 0
    for name, r in (("mask", ref(lens_r=off_by_one)), ("tap", ref(w_r=shifted)), ("bias", ref(b_r=dropped))):
        assert worst(y, *r) > 1, name


# ---- layernorm_kernel --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("Cc", [16, 24, 192, 256])
@pytest.mark.parametrize("variant", ["plain", "b2_mask", "gelu_res_mask"])
def test_layernorm(Cc, variant):
    m, _, _ = model("odd")
    gen = torch.Generator().manual_seed(Cc)
    T = 300
    lens = lens_of(T)
    a = ragged(gen, 3, Cc, T, lens, scale=3.0)
    b2 = torch.randn(3, Cc, T, generator=gen) if variant != "plain" else None
    res = torch.randn(3, Cc, T, generator=gen) if variant == "gelu_res_mask" else None
    gelu = variant == "gelu_res_mask"
    masked = variant != "plain"
    gamma = 1 + 0.1 * torch.randn(Cc, generator=gen)
    beta = 0.1 * torch.randn(Cc, generator=gen)
    y = nan(3, Cc, T)
    assert debug(m, "layernorm", 3, T, lengths=torch.tensor(lens, dtype=torch.int32).cuda() if masked else None, x=a.cuda(),
                 x2=b2.cuda() if b2 is not None else None, res=res.cuda() if res is not None else None, w=gamma.cuda(),
                 bias=beta.cuda(), y=y, cin=Cc, gelu=int(gelu)) == 0
    xs = (a + b2 if b2 is not None else a).double()  # the kernel's first operation, a + b2 rounded to float32
    mu = xs.mean(1, keepdim=True)
    xh = (xs - mu) / torch.sqrt(((xs - mu) ** 2).mean(1, keepdim=True) + 1e-5)
    g, be = gamma.double()[None, :, None], beta.double()[None, :, None]
    pre = xh * g + be
    ref = vo.gelu(pre) if gelu else pre
    if res is not None:
        ref = res.double() + ref
    # test_wav2emo_kernels.test_ln_act's bound (mean and variance C-term sums, rstd / normalise / affine roundings, GELU
    # 1.13-Lipschitz) plus the residual add's rounding
    bound = 1.2 * (2 * Cc * U * g.abs() * (xh.abs() + 1) + 8 * U * (pre.abs() + be.abs())) + 2 * U * ref.abs()
    if masked:
        msk = mask(lens, T)
        ref, bound = ref * msk, bound * msk
        assert padded_zero(y, lens)
    r = worst(y, ref, bound)
    print("layernorm", Cc, variant, "worst err / bound", r)
    assert r <= 1, r


# ---- rel_attn_kernel ---------------------------------------------------------------------------------------------------
def attention_reference(q, k, v, erk, erv, L, nh):
    """one row in float64: (out [H, T], per-element bound [H, T]).  The kernel rounds q / sqrt(dk), sums dk products per
    score and per relative term, adds them; a score error ds moves each softmax weight by at most 2 ds relative; the max /
    exp / sum (per-thread runs of ceil(T / 128) then a 7-level tree) and the division add a few u more, the exponent's
    rounding at most u (log T + 2) of the weighted sum; P V and the 9 relative terms are sums of T + 9 terms."""
    H, T = q.shape
    dk = H // nh
    W = vo.WINDOW
    qs = q.double().view(nh, dk, T).transpose(1, 2) / math.sqrt(dk)
    kk, vv = (a.double().view(nh, dk, T).transpose(1, 2) for a in (k, v))
    ek, ev = erk.double()[0], erv.double()[0]
    S, Sa = qs @ kk.transpose(1, 2), qs.abs() @ kk.abs().transpose(1, 2)
    rl, rla = qs @ ek.T, qs.abs() @ ek.abs().T
    t = torch.arange(T)
    band = [(r, t[(t + r >= 0) & (t + r < T)]) for r in range(-W, W + 1)]
    for r, tt in band:
        S[:, tt, tt + r] += rl[:, tt, r + W]
        Sa[:, tt, tt + r] += rla[:, tt, r + W]
    valid = (t[:, None] < L) & (t[None, :] < L)
    ds = torch.where(valid, (dk + 2) * U * Sa + 2 * U * S.abs(), torch.zeros(())).amax(-1)  # [nh, T]
    S = torch.where(valid, S, torch.full_like(S, -1e4))
    p = torch.softmax(S, -1)
    out = p @ vv
    for r, tt in band:
        out[:, tt] += p[:, tt, tt + r, None] * ev[r + W]
    vmax = torch.where((t < L)[None, :, None], vv[:, :L].abs().amax(1, keepdim=True), vv.abs().amax(1, keepdim=True))
    mag = vmax + ev.abs().amax(0)
    nsum = math.ceil(T / 128) + 7
    bound = ((2 * ds + (nsum + math.log(T) + 12) * U)[..., None] + (T + 12) * U) * mag * 1.01
    return out.transpose(1, 2).reshape(H, T), bound.transpose(1, 2).reshape(H, T)


@pytest.mark.parametrize("name", ["odd", "full", "wide"])
@pytest.mark.parametrize("T", [127, 128, 129, 300, 1024])
def test_attention(name, T):
    m, cfg, sd = model(name)
    H, nh = cfg["hidden_channels"], cfg["n_heads"]
    gen = torch.Generator().manual_seed(T)
    lens = lens_of(T)
    q, k, v = (ragged(gen, 3, H, T, lens) for _ in range(3))
    layer = cfg["n_layers"] - 1
    y = nan(3, H, T)
    assert debug(m, "attn", 3, T, lengths=torch.tensor(lens, dtype=torch.int32).cuda(), x=q.cuda(), x2=k.cuda(), x3=v.cuda(), y=y,
                 index=layer) == 0
    a = f"enc_p.encoder.attn_layers.{layer}"
    r = 0.0
    for b, L in enumerate(lens):
        ref, bound = attention_reference(q[b], k[b], v[b], sd[a + ".emb_rel_k"], sd[a + ".emb_rel_v"], L, nh)
        r = max(r, worst(y[b], ref, bound))
    print("attention", name, T, "dk", H // nh, "worst err / bound", r)
    assert r <= 1, r


def test_attention_bound_is_sharp():
    """the attention bound rejects a reference whose key mask is one frame longer"""
    m, cfg, sd = model("full")
    H, nh, T, L = cfg["hidden_channels"], cfg["n_heads"], 129, 70
    gen = torch.Generator().manual_seed(3)
    q, k, v = (ragged(gen, 1, H, T, [L], scale=2.0) for _ in range(3))
    k[:, :, L:] = 0  # an off-by-one key must not be hidden by garbage scores saturating the softmax
    y = nan(1, H, T)
    assert debug(m, "attn", 1, T, lengths=torch.tensor([L], dtype=torch.int32).cuda(), x=q.cuda(), x2=k.cuda(), x3=v.cuda(), y=y) == 0
    a = "enc_p.encoder.attn_layers.0"
    assert worst(y[0], *attention_reference(q[0], k[0], v[0], sd[a + ".emb_rel_k"], sd[a + ".emb_rel_v"], L, nh)) <= 1
    ref, _ = attention_reference(q[0], k[0], v[0], sd[a + ".emb_rel_k"], sd[a + ".emb_rel_v"], L + 1, nh)
    _, bound = attention_reference(q[0], k[0], v[0], sd[a + ".emb_rel_k"], sd[a + ".emb_rel_v"], L, nh)
    assert worst(y[0, :, :L], ref[:, :L], bound[:, :L]) > 1


# ---- encoder layers, the whole text encoder ----------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["full", "odd", "wide"])
def test_encoder_layer(name):
    """ENC_LAYER for layer 0 and the last layer on inputs with +-1e3 garbage past each length: the valid outputs do not
    depend on the garbage, the last layer's padded outputs are exactly 0"""
    m, cfg, sd = model(name)
    H, T = cfg["hidden_channels"], 300
    lens = lens_of(T)
    gen = torch.Generator().manual_seed(2)
    x = ragged(gen, 3, H, T, lens)
    x2 = torch.where(mask(lens, T).float() > 0, x, -ragged(gen, 3, H, T, [0, 0, 0]))  # other garbage
    ld = torch.tensor(lens, dtype=torch.int32).cuda()
    for l in (0, cfg["n_layers"] - 1):
        last = l == cfg["n_layers"] - 1
        y, y2 = nan(3, H, T), nan(3, H, T)
        assert debug(m, "enc_layer", 3, T, lengths=ld, x=x.cuda(), y=y, index=l) == 0
        assert debug(m, "enc_layer", 3, T, lengths=ld, x=x2.cuda(), y=y2, index=l) == 0
        for b, L in enumerate(lens):
            assert torch.equal(y[b, :, :L], y2[b, :, :L]), (l, b)
        ref = vo.text_encoder_layer(sd, cfg, l, x.double(), torch.tensor(lens), last)
        r = row_rel(y, ref, lens)
        print("encoder layer", name, l, "worst row rel", r)
        assert r <= COMPOSITE, (l, r)
        if last:
            assert padded_zero(y, lens)


def call_durations(m, x, lens, sid, emo, noise, nsw, ls):
    """mb_vits_durations with outputs pre-filled with NaN / -7"""
    B, T = x.shape
    I = m.inter_channels
    m_p, logs_p = nan(B, I, T), nan(B, I, T)
    w_ceil = torch.full((B, T), -7, dtype=torch.int32, device="cuda")
    y_len = torch.full((B,), -7, dtype=torch.int32, device="cuda")
    L = _lib.lib()
    need = int(L.mb_vits_durations_workspace_bytes(m._handle, B, T))
    ws = torch.empty(max(need, 1), dtype=torch.uint8, device="cuda")
    p = lambda t: C.c_void_p(t.data_ptr()) if t is not None else None  # noqa: E731
    rc = L.mb_vits_durations(m._handle, p(x), p(lens), B, T, p(sid), p(emo), p(noise), float(nsw), float(ls), p(m_p), p(logs_p),
                             p(w_ceil), p(y_len), p(ws), ws.numel(), C.c_void_p(torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    return rc, m_p, logs_p, w_ceil, y_len


def token_batch(cfg, lens, T, seed):
    """random valid ids everywhere (past each length too), emo, sid, SDP noise with garbage past each length"""
    gen = torch.Generator().manual_seed(seed)
    B = len(lens)
    x = torch.randint(0, cfg["n_vocab"], (B, T), generator=gen, dtype=torch.int32)
    emo = torch.randn(B, 1024, generator=gen)
    sid = torch.arange(B, dtype=torch.int32) % max(cfg["n_speakers"], 1)
    noise = ragged(gen, B, 2, T, lens)
    return x, emo, sid, noise


@pytest.mark.parametrize("name,T,lens", [("full", 65, [65, 64, 33, 1]), ("full", 1024, [1024, 700, 129, 1]),
                                         ("odd", 1024, [1024, 700, 129, 1])])
def test_text_encoder_and_durations(name, T, lens):
    """m_p / logs_p of mb_vits_durations against the float64 text encoder, padded positions exactly 0; w_ceil against the
    float64 ceil except within 1e-4 of an integer; y_len = max(1, sum w_ceil)"""
    m, cfg, sd = model(name)
    x, emo, sid, noise = token_batch(cfg, lens, T, T)
    nsw, ls = 0.8, 1.13
    rc, m_p, logs_p, w_ceil, y_len = call_durations(m, x.cuda(), torch.tensor(lens, dtype=torch.int32).cuda(), sid.cuda(),
                                                    emo.cuda(), noise.cuda(), nsw, ls)
    assert rc == 0
    lt = torch.tensor(lens)
    with torch.no_grad():
        h, rm, rl = vo.text_encoder(sd, cfg, x, lt, emo)
        g = vo._d(sd["emb_g.weight"])[sid.long()] if cfg["n_speakers"] > 1 else None
        w = vo.durations(sd, cfg, h, lt, g, noise.double(), nsw, ls)[:, 0]
    r = max(row_rel(m_p, rm, lens), row_rel(logs_p, rl, lens))
    print("text encoder", name, T, "worst row rel", r)
    assert r <= COMPOSITE, r
    assert padded_zero(m_p, lens) and padded_zero(logs_p, lens)
    wc = w_ceil.cpu()
    assert padded_zero(wc, lens)
    valid = mask(lens, T)[:, 0] > 0
    near = (w - torch.round(w)).abs() < 1e-4
    keep = valid & ~near
    print("durations", name, T, "tokens excluded within 1e-4 of an integer:", int((valid & near).sum()), "of", int(valid.sum()))
    assert torch.equal(wc[keep].long(), torch.ceil(w)[keep].long())
    assert torch.equal(y_len.cpu().long(), wc.long().sum(1).clamp_min(1))


def test_the_token_limit():
    """1024 tokens run (test_text_encoder_and_durations); 1025 are refused by mb_vits_durations, ATTN, ENC_LAYER and
    Vits.infer before anything is launched"""
    m, cfg, _ = model("full")
    assert int(_lib.lib().mb_vits_max_tokens()) == 1024
    T = 1025
    x, emo, sid, noise = token_batch(cfg, [T], T, 1)
    rc, m_p, *_ = call_durations(m, x.cuda(), torch.tensor([T], dtype=torch.int32).cuda(), sid.cuda(), emo.cuda(), noise.cuda(), 1,
                                 1)
    assert rc == MB_ERR_INVALID and torch.isnan(m_p).all()
    q = torch.zeros(1, cfg["hidden_channels"], T, device="cuda")
    y = nan(1, cfg["hidden_channels"], T)
    ld = torch.tensor([T], dtype=torch.int32).cuda()
    assert debug(m, "attn", 1, T, lengths=ld, x=q, x2=q, x3=q, y=y) == MB_ERR_INVALID
    assert debug(m, "enc_layer", 1, T, lengths=ld, x=q, y=y) == MB_ERR_INVALID
    assert torch.isnan(y).all()
    with pytest.raises(ValueError, match="1025 tokens"):
        m.infer(x.long(), [T], sid=sid.long(), emo=emo)


# ---- duration predictors -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["full", "odd"])  # the stochastic predictor, the DurationPredictor
@pytest.mark.parametrize("with_g", [True, False])
def test_logw(name, with_g):
    """LOGW against the float64 logw; the kernel's w_ceil is ceil(float32(exp(logw)) * length_scale) except within 4 ulp of
    an integer and y_len = max(1, sum); garbage in the SDP noise past each length changes nothing"""
    m, cfg, sd = model(name)
    H, T = cfg["hidden_channels"], 300
    lens = [300, 129, 1]
    B = len(lens)
    gen = torch.Generator().manual_seed(8)
    x = (torch.randn(B, H, T, generator=gen) * mask(lens, T).float()).contiguous()  # an encoder output: masked
    noise = ragged(gen, B, 2, T, lens)
    noise2 = torch.where(mask(lens, T).float() > 0, noise, ragged(gen, B, 2, T, [0] * B))
    sid = torch.tensor([2, 0, 1], dtype=torch.int32)
    nsw, ls = 0.8, 1.37
    outs = []
    for nz in (noise, noise2):
        y = nan(B, 1, T)
        y2 = torch.full((B * T + B,), -7, dtype=torch.int32, device="cuda")
        assert debug(m, "logw", B, T, lengths=torch.tensor(lens, dtype=torch.int32).cuda(), x=x.cuda(),
                     x2=sid.cuda() if with_g else None, x3=nz.cuda(), y=y, y2=y2, noise_scale_w=nsw, length_scale=ls) == 0
        outs.append((y.cpu(), y2.cpu()))
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])
    lw, ints = outs[0]
    g = vo._d(sd["emb_g.weight"])[sid.long()] if with_g else None
    ref = vo.logw(sd, cfg, x.double(), torch.tensor(lens), g, noise.double(), nsw)
    r = row_rel(lw, ref, lens)
    print("logw", name, "g" if with_g else "no g", "worst row rel", r)
    assert r <= COMPOSITE, r
    assert padded_zero(lw, lens)
    wc, yl = ints[:B * T].view(B, T), ints[B * T:]
    w32 = (np.exp(lw[:, 0].numpy().astype(np.float32)) * np.float32(ls)).astype(np.float32)
    near = np.abs(w32 - np.round(w32)) <= 4 * np.spacing(np.abs(w32))
    valid = (mask(lens, T)[:, 0] > 0).numpy()
    keep = valid & ~near
    assert np.array_equal(wc.numpy()[keep], np.ceil(w32)[keep].astype(np.int32))
    assert (wc.numpy()[~valid] == 0).all()
    assert torch.equal(yl.long(), wc.long().sum(1).clamp_min(1))
    w64 = torch.exp(ref[:, 0]) * ls
    near64 = (w64 - torch.round(w64)).abs() < 1e-4
    k64 = torch.from_numpy(valid) & ~near64
    print("logw", name, "tokens excluded from the float64 ceil:", int((torch.from_numpy(valid) & near64).sum()))
    assert torch.equal(wc[k64].long(), torch.ceil(w64)[k64].long())


# ---- the coupling flow -------------------------------------------------------------------------------------------------
def coupling_cases():
    for name in ("odd", "full"):
        for T in (1, 63, 64, 65, 1000, 4096):
            if name == "full" and T == 4096:  # the float64 reference of the full model at 4096 frames: two layers
                yield name, T, ((0, True), (3, False))
            else:
                yield name, T, tuple((f, g) for f in range(4) for g in (True, False))


@pytest.mark.parametrize("name,T,layers", list(coupling_cases()))
def test_coupling(name, T, layers):
    """COUPLING against the float64 coupling_reverse: x0 passes through bitwise (garbage included), x1 is within 1e-5 of
    each row's maximum and exactly 0 past each length"""
    m, cfg, sd = model(name)
    I, G = cfg["inter_channels"], cfg["gin_channels"]
    B = 2 if T == 4096 else 3
    lens = lens_of(T, B)
    gen = torch.Generator().manual_seed(T + I)
    z = ragged(gen, B, I, T, lens)
    gv = torch.randn(B, G, generator=gen)
    ld = torch.tensor(lens, dtype=torch.int32).cuda()
    r = 0.0
    for f, with_g in layers:
        y = nan(B, I, T)
        assert debug(m, "coupling", B, T, lengths=ld, x=z.cuda(), x2=gv.cuda() if with_g else None, y=y, index=f) == 0
        y = y.cpu()
        assert torch.equal(y[:, :I // 2], z[:, :I // 2])
        ref = vo.coupling_reverse(sd, f, z.double(), torch.tensor(lens), gv.double() if with_g else None)
        r = max(r, row_rel(y[:, I // 2:], ref[:, I // 2:], lens))
        assert padded_zero(y[:, I // 2:], lens)
    print("coupling", name, T, "worst row rel", r)
    assert r <= COMPOSITE, r


def decode_inputs(cfg, x_lens, Tx, seed, dur_max=16):
    gen = torch.Generator().manual_seed(seed)
    B, I = len(x_lens), cfg["inter_channels"]
    w_ceil = torch.randint(0, dur_max + 1, (B, Tx), generator=gen, dtype=torch.int32)
    m_p = torch.randn(B, I, Tx, generator=gen)
    logs_p = torch.randn(B, I, Tx, generator=gen) * 0.3
    sid = torch.arange(B, dtype=torch.int32) % cfg["n_speakers"]
    return w_ceil, m_p, logs_p, sid


def test_expansion_and_flow_at_length():
    """mb_vits_decode at about 2600 frames: attn, m_p_y, logs_p_y bitwise the float64 gather, z_p within a few ulp of m +
    eps exp(logs) noise_scale, z against the float64 flow_reverse of the kernel's z_p; the same with t_dec < T_y"""
    m, cfg, sd = model("full")
    Tx, x_lens = 320, [320, 251]
    w_ceil, m_p, logs_p, sid = decode_inputs(cfg, x_lens, Tx, 4)
    x_len = torch.tensor(x_lens, dtype=torch.int32)
    _, _, _, _, y_len = vo.expand(m_p.double(), logs_p.double(), w_ceil, x_len, torch.zeros(2, 1, 1, dtype=torch.float64), 0)
    Ty = int(y_len.max())
    assert Ty > 2400
    eps = torch.randn(2, cfg["inter_channels"], Ty, generator=torch.Generator().manual_seed(6))
    ns = 0.667
    attn_r, z_p_r, m_y_r, l_y_r, y_len = vo.expand(m_p.double(), logs_p.double(), w_ceil, x_len, eps.double(), ns)
    g = vo._d(sd["emb_g.weight"])[sid.long()]
    z_first = None
    for t_dec in (Ty, Ty - 333):
        with torch.cuda.device(m._device):
            _, attn, z_p, z, m_y, l_y = m._decode(m_p.cuda(), logs_p.cuda(), w_ceil.cuda(), x_len.cuda(), sid.cuda(), eps.cuda(), ns,
                                                  t_dec, False, True)
        assert torch.equal(attn.cpu().double(), attn_r)
        assert torch.equal(m_y.cpu().double(), m_y_r.float().double()) and torch.equal(l_y.cpu().double(), l_y_r.float().double())
        # expf (2 ulp), two products, the sum, and noise_scale rounded to float32
        zb = 8 * U * (m_y_r.abs() + (eps.double() * torch.exp(l_y_r) * ns).abs())
        assert worst(z_p, z_p_r, zb) <= 1
        if z_first is None:
            z_first = z.cpu()
            ref = vo.flow_reverse(sd, z_p.cpu().double(), y_len, g)
            r = row_rel(z, ref, y_len.tolist())
            print("flow", Ty, "frames, worst row rel", r)
            assert r <= COMPOSITE, r
        else:
            assert torch.equal(z.cpu(), z_first)


# ---- rows bitwise their B = 1 calls ------------------------------------------------------------------------------------
def test_durations_rows_bitwise_their_single_calls():
    m, cfg, _ = model("full")
    lens, T = [1024, 700, 129, 1], 1024
    x, emo, sid, noise = token_batch(cfg, lens, T, 9)
    batch = call_durations(m, x.cuda(), torch.tensor(lens, dtype=torch.int32).cuda(), sid.cuda(), emo.cuda(), noise.cuda(), 0.8, 1.0)
    assert batch[0] == 0
    for b, L in enumerate(lens):
        one = call_durations(m, x[b:b + 1, :L].contiguous().cuda(), torch.tensor([L], dtype=torch.int32).cuda(), sid[b:b + 1].cuda(),
                             emo[b:b + 1].cuda(), noise[b:b + 1, :, :L].contiguous().cuda(), 0.8, 1.0)
        assert one[0] == 0
        for got, alone in zip(batch[1:4], one[1:4]):
            assert torch.equal(got[b, ..., :L].cpu(), alone[0].cpu()), b
        assert int(batch[4][b]) == int(one[4][0])


def test_decode_rows_bitwise_their_single_calls():
    m, cfg, _ = model("full")
    x_lens, Tx = [300, 210, 37, 1], 300
    w_ceil, m_p, logs_p, sid = decode_inputs(cfg, x_lens, Tx, 12, dur_max=20)
    w_ceil[3, 0] = 5
    x_len = torch.tensor(x_lens, dtype=torch.int32)
    y_len = (w_ceil.long() * mask(x_lens, Tx)[:, 0].long()).sum(1).clamp_min(1).tolist()
    Ty = max(y_len)
    assert Ty > 2000
    eps = torch.randn(4, cfg["inter_channels"], Ty, generator=torch.Generator().manual_seed(13))
    with torch.cuda.device(m._device):
        wav, _, _, z, _, _ = m._decode(m_p.cuda(), logs_p.cuda(), w_ceil.cuda(), x_len.cuda(), sid.cuda(), eps.cuda(), 0.667, Ty, True,
                                       True)
        for b, (L, Y) in enumerate(zip(x_lens, y_len)):
            w1, _, _, z1, _, _ = m._decode(m_p[b:b + 1, :, :L].contiguous().cuda(), logs_p[b:b + 1, :, :L].contiguous().cuda(),
                                           w_ceil[b:b + 1, :L].contiguous().cuda(), x_len[b:b + 1].cuda(), sid[b:b + 1].cuda(),
                                           eps[b:b + 1, :, :Y].contiguous().cuda(), 0.667, Y, True, True)
            assert torch.equal(wav[b, :, :Y * m.hop].cpu(), w1[0].cpu()), b
            assert torch.equal(z[b, :, :Y].cpu(), z1[0].cpu()), b


def test_every_conv_variant_ran():
    """the conv tests above reached every listed branch"""
    assert CONV_RAN["K"] >= {1, 3, 5, 7} and CONV_RAN["dil"] >= {1, 2, 3, 7}
    assert CONV_RAN["cin"] >= {1, 9, 16, 17, 1024} and CONV_RAN["cout"] >= {1, 29, 32, 33, 768}
    assert CONV_RAN["T"] >= {1, 63, 64, 65, 1000} and CONV_RAN["mode"] >= {0, 1, 2}
    assert CONV_RAN["flags"] >= {"relu", "in_mask", "out_mask", "bbias", "convflow_pre", "coupling_post", "emo_proj", "refused"}
