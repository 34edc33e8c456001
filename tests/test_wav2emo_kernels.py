"""The emotion model's kernels one launch at a time (mb_emo_debug) against float64 references.  Each bound is derived from the
kernel's roundings: u = 2^-24 per float32 operation, a sum of n terms in float32 errs by at most n u sum|terms|, and the 3-term
fp16 split (hi hi + lo hi + hi lo) of a product errs by at most 3 2^-22 of |product| (the dropped lo lo term and the roundings
of the two halves).  Every launch mixes clip lengths (T = 1, T not a multiple of the 64-row tiles, 1500), fills the rows past
each clip with large non-zero values and the output with NaN, so a read past a clip or an unwritten row shows."""
from __future__ import annotations

import ctypes as C
import math
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "oracle"))

import wav2emo_oracle as wo  # noqa: E402

pytestmark = pytest.mark.gpu
U = 2.0 ** -24
SPLIT = 3 * 2.0 ** -22
KIND = dict(norm=0, conv0=1, ln_act=2, posconv=3, attn=4, mean=5, head=6)
LENS = [1, 70, 1500, 64, 129]  # frames: T = 1, not a tile multiple, 1500, one tile, two tiles + 1
S = 1500


def run(kind, lengths, x, out_shape, w=None, bias=None, gamma=None, beta=None, **kw):
    from mockingbird_b200 import _lib

    L = _lib.lib()
    dev = torch.device("cuda")
    keep = [torch.as_tensor(np.ascontiguousarray(a), dtype=torch.float32).to(dev) if a is not None else None
            for a in (x, w, bias, gamma, beta)]
    y = torch.full(out_shape, float("nan"), device=dev)
    lens = (C.c_int32 * len(lengths))(*lengths)
    p = lambda t: C.c_void_p(t.data_ptr()) if t is not None else None  # noqa: E731
    s = _lib.EmoDebugSpec(kind=KIND[kind], batch=len(lengths), lengths=lens, x=p(keep[0]), w=p(keep[1]), bias=p(keep[2]),
                          gamma=p(keep[3]), beta=p(keep[4]), y=p(y), **kw)
    need = int(L.mb_emo_debug_workspace_bytes(C.byref(s)))
    ws = torch.empty(need, dtype=torch.uint8, device=dev)
    _lib.check(L.mb_emo_debug(C.byref(s), C.c_void_p(ws.data_ptr()), need, C.c_void_p(torch.cuda.current_stream().cuda_stream)))
    return y.cpu().double().numpy()


def rows(rng, lengths, D, scale=1.0, garbage=1e3):
    """[B][S][D]: the clips' frames from N(0, scale), rows past each clip filled with `garbage`-sized values"""
    x = rng.uniform(-garbage, garbage, (len(lengths), S, D))
    for b, T in enumerate(lengths):
        x[b, :T] = rng.standard_normal((T, D)) * scale
    return x.astype(np.float32)


def check(got, ref, bound, lengths=None):
    assert not np.isnan(got).any()
    err = np.abs(got - ref)
    assert (err <= bound + 1e-30).all(), float((err / (bound + 1e-30)).max())
    if lengths is not None:
        for b, T in enumerate(lengths):
            assert (got[b, T:] == 0).all(), b


def test_norm_bitwise_numpy():
    rng = np.random.default_rng(0)
    clips = [(rng.standard_normal(n) * 0.3 + 0.01).astype(np.float32) for n in (400, 1001, 16000, 480000, 129)]
    got = run("norm", [c.size for c in clips], np.concatenate(clips), (sum(c.size for c in clips),))
    ref = np.concatenate([wo.normalize(c) for c in clips])
    assert np.array_equal(got.astype(np.float32).view(np.int32), ref.view(np.int32))


@pytest.mark.parametrize("bias", [True, False])
def test_conv0(bias):
    rng = np.random.default_rng(1)
    n = [400, 405, 2000, 640 * 5 + 5]
    k, s, D, Sx = 10, 5, 128, 700
    clips = [rng.standard_normal(m).astype(np.float32) for m in n]
    w = (rng.standard_normal((D, 1, k)) / math.sqrt(k)).astype(np.float32)
    b = (rng.standard_normal(D) * 0.1).astype(np.float32) if bias else None
    got = run("conv0", n, np.concatenate(clips), (len(n), Sx, D), w=w, bias=b, frames=Sx, dim=D, kernel=k, stride=s)
    T = [(m - k) // s + 1 for m in n]
    for i, c in enumerate(clips):
        ref = torch.nn.functional.conv1d(torch.from_numpy(c).double()[None, None], torch.from_numpy(w).double(),
                                         torch.from_numpy(b).double() if bias else None, stride=s)[0].T.numpy()
        fr = np.lib.stride_tricks.sliding_window_view(c.astype(np.float64), k)[::s][:T[i]]
        mag = np.abs(fr) @ np.abs(w[:, 0, :].astype(np.float64)).T + (np.abs(b) if bias else 0)
        check(got[i, :T[i]], ref, (k + 1) * U * mag)
        assert (got[i, T[i]:] == 0).all()


@pytest.mark.parametrize("act", [0, 3])
def test_ln_act(act):
    rng = np.random.default_rng(2)
    D = 512
    x = rows(rng, LENS, D, scale=3.0)
    g = (1 + 0.1 * rng.standard_normal(D)).astype(np.float32)
    be = (0.1 * rng.standard_normal(D)).astype(np.float32)
    got = run("ln_act", LENS, x, x.shape, gamma=g, beta=be, frames=S, dim=D, eps=1e-5, act=act)
    xd = x.astype(np.float64)
    mu = xd.mean(-1, keepdims=True)
    xh = (xd - mu) / np.sqrt(xd.var(-1, keepdims=True) + 1e-5)
    pre = xh * g + be
    ref = torch.nn.functional.gelu(torch.from_numpy(pre)).numpy() if act == 3 else pre
    # mean and variance: D-term sums (D u); rstd, normalise and affine: a few roundings more; GELU is 1.13-Lipschitz
    bound = 1.2 * (2 * D * U * np.abs(g) * (np.abs(xh) + 1) + 8 * U * (np.abs(pre) + np.abs(be)))
    for b, T in enumerate(LENS):
        check(got[b, :T], ref[b, :T], bound[b, :T])
        assert (got[b, T:] == 0).all()


@pytest.mark.parametrize("D,G,k", [(1024, 16, 128), (128, 1, 15), (256, 2, 16)])
def test_posconv(D, G, k):
    rng = np.random.default_rng(3)
    lens = [1, 70, 1500, 40, 129] if D == 1024 else [1, 30, 700, 64, 5]  # rows shorter than 64 included
    x = rows(rng, lens, D)
    cg = D // G
    w = (rng.standard_normal((D, cg, k)) / math.sqrt(cg * k)).astype(np.float32)
    bias = (0.05 * rng.standard_normal(D)).astype(np.float32)
    got = run("posconv", lens, x, x.shape, w=w, bias=bias, frames=S, dim=D, groups=G, kernel=k)
    wd = torch.from_numpy(w).double()
    for b, T in enumerate(lens):
        xb = torch.from_numpy(x[b, :T]).double().T[None]
        conv = torch.nn.functional.conv1d(xb, wd, torch.from_numpy(bias).double(), padding=k // 2, groups=G)[0, :, :T]
        mag = torch.nn.functional.conv1d(xb.abs(), wd.abs(), None, padding=k // 2, groups=G)[0, :, :T]
        ref = (xb[0] + torch.nn.functional.gelu(conv)).T.numpy()
        # the split product errs by SPLIT, the cg k-term FP32 sum by cg k u; GELU (1.13-Lipschitz) and the residual add
        bound = 1.2 * (SPLIT + cg * k * U) * mag.T.numpy() + 4 * U * np.abs(ref) + 1e-7
        check(got[b, :T], ref, bound)
        assert (got[b, T:] == 0).all(), b


def test_attention():
    rng = np.random.default_rng(4)
    H, D = 4, 256
    qkv = rows(rng, LENS, 3 * D)
    got = run("attn", LENS, qkv, (len(LENS), S, D), frames=S, dim=D, heads=H)
    for b, T in enumerate(LENS):
        q, kk, v = (torch.from_numpy(qkv[b, :T, i * D:(i + 1) * D]).double().reshape(T, H, 64).transpose(0, 1) for i in range(3))
        sc = q @ kk.transpose(1, 2) / 8
        ref = (torch.softmax(sc, -1) @ v).transpose(0, 1).reshape(T, D).numpy()
        # score error ds <= (SPLIT + 64 u) sum|q k| / 8, which moves each softmax weight by at most 2 max ds relative; P V then
        # adds SPLIT + T u of sum p |v|
        ds = ((SPLIT + 64 * U) * (q.abs() @ kk.abs().transpose(1, 2)) / 8).amax(-1)  # [H][T]
        vmax = v.abs().amax(1)  # [H][64]
        bound = ((2 * ds + 2 * U)[:, :, None] * vmax[:, None, :] * 1.01 + (SPLIT + (T + 64) * U) * vmax[:, None, :])
        check(got[b, :T], ref, bound.transpose(0, 1).reshape(T, D).numpy())
        assert (got[b, T:] == 0).all(), b


def test_mean_and_head():
    rng = np.random.default_rng(5)
    D, N = 1024, 3
    x = rows(rng, LENS, D)
    got = run("mean", LENS, x, (len(LENS), D), frames=S, dim=D)
    ref = np.stack([x[b, :T].astype(np.float64).mean(0) for b, T in enumerate(LENS)])
    mag = np.stack([np.abs(x[b, :T].astype(np.float64)).mean(0) for b, T in enumerate(LENS)])
    check(got, ref, (S + 1) * U * mag + U * np.abs(ref))
    w = (rng.standard_normal((N, D)) / math.sqrt(D)).astype(np.float32)
    bias = (0.1 * rng.standard_normal(N)).astype(np.float32)
    for act in (0, 1):
        e = rng.standard_normal((len(LENS), D)).astype(np.float32)
        got = run("head", LENS, e, (len(LENS), N), w=w, bias=bias, frames=S, dim=D, n_out=N, act=act)
        pre = e.astype(np.float64) @ w.T.astype(np.float64) + bias
        ref = np.tanh(pre) if act else pre
        mag = np.abs(e.astype(np.float64)) @ np.abs(w.T.astype(np.float64)) + np.abs(bias)
        check(got, ref, (D + 2) * U * mag + 2 * U * np.abs(ref) + 1e-7)
