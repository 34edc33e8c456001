"""The signal-processing kernels against float64 references at every size their handles accept: the shared Stockham FFT
(csrc/mb_fft.cuh, through mb_fft_debug), log-MMSE (csrc/logmmse.cu), Griffin-Lim (csrc/griffinlim.cu) and the mel front-end
(csrc/melspec.cu).  Every GPU case prints its measured error next to its bound.

Bounds.
- Double FFT: max|y - numpy.fft| <= 1e-13 max|X| on every row.  Float FFT: numpy complex64 (pocketfft computes it in float32)
  on the same rounded input drifts from float64 by d, relative to the row's max|X|; the kernel is held to 20 d per row, and
  never below 20 * 2^-24 = 1.2e-6 (the outputs' own fp32 rounding; an impulse at 0 is exact in both, d = 0).  d measured on
  the CPU (numpy 2.3.5), max over the rows of a kind at each of the 11 sizes, the same in both directions: random rows
  3.4e-8 .. 5.1e-8, impulses 2.9e-8 .. 4.2e-8, tones 5.4e-10 .. 7.8e-9 (so tone rows are held to the 1.2e-6 floor).
- log-MMSE: the bars of tests/test_logmmse_gpu.py: output within 1 fp32 ulp of oracle/logmmse_oracle.py, VAD statistic
  within 1e-12 and on the same side of eta on every frame, noise profile within 1e-13 relative.
- Griffin-Lim: the staged check of tests/test_griffinlim_gpu.py (initial ISTFT with n_iters = 0, then one teacher-forced
  iteration), each held to 20x the drift of oracle/griffinlim_oracle.py run in numpy float32 from the same magnitudes, phases
  and previous waveform, max|d| / max|ref|.  Measured on the CPU (initial / one iteration, the iteration from the float64
  initial waveform): 1.3e-7 .. 2.2e-7 / 1.3e-7 .. 2.4e-7 over the configurations below (largest: power 2 initial, odd
  win_length 1023 iteration), bounds 2.6e-6 .. 4.8e-6; the test recomputes the drift from the kernel's own waveform and
  prints it.  The inverse pre-emphasis restarts each two-hop chunk's recursion W samples early with k^W < 2^-30: its error
  against scipy.signal.lfilter of the kernel's own waveform is bounded by the dropped state, k^W max|out|, plus the output's
  fp32 rounding, 2^-24 max|out|, plus float64 rounding amplified by at most 1 / (1 - k): 6.1e-8 of max|out| at k = 0.99.
- Mel front-end: the DFT is a sequential fp32 sum of n_fft terms, so its error grows with n_fft.  The bound is 20x the drift of
  a float32 numpy restatement of the kernel (same window, twiddle and basis tables, the same n_fft-term sums in the same
  order) from the float64 oracle; relative to max|ref| for linear outputs, absolute for dB and normalised ones.  Measured on
  the CPU: linear 7.3e-8 (n_fft 16, 9 samples), 1.7e-7 (16), 2.3e-7 .. 1.0e-6 (400), 3.2e-7 .. 8.6e-7 (512), 8.3e-7 (1024),
  2.0e-6 (2048); normalised 5.7e-6 (symmetric) and 2.7e-6 (asymmetric); 9.2e-5 dB without normalisation.
"""
import ctypes as C
from types import SimpleNamespace

import numpy as np
import pytest
import torch
from scipy.signal import lfilter

import griffinlim_oracle as go
import logmmse_oracle as lo
import melspec_oracle as mo
from mockingbird_b200 import _lib

gpu = pytest.mark.gpu
MB_ERR_INVALID = 1  # include/mockingbird_b200.h
FACTOR = 20  # float bounds: this many times the numpy float32 drift measured on the same inputs

FFT_SIZES = [64, 80, 128, 160, 256, 320, 512, 640, 1024, 1280, 2048]  # log-MMSE's n_fft set; Griffin-Lim's is 256 .. 2048


# --------------------------------------------------------------------------------------------------------- shared FFT


def fft_rows(n):
    """the test rows of one size -> (complex128 [rows, n], kind of each row): 4 random rows, impulses at 0, 1 and n - 1,
    tones at bins 0, 1, n / 2 and n - 1"""
    rng = np.random.default_rng(n)
    rows, kinds = [], []
    for _ in range(4):
        rows.append(rng.standard_normal(n) + 1j * rng.standard_normal(n))
        kinds.append("random")
    for p in (0, 1, n - 1):
        e = np.zeros(n, np.complex128)
        e[p] = 1.0
        rows.append(e)
        kinds.append("impulse")
    j = np.arange(n)
    for b in (0, 1, n // 2, n - 1):
        rows.append(np.exp(2j * np.pi * b * j / n))
        kinds.append("tone")
    return np.stack(rows), kinds


def numpy_fft(x, inverse):
    """the unscaled transform of each row, in x's precision (complex64 runs in float32)"""
    return np.fft.ifft(x, axis=1, norm="forward") if inverse else np.fft.fft(x, axis=1)


def device_fft(x, inverse):
    rows, n = x.shape
    xd = torch.from_numpy(np.ascontiguousarray(x)).cuda()
    yd = torch.empty_like(xd)
    dtype = 0 if x.dtype == np.complex64 else 1
    _lib.check(_lib.lib().mb_fft_debug(C.c_void_p(xd.data_ptr()), C.c_void_p(yd.data_ptr()), n, rows, dtype, int(inverse),
                                       None))
    return yd.cpu().numpy()


def row_errors(got, ref):
    """max |got - ref| / max |ref| of each row"""
    return np.abs(got - ref).max(axis=1) / np.abs(ref).max(axis=1)


@gpu
@pytest.mark.parametrize("inverse", [False, True])
@pytest.mark.parametrize("n", FFT_SIZES)
@pytest.mark.parametrize("prec", ["double", "float"])
def test_fft_against_numpy(prec, n, inverse):
    x, kinds = fft_rows(n)
    kinds = np.array(kinds)
    if prec == "float":
        x = x.astype(np.complex64)
    ref = numpy_fft(x.astype(np.complex128), inverse)
    err = row_errors(device_fft(x, inverse), ref)
    if prec == "double":
        bound = np.full(len(err), 1e-13)
    else:
        drift = row_errors(numpy_fft(x, inverse), ref)
        bound = FACTOR * np.maximum(drift, 2.0 ** -24)
    worst = "  ".join(f"{k} {err[kinds == k].max():.1e} (bound {bound[kinds == k].min():.1e})"
                      for k in ("random", "impulse", "tone"))
    print(f"fft {prec} n {n} {'inverse' if inverse else 'forward'}: {worst}")
    bad = [(k, float(e), float(b)) for k, e, b in zip(kinds, err, bound) if not e <= b]
    assert not bad, bad


def test_fft_debug_refuses_unsupported_sizes_without_launching():
    L = _lib.lib()
    before = L.mb_launch_count()
    for n, dtype in ((32, 1), (96, 1), (2560, 1), (4096, 0), (200, 0), (256, 2)):
        assert L.mb_fft_debug(C.c_void_p(256), C.c_void_p(256), n, 1, dtype, 0, None) == MB_ERR_INVALID, n
        assert b"mb_fft_debug" in L.mb_last_error()
    assert L.mb_launch_count() == before


def test_logmmse_and_griffinlim_refuse_other_sizes():
    L = _lib.lib()
    for n in (32, 96, 2560, 4096):
        cfg = _lib.LogMmseConfig()
        cfg.window_size, cfg.n_fft = min(n, 2048) // 2, n
        cfg.len1 = cfg.len2 = cfg.window_size // 2
        h = C.c_void_p()
        assert L.mb_logmmse_create(C.byref(cfg), C.byref(h)) == MB_ERR_INVALID, n
        assert f"n_fft = {n}".encode() in L.mb_last_error()
    for n in (128, 320, 4096):
        cfg = _lib.GriffinLimConfig()
        cfg.n_fft, cfg.win_length, cfg.hop_length, cfg.n_mels, cfg.power = n, n, n // 4, 80, 1.5
        h = C.c_void_p()
        assert L.mb_griffinlim_create(C.byref(cfg), C.byref(h)) == MB_ERR_INVALID, n
        assert f"n_fft = {n}".encode() in L.mb_last_error()


# ---------------------------------------------------------------------------------------------------------- log-MMSE


def _ulps(got, ref):
    """fp32 ulps between two finite fp32 arrays"""
    a = got.view(np.int32).astype(np.int64)
    b = ref.view(np.int32).astype(np.int64)
    a = np.where(a < 0, -(a & 0x7FFFFFFF), a)
    b = np.where(b < 0, -(b & 0x7FFFFFFF), b)
    return np.abs(a - b)


def _check_denoise(x, prof, win, n_fft, what):
    from mockingbird_b200 import logmmse

    for eta in (0.15, 0.0):
        vads = []
        got = logmmse.denoise_many([x], [prof], eta, vad_out=vads)[0]
        ref, v_ref, _, _ = lo.denoise_loop(x, win, n_fft, prof.noise_mu2, eta)
        assert got.dtype == np.float32 and got.shape == ref.shape
        u = _ulps(got, ref)
        dv = float(np.abs(vads[0] - v_ref).max())
        print(f"{what} eta {eta}: {int(np.count_nonzero(u))} of {u.size} samples differ, max {int(u.max())} ulp (bound 1); "
              f"vad {dv:.1e} (bound 1e-12), smallest |vad - eta| {float(np.min(np.abs(v_ref - eta))):.1e}")
        assert u.max() <= 1
        assert dv <= 1e-12 and np.array_equal(vads[0] < eta, v_ref < eta)


@gpu
@pytest.mark.parametrize("n_fft", FFT_SIZES)
def test_logmmse_every_size(n_fft):
    """window_size = n_fft / 2 reaches every n_fft the handle accepts; the clip ends half a hop past its last whole frame"""
    from mockingbird_b200 import logmmse

    sr = 16000
    W, _, hop, win, n = lo.params(sr, n_fft // 2)
    assert n == n_fft
    x = lo.speechlike(n_fft, 211 * hop + hop // 2 + 1, sr)
    noise = lo.speechlike(n_fft + 1, 5 * W + 7, sr)
    p = logmmse.profile_noise(noise, sr, W)
    mu_ref = lo.profile_mu2(noise, win, n)
    rel = float(np.max(np.abs(p.noise_mu2 - mu_ref) / mu_ref))
    print(f"logmmse n_fft {n_fft}: noise profile {rel:.1e} relative (bound 1e-13)")
    assert p.n_fft == n_fft and rel <= 1e-13
    _check_denoise(x, p, win, n, f"logmmse n_fft {n_fft}")


@gpu
def test_logmmse_window_shorter_than_half_n_fft():
    """create() takes window_size < n_fft / 2; the Python layer always asks for n_fft = 2 W, so the handle is made here"""
    from mockingbird_b200 import logmmse

    sr, W, n_fft = 16000, 160, 512
    _, l1, l2, win, _ = lo.params(sr, W)
    h = logmmse._handle(W, l1, l2, n_fft)
    noise = lo.speechlike(7, 6 * W + 3, sr)
    T, ws = h.workspace([len(noise)])
    xd = torch.from_numpy(noise).cuda()
    wd = torch.from_numpy(win).cuda()
    mu2 = torch.empty(1, n_fft, dtype=torch.float64, device="cuda")
    _lib.check(_lib.lib().mb_logmmse_profile(h._handle, C.c_void_p(xd.data_ptr()), T, 1, C.c_void_p(wd.data_ptr()),
                                             C.c_void_p(mu2.data_ptr()), C.c_void_p(ws.data_ptr()), ws.numel(), None))
    mu2 = mu2.cpu().numpy()[0]
    mu_ref = lo.profile_mu2(noise, win, n_fft)
    rel = float(np.max(np.abs(mu2 - mu_ref) / mu_ref))
    print(f"logmmse W {W} n_fft {n_fft}: noise profile {rel:.1e} relative (bound 1e-13)")
    assert rel <= 1e-13
    prof = logmmse.NoiseProfile(sr, W, l1, l2, win, n_fft, mu2)
    _check_denoise(lo.speechlike(8, 3 * sr + 37, sr), prof, win, n_fft, f"logmmse W {W} n_fft {n_fft}")


# ------------------------------------------------------------------------------------------------------- Griffin-Lim


def _gl_hp(**kw):
    from mockingbird_b200.synthesizer.hparams import hparams

    base = {k: getattr(hparams, k) for k in ("sample_rate", "n_fft", "num_mels", "hop_size", "win_size", "fmin", "fmax",
                                             "min_level_db", "ref_level_db", "max_abs_value", "signal_normalization",
                                             "allow_clipping_in_normalization", "symmetric_mels", "power")}
    base.update(kw)
    return SimpleNamespace(**base)


def _gl_handle(hp, pad_mode="reflect", preemphasis=0.0):
    from mockingbird_b200.griffinlim import GriffinLim

    return GriffinLim(go.inv_basis(hp), hp.n_fft, hp.hop_size, hp.win_size, pad_mode=pad_mode, power=hp.power,
                      preemphasis=preemphasis, signal_normalization=hp.signal_normalization,
                      allow_clipping=hp.allow_clipping_in_normalization, symmetric=hp.symmetric_mels,
                      max_abs_value=hp.max_abs_value, min_level_db=hp.min_level_db, ref_level_db=hp.ref_level_db)


def _gl_run(g, mels, n_iters, us):
    ys = g(mels, n_iters, uniforms=us)
    return [y.cpu().numpy().astype(np.float64) for y in ys]


def _rel(got, ref):
    assert got.shape == ref.shape, (got.shape, ref.shape)
    return float(np.abs(got - ref).max() / np.abs(ref).max())


def _gl_mel(n_mels, T, seed):
    return (np.random.RandomState(seed).rand(n_mels, T) * 9 - 4.5).astype(np.float32)


def _gl_staged(hp, mel, u, y0, y1, pad_mode, what):
    """initial ISTFT and one teacher-forced iteration of one utterance against the oracle, bounds from its float32 drift"""
    S = go.magnitudes(mel, hp)
    args = (hp.n_fft, hp.hop_size, hp.win_size)
    r0 = go.griffin_lim(S, u, 0, *args, pad_mode)
    d0 = _rel(go.griffin_lim(S, u, 0, *args, pad_mode, dtype=np.float32).astype(np.float64), r0)
    r1 = go.iterate(S, y0, *args, pad_mode)
    d1 = _rel(go.iterate(S, y0.astype(np.float32), *args, pad_mode, dtype=np.float32).astype(np.float64), r1)
    e0, e1 = _rel(y0, r0), _rel(y1, r1)
    print(f"griffinlim {what}: initial {e0:.2e} (float32 drift {d0:.1e}, bound {FACTOR * d0:.1e}), "
          f"one iteration {e1:.2e} (drift {d1:.1e}, bound {FACTOR * d1:.1e})")
    assert e0 <= FACTOR * d0 and e1 <= FACTOR * d1


GL_CONFIGS = {
    "n_fft256": dict(n_fft=256, win_size=256, hop_size=64),
    "odd_win_1023": dict(win_size=1023),
    "odd_win_801": dict(win_size=801, hop_size=200),
    "hop_eq_win": dict(n_fft=512, win_size=400, hop_size=400),
    "n_mels1": dict(num_mels=1),
    "n_mels40": dict(num_mels=40),
    "n_mels128": dict(num_mels=128, fmin=0, fmax=8000),
    "power2": dict(power=2.0),
}


@gpu
@pytest.mark.parametrize("name", list(GL_CONFIGS))
def test_griffinlim_configs(name):
    hp = _gl_hp(**GL_CONFIGS[name])
    T = 41
    mel = _gl_mel(hp.num_mels, T, 3)
    u = np.random.RandomState(4).rand(hp.n_fft // 2 + 1, T)
    g = _gl_handle(hp)
    y0 = _gl_run(g, [mel], 0, [u])[0]
    y1 = _gl_run(g, [mel], 1, [u])[0]
    _gl_staged(hp, mel, u, y0, y1, "reflect", name)


@gpu
def test_griffinlim_constant_padding_ragged_with_two_frames():
    hp = _gl_hp()
    Ts = [2, 7, 3, 30]
    mels = [_gl_mel(hp.num_mels, T, 10 + T) for T in Ts]
    us = [np.random.RandomState(20 + T).rand(hp.n_fft // 2 + 1, T) for T in Ts]
    g = _gl_handle(hp, "constant")
    y0s = _gl_run(g, mels, 0, us)
    y1s = _gl_run(g, mels, 1, us)
    for T, mel, u, y0, y1 in zip(Ts, mels, us, y0s, y1s):
        assert y0.shape == (hp.hop_size * (T - 1),)
        _gl_staged(hp, mel, u, y0, y1, "constant", f"constant padding T {T}")


@gpu
def test_griffinlim_inverse_preemphasis_long_warmup():
    """k = 0.99 needs a 2070-sample warm-up (the smallest W with k^W < 2^-30), more than two hops (512): chunks restart
    their recursion in earlier chunks, and the utterances of 768 and 1792 samples are shorter than the warm-up"""
    k = 0.99
    warm = int(np.ceil(30 * np.log(2) / -np.log(k)))  # mb_griffinlim_create's rule
    assert warm == 2070 and k ** warm < 2.0 ** -30 <= k ** (warm - 1)
    hp = _gl_hp()
    Ts = [4, 8, 40, 120]
    mels = [_gl_mel(hp.num_mels, T, 40 + T) for T in Ts]
    us = [np.random.RandomState(50 + T).rand(hp.n_fft // 2 + 1, T) for T in Ts]
    ys = _gl_run(_gl_handle(hp), mels, 1, us)
    outs = _gl_run(_gl_handle(hp, preemphasis=k), mels, 1, us)
    rel_bound = k ** warm + 2.0 ** -24 + 2 * 2.0 ** -53 / (1 - k)
    for T, y, out in zip(Ts, ys, outs):
        e = _rel(out, lfilter([1], [1, -k], y))
        print(f"griffinlim inverse pre-emphasis k {k} T {T} ({len(y)} samples): {e:.2e} (bound {rel_bound:.2e})")
        assert e <= rel_bound


# ----------------------------------------------------------------------------------------------------- mel front-end

MEL_BASE = dict(sample_rate=16000, fmin=55.0, fmax=7600.0, pad_mode="reflect", preemphasis=0.0, to_db=False,
                normalize=False, symmetric=True, min_level_db=-100.0, ref_level_db=20.0, max_abs_value=4.0)

MEL_CASES = {  # n: the signal's length
    "n16_shortest": dict(n_fft=16, hop_length=4, win_length=16, n_mels=4, fmin=0.0, fmax=8000.0, power=2,
                         transpose_out=True, n=9),
    "n16_mels1": dict(n_fft=16, hop_length=5, win_length=13, n_mels=1, fmin=0.0, fmax=8000.0, power=1,
                      transpose_out=False, n=300),
    "n400_win301": dict(n_fft=400, hop_length=160, win_length=301, n_mels=40, power=2, transpose_out=True, n=4000),
    "n400_shortest": dict(n_fft=400, hop_length=160, win_length=400, n_mels=40, power=2, transpose_out=False, n=201),
    "n512_hop_gt_win": dict(n_fft=512, hop_length=400, win_length=300, n_mels=40, power=1, transpose_out=True, n=6001),
    "n512_mels1": dict(n_fft=512, hop_length=128, win_length=512, n_mels=1, power=2, transpose_out=False, n=3000),
    "n1024_power1_constant": dict(n_fft=1024, hop_length=256, win_length=1024, n_mels=80, power=1, transpose_out=False,
                                  pad_mode="constant", n=5000),
    "n2048_fmax_half_mels128": dict(n_fft=2048, hop_length=512, win_length=2048, n_mels=128, fmin=0.0, fmax=8000.0,
                                    power=2, transpose_out=True, n=12000),
    "db_symmetric": dict(n_fft=1024, hop_length=256, win_length=1024, n_mels=80, power=1, preemphasis=0.97, to_db=True,
                         normalize=True, transpose_out=False, n=8000),
    "db_asymmetric": dict(n_fft=800, hop_length=200, win_length=800, n_mels=80, power=1, preemphasis=0.97, to_db=True,
                          normalize=True, symmetric=False, transpose_out=True, n=8000),
    "db_not_normalized": dict(n_fft=1024, hop_length=256, win_length=1024, n_mels=80, power=2, to_db=True,
                              transpose_out=True, n=5000),
}


def _mel_cfg(name):
    c = dict(MEL_BASE)
    c.update(MEL_CASES[name])
    return c


def _mel_wav(n, seed):
    rng = np.random.default_rng(seed)
    t = np.arange(n) / 16000.0
    return (0.3 * np.sin(2 * np.pi * 220 * t) + 0.05 * rng.standard_normal(n)).astype(np.float32)


def mel_reference(wav, c):
    """oracle/melspec_oracle.py float64 -> the kernel's layout"""
    hp = dict(sample_rate=c["sample_rate"], n_fft=c["n_fft"], num_mels=c["n_mels"], hop_size=c["hop_length"],
              win_size=c["win_length"], fmin=c["fmin"], fmax=c["fmax"], min_level_db=c["min_level_db"],
              ref_level_db=c["ref_level_db"], max_abs_value=c["max_abs_value"], preemphasis=c["preemphasis"],
              preemphasize=c["preemphasis"] != 0, symmetric_mels=c["symmetric"], power=c["power"], to_db=c["to_db"],
              signal_normalization=c["normalize"])
    r = mo.synthesizer_mel(wav, hp, c["pad_mode"]).astype(np.float64)
    return r.T if c["transpose_out"] else r


def _hz_to_mel(f):
    return np.where(f >= 1000.0, 15.0 + np.log(np.maximum(f, 1e-30) / 1000.0) / (np.log(6.4) / 27.0), f * 3.0 / 200.0)


def _mel_to_hz(m):
    return np.where(m >= 15.0, 1000.0 * np.exp(np.log(6.4) / 27.0 * (m - 15.0)), m * 200.0 / 3.0)


def mel_float32(wav, c):
    """the kernel's algorithm in numpy float32: its window, twiddle and basis tables (float64, rounded once), the padded
    pre-emphasised frame, the n_fft-term DFT sums in the kernel's order, |.| or |.|^2, the mel projection, dB and
    normalisation; for the bound only"""
    f32 = np.float32
    N, H, Wl, nb = c["n_fft"], c["hop_length"], c["win_length"], c["n_fft"] // 2 + 1
    win = np.zeros(N, f32)
    lpad = (N - Wl) // 2
    win[lpad:lpad + Wl] = (0.5 - 0.5 * np.cos(2 * np.pi * np.arange(Wl) / Wl)).astype(f32)
    cs = np.cos(2 * np.pi * np.arange(N) / N).astype(f32)
    sn = (-np.sin(2 * np.pi * np.arange(N) / N)).astype(f32)
    edges = _mel_to_hz(_hz_to_mel(c["fmin"]) + (_hz_to_mel(c["fmax"]) - _hz_to_mel(c["fmin"])) *
                       np.arange(c["n_mels"] + 2) / (c["n_mels"] + 1))
    fk = np.arange(nb) * c["sample_rate"] / N
    lo_, ce, hi = edges[:-2, None], edges[1:-1, None], edges[2:, None]
    basis = (np.maximum(0.0, np.minimum((fk - lo_) / (ce - lo_), (hi - fk) / (hi - ce))) * (2.0 / (hi - lo_))).astype(f32)
    x = np.asarray(wav, f32)
    k = f32(c["preemphasis"])
    y = np.concatenate([x[:1], x[1:] - k * x[:-1]]) if k != 0 else x
    yp = np.pad(y, N // 2, mode=c["pad_mode"])
    nf = 1 + len(x) // H
    fr = np.stack([yp[f * H:f * H + N] for f in range(nf)]) * win
    re = np.zeros((nf, nb), f32)
    im = np.zeros((nf, nb), f32)
    kk = np.arange(nb)
    for j in range(N):
        idx = (j * kk) % N
        re = re + fr[:, j:j + 1] * cs[idx]
        im = im + fr[:, j:j + 1] * sn[idx]
    pw = re * re + im * im
    mag = pw if c["power"] == 2 else np.sqrt(pw)
    v = mag @ basis.T  # [frames, n_mels]
    if c["to_db"]:
        min_level = np.exp(f32(c["min_level_db"]) / f32(20) * np.log(f32(10)))
        v = f32(20) * np.log10(np.maximum(min_level, v)) - f32(c["ref_level_db"])
    if c["normalize"]:
        A, lo_db = f32(c["max_abs_value"]), f32(c["min_level_db"])
        s = (v - lo_db) / -lo_db
        v = np.clip(f32(2) * A * s - A, -A, A) if c["symmetric"] else np.clip(A * s, f32(0), A)
    return (v if c["transpose_out"] else v.T).astype(np.float64)


def _mel_err(got, ref, c):
    """relative to max|ref| for linear outputs, absolute for dB or normalised ones"""
    assert got.shape == ref.shape, (got.shape, ref.shape)
    e = float(np.abs(got - ref).max())
    return e if (c["to_db"] or c["normalize"]) else e / float(np.abs(ref).max())


@gpu
@pytest.mark.parametrize("name", list(MEL_CASES))
def test_melspec_configs(name):
    from mockingbird_b200.melspec import MelSpectrogram

    c = _mel_cfg(name)
    n = c.pop("n")
    m = MelSpectrogram(**c)
    wav = _mel_wav(n, n)
    got = m(wav).cpu().numpy()
    assert got.dtype == np.float32
    ref = mel_reference(wav, c)
    err = _mel_err(got.astype(np.float64), ref, c)
    drift = _mel_err(mel_float32(wav, c), ref, c)
    unit = "" if (c["to_db"] or c["normalize"]) else " relative"
    print(f"melspec {name}: {err:.2e}{unit} (float32 drift {drift:.1e}, bound {FACTOR * drift:.1e})")
    assert err <= FACTOR * drift
    # the ragged launch: each utterance bitwise its single call, the shortest accepted signal among them
    wavs = [_mel_wav(n + 37, 1), wav, _mel_wav(c["n_fft"] // 2 + 1, 2), _mel_wav(3 * n + 1, 3)]
    for w, r in zip(wavs, m.many(wavs)):
        assert np.array_equal(r, m(w).cpu().numpy()), len(w)


def test_melspec_refuses_odd_n_fft():
    """bin k sits at k sr / n_fft; for odd n_fft librosa's grid depends on its version (oracle/melspec_oracle.py header)"""
    L = _lib.lib()
    for n_fft, win in ((401, 401), (17, 16), (1023, 800)):
        cfg = _lib.MelSpecConfig()
        cfg.sample_rate, cfg.n_fft, cfg.hop_length, cfg.win_length, cfg.n_mels = 16000, n_fft, 160, win, 40
        cfg.fmin, cfg.fmax, cfg.power = 0.0, 8000.0, 2
        h = C.c_void_p()
        assert L.mb_melspec_create(C.byref(cfg), C.byref(h)) == MB_ERR_INVALID, n_fft
        assert b"is odd" in L.mb_last_error()
        cfg.n_fft = n_fft + 1
        assert L.mb_melspec_create(C.byref(cfg), C.byref(h)) == 0, n_fft + 1
        L.mb_melspec_destroy(h)
