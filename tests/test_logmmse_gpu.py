"""Log-MMSE on the H100 (mb_logmmse_*, mockingbird_b200.logmmse) against the outputs of the live reference recorded in
tests/golden/logmmse_seed0.npz and against the float64 restatement oracle/logmmse_oracle.py.

Bars.  The device computes in float64 like the reference and rounds once to fp32, and no frame's VAD statistic lies near
eta (the smallest gap on these clips is about 1e-3), so the fp32 output is held to the reference's own: at most 1 fp32 ulp
on any sample, the count of such samples printed (expected 0).  The VAD statistics are held to 1e-12 of the oracle's and to
the same side of eta on every frame, the noise profiles to 1e-13 relative, E1 to 5 ulp of its 40-digit value."""
import ctypes as C
import hashlib

import numpy as np
import pytest
import torch
from scipy.special import exp1

import golden_io
import logmmse_oracle as lo
from mockingbird_b200 import _lib
from mockingbird_b200 import logmmse

pytestmark = pytest.mark.gpu

SR = 16000
W, LEN1, LEN2, WIN, N_FFT = lo.params(SR)


@pytest.fixture(scope="module")
def golden(golden_dir):
    z = golden_io.load(golden_dir / "logmmse_seed0.npz")
    return z, sum(1 for k in z if k.startswith("clip_"))


def _profile(mu2):
    return logmmse.NoiseProfile(SR, W, LEN1, LEN2, WIN, N_FFT, mu2)


def _edges(x):
    return np.concatenate([x[:2400], x[-2400:]])


def _ulps(got, ref):
    """fp32 ulps between two fp32 arrays (both finite)"""
    a = got.view(np.int32).astype(np.int64)
    b = ref.view(np.int32).astype(np.int64)
    a = np.where(a < 0, -(a & 0x7FFFFFFF), a)
    b = np.where(b < 0, -(b & 0x7FFFFFFF), b)
    return np.abs(a - b)


def _check_output(got, ref, what):
    assert got.dtype == np.float32 and got.shape == ref.shape, what
    u = _ulps(got, ref)
    print(f"{what}: {int(np.count_nonzero(u))} of {u.size} samples differ, max {int(u.max(initial=0))} ulp")
    assert u.max(initial=0) <= 1, what
    return int(np.count_nonzero(u))


@pytest.mark.parametrize("eta", [0.15, 0.0])
def test_golden_clips_equal_reference(golden, eta):
    z, n = golden
    key = "out015" if eta == 0.15 else "out0"
    clips = [z[f"clip_{i}"] for i in range(n)]
    vads = []
    outs = logmmse.denoise_many(clips, [_profile(z[f"mu2_{i}"]) for i in range(n)], eta, vad_out=vads)
    for i in range(n):
        _check_output(outs[i], z[f"{key}_{i}"], f"clip {i} ({len(clips[i])} samples) eta {eta}")
        _, v_ref, _, _ = lo.denoise_loop(clips[i], WIN, N_FFT, z[f"mu2_{i}"], eta)
        assert vads[i].shape == v_ref.shape
        if len(v_ref):
            assert np.abs(vads[i] - v_ref).max() <= 1e-12
            assert np.array_equal(vads[i] < eta, v_ref < eta)


def test_profiles_match_reference(golden):
    z, n = golden
    profs = logmmse.profile_noise_many([_edges(z[f"clip_{i}"]) for i in range(n)], SR)
    worst = 0.0
    for i, p in enumerate(profs):
        assert p.noise_mu2.shape == (N_FFT,) and np.array_equal(p.win, WIN) and (p.window_size, p.n_fft) == (W, N_FFT)
        worst = max(worst, float(np.max(np.abs(p.noise_mu2 - z[f"mu2_{i}"]) / z[f"mu2_{i}"])))
    print(f"device noise_mu2 vs reference: max relative {worst:.1e}")
    assert worst <= 1e-13
    single = logmmse.profile_noise(_edges(z["clip_4"]), SR)
    assert np.array_equal(single.noise_mu2, profs[4].noise_mu2)


@pytest.mark.parametrize("eta", [0.15, 0.0])
def test_ten_second_clip_against_oracle(eta):
    x = lo.speechlike(10, 10 * SR)
    p = logmmse.profile_noise(_edges(x), SR)
    mu_ref = lo.profile_mu2(_edges(x), WIN, N_FFT)
    assert np.max(np.abs(p.noise_mu2 - mu_ref) / mu_ref) <= 1e-13
    vads = []
    got = logmmse.denoise_many([x], [p], eta, vad_out=vads)[0]
    ref, v_ref, _, _ = lo.denoise_loop(x, WIN, N_FFT, p.noise_mu2, eta)
    _check_output(got, ref, f"10 s clip eta {eta}")
    margin = float(np.min(np.abs(v_ref - eta)))
    print(f"10 s clip eta {eta}: max |vad - oracle| {np.abs(vads[0] - v_ref).max():.1e}, smallest |vad - eta| {margin:.1e}")
    assert np.abs(vads[0] - v_ref).max() <= 1e-12 and np.array_equal(vads[0] < eta, v_ref < eta)


def test_exp1_against_40_digits():
    """scipy.special.exp1 is itself up to 17 ulp away from E1 near x = 1 (against mpmath at 40 digits), so the device
    function is held to the 40-digit value, 5 ulp, and its distance to scipy is reported"""
    from mpmath import mp

    x = np.concatenate([np.geomspace(1e-8, 60.0, 6001), np.linspace(0.5, 2.0, 1501), [1.0, np.nextafter(1.0, 2.0)]])
    xd = torch.from_numpy(x).cuda()
    yd = torch.empty_like(xd)
    _lib.check(_lib.lib().mb_logmmse_exp1(C.c_void_p(xd.data_ptr()), C.c_void_p(yd.data_ptr()), x.size, None))
    y = yd.cpu().numpy()
    mp.dps = 40
    exact = np.array([float(mp.e1(mp.mpf(float(v)))) for v in x])
    ulps = np.abs(y - exact) / np.spacing(exact)
    ulps_scipy = np.abs(y - exp1(x)) / np.spacing(exact)
    print(f"E1 over [1e-8, 60]: max {ulps.max():.0f} ulp from the 40-digit value, {ulps_scipy.max():.0f} ulp from scipy")
    assert ulps.max() <= 5 and ulps_scipy.max() <= 24


RAGGED = [320, 479, 480, 481, 640, 6401, 160, 0, 12345, 16000, 33333, 799, 96000, 5000, 2, 48001]


def test_ragged_batch_bitwise_equal_to_single_calls():
    lengths = [n if n >= 320 else 320 + n for n in RAGGED]
    clips = [lo.speechlike(40 + i, n) for i, n in enumerate(lengths)]
    profs = logmmse.profile_noise_many([lo.speechlike(80 + i, 960 + 320 * i) for i in range(len(clips))], SR)
    for eta in (0.15, 0.0):
        vads = []
        batch = logmmse.denoise_many(clips, profs, eta, vad_out=vads)
        for i, (x, p) in enumerate(zip(clips, profs)):
            v1 = []
            one = logmmse.denoise_many([x], [p], eta, vad_out=v1)[0]
            assert np.array_equal(batch[i], one), (i, len(x))
            assert np.array_equal(vads[i], v1[0]), i
    # a clip's output does not depend on its neighbours
    other = [lo.speechlike(120 + i, n) for i, n in enumerate(lengths)]
    other[5] = clips[5]
    assert np.array_equal(logmmse.denoise_many(other, profs)[5], logmmse.denoise(clips[5], profs[5]))


def test_launch_count_independent_of_batch():
    L = _lib.lib()
    counts = []
    for B in (1, 16, 64):
        clips = [lo.speechlike(b, 3000 + 997 * b) for b in range(B)]
        logmmse.denoise_many(clips[:1], logmmse.profile_noise_many([_edges(clips[0])], SR))  # handle and workspace set up
        before = L.mb_launch_count()
        profs = logmmse.profile_noise_many([_edges(c) for c in clips], SR)
        mid = L.mb_launch_count()
        logmmse.denoise_many(clips, profs)
        counts.append((mid - before, L.mb_launch_count() - mid))
    assert counts == [(1, 4)] * 3


def test_refusals_queue_nothing():
    L = _lib.lib()
    p = logmmse.profile_noise(lo.speechlike(1, 4800), SR)
    logmmse.denoise(lo.speechlike(2, 1000), p)
    before = L.mb_launch_count()
    with pytest.raises(ValueError, match="wav 1 has 319 samples"):
        logmmse.denoise_many([lo.speechlike(2, 1000), lo.speechlike(3, 319)], [p, p])
    with pytest.raises(ValueError, match="float64"):
        logmmse.denoise(lo.speechlike(2, 1000).astype(np.float64), p)
    with pytest.raises(ValueError, match="int16"):
        logmmse.denoise((lo.speechlike(2, 1000) * 32767).astype(np.int16), p)
    assert L.mb_launch_count() == before
    # the C entry point refuses on its own too, naming the utterance
    h = logmmse._handle(W, LEN1, LEN2, N_FFT)
    T, ws = h.workspace([1000, 1000])
    T[1] = 319
    x = torch.zeros(2000, device="cuda")
    w = torch.from_numpy(WIN).cuda()
    mu2 = torch.ones(2, N_FFT, dtype=torch.float64, device="cuda")
    rc = L.mb_logmmse_denoise(h._handle, C.c_void_p(x.data_ptr()), T, 2, C.c_void_p(w.data_ptr()), C.c_void_p(mu2.data_ptr()),
                              0.15, C.c_void_p(x.data_ptr()), None, C.c_void_p(ws.data_ptr()), ws.numel(), None)
    assert rc != 0 and b"utterance 1" in L.mb_last_error()
    T[1] = 300
    rc = L.mb_logmmse_profile(h._handle, C.c_void_p(x.data_ptr()), T, 2, C.c_void_p(w.data_ptr()), C.c_void_p(mu2.data_ptr()),
                              C.c_void_p(ws.data_ptr()), ws.numel(), None)
    assert rc != 0 and b"noise 1" in L.mb_last_error()
    assert L.mb_launch_count() == before


def test_load_preprocess_wavs_equals_reference(golden):
    from mockingbird_b200.synthesizer.inference import Synthesizer

    z, n = golden
    clips = [z[f"clip_{i}"] for i in range(n)]
    got = Synthesizer.load_preprocess_wavs(clips)
    for i, x in enumerate(clips):
        _check_output(got[i], z[f"pre_{i}"], f"load_preprocess_wavs clip {i}")
        if len(x) <= SR * 0.4:  # only rescaled
            assert np.array_equal(got[i], x / np.abs(x).max() * 0.9)


def test_other_sizes_against_oracle():
    """8 kHz (n_fft 320 = 5 * 64) and 32 kHz (1280 = 5 * 256): the radix-5 stage at both ends of the range in use, and the
    two-bins-per-thread scan at n_fft 2048 (window_size 1024)"""
    for sr, ws in ((8000, 0), (32000, 0), (16000, 1024)):
        Wd, l1, l2, win, n = lo.params(sr, ws)
        x = lo.speechlike(sr + ws, 3 * sr, sr)
        noise = lo.speechlike(sr + ws + 1, 4 * Wd, sr)
        p = logmmse.profile_noise(noise, sr, ws)
        mu_ref = lo.profile_mu2(noise, win, n)
        assert p.n_fft == n and np.max(np.abs(p.noise_mu2 - mu_ref) / mu_ref) <= 1e-13
        for eta in (0.15, 0.0):
            vads = []
            got = logmmse.denoise_many([x], [p], eta, vad_out=vads)[0]
            ref, v_ref, _, _ = lo.denoise_loop(x, win, n, p.noise_mu2, eta)
            _check_output(got, ref, f"sr {sr} n_fft {n} eta {eta}")
            assert np.abs(vads[0] - v_ref).max() <= 1e-12 and np.array_equal(vads[0] < eta, v_ref < eta)


# sha256 of the fp32 output below, recorded on an H100 from the Griffin-Lim build that had its own FFT, before the FFT moved
# into csrc/mb_fft.cuh
GRIFFINLIM_SHA256 = "7c963548a270d54afb290a884ae29ab70b338fb6661be4b187126f4384ab173d"


def griffinlim_digest():
    """sha256 of Griffin-Lim's fp32 outputs for n_fft 1024, 512 and 2048 (3 seeded mels each, 5 iterations, pre-emphasis)"""
    from types import SimpleNamespace

    import griffinlim_oracle as go
    from mockingbird_b200.griffinlim import GriffinLim
    from mockingbird_b200.synthesizer.hparams import hparams as hp

    outs = []
    for n_fft, hop in ((1024, 256), (512, 128), (2048, 512)):
        h = SimpleNamespace(**{k: getattr(hp, k) for k in ("sample_rate", "num_mels", "fmin", "fmax")}, n_fft=n_fft)
        g = GriffinLim(go.inv_basis(h), n_fft, hop, n_fft, preemphasis=0.97)
        mels = [(np.random.RandomState(60 + T).rand(80, T) * 8 - 4).astype(np.float32) for T in (9, 64, 313)]
        outs += [y.cpu().numpy() for y in g(mels, 5, seeds=[1, 2, 3])]
    return hashlib.sha256(b"".join(o.tobytes() for o in outs)).hexdigest()


def test_griffinlim_unchanged_by_shared_fft():
    digest = griffinlim_digest()
    print("griffinlim sha256", digest)
    assert digest == GRIFFINLIM_SHA256
