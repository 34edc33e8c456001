"""Log-MMSE without a GPU: the float64 restatement (oracle/logmmse_oracle.py) against the golden outputs of the live
reference and, where the reference tree is present, against the reference itself; the frame-count and tail rules; the
input checks of mockingbird_b200.logmmse that run before any device work; the handle's create-time checks and workspace
arithmetic."""
import ctypes as C
import importlib.util

import numpy as np
import pytest

import golden_io
import logmmse_oracle as lo
import ref_harness as rh
from mockingbird_b200 import _lib
from mockingbird_b200 import logmmse

MB_ERR_INVALID = 1
SR = 16000
W, LEN1, LEN2, WIN, N_FFT = lo.params(SR)


@pytest.fixture(scope="module")
def golden(golden_dir):
    z = golden_io.load(golden_dir / "logmmse_seed0.npz")
    n = sum(1 for k in z if k.startswith("clip_"))
    return z, n


def _edges(x):
    return np.concatenate([x[:2400], x[-2400:]])


def test_params_match_reference_defaults():
    assert (W, LEN1, LEN2, N_FFT) == (320, 160, 160, 640)
    assert np.array_equal(WIN, np.hanning(320) * 160 / np.sum(np.hanning(320)))
    assert logmmse._params(SR, 0)[:3] == (320, 160, 160) and np.array_equal(logmmse._params(SR, 0)[3], WIN)
    assert logmmse._params(22050, 0)[0] == 442 and logmmse._params(8000, 0)[4] == 320 and logmmse._params(32000, 0)[4] == 1280


@pytest.mark.parametrize("eta", [0.15, 0.0])
def test_oracle_equals_golden(golden, eta):
    z, n = golden
    key = "out015" if eta == 0.15 else "out0"
    for i in range(n):
        got = lo.denoise(z[f"clip_{i}"], WIN, N_FFT, z[f"mu2_{i}"], eta)
        assert got.dtype == np.float32 and np.array_equal(got, z[f"{key}_{i}"]), (i, len(got))


def test_oracle_profile_matches_golden(golden):
    z, n = golden
    worst = 0.0
    for i in range(n):
        mu2 = lo.profile_mu2(_edges(z[f"clip_{i}"]), WIN, N_FFT)
        worst = max(worst, float(np.max(np.abs(mu2 - z[f"mu2_{i}"]) / z[f"mu2_{i}"])))
    print(f"oracle noise_mu2 vs reference: max relative {worst:.1e}")
    assert worst <= 1e-13


def test_oracle_load_preprocess_equals_golden(golden):
    z, n = golden
    for i in range(n):
        assert np.array_equal(lo.load_preprocess(z[f"clip_{i}"]), z[f"pre_{i}"]), i


@pytest.mark.skipif(not rh.reference_available(), reason="needs the reference tree")
@pytest.mark.parametrize("seed,n", [(7, 4321), (8, 160000), (9, 481)])
def test_oracle_equals_live_reference(seed, n):
    spec = importlib.util.spec_from_file_location("ref_logmmse", rh.REFERENCE_ROOT / "utils" / "logmmse.py")
    ref = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(ref)
    x = lo.speechlike(seed, n)
    noise = lo.speechlike(seed + 1, 4800)
    p = ref.profile_noise(noise.copy(), SR)
    assert np.max(np.abs(lo.profile_mu2(noise, WIN, N_FFT) - p.noise_mu2) / p.noise_mu2) <= 1e-13
    for eta in (0.15, 0.0):
        assert np.array_equal(lo.denoise(x, p.win, p.n_fft, p.noise_mu2, eta), ref.denoise(x, p, eta=eta))


@pytest.mark.parametrize("L", [320, 479, 480, 481, 639, 640, 6401])
def test_frame_count_and_zero_tail(L):
    x = lo.speechlike(3, L)
    out, vad, hw, _ = lo.denoise_loop(x, WIN, N_FFT, lo.profile_mu2(lo.speechlike(4, 960), WIN, N_FFT))
    nf = L // LEN2 - W // LEN2
    assert len(vad) == nf == hw.shape[0] and out.shape == (L,)
    assert not np.any(out[nf * LEN2:])
    if nf > 0:
        assert np.any(out[:nf * LEN2])


def test_too_short_and_dtypes_refused_before_device_work():
    prof = logmmse.NoiseProfile(SR, W, LEN1, LEN2, WIN, N_FFT, np.ones(N_FFT))
    with pytest.raises(ValueError):
        lo.denoise(np.zeros(319, np.float32), WIN, N_FFT, np.ones(N_FFT))
    with pytest.raises(ValueError, match="wav 1 has 319 samples"):
        logmmse.denoise_many([np.zeros(400, np.float32), np.zeros(319, np.float32)], [prof, prof])
    with pytest.raises(ValueError, match="float64"):
        logmmse.denoise(np.zeros(1000), prof)
    with pytest.raises(ValueError, match="int16"):
        logmmse.denoise(np.zeros(1000, np.int16), prof)
    with pytest.raises(ValueError, match="noise 0 has 300 samples"):
        logmmse.profile_noise(np.zeros(300, np.float32), SR)
    with pytest.raises(ValueError, match="another window"):
        other = prof._replace(win=WIN * 2)
        logmmse.denoise_many([np.zeros(400, np.float32)] * 2, [prof, other])


def _create(window_size=320, len1=160, len2=160, n_fft=640):
    cfg = _lib.LogMmseConfig()
    cfg.window_size, cfg.len1, cfg.len2, cfg.n_fft = window_size, len1, len2, n_fft
    h = C.c_void_p()
    return _lib.lib().mb_logmmse_create(C.byref(cfg), C.byref(h)), h


@pytest.mark.parametrize("kw,needle", [
    (dict(window_size=442, len1=221, len2=221, n_fft=884), b"n_fft = 884"),  # 22 050 Hz
    (dict(n_fft=32), b"n_fft = 32"), (dict(n_fft=4096), b"n_fft = 4096"), (dict(n_fft=768), b"n_fft = 768"),
    (dict(window_size=321), b"window_size"), (dict(window_size=700), b"window_size"), (dict(len1=150), b"len1"),
])
def test_create_rejects(kw, needle):
    rc, _ = _create(**kw)
    assert rc == MB_ERR_INVALID
    assert needle in _lib.lib().mb_last_error()


@pytest.mark.parametrize("sr", [8000, 16000, 32000, 12800])
def test_create_accepts_rates_of_supported_sizes(sr):
    W_, l1, l2, _, n = lo.params(sr)
    rc, h = _create(W_, l1, l2, n)
    assert rc == 0
    L = _lib.lib()
    assert L.mb_logmmse_arena_bytes(h) == 4 * ((4 * n + 63) // 64 * 64)
    L.mb_logmmse_destroy(h)


@pytest.mark.parametrize("lengths", [[320], [320, 479, 480, 6401, 160000], [481] * 16])
def test_workspace_arithmetic(lengths):
    L = _lib.lib()
    rc, h = _create()
    assert rc == 0
    a = lambda n: (n + 255) // 256 * 256  # noqa: E731
    nfs = [n // 160 - 2 for n in lengths]
    pairs = sum(max(1, (f + 1) // 2) for f in nfs)
    F = sum(nfs)
    want = a(8 * pairs) + a(24 * len(lengths)) + a(8 * F * 322) + a(8 * F * 320) + 256
    T = lambda ls: (C.c_int32 * len(ls))(*ls)  # noqa: E731
    assert L.mb_logmmse_workspace_bytes(h, len(lengths), T(lengths)) == want
    assert L.mb_logmmse_workspace_bytes(h, len(lengths) + 1, T(lengths + [319])) == 0
    assert L.mb_logmmse_workspace_bytes(h, 0, T([320])) == 0
    L.mb_logmmse_destroy(h)
