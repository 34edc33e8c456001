"""Griffin-Lim without a GPU: the float64 restatement against the host path and torch.istft, the handle's create-time
checks, the weight-table and call-order errors, the workspace arithmetic and the numpy phase draw."""
import ctypes as C
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import griffinlim_oracle as go
from mockingbird_b200 import _lib
from mockingbird_b200.griffinlim import GriffinLim
from mockingbird_b200.synthesizer import audio_host
from mockingbird_b200.synthesizer.hparams import hparams

MB_ERR_INVALID, MB_ERR_STATE = 1, 2


def _hp(**kw):
    base = {k: getattr(hparams, k) for k in ("sample_rate", "n_fft", "num_mels", "hop_size", "win_size", "fmin", "fmax",
                                             "min_level_db", "ref_level_db", "max_abs_value", "preemphasis", "preemphasize",
                                             "signal_normalization", "allow_clipping_in_normalization", "symmetric_mels",
                                             "power", "griffin_lim_iters", "frame_shift_ms", "use_lws")}
    base.update(kw)
    return SimpleNamespace(**base)


def _config(**kw):
    c = dict(n_fft=1024, hop_length=256, win_length=1024, n_mels=80, pad_mode=0, power=1.5, preemphasis=0.97,
             signal_normalization=1, allow_clipping=1, symmetric=1, max_abs_value=4.0, min_level_db=-100.0, ref_level_db=20.0)
    c.update(kw)
    cfg = _lib.GriffinLimConfig()
    for k, v in c.items():
        setattr(cfg, k, v)
    return cfg


def _create(**kw):
    h = C.c_void_p()
    rc = _lib.lib().mb_griffinlim_create(C.byref(_config(**kw)), C.byref(h))
    return rc, h


@pytest.mark.parametrize("iters", [0, 3])
def test_oracle_matches_host_path(iters):
    """the numpy restatement and audio_host (torch float64 STFT / ISTFT) from the same np.random.seed"""
    hp = _hp(griffin_lim_iters=iters)
    mel = np.random.RandomState(0).rand(80, 37) * 8 - 4
    np.random.seed(11)
    ref = audio_host.inv_mel_spectrogram(mel, hp)
    np.random.seed(11)
    u = np.random.rand(hp.n_fft // 2 + 1, mel.shape[1])
    got = go.inv_mel_spectrogram(mel, hp, u)
    assert got.shape == ref.shape == (256 * 36,)
    assert np.abs(got - ref).max() <= 1e-9 * np.abs(ref).max()


@pytest.mark.parametrize("n_fft,win", [(1024, 1024), (512, 400), (2048, 2048)])
def test_oracle_istft_matches_torch(n_fft, win):
    rng = np.random.RandomState(n_fft)
    Cx = rng.randn(n_fft // 2 + 1, 23) + 1j * rng.randn(n_fft // 2 + 1, 23)
    window = torch.hann_window(win, periodic=True, dtype=torch.float64)
    ref = torch.istft(torch.from_numpy(Cx), n_fft, 256, win, window, center=True).numpy()
    got = go.istft(Cx, n_fft, 256, win)
    assert got.shape == ref.shape
    assert np.abs(got - ref).max() <= 1e-12


@pytest.mark.parametrize("kw,needle", [
    (dict(n_fft=1000), b"n_fft = 1000"), (dict(n_fft=128), b"n_fft = 128"), (dict(n_fft=4096), b"n_fft = 4096"),
    (dict(win_length=1025), b"win_length"), (dict(hop_length=0), b"hop_length"), (dict(win_length=200), b"hop_length"),
    (dict(n_mels=0), b"n_mels"), (dict(pad_mode=2), b"pad_mode"), (dict(power=0.0), b"power"),
    (dict(preemphasis=1.0), b"preemphasis"), (dict(preemphasis=0.999), b"warm-up"), (dict(max_abs_value=0.0), b"max_abs"),
])
def test_create_rejects(kw, needle):
    rc, _ = _create(**kw)
    assert rc == MB_ERR_INVALID
    assert needle in _lib.lib().mb_last_error()


@pytest.mark.parametrize("n_fft", [256, 512, 1024, 2048])
def test_create_accepts_powers_of_two(n_fft):
    rc, h = _create(n_fft=n_fft, win_length=n_fft, hop_length=n_fft // 4)
    assert rc == 0
    _lib.lib().mb_griffinlim_destroy(h)


def test_weight_table_and_call_order():
    L = _lib.lib()
    rc, h = _create()
    assert rc == 0
    t = torch.zeros(513, 80)
    dims = lambda *d: (C.c_int64 * len(d))(*d)  # noqa: E731
    p = C.c_void_p(t.data_ptr())
    assert L.mb_griffinlim_set_weight(h, b"inv_mel_basis", p, dims(513, 80), 2, None) == MB_ERR_STATE  # no arena yet
    assert L.mb_griffinlim_set_weight(h, b"inv_mel_basis", p, dims(80, 513), 2, None) == MB_ERR_INVALID
    assert L.mb_griffinlim_set_weight(h, b"inv_mel_basis", p, dims(513 * 80), 1, None) == MB_ERR_INVALID
    assert L.mb_griffinlim_set_weight(h, b"mel_basis", p, dims(513, 80), 2, None) == MB_ERR_INVALID
    for derived in (b"window", b"twiddles"):
        assert L.mb_griffinlim_set_weight(h, derived, p, dims(1024), 1, None) == MB_ERR_INVALID
        assert b"unknown" in L.mb_last_error()
    assert L.mb_griffinlim_finalize(h, None) == MB_ERR_STATE
    big = C.c_void_p(1 << 32)  # never dereferenced: refused before anything is read
    T = (C.c_int32 * 1)(313)
    before = L.mb_launch_count()
    assert L.mb_griffinlim_forward(h, big, T, 1, big, None, 60, big, big, 1 << 30, None) == MB_ERR_STATE
    assert b"finalized" in L.mb_last_error()
    assert L.mb_launch_count() == before
    nbytes = int(L.mb_griffinlim_arena_bytes(h))
    assert nbytes == 4 * (((513 * 80 + 63) // 64 + (1024 + 63) // 64 + (2048 + 63) // 64) * 64)
    L.mb_griffinlim_destroy(h)


def _expected_workspace(frames, n_fft=1024, hop=256):
    a = lambda n: (n + 255) // 256 * 256  # noqa: E731
    pairs = sum((t + 1) // 2 for t in frames)
    F = sum(frames)
    samples = sum(hop * (t - 1) for t in frames)
    return a(8 * pairs) + a(24 * len(frames)) + a(4 * F * (n_fft // 2 + 1)) + a(4 * F * n_fft) + a(4 * samples) + 256


@pytest.mark.parametrize("frames", [[313], [4, 5, 17, 63, 313, 1000], [1], [2, 3]])
def test_workspace_arithmetic(frames):
    g = GriffinLim(np.zeros((513, 80), np.float32), 1024, 256, 1024)
    assert g.workspace_bytes(frames) == _expected_workspace(frames)
    assert g.workspace_bytes(frames + [0]) == 0
    assert g.workspace_bytes([]) == 0


def test_numpy_phase_draw_matches_per_mel_calls():
    """the draw inv_mel_spectrograms makes: np.random.rand(n_bins, T) per mel in list order, which is what the reference's
    np.random.rand(*S.shape) consumes call after call"""
    frames = [17, 5, 63]
    np.random.seed(7)
    batch = [np.random.rand(513, t) for t in frames]
    state_batch = np.random.get_state()
    np.random.seed(7)
    single = [np.random.rand(*(go.magnitudes(np.zeros((80, t)), _hp()).shape)) for t in frames]
    assert all(np.array_equal(a, b) for a, b in zip(batch, single))
    st = np.random.get_state()
    assert np.array_equal(st[1], state_batch[1]) and st[2] == state_batch[2]


def test_use_lws_refused():
    from mockingbird_b200.synthesizer import audio

    with pytest.raises(NotImplementedError):
        audio.inv_mel_spectrograms([np.zeros((80, 10), np.float32)], _hp(use_lws=True))
