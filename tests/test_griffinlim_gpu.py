"""Griffin-Lim on the H100 (mb_griffinlim_*) against the float64 restatement oracle/griffinlim_oracle.py, fed the same
uniforms.  Every error is max|gpu - oracle| / max|oracle|.

Bounds.  The oracle's own algorithm run in numpy float32 (pocketfft) instead of float64, from the same phases, drifts by
(measured on the CPU on the inputs below, reference hparams):
  harmonic 3 s mel:  2.1e-7 after the initial ISTFT, 3.3e-7 after 1 iteration, 8.5e-6 after 60
  random mel (63 frames, uniform in [-4, 4]):  1.8e-7, 2.8e-7, 2.2e-6
The bounds are the initial ISTFT 1e-6, one teacher-forced iteration (the oracle's step applied to the kernel's own
previous output) 2e-6, and 60 iterations 1e-4 (harmonic) / 4e-5 (random), each under 20x the measured drift, with the
spectral convergence within 1e-3 of the oracle's.  The magnitude stage is not read back on its own: the initial ISTFT is
linear in S, so its 1e-6 bound also bounds S.  Inverse pre-emphasis is checked against scipy.signal.lfilter in float64
applied to the kernel's own waveform, to 1e-5."""
import ctypes as C
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import griffinlim_oracle as go
import melspec_oracle as mo
from mockingbird_b200 import _lib
from mockingbird_b200.griffinlim import GriffinLim
from mockingbird_b200.synthesizer.hparams import hparams

pytestmark = pytest.mark.gpu


def _hp(**kw):
    base = {k: getattr(hparams, k) for k in ("sample_rate", "n_fft", "num_mels", "hop_size", "win_size", "fmin", "fmax",
                                             "min_level_db", "ref_level_db", "max_abs_value", "preemphasis", "preemphasize",
                                             "signal_normalization", "allow_clipping_in_normalization", "symmetric_mels",
                                             "power", "griffin_lim_iters", "frame_shift_ms", "use_lws")}
    base.update(kw)
    return SimpleNamespace(**base)


def _handle(hp, pad_mode="reflect"):
    return GriffinLim(go.inv_basis(hp), hp.n_fft, hp.hop_size, hp.win_size, pad_mode=pad_mode, power=hp.power,
                      preemphasis=hp.preemphasis if hp.preemphasize else 0.0, signal_normalization=hp.signal_normalization,
                      allow_clipping=hp.allow_clipping_in_normalization, symmetric=hp.symmetric_mels,
                      max_abs_value=hp.max_abs_value, min_level_db=hp.min_level_db, ref_level_db=hp.ref_level_db)


def _run(g, mels, n_iters, uniforms=None, seeds=None):
    ys = g(mels, n_iters, uniforms=uniforms, seeds=seeds)
    torch.cuda.synchronize()
    return [y.cpu().numpy().astype(np.float64) for y in ys]


def _err(got, ref):
    assert got.shape == ref.shape, (got.shape, ref.shape)
    return float(np.abs(got - ref).max() / np.abs(ref).max())


def _harmonic_mel(seconds=3.0):
    t = np.arange(int(16000 * seconds)) / 16000
    w = sum(np.sin(2 * np.pi * f * t) / (i + 1) for i, f in enumerate([220, 440, 660, 990])) * 0.3
    return mo.synthesizer_mel(w, mo.SYNTH_HP)


def _random_mel(T, seed, lo=-4.0, hi=4.0):
    return (np.random.RandomState(seed).rand(80, T) * (hi - lo) + lo).astype(np.float32)


MELS = {"harmonic": (_harmonic_mel, 1e-4), "random": (lambda: _random_mel(63, 1), 4e-5)}


@pytest.mark.parametrize("pad_mode", ["reflect", "constant"])
@pytest.mark.parametrize("which", list(MELS))
def test_initial_istft_and_one_iteration(which, pad_mode):
    hp = _hp(preemphasize=False)
    mel = MELS[which][0]()
    g = _handle(hp, pad_mode)
    S = go.magnitudes(mel, hp)
    u = np.random.RandomState(5).rand(*S.shape)
    y0 = _run(g, [mel], 0, [u])[0]
    e0 = _err(y0, go.griffin_lim(S, u, 0, 1024, 256, 1024, pad_mode))
    y1 = _run(g, [mel], 1, [u])[0]
    e1 = _err(y1, go.iterate(S, y0, 1024, 256, 1024, pad_mode))
    print(f"{which} {pad_mode}: initial {e0:.2e}, one iteration {e1:.2e}")
    assert e0 <= 1e-6 and e1 <= 2e-6


@pytest.mark.parametrize("which", list(MELS))
def test_sixty_iterations(which):
    make, bound = MELS[which]
    hp = _hp(preemphasize=False)
    mel = make()
    S = go.magnitudes(mel, hp)
    u = np.random.RandomState(5).rand(*S.shape)
    y = _run(_handle(hp), [mel], 60, [u])[0]
    ref = go.griffin_lim(S, u, 60, 1024, 256, 1024)
    e = _err(y, ref)
    sc, sc_ref = go.spectral_convergence(S, y, 1024, 256, 1024), go.spectral_convergence(S, ref, 1024, 256, 1024)
    print(f"{which}: 60 iterations {e:.2e}, spectral convergence {sc:.5f} vs {sc_ref:.5f}")
    assert e <= bound and abs(sc - sc_ref) <= 1e-3


def test_inverse_preemphasis():
    mel = _random_mel(313, 3)
    u = np.random.RandomState(4).rand(513, 313)
    y = _run(_handle(_hp(preemphasize=False)), [mel], 2, [u])[0]
    out = _run(_handle(_hp(preemphasize=True)), [mel], 2, [u])[0]
    assert _err(out, go.inv_preemphasis(y, 0.97)) <= 1e-5


CONFIGS = {
    "n_fft512": dict(n_fft=512, win_size=512, hop_size=128),
    "n_fft2048": dict(n_fft=2048, win_size=2048, hop_size=512),
    "win_lt_n_fft": dict(win_size=800, hop_size=200),
    "power1": dict(power=1.0),
    "asymmetric": dict(symmetric_mels=False),
    "no_normalization": dict(signal_normalization=False),
    "no_clipping": dict(allow_clipping_in_normalization=False),
}


@pytest.mark.parametrize("name", list(CONFIGS))
def test_configs(name):
    hp = _hp(preemphasize=False, **CONFIGS[name])
    if not hp.symmetric_mels:
        mel = _random_mel(57, 6, 0.0, 4.0)
    elif not hp.signal_normalization:
        mel = _random_mel(57, 6, -100.0, -20.0)  # dB - ref_level_db
    else:
        mel = _random_mel(57, 6, -4.5, 4.5)
    g = _handle(hp)
    S = go.magnitudes(mel, hp)
    u = np.random.RandomState(8).rand(*S.shape)
    y0 = _run(g, [mel], 0, [u])[0]
    e0 = _err(y0, go.griffin_lim(S, u, 0, hp.n_fft, hp.hop_size, hp.win_size))
    y1 = _run(g, [mel], 1, [u])[0]
    e1 = _err(y1, go.iterate(S, y0, hp.n_fft, hp.hop_size, hp.win_size))
    print(f"{name}: initial {e0:.2e}, one iteration {e1:.2e}")
    assert e0 <= 1e-6 and e1 <= 2e-6


RAGGED = [4, 5, 17, 63, 313, 1000]


def test_ragged_rows_bitwise_equal_to_single_calls():
    g = _handle(_hp())
    mels = [_random_mel(T, 10 + i) for i, T in enumerate(RAGGED)]
    us = [np.random.RandomState(20 + i).rand(513, T) for i, T in enumerate(RAGGED)]
    seeds = [1000 + i for i in range(len(RAGGED))]
    batch_u = _run(g, mels, 3, uniforms=us)
    batch_s = _run(g, mels, 3, seeds=seeds)
    for i, T in enumerate(RAGGED):
        assert batch_u[i].shape == (256 * (T - 1),)
        assert np.array_equal(batch_u[i], _run(g, [mels[i]], 3, uniforms=[us[i]])[0]), T
        assert np.array_equal(batch_s[i], _run(g, [mels[i]], 3, seeds=[seeds[i]])[0]), T
    # with seeds, a row does not depend on its neighbours
    other = [_random_mel(T, 50 + i) for i, T in enumerate(RAGGED)]
    other[2] = mels[2]
    swapped = _run(g, other, 3, seeds=[7, 8, seeds[2], 9, 10, 11])
    assert np.array_equal(swapped[2], batch_s[2])
    assert not np.array_equal(batch_s[0], _run(g, [mels[0]], 3, seeds=[seeds[0] + 1])[0])


def test_launch_count_independent_of_batch():
    L = _lib.lib()
    g = _handle(_hp())
    counts = []
    for B in (1, 64):
        mels = [_random_mel(20 + b % 7, b) for b in range(B)]
        _run(g, mels, 2, seeds=list(range(B)))  # first call uploads the weights
        before = L.mb_launch_count()
        _run(g, mels, 5, seeds=list(range(B)))
        counts.append(L.mb_launch_count() - before)
    assert counts[0] == counts[1] == 2 * 5 + 4


def test_too_short_refused_without_queuing():
    L = _lib.lib()
    for pad_mode, T in (("reflect", 3), ("constant", 1)):
        g = _handle(_hp(), pad_mode)
        _run(g, [_random_mel(8, 0)], 0, seeds=[0])
        before = L.mb_launch_count()
        with pytest.raises(_lib.MbError, match="utterance 1"):
            g([_random_mel(8, 0), _random_mel(T, 1)], 1, seeds=[0, 1])
        assert L.mb_launch_count() == before
    assert len(_run(_handle(_hp(), "constant"), [_random_mel(2, 0)], 1, seeds=[0])[0]) == 256


def test_drop_in_matches_host_path():
    """np.random.seed(s) then audio.inv_mel_spectrogram against the same on audio_host (torch float64, reflect padding, 60
    iterations and inverse pre-emphasis): same length, dtype float64, final numpy state, within the 60-iteration bound"""
    from mockingbird_b200.synthesizer import audio, audio_host

    mel = _harmonic_mel(1.5)
    np.random.seed(123)
    ref = audio_host.inv_mel_spectrogram(mel, hparams)
    st_ref = np.random.get_state()
    np.random.seed(123)
    got = audio.inv_mel_spectrogram(mel, hparams)
    st = np.random.get_state()
    assert got.dtype == np.float64 and got.shape == ref.shape
    assert np.array_equal(st[1], st_ref[1]) and st[2] == st_ref[2]
    e = _err(got, ref)
    print(f"drop-in vs host: {e:.2e}")
    assert e <= 1e-4


def test_griffin_lim_many_equals_single_calls():
    from mockingbird_b200.synthesizer import audio
    from mockingbird_b200.synthesizer.inference import Synthesizer

    mels = [_random_mel(T, 30 + T) for T in (17, 40, 9)]
    np.random.seed(5)
    many = Synthesizer.griffin_lim_many(mels)
    st_many = np.random.get_state()
    np.random.seed(5)
    single = [audio.inv_mel_spectrogram(m, hparams) for m in mels]
    st = np.random.get_state()
    assert all(np.array_equal(a, b) for a, b in zip(many, single))
    assert np.array_equal(st[1], st_many[1]) and st[2] == st_many[2]
    seeded = Synthesizer.griffin_lim_many(mels, seeds=[1, 2, 3])
    assert all(np.array_equal(a, audio.inv_mel_spectrograms([m], hparams, seeds=[s])[0])
               for a, m, s in zip(seeded, mels, [1, 2, 3]))
