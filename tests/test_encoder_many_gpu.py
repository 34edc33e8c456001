"""GPU tests of the many-utterance speaker-encoder path: the ragged mel front-end against its single calls (bitwise), the
virtual zero tail against np.pad (bitwise), embed_utterances against the CPU oracle chain and embed_utterance (2e-4), and
every result's independence of the list around it (bitwise), with the tensor-core and the FFMA routes."""
import hashlib
import os
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

import encoder_oracle as eo
import melspec_oracle as mo
import ref_init as ri

pytestmark = pytest.mark.gpu
TOL = 2e-4
ROOT = Path(__file__).resolve().parent.parent


def _wav(n, seed):
    """speech-like: a few harmonics under a slow amplitude envelope, plus noise"""
    rng = np.random.default_rng(seed)
    t = np.arange(n) / 16000.0
    f0 = 100 + 120 * rng.random()
    env = 0.5 + 0.5 * np.sin(2 * np.pi * (1 + 3 * rng.random()) * t + rng.random() * 6) ** 2
    y = sum(np.sin(2 * np.pi * f0 * k * t + rng.random() * 6) / k for k in range(1, 6))
    return (0.1 * env * y + 0.01 * rng.standard_normal(n)).astype(np.float32)


@pytest.fixture
def pad_mode():
    from mockingbird_b200.encoder import audio
    from mockingbird_b200.synthesizer import audio as saudio

    yield lambda m: (setattr(audio, "pad_mode", m), setattr(saudio, "pad_mode", m))
    audio.pad_mode = saudio.pad_mode = "reflect"


@pytest.fixture(scope="module")
def enc():
    from mockingbird_b200.encoder import inference as enc_inf
    from mockingbird_b200.encoder.model import SpeakerEncoder

    m = SpeakerEncoder()
    m.load_state_dict(ri.encoder_state_dict(0))
    m.eval()
    enc_inf.set_model(m)
    return enc_inf


def _ragged_lengths(k, lo, hi, seed):
    return [int(n) for n in np.random.default_rng(seed).integers(lo, hi, k)]


@pytest.mark.parametrize("mode", ["reflect", "constant"])
def test_encoder_mels_equal_single_calls(mode, pad_mode):
    from mockingbird_b200.encoder import audio

    pad_mode(mode)
    lengths = [201, 1600, 16000, 48123] + _ragged_lengths(64, 201, 48124, 1)
    if mode == "constant":
        lengths = [1, 5] + lengths
    wavs = [_wav(n, i) for i, n in enumerate(lengths)]
    got = audio.wav_to_mel_spectrograms(wavs)
    assert len(got) == len(wavs)
    for w, g in zip(wavs, got):
        one = audio.wav_to_mel_spectrogram(w)
        assert g.shape == one.shape == (1 + len(w) // 160, 40) and g.dtype == np.float32
        assert np.array_equal(g, one)


@pytest.mark.parametrize("mode", ["reflect", "constant"])
def test_synthesizer_mels_equal_single_calls(mode, pad_mode):
    """the synthesizer front-end: pre-emphasis must start afresh at each utterance's first sample"""
    from mockingbird_b200.synthesizer import audio
    from mockingbird_b200.synthesizer.hparams import hparams

    pad_mode(mode)
    lengths = [513, 4000, 32000, 48123] + _ragged_lengths(64, 513, 48124, 2)
    wavs = [_wav(n, 100 + i) + 0.5 for i, n in enumerate(lengths)]  # an offset makes a wrong carried-over sample visible
    got = audio.melspectrograms(wavs, hparams)
    for w, g in zip(wavs, got):
        one = audio.melspectrogram(w, hparams)
        assert g.shape == one.shape == (80, 1 + len(w) // hparams.hop_size)
        assert np.array_equal(g, one)
    assert audio.melspectrograms([], hparams) == []


@pytest.mark.parametrize("mode", ["reflect", "constant"])
def test_virtual_zero_tail_equals_np_pad(mode, pad_mode):
    """signal lengths past the stored samples read zeros: bitwise np.pad then a single call, for tails shorter than n_fft / 2
    (the end reflection reaches back into real samples) and longer"""
    from mockingbird_b200.encoder import audio
    from mockingbird_b200.synthesizer import audio as saudio
    from mockingbird_b200.synthesizer.hparams import hparams

    pad_mode(mode)
    w = _wav(3000, 7) + 0.25
    pads = list(range(1, 200)) + [200, 201, 399, 400, 1000, 25600]
    got = audio.mel_front().many([w] * len(pads), [len(w) + p for p in pads])
    for p, g in zip(pads, got):
        assert np.array_equal(g, audio.wav_to_mel_spectrogram(np.pad(w, (0, p)))), p
    pads = [1, 2, 255, 256, 511, 512, 513, 3000]
    got = saudio._mel_front(hparams).many([w] * len(pads), [len(w) + p for p in pads])
    for p, g in zip(pads, got):
        assert np.array_equal(g, saudio.melspectrogram(np.pad(w, (0, p)), hparams)), p


# sha256 of the single-call outputs below, recorded on an H100 from the build before mb_melspec_forward became a
# one-utterance call of the ragged kernel; the same digest came from this build in the same run
MELSPEC_SHA256 = "4a5af318278d84e7631f3042d675de8e72435f24c0a0072a69101bc17c33cd24"


def melspec_digest():
    """sha256 of wav_to_mel_spectrogram and melspectrogram single calls in both pad modes over seeded signals"""
    from mockingbird_b200.encoder import audio
    from mockingbird_b200.synthesizer import audio as saudio
    from mockingbird_b200.synthesizer.hparams import hparams

    outs = []
    try:
        for mode in ("reflect", "constant"):
            audio.pad_mode = saudio.pad_mode = mode
            for i, n in enumerate([201, 1600, 16000, 48123, 160 * 251]):
                outs.append(audio.wav_to_mel_spectrogram(_wav(n, 300 + i)))
            for i, n in enumerate([513, 4000, 32000, 48123]):
                outs.append(saudio.melspectrogram(_wav(n, 400 + i) + 0.5, hparams))
    finally:
        audio.pad_mode = saudio.pad_mode = "reflect"
    return hashlib.sha256(b"".join(o.tobytes() for o in outs)).hexdigest()


def test_single_call_outputs_unchanged():
    digest = melspec_digest()
    print("melspec sha256", digest)
    assert digest == MELSPEC_SHA256


def _oracle_partials(wav, **kwargs):
    from mockingbird_b200.encoder import inference as enc_inf

    wave_slices, mel_slices = enc_inf.compute_partial_slices(len(wav), **kwargs)
    wpad = np.pad(wav, (0, max(0, wave_slices[-1].stop - len(wav))), "constant")
    frames = mo.encoder_mel(wpad)
    pf = torch.from_numpy(np.stack([frames[s] for s in mel_slices]))
    return eo.embed_utterance_partials(ri.encoder_state_dict(0), pf), eo.embed_frames(ri.encoder_state_dict(0), pf).numpy()


@pytest.mark.parametrize("kwargs", [{}, {"overlap": 0.25}, {"rate": 1.3}])
def test_embeddings_match_oracle_and_embed_utterance(enc, kwargs):
    lengths = [16000 * 2, 16000 * 3 + 80, 52340, 25600, 160 * 300, 16000 * 10 - 7]
    wavs = [_wav(n, 500 + i) for i, n in enumerate(lengths)]
    got = enc.embed_utterances(wavs, return_partials=True, **kwargs)
    embeds = enc.embed_utterances(wavs, **kwargs)
    assert embeds.shape == (len(wavs), 256) and embeds.dtype == np.float32
    for w, (e, pe, ws), e2 in zip(wavs, got, embeds):
        assert np.array_equal(e, e2)
        ref, ref_pe = _oracle_partials(w, **kwargs)
        assert np.abs(e - ref).max() < TOL and np.abs(pe - ref_pe).max() < TOL
        e1, pe1, ws1 = enc.embed_utterance(w, return_partials=True, **kwargs)
        assert ws == ws1 == enc.compute_partial_slices(len(w), **kwargs)[0]
        assert np.abs(e - e1).max() < TOL and np.abs(pe - pe1).max() < TOL


def test_whole_utterances_match_oracle(enc):
    """using_partials=False: one row per utterance over all its frames, rows of different lengths in one call"""
    lengths = [16000 * 30, 201, 4000, 16000 * 2 + 33, 16000 * 7]
    wavs = [_wav(n, 600 + i) for i, n in enumerate(lengths)]
    got = enc.embed_utterances(wavs, using_partials=False)
    parts = enc.embed_utterances(wavs, using_partials=False, return_partials=True)
    for w, e, (e2, pe, ws) in zip(wavs, got, parts):
        assert np.array_equal(e, e2) and pe is None and ws is None
        ref = eo.embed_frames(ri.encoder_state_dict(0), torch.from_numpy(mo.encoder_mel(w))[None]).numpy()[0]
        assert np.abs(e - ref).max() < TOL
        assert np.abs(e - enc.embed_utterance(w, using_partials=False)).max() < TOL


def test_empty_list(enc):
    assert enc.embed_utterances([]).shape == (0, 256)
    assert enc.embed_utterances([], return_partials=True) == []


def _independence_lists():
    base = [16000 * 2, 16000 * 10, 26000, 48123, 16000 * 5 + 1, 160 * 400, 31999, 16000 * 3]
    wavs = [_wav(n, 700 + i) for i, n in enumerate(base)]
    big = [_wav(n, 900 + i) for i, n in enumerate(_ragged_lengths(200, 32000, 160000, 3))]
    return wavs, big


def check_batch_independence(enc, using_partials):
    """every result bitwise the same across permutations, subsets, one-element lists, duplicates and a list of more than
    1024 partial rows (several library calls); returns the base results"""
    wavs, big = _independence_lists()
    U = len(wavs)
    ref = enc.embed_utterances(wavs, using_partials=using_partials)
    perm = np.random.default_rng(5).permutation(U)
    assert np.array_equal(enc.embed_utterances([wavs[i] for i in perm], using_partials=using_partials), ref[perm])
    sub = [1, 4, 6]
    assert np.array_equal(enc.embed_utterances([wavs[i] for i in sub], using_partials=using_partials), ref[sub])
    for i in range(U):
        assert np.array_equal(enc.embed_utterances([wavs[i]], using_partials=using_partials)[0], ref[i]), i
    dup = [3, 0, 3, 5, 0]
    assert np.array_equal(enc.embed_utterances([wavs[i] for i in dup], using_partials=using_partials), ref[dup])
    mixed = big[:100] + wavs + big[100:]
    rows = sum(len(enc.utterance_rows(len(w), using_partials)[2]) for w in mixed)
    calls = enc.many_plan([enc.utterance_rows(len(w), using_partials)[3] for w in mixed])
    if using_partials:
        assert rows > 1024 and len(calls) > 1
    got = enc.embed_utterances(mixed, using_partials=using_partials)
    assert np.array_equal(got[100:100 + U], ref)
    return ref


@pytest.mark.parametrize("using_partials", [True, False])
def test_results_independent_of_the_list(enc, using_partials):
    ref = check_batch_independence(enc, using_partials)
    wavs, _ = _independence_lists()
    for w, e in zip(wavs[:3], ref[:3]):
        assert np.abs(e - enc.embed_utterance(w, using_partials=using_partials)).max() < TOL


_FFMA_SCRIPT = """
import sys
sys.path[:0] = [{root!r}, {root!r} + '/oracle', {root!r} + '/synth_weights', {root!r} + '/tests']
import numpy as np
import ref_init as ri
import test_encoder_many_gpu as t
from mockingbird_b200.encoder import inference as enc
from mockingbird_b200.encoder.model import SpeakerEncoder
m = SpeakerEncoder()
m.load_state_dict(ri.encoder_state_dict(0))
enc.set_model(m)
for up in (True, False):
    ref = t.check_batch_independence(enc, up)
    wavs, _ = t._independence_lists()
    for w, e in zip(wavs[:3], ref[:3]):
        assert np.abs(e - enc.embed_utterance(w, using_partials=up)).max() < t.TOL
print("ffma route independent")
"""


def test_results_independent_of_the_list_ffma_route():
    """the same with MB_ENC_TC=0 (FP32 GEMMs of one fmaf chain per output at every row count); the switch is read once per
    process"""
    env = dict(os.environ, MB_ENC_TC="0")
    proc = subprocess.run([sys.executable, "-c", _FFMA_SCRIPT.format(root=str(ROOT))], env=env, capture_output=True, text=True,
                          timeout=1800)
    assert proc.returncode == 0, proc.stdout[-2000:] + proc.stderr[-4000:]
    assert "ffma route independent" in proc.stdout


def test_frames_must_be_on_the_model_device(enc):
    """embed_rows refuses frames it cannot read in place (another device, the host, another dtype or layout) before
    anything is queued; embed_utterances computes its frames on the model's device, also for a device given without index"""
    from mockingbird_b200 import _lib
    from mockingbird_b200.encoder import audio

    m = enc._model
    dev = m.resolved_device()
    assert dev.index is not None and audio.mel_front(dev)._device == dev
    good = torch.zeros(320, 40, device=dev)
    assert m.embed_rows(good, [0, 160], [160, 160]).shape == (2, 256)
    for bad in (torch.zeros(320, 40), good.double(), good[:, :20],
                torch.zeros(320, 40, device=dev).t()):
        with pytest.raises(_lib.MbError, match="embed_rows: frames must be"):
            m.embed_rows(bad, [0], [160])
    w = _wav(16000 * 3, 11)
    ref = enc.embed_utterances([w])
    enc.set_model(m, "cuda")  # no device index: the current device
    try:
        assert np.array_equal(enc.embed_utterances([w]), ref)
    finally:
        enc.set_model(m, dev)
