"""Resampling and levelling on the H100 (mb_resample_*, mockingbird_b200.resample) and the loaders built on it, every clip
held bitwise to the host functions it replaces: scipy's resample_poly, numpy's mean square and normalize_volume,
audio_host.preprocess_wav, the host route of Synthesizer.load_preprocess_wav, and the models fed from host arrays."""
import numpy as np
import pytest
import torch
from scipy.io import wavfile
from scipy.signal import resample_poly

import ref_init as ri
from mockingbird_b200 import resample as rs
from mockingbird_b200.synthesizer import audio_host

pytestmark = pytest.mark.gpu

RATIOS = [(44100, 16000), (48000, 16000), (22050, 16000), (24000, 16000), (11025, 16000), (8000, 16000), (16000, 24000),
          (16000, 16000), (44056, 16000)]


def _bits(a, b, what):
    """bitwise equal; a NaN matches a NaN (a silent clip's 0 * inf: the host's and the device's NaN payloads differ)"""
    assert a.dtype == np.float32 and b.dtype == np.float32 and a.shape == b.shape, (what, a.dtype, b.dtype, a.shape, b.shape)
    bad = np.flatnonzero((a.view(np.int32) != b.view(np.int32)) & ~(np.isnan(a) & np.isnan(b)))
    assert bad.size == 0, f"{what}: {bad.size} of {a.size} samples differ, first at {bad[0]}"


def _speechlike(n, seed, peak=0.3):
    rng = np.random.default_rng(seed)
    t = np.arange(n) / 16000.0
    x = np.sin(2 * np.pi * 180 * t) * (0.5 + 0.5 * np.sin(2 * np.pi * 3 * t)) + 0.3 * rng.standard_normal(n)
    return (x / np.abs(x).max() * peak).astype(np.float32)


def _pcm(n, seed):
    return (_speechlike(n, seed, 0.5) * 32767).astype(np.int16)


def _host(x, src, dst):
    up, down = rs.ratio(src, dst)
    xf = x.astype(np.float32) / np.float32(32768) if x.dtype == np.int16 else x
    return xf.copy() if up == down else resample_poly(xf, up, down)


@pytest.mark.parametrize("smem", [-1, 0], ids=["smem_filter", "l2_filter"])
@pytest.mark.parametrize("dtype", ["float32", "int16"])
def test_every_ratio_is_resample_poly(smem, dtype):
    """float32 and int16 input, the default handle (tables up to 64 KB staged in shared memory; 44056 -> 16000 read through
    L2) and a handle that reads every table through L2; lengths 1, 2, shorter than one phase of the filter, and 3 s"""
    h = rs.resampler(filter_smem_bytes=smem)
    for src, dst in RATIOS:
        up, down = rs.ratio(src, dst)
        if up != down:
            assert h.in_smem(up, down) == (smem != 0 and up * -(-(20 * max(up, down) + 1) // up) * 4 <= 64 * 1024)
        per_phase = -(-(20 * max(up, down) + 1) // up)
        lens = [1, 2, max(1, per_phase // 2), 3 * src + 17]
        clips = [_pcm(n, src + n) if dtype == "int16" else _speechlike(n, src + n) for n in lens]
        got = rs.resample_many(clips, src, dst, filter_smem_bytes=smem)
        for n, x, y in zip(lens, clips, got):
            _bits(y, _host(x, src, dst), f"{src} -> {dst}, {dtype}, n = {n}")


def test_mixed_batch_equals_single_calls_in_any_order():
    rng = np.random.default_rng(5)
    items = []
    for k in range(24):
        src = RATIOS[k % len(RATIOS)][0]
        n = int(rng.integers(1, 3 * src))
        items.append((_speechlike(n, 100 + k), src))
    single = [rs.resample_many([x], sr, 16000)[0] for x, sr in items]
    for (x, sr), y in zip(items, single):
        _bits(y, _host(x, sr, 16000), f"single {sr}")
    for seed in (0, 1):
        order = np.random.default_rng(seed).permutation(len(items))
        got = rs.resample_many([items[i][0] for i in order], [items[i][1] for i in order], 16000)
        for i, y in zip(order, got):
            _bits(y, single[i], f"clip {i} in shuffled batch {seed}")
    # different neighbours: every other clip with a 60 s clip at 44.1 kHz in between
    long = _speechlike(60 * 44100, 7)
    sub = items[::2]
    got = rs.resample_many([c for x, sr in sub for c in (x, long)], [s for x, sr in sub for s in (sr, 44100)], 16000)
    for k, (y, ref) in enumerate(zip(got[::2], single[::2])):
        _bits(y, ref, f"clip {2 * k} next to a 60 s clip")
    _bits(got[1], _host(long, 44100, 16000), "60 s clip")


def test_levelling_is_numpy():
    clips = [_speechlike(n, n) * s for n, s in ((1, 1.0), (7, 0.5), (129, 0.01), (16000, 0.001), (960_000, 0.2), (33_333, 1))]
    clips.append(np.zeros(300, np.float32))  # silent: -inf dB, NaN after the gain, as on the host
    dc = rs.DeviceClips(torch.from_numpy(np.concatenate(clips)).cuda(), [c.size for c in clips], 16000)
    ms = rs.mean_squares(dc)
    for i, c in enumerate(clips):
        assert ms[i] == np.mean(c ** 2), i
    with np.errstate(divide="ignore", invalid="ignore"):
        for kw in ({"increase_only": True}, {}, {"decrease_only": True}):
            got = rs.normalize_volume_device(dc, -30, **kw).numpy()
            for i, c in enumerate(clips):
                _bits(got[i], audio_host.normalize_volume(c, -30, **kw), f"normalize_volume {kw} clip {i}")
    got = rs.rescale_device(dc, 0.9).numpy()
    with np.errstate(invalid="ignore"):
        for i, c in enumerate(clips):
            _bits(got[i], c / np.abs(c).max() * 0.9, f"rescale clip {i}")


def _write_wavs(tmp_path, rates, seconds):
    paths = []
    for k, (sr, sec) in enumerate(zip(rates, seconds)):
        p = tmp_path / f"clip{k}_{sr}.wav"
        wavfile.write(p, sr, _pcm(int(sr * sec), 40 + k))
        paths.append(p)
    return paths


def test_preprocess_wavs_is_preprocess_wav(tmp_path):
    from mockingbird_b200.encoder import inference as enc

    paths = _write_wavs(tmp_path, [44100, 48000, 16000, 22050], [2.5, 1.3, 3.0, 0.7])
    arrays = [(_speechlike(30_000, 1), 44100), (_speechlike(9_000, 2) * 0.01, 24000), (_speechlike(5_000, 3), None)]
    items = paths + [a for a, _ in arrays]
    srs = [None] * len(paths) + [sr for _, sr in arrays]
    for normalize in (True, False):
        got = enc.preprocess_wavs(items, srs, normalize=normalize).numpy()
        for i, (x, sr) in enumerate(zip(items, srs)):
            _bits(got[i], enc.preprocess_wav(x, sr, normalize=normalize), f"preprocess_wavs clip {i} normalize={normalize}")


def test_embeddings_from_device_clips(tmp_path):
    from mockingbird_b200.encoder import inference as enc
    from mockingbird_b200.encoder.model import SpeakerEncoder

    m = SpeakerEncoder()
    m.load_state_dict(ri.encoder_state_dict(0))
    m.eval()
    enc.set_model(m)
    paths = _write_wavs(tmp_path, [44100, 48000], [3.2, 2.1])
    items = paths + [_speechlike(44100 * 4, 9), _speechlike(22050 * 2, 10)]
    srs = [None, None, 44100, 22050]
    dc = enc.preprocess_wavs(items, srs)
    got = enc.embed_utterances(dc)
    for i, (x, sr) in enumerate(zip(items, srs)):
        ref = enc.embed_utterances([enc.preprocess_wav(x, sr)])[0]
        _bits(got[i], ref, f"embedding {i}")


def test_load_preprocess_wavs_is_the_host_route(tmp_path):
    from mockingbird_b200 import logmmse
    from mockingbird_b200.synthesizer.hparams import hparams
    from mockingbird_b200.synthesizer.inference import Synthesizer

    sr = hparams.sample_rate
    paths = _write_wavs(tmp_path, [44100, 48000, 16000, 44100, 48000], [2.0, 1.5, 1.2, 0.3, 0.35])
    arr = _speechlike(3 * 22050, 11)
    got = Synthesizer.load_preprocess_wavs(paths + [arr], [None] * len(paths) + [22050])
    host = [audio_host.load_wav(p, sr)[0] for p in paths] + [resample_poly(arr, *rs.ratio(22050, sr))]
    host = [w / np.abs(w).max() * hparams.rescaling_max for w in host]
    edge = int(sr * 0.15)
    for i, w in enumerate(host):
        if len(w) > sr * 0.4:
            p = logmmse.profile_noise(np.concatenate([w[:edge], w[-edge:]]), sr)
            w = logmmse.denoise(w, p)
        _bits(got[i], w, f"load_preprocess_wavs clip {i}")


def test_ppg_extractor_from_device_clips():
    from mockingbird_b200.ppg_extractor import build_model

    m = build_model(ri.PPGX_CONFIG)
    m.load_state_dict(ri.ppg_extractor_state_dict(ri.PPGX_CONFIG, 0))
    m = m.cuda().eval()
    clips = [_speechlike(int(22050 * s), 20 + k) for k, s in enumerate((1.5, 0.8))]
    clips += [_speechlike(int(44100 * s), 30 + k) for k, s in enumerate((1.1, 2.0))]
    srs = [22050, 22050, 44100, 44100]
    dc = rs.resample_device(clips, srs, 16000)
    host = [resample_poly(x, *rs.ratio(sr, 16000)) for x, sr in zip(clips, srs)]
    got = m.extract_batch(dc)
    ref = m.extract_batch(host)
    for i, (a, b) in enumerate(zip(got, ref)):
        assert torch.equal(a, b), f"PPG of clip {i}"
