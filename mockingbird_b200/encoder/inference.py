"""Drop-in for ``models/encoder/inference.py`` (reference :15-172): module-global model,
``load_model`` / ``set_model`` / ``is_loaded`` / ``embed_frames_batch`` / ``compute_partial_slices`` /
``embed_utterance``.  The network runs on the H100 (mb_encoder_*); outputs are host numpy like the
reference.  Extensions: ``embed_utterances_frames`` embeds many utterances' partial stacks in one batch, and
``embed_utterances`` is ``embed_utterance`` for a list of waveforms, mels and rows on the device, each result independent
of the list around it.
"""
from __future__ import annotations

from pathlib import Path
from typing import List, Sequence

import numpy as np
import torch

from .. import _lib
from .model import SpeakerEncoder
from .params_data import *  # noqa: F401,F403  (the reference re-exports these, inference.py:1)
from .params_data import mel_n_channels, mel_window_step, partials_n_frames, sampling_rate
from ..synthesizer import audio_host as _audio_host

_model = None  # type: SpeakerEncoder
_device = None  # type: torch.device


def preprocess_wav(fpath_or_wav, source_sr=None, normalize=True, trim_silence=True):
    """re-exported like the reference does from models/encoder/audio.py:19-53 (host utility: load / resample / volume
    normalisation / optional webrtcvad trim)"""
    from .params_data import audio_norm_target_dBFS

    return _audio_host.preprocess_wav(fpath_or_wav, source_sr, normalize, trim_silence, sampling_rate, audio_norm_target_dBFS)


def _have_webrtcvad():
    try:
        import webrtcvad  # noqa: F401
    except Exception:
        return False
    return True


def preprocess_wavs(fpaths_or_wavs, source_srs=None, normalize=True, trim_silence=True, device=None):
    """preprocess_wav for a list of paths and float32 arrays, resampled to 16 kHz and volume-normalised on the device
    (mockingbird_b200.resample): a path is read at its own rate (16-bit mono PCM uploaded as int16), an array is at
    source_srs (one int, or one per clip; None: already 16 kHz).  -> a resample.DeviceClips whose clip i is bitwise
    preprocess_wav(fpaths_or_wavs[i], source_srs[i]) (``.numpy()`` for host arrays; ``embed_utterances`` takes it as it
    is).  Silence trimming runs on the host, clip by clip, and only where webrtcvad is installed, as in preprocess_wav."""
    from .. import resample
    from .params_data import audio_norm_target_dBFS

    clips, rates = resample.load_clips(fpaths_or_wavs, source_srs, sampling_rate)
    out = resample.resample_device(clips, rates, sampling_rate, device)
    if normalize:
        out = resample.normalize_volume_device(out, audio_norm_target_dBFS, increase_only=True)
    if trim_silence and len(out) and _have_webrtcvad():
        trimmed = [_audio_host.trim_long_silences(w, sampling_rate) for w in out.numpy()]
        out = resample.DeviceClips(torch.from_numpy(np.concatenate(trimmed)).to(out.device), [len(w) for w in trimmed],
                                   sampling_rate)
    return out


def load_model(weights_fpath: Path, device=None):
    """inference.py:15-37: checkpoint['model_state'] -> module-global model; returns the model"""
    global _model, _device
    _device = _lib.require_cuda() if device is None or str(device) == "cuda" else torch.device(device)
    _model = SpeakerEncoder(_device, torch.device("cpu"))
    checkpoint = torch.load(weights_fpath, map_location="cpu")
    _model.load_state_dict(checkpoint["model_state"])
    _model.eval()
    _model.to(_device)
    print("Loaded encoder \"%s\" trained to step %d" % (Path(weights_fpath).name, checkpoint["step"]))
    return _model


def set_model(model, device=None):
    global _model, _device
    _model = model
    _device = _lib.require_cuda() if device is None else torch.device(device)
    _model.to(_device)


def is_loaded():
    return _model is not None


def embed_frames_batch(frames_batch):
    """(batch, n_frames, 40) float32 numpy -> (batch, 256) float32 numpy (inference.py:51-64)"""
    if _model is None:
        raise Exception("Model was not loaded. Call load_model() before inference.")
    frames = torch.from_numpy(np.ascontiguousarray(frames_batch, dtype=np.float32))
    return _model.forward(frames).cpu().numpy()


def compute_partial_slices(n_samples, partial_utterance_n_frames=partials_n_frames, min_pad_coverage=0.75, overlap=0.5,
                           rate=None):
    """Where to cut an utterance (waveform samples and mel frames) into partial utterances; same rule
    and defaults as inference.py:66-125."""
    assert 0 <= overlap < 1
    assert 0 < min_pad_coverage <= 1
    samples_per_frame = int(sampling_rate * mel_window_step / 1000)
    n_frames = int(np.ceil((n_samples + 1) / samples_per_frame))
    if rate is not None:
        frame_step = int(np.round((sampling_rate / rate) / samples_per_frame))
    else:
        frame_step = max(int(np.round(partial_utterance_n_frames * (1 - overlap))), 1)
    assert 0 < frame_step, "The rate is too high"
    assert frame_step <= partials_n_frames, "The rate is too low, it should be %f at least" % \
        (sampling_rate / (samples_per_frame * partials_n_frames))
    wav_slices, mel_slices = [], []
    last = max(1, n_frames - partial_utterance_n_frames + frame_step + 1)
    for start in range(0, last, frame_step):
        stop = start + partial_utterance_n_frames
        mel_slices.append(slice(start, stop))
        wav_slices.append(slice(start * samples_per_frame, stop * samples_per_frame))
    tail = wav_slices[-1]
    coverage = (n_samples - tail.start) / (tail.stop - tail.start)
    if coverage < min_pad_coverage and len(mel_slices) > 1:
        mel_slices, wav_slices = mel_slices[:-1], wav_slices[:-1]
    return wav_slices, mel_slices


def embed_utterances_frames(partials: Sequence[np.ndarray]) -> np.ndarray:
    """Batched embed_utterance: partials[u] is the stack of utterance u's partial mel windows
    [P_u, n_frames, 40]; returns [U, 256] = L2(mean_p embed(partial)) (inference.py:160-166)."""
    if _model is None:
        raise Exception("Model was not loaded. Call load_model() before inference.")
    counts = [int(p.shape[0]) for p in partials]
    offsets = np.concatenate([[0], np.cumsum(counts)]).astype(np.int32)
    frames = torch.from_numpy(np.ascontiguousarray(np.concatenate(list(partials), axis=0), dtype=np.float32))
    part = _model.forward(frames)
    return _model.reduce_partials(part, offsets).cpu().numpy()


def embed_utterance_frames(frames: np.ndarray, wav_len: int = None, using_partials=True, return_partials=False, **kwargs):
    """embed_utterance (inference.py:128-172) from the utterance's mel frames [n_frames, 40] (for callers that already
    hold them; embed_utterance(wav) computes them with mockingbird_b200.encoder.audio)."""
    if not using_partials:
        embed = embed_frames_batch(frames[None, ...])[0]
        return (embed, None, None) if return_partials else embed
    samples_per_frame = int(sampling_rate * mel_window_step / 1000)
    n_samples = wav_len if wav_len is not None else max(0, (frames.shape[0] - 1) * samples_per_frame)
    wave_slices, mel_slices = compute_partial_slices(n_samples, **kwargs)
    need = mel_slices[-1].stop
    if need > frames.shape[0]:
        raise ValueError("frames must cover the padded waveform (pad the wav to wave_slices[-1].stop first)")
    frames_batch = np.array([frames[s] for s in mel_slices])
    partial_embeds = embed_frames_batch(frames_batch)
    raw_embed = np.mean(partial_embeds, axis=0)
    embed = raw_embed / np.linalg.norm(raw_embed, 2)
    return (embed, partial_embeds, wave_slices) if return_partials else embed


def embed_utterance(wav, using_partials=True, return_partials=False, **kwargs):
    """inference.py:128-172: wav -> 40-mel frames (device kernel) -> partial slices -> embeddings -> L2(mean)."""
    from . import audio

    if not using_partials:
        frames = audio.wav_to_mel_spectrogram(wav)
        return embed_utterance_frames(frames, using_partials=False, return_partials=return_partials)
    wave_slices, mel_slices = compute_partial_slices(len(wav), **kwargs)
    max_wave_length = wave_slices[-1].stop
    if max_wave_length >= len(wav):
        wav = np.pad(wav, (0, max_wave_length - len(wav)), "constant")
    frames = audio.wav_to_mel_spectrogram(wav)
    frames_batch = np.array([frames[s] for s in mel_slices])
    partial_embeds = embed_frames_batch(frames_batch)
    raw_embed = np.mean(partial_embeds, axis=0)
    embed = raw_embed / np.linalg.norm(raw_embed, 2)
    return (embed, partial_embeds, wave_slices) if return_partials else embed


# rows per mb_encoder_embed_rows call, and rows x longest row per call: a full call's workspace is ~1.2 GB
# (mb_encoder_rows_workspace_bytes(1024, 160), which the model keeps for its lifetime); see DESIGN.md section 4c
MANY_ROWS = 1024
MANY_FRAMES = MANY_ROWS * partials_n_frames


def utterance_rows(n_samples, using_partials=True, **kwargs):
    """How embed_utterance cuts an utterance of n_samples samples: (signal length, wave_slices, row starts, row lengths).
    With partials the rows are the mel_slices of compute_partial_slices over the waveform zero-padded to
    wave_slices[-1].stop (the signal length when that is longer); without, one row of all 1 + n // hop frames."""
    samples_per_frame = int(sampling_rate * mel_window_step / 1000)
    if not using_partials:
        return n_samples, None, [0], [1 + n_samples // samples_per_frame]
    wave_slices, mel_slices = compute_partial_slices(n_samples, **kwargs)
    return (max(n_samples, wave_slices[-1].stop), wave_slices, [s.start for s in mel_slices],
            [s.stop - s.start for s in mel_slices])


def many_plan(row_lens, max_rows=MANY_ROWS, max_frames=MANY_FRAMES):
    """embed_utterances' library calls.  row_lens[u]: utterance u's row lengths.  Utterances are taken longest row first
    (then most rows, then input order) and their rows packed into calls of at most max_rows rows and max_frames rows x
    longest row; an utterance may span calls.  Returns a list of calls, each a list of (u, first row, end row)."""
    if max_rows < 1 or max_frames < 1:
        raise ValueError(f"max_rows = {max_rows} and max_frames = {max_frames} must be positive")
    order = sorted(range(len(row_lens)), key=lambda u: (-max(row_lens[u]), -len(row_lens[u]), u))
    calls, cur, rows, T = [], [], 0, 0
    for u in order:
        for r, n in enumerate(row_lens[u]):
            if rows and (rows + 1 > max_rows or (rows + 1) * max(T, n) > max_frames):
                calls.append(cur)
                cur, rows, T = [], 0, 0
            if cur and cur[-1][0] == u and cur[-1][2] == r:
                cur[-1] = (u, cur[-1][1], r + 1)
            else:
                cur.append((u, r, r + 1))
            rows, T = rows + 1, max(T, n)
    if cur:
        calls.append(cur)
    return calls


def embed_utterances(wavs, using_partials=True, return_partials=False, **kwargs):
    """embed_utterance (inference.py:128-172) for a list of waveforms: [U, 256] float32, or with return_partials a list of
    (embed, partial_embeds, wave_slices) per utterance.  The slices come from compute_partial_slices with the same kwargs for
    every utterance.  Utterances are sorted by length and their mels and rows computed in a few library calls
    (``many_plan``): one mel launch and one mb_encoder_embed_rows per call, the frames never leaving the device.  A result
    is bitwise the same whatever the list around it (order, neighbours, chunking), and within FP32 rounding of
    embed_utterance on the same waveform.  `wavs` may be a resample.DeviceClips (what preprocess_wavs returns): its
    samples go to the mel front-end without leaving the device, with the same results as the same samples from the host."""
    if _model is None:
        raise Exception("Model was not loaded. Call load_model() before inference.")
    from . import audio
    from ..melspec import as_wavs
    from ..resample import DeviceClips

    resident = isinstance(wavs, DeviceClips)
    if not resident:
        wavs = as_wavs(wavs)
    plans = [utterance_rows(len(w), using_partials, **kwargs) for w in wavs]
    audio.check(wavs, [p[0] for p in plans])
    E = _model._cfg.embedding_size
    if not wavs:
        return [] if return_partials else np.zeros((0, E), np.float32)
    offsets = np.concatenate([[0], np.cumsum([len(p[2]) for p in plans])]).astype(np.int64)
    dev = _model.resolved_device()
    part = torch.empty(int(offsets[-1]), E, dtype=torch.float32, device=dev)
    front = audio.mel_front(dev)  # the frames are computed where the encoder reads them
    for call in many_plan([p[3] for p in plans]):
        utts = list(dict.fromkeys(u for u, _, _ in call))
        if resident:
            sel = wavs.select(utts)
            flat, counts = front.many_flat_device(sel.data, sel.lengths, [plans[u][0] for u in utts])
        else:
            flat, counts = front.many_flat([wavs[u] for u in utts], [plans[u][0] for u in utts])
        first = dict(zip(utts, np.concatenate([[0], np.cumsum(counts)[:-1]]).tolist()))
        starts, lens, dst = [], [], []
        for u, r0, r1 in call:
            starts += [first[u] + s for s in plans[u][2][r0:r1]]
            lens += plans[u][3][r0:r1]
            dst += range(int(offsets[u]) + r0, int(offsets[u]) + r1)
        rows = _model.embed_rows(flat.view(-1, mel_n_channels), starts, lens)
        part.index_copy_(0, torch.tensor(dst, dtype=torch.long, device=dev), rows)
    embeds = (_model.reduce_partials(part, offsets.astype(np.int32)) if using_partials else part).cpu().numpy()
    if not return_partials:
        return embeds
    if not using_partials:
        return [(embeds[u], None, None) for u in range(len(wavs))]
    pe = part.cpu().numpy()
    return [(embeds[u], pe[offsets[u]:offsets[u + 1]], plans[u][1]) for u in range(len(wavs))]
