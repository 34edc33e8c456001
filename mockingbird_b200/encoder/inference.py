"""Drop-in for ``models/encoder/inference.py`` (reference :15-172): module-global model,
``load_model`` / ``set_model`` / ``is_loaded`` / ``embed_frames_batch`` / ``compute_partial_slices`` /
``embed_utterance``.  The network runs on the H100 (mb_encoder_*); outputs are host numpy like the
reference.  Extension: ``embed_utterances_frames`` embeds many utterances' partial stacks in one batch.
"""
from __future__ import annotations

from pathlib import Path
from typing import List, Sequence

import numpy as np
import torch

from .. import _lib
from .model import SpeakerEncoder
from .params_data import *  # noqa: F401,F403  (the reference re-exports these, inference.py:1)
from .params_data import mel_window_step, partials_n_frames, sampling_rate
from ..synthesizer import audio_host as _audio_host

_model = None  # type: SpeakerEncoder
_device = None  # type: torch.device


def preprocess_wav(fpath_or_wav, source_sr=None, normalize=True, trim_silence=True):
    """re-exported like the reference does from models/encoder/audio.py:19-53 (host utility: load / resample / volume
    normalisation / optional webrtcvad trim)"""
    from .params_data import audio_norm_target_dBFS

    return _audio_host.preprocess_wav(fpath_or_wav, source_sr, normalize, trim_silence, sampling_rate, audio_norm_target_dBFS)


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
