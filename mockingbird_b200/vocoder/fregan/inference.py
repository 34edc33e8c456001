"""Drop-in for ``models.vocoder.fregan.inference`` (reference: models/vocoder/fregan/inference.py:22-73).

Same module-level protocol: ``load_model(weights_fpath, config_fpath=None, verbose=True)``,
``is_loaded()``, ``infer_waveform(mel, progress_callback=None) -> (wav, sample_rate)`` with module
globals ``generator``, ``_device``, ``output_sample_rate``.  Extension: ``infer_waveforms`` vocodes
a list of utterances as padded batches (the reference vocodes one utterance per call).
"""
from __future__ import annotations

import json
import os
from pathlib import Path
from typing import List, Optional, Sequence

import numpy as np
import torch

from ... import _lib
from ...utils import AttrDict
from .._gan import infer_waveforms_batched
from .models import DEFAULT_CONFIG as DEFAULT_CONFIG_16K, FreGAN as Generator

generator = None  # type: Optional[Generator]
output_sample_rate = None
_device = None
_precision = os.environ.get("MOCKINGBIRD_B200_GAN_PRECISION", "auto")  # auto | f16tc | f16x3 | fp32 (see vocoder/_gan.py)


def set_precision(precision: str) -> None:
    """'auto' (default: f16tc if a load-time probe shows it within 5e-4 of f16x3 for the checkpoint, else f16x3), 'f16tc',
    'f16x3' or 'fp32'; takes effect at the next load_model."""
    global _precision
    if precision != "auto" and precision not in _lib.PRECISIONS:
        raise ValueError(precision)
    _precision = precision


def load_checkpoint(filepath, device):
    assert os.path.isfile(filepath)
    print("Loading '{}'".format(filepath))
    checkpoint_dict = torch.load(filepath, map_location=device)
    print("Complete.")
    return checkpoint_dict


def load_model(weights_fpath, config_fpath=None, verbose=True):
    global generator, _device, output_sample_rate

    if verbose:
        print("Building fregan")
    weights_fpath = Path(weights_fpath)
    if config_fpath is None:
        model_config_fpaths = list(weights_fpath.parent.rglob("*.json"))
        if len(model_config_fpaths) > 0:
            config_fpath = model_config_fpaths[0]
    if config_fpath is not None:
        with open(config_fpath) as f:
            h = AttrDict(json.loads(f.read()))
    else:
        h = AttrDict(DEFAULT_CONFIG_16K)
    output_sample_rate = h.sampling_rate
    torch.manual_seed(h.seed)  # side effect kept: reference reseeds the global RNG here (inference.py:39)

    _device = _lib.require_cuda()
    generator = Generator(h, precision=_precision).to(_device)
    state_dict_g = load_checkpoint(weights_fpath, "cpu")
    generator.load_state_dict(state_dict_g["generator"])
    generator.eval()
    generator.remove_weight_norm()


def load_state(state_dict, h=None, precision: Optional[str] = None):
    """Install a generator from an in-memory ``ckpt['generator']`` dict (no file)."""
    global generator, _device, output_sample_rate
    h = AttrDict(h or DEFAULT_CONFIG_16K)
    output_sample_rate = h.sampling_rate
    _device = _lib.require_cuda()
    generator = Generator(h, precision=precision or _precision).to(_device)
    generator.load_state_dict(state_dict)
    generator.eval()
    generator.remove_weight_norm()
    return generator


def is_loaded():
    return generator is not None


def infer_waveform(mel, progress_callback=None):
    if generator is None:
        raise Exception("Please load fre-gan in memory before using it")

    mel = torch.as_tensor(np.asarray(mel), dtype=torch.float32)
    mel = mel.to(_device, non_blocking=True).unsqueeze(0)
    with torch.no_grad():
        y_g_hat = generator(mel)
        audio = y_g_hat.squeeze()
    audio = audio.cpu().numpy()
    return audio, output_sample_rate


def infer_waveforms(mels: Sequence[np.ndarray], batch_size: int = 32, max_frames: Optional[int] = None) -> List[np.ndarray]:
    """Vocode many utterances as length-sorted padded batches; each result equals the per-utterance
    call (padding is masked at every layer on the device).  ``max_frames`` also bounds each batch's padded frames (rows x
    longest row; default None: no bound).  See ``_gan.infer_waveforms_batched``."""
    if generator is None:
        raise Exception("Please load fre-gan in memory before using it")
    return infer_waveforms_batched(generator, _device, mels, batch_size, max_frames)
