"""Drop-in for ``models.vocoder.wavernn.inference`` (reference: models/vocoder/wavernn/inference.py:8-64).

``load_model(weights_fpath, verbose=True)`` (the toolbox also passes a config path positionally,
control/toolbox/__init__.py:471, hence ``*ignored``), ``is_loaded()``,
``infer_waveform(mel, normalize=True, batched=True, target=8000, overlap=800, progress_callback=None)``.

Extension: ``infer_waveforms(mels, ...)`` vocodes a list of utterances in one sample loop (the counterpart of the GAN
modules' ``infer_waveforms``).
"""
from __future__ import annotations

from typing import List, Optional, Sequence

import numpy as np
import torch

from ... import _lib
from . import hparams as hp
from .models.fatchord_version import WaveRNN

_model = None  # type: WaveRNN
_device = None


def _build():
    return WaveRNN(
        rnn_dims=hp.voc_rnn_dims,
        fc_dims=hp.voc_fc_dims,
        bits=hp.bits,
        pad=hp.voc_pad,
        upsample_factors=hp.voc_upsample_factors,
        feat_dims=hp.num_mels,
        compute_dims=hp.voc_compute_dims,
        res_out_dims=hp.voc_res_out_dims,
        res_blocks=hp.voc_res_blocks,
        hop_length=hp.hop_length,
        sample_rate=hp.sample_rate,
        mode=hp.voc_mode,
    )


def load_model(weights_fpath, *ignored, verbose=True):
    global _model, _device

    if verbose:
        print("Building Wave-RNN")
    _model = _build()
    _device = _lib.require_cuda()
    _model = _model.cuda()
    if verbose:
        print("Loading model weights at %s" % weights_fpath)
    checkpoint = torch.load(weights_fpath, "cpu")
    _model.load_state_dict(checkpoint['model_state'])
    _model.eval()


def load_state(model_state, rng: str = "torch", seed: int = 0):
    """Install a model from an in-memory ``ckpt['model_state']`` dict (no file)."""
    global _model, _device
    _model = _build()
    _device = _lib.require_cuda()
    _model = _model.cuda()
    _model.load_state_dict(model_state)
    _model.eval()
    _model.rng = rng
    _model.seed = seed
    return _model


def is_loaded():
    return _model is not None


def infer_waveform(mel, normalize=True, batched=True, target=8000, overlap=800, progress_callback=None):
    """Infers the waveform of a mel spectrogram output by the synthesizer (inference.py:45-64)."""
    if _model is None:
        raise Exception("Please load Wave-RNN in memory before using it")

    if normalize:
        mel = mel / hp.mel_max_abs_value
    mel = torch.from_numpy(mel[None, ...])
    wav = _model.generate(mel, batched, target, overlap, hp.mu_law, progress_callback)
    return wav, hp.sample_rate


def split_by_rows(rows: Sequence[int], max_rows: Optional[int]) -> List[List[int]]:
    """Consecutive groups of utterances (input order, so that ``seeds=None`` keeps drawing in the order of the Python loop) of at
    most ``max_rows`` sample-loop rows each; an utterance with more rows than that is a group of its own."""
    groups, cur, n = [], [], 0
    for i, r in enumerate(rows):
        if cur and max_rows is not None and n + r > max_rows:
            groups.append(cur)
            cur, n = [], 0
        cur.append(i)
        n += r
    if cur:
        groups.append(cur)
    return groups


def infer_waveforms(mels: Sequence[np.ndarray], normalize=True, batched=True, target=8000, overlap=800, seeds=None,
                    max_rows=None, progress_callback=None) -> List[np.ndarray]:
    """Vocode many utterances ``[80, T_u]`` in one WaveRNN sample loop (``WaveRNN.generate_many``); the waveforms in input
    order, each equal to ``infer_waveform`` on that utterance alone.  ``seeds=None``: the noise of ``[infer_waveform(m) for m
    in mels]`` under the global torch generator; ``seeds=[s_u]``: utterance u as under ``torch.manual_seed(s_u)``, the
    global generator untouched.  ``max_rows`` splits the list into several loops of at most that many rows (folds, or one
    row per unbatched utterance); the default runs everything in one loop (throughput still rises at 256 rows, DESIGN.md
    section 4.7) - set it to bound the workspace.  In a process group with ``seeds`` given, the utterances are dealt
    to the ranks and rank 0 returns the list (the others ``None``); the result does not depend on the world size."""
    if _model is None:
        raise Exception("Please load Wave-RNN in memory before using it")
    from ... import distributed as mbd
    from .models.fatchord_version import fold_geometry

    mels = [torch.from_numpy((m / hp.mel_max_abs_value if normalize else m)[None, ...]) for m in mels]
    rank, world = mbd.world()
    if world > 1 and seeds is None:
        raise ValueError("infer_waveforms in a process group needs per-utterance seeds: the single global noise stream of "
                         "seeds=None cannot be dealt to ranks")
    mine = mbd.shard_utterances([int(m.shape[-1]) for m in mels], rank, world) if world > 1 else list(range(len(mels)))
    scale = int(np.prod(hp.voc_upsample_factors))  # samples per frame (not hp.hop_length: hparams.py)
    rows = [fold_geometry(int(mels[i].shape[-1]) * scale, target, overlap)[0] if batched else 1 for i in mine]
    local = []
    for group in split_by_rows(rows, max_rows):
        idx = [mine[k] for k in group]
        local += _model.generate_many([mels[i] for i in idx], batched, target, overlap, hp.mu_law,
                                      None if seeds is None else [seeds[i] for i in idx], progress_callback)
    if world == 1:
        return local
    gathered = mbd.gather_object_lists(local, dst=0)
    if rank != 0:
        return None
    shards = [mbd.shard_utterances([int(m.shape[-1]) for m in mels], r, world) for r in range(world)]
    return mbd.merge_sharded(gathered, shards, len(mels))
