"""The emotion-vector part of models/synthesizer/preprocess_audio.py (extract_emo) and of preprocess.py (create_emo) on the GPU.

``load_model(dir_or_model)`` takes a downloaded snapshot directory of the emotion model (config.json plus
pytorch_model.bin or model.safetensors) or a loaded ``EmotionExtractorModel``.  ``extract_emo`` is the drop-in: the
feature extractor's normalisation and the model run on the device and the result comes back as numpy, [1, hidden]
(embeddings=True) or [1, num_labels].  The reference passes its model a 1-D tensor, which the conv stack rejects; this
follows the model card's [1, n] batch, the shape both callers expect.  ``extract_emos`` runs a ragged list in batched
device calls, each row bitwise its ``extract_emo``.
"""
from __future__ import annotations

from pathlib import Path
from typing import List, Sequence

import numpy as np
import torch

from .models.wav2emo import EmotionExtractorModel

_model: EmotionExtractorModel | None = None
SAMPLING_RATE = 16000


def load_model(dir_or_model, device=None) -> EmotionExtractorModel:
    global _model
    m = dir_or_model if isinstance(dir_or_model, EmotionExtractorModel) else EmotionExtractorModel.from_pretrained(dir_or_model)
    _model = m.to(device) if device is not None else m.cuda()
    return _model


def is_loaded() -> bool:
    return _model is not None


def _require():
    if _model is None:
        raise RuntimeError("no emotion model: call load_model(<snapshot directory>) first")
    return _model


def _check_rate(sampling_rate: int) -> None:
    if sampling_rate != SAMPLING_RATE:  # Wav2Vec2FeatureExtractor's message
        raise ValueError(f"The model corresponding to this feature extractor: Wav2Vec2FeatureExtractor was trained using a "
                         f"sampling rate of {SAMPLING_RATE}. Please make sure that the provided `raw_speech` input was "
                         f"sampled with {SAMPLING_RATE} and not {sampling_rate}.")


def _clip(x) -> np.ndarray:
    x = np.asarray(x, dtype=np.float32)
    if x.ndim == 2 and x.shape[0] == 1:  # create_emo's np.expand_dims(wav, 0)
        x = x[0]
    if x.ndim != 1:
        raise ValueError(f"expected one clip of samples, got shape {x.shape}")
    return x


def extract_emos(wavs: Sequence, sampling_rate: int = SAMPLING_RATE, embeddings: bool = True, as_tensor: bool = False):
    """emotion embeddings (or logits) of many clips: a list of [hidden] numpy arrays, or with as_tensor a [B, hidden] CUDA
    tensor (what Vits.infer_many(emos=...) takes)"""
    _check_rate(sampling_rate)
    m = _require()
    rows = m.run_clips([_clip(w) for w in wavs])
    out = torch.stack([r[0 if embeddings else 1] for r in rows])
    return out if as_tensor else list(out.cpu().numpy())


def extract_emo(x: np.ndarray, sampling_rate: int, embeddings: bool = False) -> np.ndarray:
    r"""Predict emotions or extract embeddings from raw audio signal: [1, hidden] with embeddings, else [1, num_labels]."""
    return extract_emos([x], sampling_rate, embeddings)[0][None]


def create_emo(synthesizer_root: Path, skip_existing: bool, hparams, n_processes: int | None = None,
               batch_clips: int = 64) -> List[Path]:
    """preprocess.py create_emo: emo/emo-*.npy of shape (hidden,) float32 for every audio-*.npy listed in train.txt, in
    ragged batches of `batch_clips` clips on the device, in this process.  n_processes is accepted for pre.py's keyword call
    and ignored: the reference's process pool cannot share a CUDA context with forked workers, and batching replaces it.
    Returns the files written."""
    wav_dir = Path(synthesizer_root).joinpath("audio")
    metadata_fpath = Path(synthesizer_root).joinpath("train.txt")
    assert wav_dir.exists() and metadata_fpath.exists()
    emo_dir = Path(synthesizer_root).joinpath("emo")
    emo_dir.mkdir(exist_ok=True)
    with metadata_fpath.open("r", encoding="utf-8") as metadata_file:
        metadata = [line.split("|") for line in metadata_file]
    fpaths = [(wav_dir.joinpath(m[0]), emo_dir.joinpath(m[0].replace("audio-", "emo-"))) for m in metadata]
    fpaths = [(w, e) for w, e in fpaths if not (skip_existing and e.exists())]
    written = []
    for i in range(0, len(fpaths), batch_clips):
        chunk = fpaths[i:i + batch_clips]
        emos = extract_emos([np.load(w) for w, _ in chunk], hparams.sample_rate, True)
        for (_, e), v in zip(chunk, emos):
            np.save(e, v.astype(np.float32), allow_pickle=False)
            written.append(e)
    return written
