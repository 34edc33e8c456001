"""Text to speech in a cloned voice on the H100: the reference's ``gen_voice.py`` (gen_one_wav and generate_wav,
gen_voice.py:15-118) over many documents in one call.  DESIGN.md section 4p.

``synthesize_wavs(synthesizer, documents, ref_wav)`` reads every document (a list of sentences) in the voice of
``ref_wav`` with one pass of every stage:

    reference   Synthesizer.load_preprocess_wavs([ref_wav]) -> encoder.inference.embed_utterances(...)[0]
    Tacotron    every sentence of every document as its own row (Synthesizer.synthesize_spectrograms_device), the trailing
                silence trimmed on the device
    join mels   each document's sentence mels concatenated on the device
    vocoder     infer_waveforms on the device mels, batches bounded by a workspace budget
    breaks      each document cut at cumsum(frames) * hop_size (numpy's clamped slicing) and 0.15 s of zeros put after every
                sentence, float64, in one launch (mb_tts_join)
    levelling   normalize_volume(wav, -30, increase_only=True) and the 0.97 peak normalisation in float64 on the device;
                webrtcvad's silence trimming on the host in between, where that package is installed

Every document's waveform is what gen_one_wav computes for it, bitwise, with these deliberate differences from the
reference:

* Tacotron runs each sentence as its own row instead of padded batches of 16: the reference's padded rows attend to pad
  tokens, so its result for a sentence depends on the batch around it.
* Dropout comes from per-row Philox seeds, not from torch's global RNG: sentence j of document d draws from row seed
  (seeds[d] + j) mod 2**64, seeds[d] defaulting to the Tacotron model's ``seed``.  A one-document call with the default
  seed is exactly ``synthesize_spectrograms_many(sentences)``, and a document is bitwise its own ``synthesize_wav``
  whatever else is in the call.
* The reference clip is read at its own rate and resampled by resample_poly's filter (DESIGN.md section 4k), as in
  ``run.convert_wavs``.

``generate_wav`` and ``main`` are gen_voice.py's command line: ``python -m mockingbird_b200.gen_voice <text file>
<reference wav>`` writes document ``seq`` (from 1) as ``"%s_%d_%s.wav" % (text file, seq, basename(reference wav))``,
16-bit PCM.
"""
from __future__ import annotations

import argparse
import ctypes as C
import os
import re
from pathlib import Path
from typing import List, Optional, Sequence, Tuple

import numpy as np
import torch

from . import _lib, resample
from .encoder import inference as encoder
from .run import write_pcm16
from .synthesizer import audio_host
from .synthesizer.inference import Synthesizer
from .vocoder.fregan import inference as fregan_inference
from .vocoder.hifigan import inference as hifigan_inference

EACH_NUM = 1500  # characters per document (gen_voice.py:78)
PUNCTUATION = "！，。、,"  # sentence breaks (gen_voice.py:80)
BREAK_SECONDS = 0.15  # silence after every sentence (gen_voice.py:33)
PEAK = 0.97  # peak normalisation (gen_voice.py:42)
VOCODER_WORKSPACE_BUDGET = 4 << 30  # bytes of vocoder workspace one batch of documents may take
_SEED_LIMIT = 1 << 64


def split_documents(text: str, each_num: int = EACH_NUM) -> List[List[str]]:
    """gen_voice.py:76-96: the text's lines split at runs of sentence punctuation; every non-empty piece is kept stripped (a
    whitespace-only piece as ""), and a document ends after the line that takes its stripped length over ``each_num``"""
    documents = []
    processed_texts: List[str] = []
    cur_num = 0
    for line in text.split("\n"):
        for piece in re.sub(r"[{}]+".format(PUNCTUATION), "\n", line).split("\n"):
            if piece:
                processed_texts.append(piece.strip())
                cur_num += len(piece.strip())
        if cur_num > each_num:
            documents.append(processed_texts)
            processed_texts = []
            cur_num = 0
    if len(processed_texts) > 0:
        documents.append(processed_texts)
    return documents


def _check_seed(v, what) -> int:
    if isinstance(v, bool) or not isinstance(v, (int, np.integer)) or not 0 <= int(v) < _SEED_LIMIT:
        raise ValueError(f"{what} = {v!r} is not an integer in [0, 2**64)")
    return int(v)


def _check_arguments(documents, seeds, vocoder):
    docs = []
    for d, doc in enumerate(documents):
        if isinstance(doc, str):
            raise ValueError(f"document {d} is a string; a document is a list of sentences")
        doc = list(doc)
        if not doc:
            raise ValueError(f"document {d} has no sentences")
        docs.append(doc)
    if not docs:
        raise ValueError("no documents to synthesize")
    if seeds is not None:
        seeds = list(seeds)
        if len(seeds) != len(docs):
            raise ValueError(f"{len(seeds)} seeds for {len(docs)} documents")
        seeds = [_check_seed(v, f"seeds[{d}]") for d, v in enumerate(seeds)]
    if vocoder is not hifigan_inference and vocoder is not fregan_inference:
        raise ValueError(f"the vocoder must be mockingbird_b200.vocoder.hifigan.inference or .fregan.inference, got {vocoder!r}")
    if not encoder.is_loaded():
        raise Exception("Model was not loaded. Call load_model() before inference.")
    if not vocoder.is_loaded():
        raise Exception("Please load %s in memory before using it" % ("hifi-gan" if vocoder is hifigan_inference else "fre-gan"))
    return docs, seeds


def reference_embedding(ref_wav, ref_sr=None) -> np.ndarray:
    """gen_voice.py:73-74 on the device: the speaker embedding [256] of the reference clip (a path, or a float32 array at
    ``ref_sr``, default the synthesizer rate)"""
    ref = Synthesizer.load_preprocess_wavs([ref_wav], None if ref_sr is None else [ref_sr])
    return encoder.embed_utterances(ref)[0]


def _join(wavs: Sequence[torch.Tensor], frames: Sequence[Sequence[int]], hop_size: int, zeros: int) -> resample.DeviceClips:
    """gen_voice.py:30-34 for every document in one mb_tts_join launch -> the float64 documents as one DeviceClips"""
    L = _lib.lib()
    pieces = []
    for wav, fr in zip(wavs, frames):
        ends = np.cumsum(np.array(fr, dtype=np.int64) * hop_size)
        starts = np.concatenate(([0], ends[:-1]))
        for a, b in zip(starts.tolist(), ends.tolist()):
            pieces.append(_lib.TtsPiece(wav.data_ptr() if wav.numel() else None, wav.numel(), a, b, zeros, 0))
    n = len(pieces)
    table = (_lib.TtsPiece * n)(*pieces)
    offsets = (C.c_int64 * (n + 1))()
    _lib.check(L.mb_tts_join_plan(table, n, offsets))
    dev = wavs[0].device
    with torch.cuda.device(dev):
        out = torch.empty(offsets[n], dtype=torch.float64, device=dev)
        ws = _lib.workspace(int(L.mb_tts_join_workspace_bytes(n)), dev)
        stream = torch.cuda.current_stream(dev).cuda_stream
        _lib.check(L.mb_tts_join(table, n, C.c_void_p(out.data_ptr()), C.c_void_p(ws.data_ptr()), ws.numel(),
                                 C.c_void_p(stream)))
    first = np.concatenate(([0], np.cumsum([len(fr) for fr in frames]))).tolist()
    lengths = [offsets[first[d + 1]] - offsets[first[d]] for d in range(len(frames))]
    return resample.DeviceClips(out, lengths, Synthesizer.sample_rate)


def _trim_long_silences(clips: resample.DeviceClips) -> resample.DeviceClips:
    """encoder.preprocess_wav's webrtcvad trim (models/encoder/audio.py:68-105), on the host document by document"""
    with np.errstate(invalid="ignore"):  # a NaN document: numpy's cast warns and gives what it gives on the host
        trimmed = [audio_host.trim_long_silences(w, encoder.sampling_rate) for w in clips.numpy()]
    return resample.DeviceClips(torch.from_numpy(np.concatenate(trimmed)).to(clips.device), [len(w) for w in trimmed],
                                clips.sample_rate)


def synthesize_wavs(synthesizer: Synthesizer, documents: Sequence[Sequence[str]], ref_wav, seeds: Optional[Sequence[int]] = None,
                    ref_sr=None, style_idx=-1, min_stop_token=4, steps=400, trim_silences=True, vocoder=hifigan_inference,
                    timeline: Optional[list] = None) -> Tuple[List[np.ndarray], int]:
    """Read every document in the voice of ``ref_wav``: (one float64 waveform per document in input order,
    Synthesizer.sample_rate).  Document i's waveform is gen_one_wav's (gen_voice.py:15-42) for its sentences.

    ``documents``: lists of sentences (``split_documents`` makes them from a text).  ``ref_wav``: a path or a float32 array
    at ``ref_sr``.  ``seeds``: one Tacotron dropout seed per document (sentence j draws from seeds[d] + j); None gives every
    document the Tacotron model's ``seed``.  ``style_idx``, ``min_stop_token``, ``steps``: gen_voice's Tacotron arguments.
    ``trim_silences=False`` skips encoder.preprocess_wav (the volume levelling and the silence trim); the peak
    normalisation still runs.  ``vocoder``: the hifigan or fregan inference module, loaded.  ``timeline`` (a list, for
    measurement): receives a CUDA event before the first stage and (stage name, CUDA event) after each stage.

    Refused with a ValueError before any work is queued: no documents, a document without sentences, a seed count other
    than the document count, a seed outside [0, 2**64), and any other vocoder module; an unloaded encoder or vocoder raises
    the reference's errors.  A document whose sentences are all trimmed to no frames comes out all NaN, as numpy's
    levelling of zeros does (without its warnings)."""
    docs, seeds = _check_arguments(documents, seeds, vocoder)
    if not synthesizer.is_loaded():
        synthesizer.load()
    if seeds is None:
        seeds = [int(synthesizer._model.seed)] * len(docs)
    hp = synthesizer.hparams

    def mark(stage=None):
        if timeline is not None:
            ev = torch.cuda.Event(enable_timing=True)
            ev.record()
            timeline.append(ev if stage is None else (stage, ev))

    mark()
    embed = reference_embedding(ref_wav, ref_sr)
    mark("reference")
    texts = [s for doc in docs for s in doc]
    row_seeds = [(seeds[d] + j) % _SEED_LIMIT for d, doc in enumerate(docs) for j in range(len(doc))]
    with torch.no_grad():
        mels = synthesizer.synthesize_spectrograms_device(texts, [embed] * len(texts), style_idx=style_idx,
                                                          min_stop_token=min_stop_token, steps=steps, seeds=row_seeds)
        mark("tacotron")
        frames, doc_mels, k = [], [], 0
        for doc in docs:
            ms = mels[k:k + len(doc)]
            k += len(doc)
            frames.append([m.shape[1] for m in ms])
            doc_mels.append(torch.cat(ms, dim=1))
        mark("join_mels")
        cap = vocoder.generator.frame_cap(VOCODER_WORKSPACE_BUDGET)
        wavs = vocoder.infer_waveforms(doc_mels, max_frames=cap)
        mark("vocoder")
        out = _join(wavs, frames, hp.hop_size, int(BREAK_SECONDS * synthesizer.sample_rate))
        if trim_silences:
            out = resample.normalize_volume_device(out, encoder.audio_norm_target_dBFS, increase_only=True)
            if encoder._have_webrtcvad():
                out = _trim_long_silences(out)
        out = resample.rescale_device(out, PEAK)
        mark("breaks_levelling")
    result = out.numpy()
    mark("to_host")
    return result, synthesizer.sample_rate


def synthesize_wav(synthesizer: Synthesizer, sentences: Sequence[str], ref_wav, seed: Optional[int] = None, ref_sr=None,
                   **kwargs) -> Tuple[np.ndarray, int]:
    """One document: ``synthesize_wavs`` with one document -> (float64 waveform, Synthesizer.sample_rate)"""
    wavs, sr = synthesize_wavs(synthesizer, [sentences], ref_wav, None if seed is None else [seed], ref_sr, **kwargs)
    return wavs[0], sr


def output_name(file_name, seq: int, in_fpath) -> str:
    """gen_voice.py:45-46: "%s_%d_%s.wav" % (file_name, seq, basename(in_fpath))"""
    return "%s_%d_%s.wav" % (file_name, seq, os.path.basename(in_fpath))


def generate_wav(enc_model_fpath, syn_model_fpath, voc_model_fpath, in_fpath, input_txt, file_name) -> List[str]:
    """gen_voice.py:52-96: load the three models, read every document of ``input_txt`` in the voice of ``in_fpath`` with one
    ``synthesize_wavs`` call and write document seq (from 1) as 16-bit PCM under ``output_name``.  -> the written paths"""
    device = _lib.require_cuda()
    props = torch.cuda.get_device_properties(device)
    print("Found %d GPUs available. Using GPU %d (%s) of compute capability %d.%d with %.1fGb total memory.\n"
          % (torch.cuda.device_count(), device.index, props.name, props.major, props.minor, props.total_memory / 1e9))
    print("Preparing the encoder, the synthesizer and the vocoder...")
    encoder.load_model(Path(enc_model_fpath))
    synthesizer = Synthesizer(Path(syn_model_fpath))
    hifigan_inference.load_model(Path(voc_model_fpath))
    documents = split_documents(input_txt)
    if not documents:
        return []
    wavs, sample_rate = synthesize_wavs(synthesizer, documents, in_fpath)
    written = []
    for seq, wav in enumerate(wavs, 1):
        filename = output_name(file_name, seq, in_fpath)
        write_pcm16(filename, wav, sample_rate)
        print("\nSaved output as %s\n\n" % filename)
        written.append(filename)
    return written


def get_parser():
    """gen_voice.py:98-113: the text file and the reference wav, and the three checkpoints gen_voice hard-codes
    (gen_voice.py:111-113), with its paths as defaults"""
    parser = argparse.ArgumentParser(description="Read a text file aloud in the voice of a reference recording")
    parser.add_argument("text_file", type=str, help="text to read; documents are written one wav each")
    parser.add_argument("wav_file", type=str, help="reference recording of the voice to clone")
    parser.add_argument("--enc_model_fpath", type=str, default="encoder/saved_models/pretrained.pt",
                        help="speaker encoder checkpoint file path")
    parser.add_argument("--syn_model_fpath", type=str, default="synthesizer/saved_models/mandarin.pt",
                        help="synthesizer checkpoint file path")
    parser.add_argument("--voc_model_fpath", type=str, default="vocoder/saved_models/pretrained/g_hifigan.pt",
                        help="HiFi-GAN checkpoint file path (its json config lies in the same directory tree)")
    return parser


def main(argv=None) -> List[str]:
    args = get_parser().parse_args(argv)
    my_txt = ""
    print("reading from :", args.text_file)
    with open(args.text_file, "r") as f:
        for line in f.readlines():
            my_txt += line
    try:  # numerals to Chinese words (gen_voice.py:108) where cn2an is installed, as pypinyin is optional
        import cn2an
    except ImportError:
        output = my_txt
    else:
        output = cn2an.transform(my_txt, "an2cn")
    print(output)
    return generate_wav(Path(args.enc_model_fpath), Path(args.syn_model_fpath), Path(args.voc_model_fpath), args.wav_file,
                        output, args.text_file)


if __name__ == "__main__":
    main()
