"""Voice conversion wav -> wav on the H100: the reference's ``run.py`` (``convert(args)``, run.py:30-94) over many clips.

``convert_wavs(extractor, convertor, src_wavs, ref_wav)`` converts a list of source clips to the reference speaker's voice
in one pass of every stage, each stage one ragged many-clip call:

    reference  encoder.inference.preprocess_wavs -> embed_utterances; compute_mean_std(f02lf0(compute_f0(ref)))
    sources    resample.load_clips -> 16 kHz on the device -> PPGModel.extract_batch
               -> f0_utils.get_converted_lf0uv_many(convert=True) -> both trimmed to min(PPG frames, lf0 frames)
               -> MelDecoderMOLv2.inference_batch(seeds=...) -> postnet mel [80, T]
               -> hifigan.inference.infer_waveforms on the device mels (24 kHz)

Every clip computes what run.py's loop body computes for it.  ppg2mel's PreNet dropout is always on; each clip draws it
from its own stream (``seeds``, default the convertor's own ``seed`` for every clip), so a clip's result is bitwise its
``convert_wav`` call whatever else is converted with it.  The speaker encoder and the vocoder are the module globals of
``encoder.inference`` and ``vocoder.hifigan.inference``, loaded as run.py loads them.

The one host stage is the lf0 / uv post-processing (f0_utils' host functions, which are bitwise the reference's); F0 itself
is tracked on the device from host copies of the 16 kHz clips.  Where the reference reads a source with librosa.load
(sr=16000), a path here is read at its own rate and resampled on the device by resample_poly's filter (DESIGN.md §4k).

``convert(args)``, ``get_parser()`` and ``main()`` are run.py's command line: every ``*.wav`` of ``--wav_dir`` converted to
``--ref_wav_path``'s voice, written as ``vc_{src}_ref_{ref}_step{step}.wav`` (16-bit PCM) under ``--output_dir``.
"""
from __future__ import annotations

import argparse
import glob
import os
import time
from pathlib import Path
from typing import List, Optional, Sequence, Tuple

import numpy as np
import torch

from . import _lib, f0_utils, resample
from .encoder import inference as speaker_encoder
from .vocoder.hifigan import inference as vocoder

SOURCE_SR = 16000  # the PPG extractor's and Harvest's rate (run.py:67)
OUTPUT_SR = 24000  # the vocoder run.py loads (run.py:48): the 24 kHz HiFi-GAN


def _check_loaded():
    if not speaker_encoder.is_loaded():
        raise Exception("Model was not loaded. Call load_model() before inference.")
    if not vocoder.is_loaded():
        raise Exception("Please load hifi-gan in memory before using it")
    if vocoder.output_sample_rate != OUTPUT_SR:
        raise ValueError(f"voice conversion vocodes with the {OUTPUT_SR} Hz HiFi-GAN; the loaded vocoder is "
                         f"{vocoder.output_sample_rate} Hz")


def trim_pair(ppg, lf0_uv):
    """run.py:74-77: the PPG frames and the lf0 / uv frames cut to the shorter of the two"""
    n = min(ppg.shape[0], len(lf0_uv))
    return ppg[:n], lf0_uv[:n]


def reference_voice(ref_wav, ref_sr=None):
    """(speaker embedding [256] float32, lf0 mean, lf0 std) of the reference clip (run.py:51-61)"""
    ref = speaker_encoder.preprocess_wavs([ref_wav], None if ref_sr is None else [ref_sr])
    embed = speaker_encoder.embed_utterances(ref)[0]
    lf0_mean, lf0_std = f0_utils.compute_mean_std(f0_utils.f02lf0(f0_utils.compute_f0(ref.numpy()[0])))
    return embed, lf0_mean, lf0_std


def convert_wavs(extractor, convertor, src_wavs: Sequence, ref_wav, seeds: Optional[Sequence[int]] = None,
                 src_srs=None, ref_sr=None, timeline: Optional[list] = None) -> Tuple[List[np.ndarray], int]:
    """Convert every source clip to the voice of ``ref_wav``: (float32 24 kHz waveforms in input order, 24000).

    ``src_wavs``: paths (read at their own rate) and float32 arrays at ``src_srs`` (one int, or one per clip; None:
    16 kHz).  ``ref_wav``: a path or a float32 array at ``ref_sr``.  ``seeds``: one ppg2mel dropout seed per clip;
    None gives every clip the convertor's ``seed``.  ``timeline`` (a list, for measurement): receives a CUDA event
    before the first stage and (stage name, CUDA event) after each stage, recorded on the current stream."""
    src_wavs = list(src_wavs)
    if not src_wavs:
        raise ValueError("no source clips to convert")
    if seeds is not None and len(seeds) != len(src_wavs):
        raise ValueError(f"{len(seeds)} seeds for {len(src_wavs)} source clips")
    _check_loaded()
    if seeds is None:
        seeds = [convertor.seed] * len(src_wavs)

    def mark(stage=None):
        if timeline is not None:
            ev = torch.cuda.Event(enable_timing=True)
            ev.record()
            timeline.append(ev if stage is None else (stage, ev))

    mark()
    embed, lf0_mean, lf0_std = reference_voice(ref_wav, ref_sr)
    mark("reference")
    clips, rates = resample.load_clips(src_wavs, src_srs, SOURCE_SR)
    src = resample.resample_device(clips, rates, SOURCE_SR)
    mark("load_resample")
    ppgs = extractor.extract_batch(src)
    mark("ppg")
    lf0_uvs = f0_utils.get_converted_lf0uv_many(src.numpy(), [lf0_mean] * len(src), [lf0_std] * len(src), convert=True)
    mark("f0")
    dev = ppgs[0].device
    utts = []
    for ppg, lf0_uv in zip(ppgs, lf0_uvs):
        ppg, lf0_uv = trim_pair(ppg, lf0_uv)
        utts.append((ppg, torch.from_numpy(lf0_uv).float().to(dev)))
    spk = torch.from_numpy(embed).to(dev).expand(len(utts), -1)
    with torch.no_grad():
        outs = convertor.inference_batch(utts, spk, seeds=seeds)
        mark("ppg2mel")
        wavs = vocoder.infer_waveforms([mel_post.transpose(0, 1) for _, mel_post, _ in outs])
        mark("vocoder")
    out = [w.cpu().numpy() for w in wavs]
    mark("to_host")
    return out, OUTPUT_SR


def convert_wav(extractor, convertor, src_wav, ref_wav, seed: Optional[int] = None, src_sr=None,
                ref_sr=None) -> Tuple[np.ndarray, int]:
    """One source clip: ``convert_wavs`` with one clip -> (float32 24 kHz waveform, 24000)"""
    wavs, sr = convert_wavs(extractor, convertor, [src_wav], ref_wav, None if seed is None else [seed],
                            None if src_sr is None else [src_sr], ref_sr)
    return wavs[0], sr


def output_name(output_dir, src_wav_path, ref_wav_path, step) -> str:
    """run.py:83: f"{output_dir}/vc_{src_fid}_ref_{ref_fid}_step{step}.wav", the ids being the file names less 4 characters"""
    src_fid = os.path.basename(src_wav_path)[:-4]
    ref_fid = os.path.basename(ref_wav_path)[:-4]
    return f"{output_dir}/vc_{src_fid}_ref_{ref_fid}_step{step}.wav"


def checkpoint_step(ppg2mel_model_file) -> str:
    """run.py:36: the last '_' field of the checkpoint's file name less its 4-character extension"""
    return os.path.basename(ppg2mel_model_file)[:-4].split("_")[-1]


def write_pcm16(path, wav: np.ndarray, sample_rate: int) -> None:
    """a float waveform as a 16-bit PCM WAV, as libsndfile writes float data as PCM_16: float32 (and any other non-float64
    input) is clipped to [-1, 1], scaled by 32767 in float32 and rounded to the nearest integer (ties to even); float64 is
    scaled by 32767 in float64, rounded the same way and clipped to [-32767, 32767]"""
    from scipy.io import wavfile

    wav = np.asarray(wav)
    if wav.dtype == np.float64:
        pcm = np.clip(np.rint(wav * 32767.0), -32767.0, 32767.0)
    else:
        pcm = np.rint(np.clip(np.asarray(wav, dtype=np.float32), -1.0, 1.0) * np.float32(32767.0))
    wavfile.write(str(path), int(sample_rate), pcm.astype(np.int16))


def _load_yaml(path):
    """utils/hparams.py load_hparams_yaml: the top-level keys of every document of the file"""
    import yaml

    out = {}
    with open(path, "r") as f:
        for doc in yaml.safe_load_all(f):
            out.update(doc)
    return out


def _build_ppg2mel_model(model_config, model_file, device):
    """run.py:20-27"""
    from .ppg2mel import MelDecoderMOLv2

    model = MelDecoderMOLv2(**model_config["model"]).to(device)
    ckpt = torch.load(model_file, map_location="cpu")
    model.load_state_dict(ckpt["model"])
    model.eval()
    return model


@torch.no_grad()
def convert(args):
    """run.py:29-94: every ``*.wav`` under args.wav_dir (sorted) converted in one ``convert_wavs`` call and written as
    16-bit PCM.  Prints the real-time factor of the conversion (its wall time over the converted audio's duration)."""
    from .ppg_extractor import load_model

    device = _lib.require_cuda()
    output_dir = args.output_dir
    os.makedirs(output_dir, exist_ok=True)
    step = checkpoint_step(args.ppg2mel_model_file)

    print("Load PPG-model, PPG2Mel-model, Vocoder-model...")
    ppg_model = load_model(Path(args.ppg_model_file), device)
    ppg2mel_model = _build_ppg2mel_model(_load_yaml(args.ppg2mel_model_train_config), args.ppg2mel_model_file, device)
    vocoder.load_model(args.vocoder_model_file)
    speaker_encoder.load_model(Path(args.encoder_model_file))

    source_file_list = sorted(glob.glob(f"{args.wav_dir}/*.wav"))
    print(f"Number of source utterances: {len(source_file_list)}.")
    start = time.time()
    wavs, sample_rate = convert_wavs(ppg_model, ppg2mel_model, source_file_list, args.ref_wav_path)
    seconds = sum(len(w) for w in wavs) / sample_rate
    for src_wav_path, y in zip(source_file_list, wavs):
        write_pcm16(output_name(output_dir, src_wav_path, args.ref_wav_path, step), y, sample_rate)
    print("RTF:")
    print((time.time() - start) / seconds)


def get_parser():
    """run.py:97-134, and the three checkpoints run.py hard-codes (run.py:40-58), with its paths as defaults"""
    parser = argparse.ArgumentParser(description="Conversion from wave input")
    parser.add_argument("--wav_dir", type=str, default=None, required=True, help="Source wave directory.")
    parser.add_argument("--ref_wav_path", type=str, required=True, help="Reference wave file path.")
    parser.add_argument("--ppg2mel_model_train_config", "-c", type=str, default=None, required=True,
                        help="Training config file (yaml file)")
    parser.add_argument("--ppg2mel_model_file", "-m", type=str, default=None, required=True,
                        help="ppg2mel model checkpoint file path")
    parser.add_argument("--output_dir", "-o", type=str, default="vc_gens_vctk_oneshot",
                        help="Output folder to save the converted wave.")
    parser.add_argument("--ppg_model_file", type=str, default="./ppg_extractor/saved_models/24epoch.pt",
                        help="PPG extractor checkpoint file path (its yaml config lies in the same directory tree)")
    parser.add_argument("--vocoder_model_file", type=str, default="./vocoder/saved_models/24k/g_02830000.pt",
                        help="24 kHz HiFi-GAN checkpoint file path (its json config lies in the same directory tree)")
    parser.add_argument("--encoder_model_file", type=str, default="encoder/saved_models/pretrained_bak_5805000.pt",
                        help="speaker encoder checkpoint file path")
    return parser


def main():
    parser = get_parser()
    args = parser.parse_args()
    convert(args)


if __name__ == "__main__":
    main()
