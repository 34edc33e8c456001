"""Drop-in for ``models.synthesizer.inference.Synthesizer`` (reference: models/synthesizer/inference.py:15-143).

Same class surface: ``Synthesizer(model_fpath, verbose=True)``, lazy ``load()``, ``is_loaded()``,
``synthesize_spectrograms(texts, embeddings, return_alignments=False, style_idx=0, min_stop_token=5,
steps=2000)``, class attributes ``sample_rate`` / ``hparams``.  The CPU audio front-end helpers
(load_preprocess_wav, make_spectrogram, griffin_lim, inference.py:144-181) are out of scope.
"""
from __future__ import annotations

from pathlib import Path
from typing import List, Union

import numpy as np
import torch

from .. import _lib
from .hparams import hparams
from .models.tacotron import Tacotron
from .utils.symbols import symbols
from .utils.text import text_to_sequence

try:  # the reference romanises Chinese text with pypinyin (inference.py:100); optional here
    from pypinyin import Style, lazy_pinyin
except Exception:  # pragma: no cover
    lazy_pinyin = None
    Style = None


def pad1d(x, max_len, pad_value=0):
    return np.pad(x, (0, max_len - len(x)), mode="constant", constant_values=pad_value)


class Synthesizer:
    sample_rate = hparams.sample_rate
    hparams = hparams

    def __init__(self, model_fpath: Path, verbose=True):
        self.model_fpath = Path(model_fpath)
        self.verbose = verbose
        self.device = _lib.require_cuda()
        if self.verbose:
            print("Synthesizer using device:", self.device)
        self._model = None

    def is_loaded(self):
        return self._model is not None

    def _build(self) -> Tacotron:
        return Tacotron(embed_dims=hparams.tts_embed_dims, num_chars=len(symbols), encoder_dims=hparams.tts_encoder_dims,
                        decoder_dims=hparams.tts_decoder_dims, n_mels=hparams.num_mels, fft_bins=hparams.num_mels,
                        postnet_dims=hparams.tts_postnet_dims, encoder_K=hparams.tts_encoder_K,
                        lstm_dims=hparams.tts_lstm_dims, postnet_K=hparams.tts_postnet_K,
                        num_highways=hparams.tts_num_highways, dropout=hparams.tts_dropout,
                        stop_threshold=hparams.tts_stop_threshold,
                        speaker_embedding_size=hparams.speaker_embedding_size).to(self.device)

    def load(self):
        model_config_fpaths = list(self.model_fpath.parent.rglob("*.json"))
        if len(model_config_fpaths) > 0 and model_config_fpaths[0].exists():
            hparams.loadJson(model_config_fpaths[0])
        self._model = self._build()
        self._model.load(self.model_fpath, self.device)
        self._model.eval()
        if self.verbose:
            print("Loaded synthesizer \"%s\" trained to step %d" % (self.model_fpath.name, self._model.get_step()))

    def load_state(self, model_state):
        """install weights from an in-memory ``ckpt['model_state']`` dict (no file)"""
        self._model = self._build()
        self._model.load_state_dict(model_state, strict=False)
        self._model.eval()
        return self._model

    def _sequences(self, texts: List[str]):
        """the text front-end of every synthesize_* method (inference.py:97-103): the model is loaded on first use, the
        texts are romanised with pypinyin where it is installed, then turned into symbol ids"""
        if not self.is_loaded():
            self.load()
        if lazy_pinyin is not None:
            texts = [" ".join(lazy_pinyin(v, style=Style.TONE3, neutral_tone_with_five=True)) for v in texts]
        return [text_to_sequence(text, hparams.tts_cleaner_names) for text in texts]

    @staticmethod
    def _embedding_rows(embeddings, n) -> torch.Tensor:
        emb = np.stack([np.asarray(e, dtype=np.float32) for e in embeddings]) if len(embeddings) else np.zeros((0, 256), np.float32)
        if emb.shape[0] != n:
            raise ValueError(f"{emb.shape[0]} speaker embeddings for {n} texts")
        return torch.from_numpy(emb)

    def synthesize_spectrograms(self, texts: List[str], embeddings: Union[np.ndarray, List[np.ndarray]],
                                return_alignments=False, style_idx=0, min_stop_token=5, steps=2000):
        inputs = self._sequences(texts)
        return self.synthesize_from_sequences(inputs, embeddings, return_alignments, style_idx, min_stop_token, steps)

    def synthesize_spectrograms_many(self, texts: List[str], embeddings: Union[np.ndarray, List[np.ndarray]],
                                     return_alignments=False, style_idx=0, min_stop_token=5, steps=2000, seeds=None):
        """synthesize_spectrograms with every text computed as its own batch of one (Tacotron.generate_many): a text's
        spectrogram does not depend on the texts around it.  Same text front-end, postnet output and trailing trim;
        -> list of [80, f_i] host arrays in input order (plus a list of per-text alignments when return_alignments)"""
        inputs = self._sequences(texts)
        emb = self._embedding_rows(embeddings, len(inputs))
        outs = self._model.generate_many(inputs, emb, steps=steps, style_idx=style_idx, min_stop_token=min_stop_token,
                                         seeds=seeds)
        specs, alignments = [], []
        for _, lin, attn in outs:
            m = lin.cpu().numpy()
            # Trim silence from end of each spectrogram (inference.py:135-138)
            while m.shape[1] > 0 and np.max(m[:, -1]) < hparams.tts_stop_threshold:
                m = m[:, :-1]
            specs.append(m)
            alignments.append(attn.cpu().numpy())
        return (specs, alignments) if return_alignments else specs

    def synthesize_spectrograms_device(self, texts: List[str], embeddings: Union[np.ndarray, List[np.ndarray]], style_idx=0,
                                       min_stop_token=5, steps=2000, seeds=None) -> List[torch.Tensor]:
        """synthesize_spectrograms_many left on the device: -> list of [80, f_i] CUDA tensors in input order, each equal to
        synthesize_spectrograms_many's i-th.  The trailing silence is trimmed on the device (mb_tacotron_trim_frames), so
        only the trimmed lengths reach the host."""
        inputs = self._sequences(texts)
        emb = self._embedding_rows(embeddings, len(inputs))
        outs = self._model.generate_many(inputs, emb, steps=steps, style_idx=style_idx, min_stop_token=min_stop_token,
                                         seeds=seeds, trim_threshold=hparams.tts_stop_threshold)
        return [lin for _, lin, _ in outs]

    def synthesize_spectrograms_stream(self, texts: List[str], embeddings: Union[np.ndarray, List[np.ndarray]], style_idx=0,
                                       min_stop_token=5, steps=2000, seeds=None, slots=128):
        """synthesize_spectrograms_many as an iterator that yields each text's spectrogram as soon as it is done
        (Tacotron.generate_stream): ``(i, [80, f_i] host array)`` in the order the texts finish, each equal to
        synthesize_spectrograms_many's i-th.  Same text front-end, postnet output and trailing trim."""
        inputs = self._sequences(texts)
        emb = self._embedding_rows(embeddings, len(inputs))
        outs = self._model.generate_stream(inputs, emb, steps=steps, style_idx=style_idx, min_stop_token=min_stop_token,
                                           seeds=seeds, slots=slots)
        return self._trimmed(outs)

    @staticmethod
    def _trimmed(outs):
        for i, _, lin, _ in outs:
            m = lin.cpu().numpy()
            # Trim silence from end of each spectrogram (inference.py:135-138)
            while m.shape[1] > 0 and np.max(m[:, -1]) < hparams.tts_stop_threshold:
                m = m[:, :-1]
            yield i, m

    @staticmethod
    def load_preprocess_wav(fpath):
        """inference.py:143-158 (host utility): load at the synthesizer rate and rescale.  The reference additionally
        runs the third-party `logmmse` denoiser when the clip is longer than 0.4 s; it is applied here only when that
        optional package is importable."""
        from . import audio_host

        wav = audio_host.load_wav(fpath, hparams.sample_rate)[0]
        if hparams.rescale:
            wav = wav / np.abs(wav).max() * hparams.rescaling_max
        if len(wav) > hparams.sample_rate * (0.3 + 0.1):
            try:
                import logmmse

                noise_wav = np.concatenate([wav[:int(hparams.sample_rate * 0.15)], wav[-int(hparams.sample_rate * 0.15):]])
                wav = logmmse.denoise(wav, logmmse.profile_noise(noise_wav, hparams.sample_rate))
            except ImportError:
                pass
        return wav

    @staticmethod
    def load_preprocess_wavs(fpaths_or_wavs, source_srs=None):
        """the reference's load_preprocess_wav (inference.py:145-159) for a list of clips, on the device from the file's
        samples to the denoised clip: each path is read at its own rate (16-bit mono PCM uploaded as int16), an array is at
        source_srs (one int, or one per clip; None: already at the synthesizer rate) and must hold float32 samples; every
        clip is resampled to the synthesizer rate (mockingbird_b200.resample, bitwise load_wav's resample_poly) and
        rescaled; every clip longer than 0.4 s is then denoised with the noise profile of its first and last 0.15 s, all
        profiles in one launch and all clips in one logmmse.denoise_many.  -> list of float32 waveforms, each bitwise the
        host route (load_wav, rescale, the same denoiser)"""
        from .. import logmmse, resample

        sr = hparams.sample_rate
        clips, rates = resample.load_clips(fpaths_or_wavs, source_srs, sr)
        if not clips:
            return []
        wavs = resample.resample_device(clips, rates, sr)
        if hparams.rescale:
            wavs = resample.rescale_device(wavs, hparams.rescaling_max)
        noisy = [i for i, n in enumerate(wavs.lengths) if n > sr * (0.3 + 0.1)]
        out = wavs.numpy() if len(noisy) < len(wavs) else [None] * len(wavs)
        if noisy:
            edge = int(sr * 0.15)
            loud = wavs.select(noisy)
            edges = resample.DeviceClips(torch.cat([t for w in loud for t in (w[:edge], w[-edge:])]), [2 * edge] * len(noisy),
                                         sr)
            profiles = logmmse.profile_noise_many(edges, sr)
            for i, w in zip(noisy, logmmse.denoise_many(loud, profiles)):
                out[i] = w
        return out

    @staticmethod
    def make_spectrogram(fpath_or_wav):
        """inference.py:160-172: mel spectrogram [80, M] as fed to the synthesizer in training (GPU front-end,
        synthesizer/audio.py)"""
        from . import audio

        wav = Synthesizer.load_preprocess_wav(fpath_or_wav) if isinstance(fpath_or_wav, (str, Path)) else fpath_or_wav
        return audio.melspectrogram(wav, hparams).astype(np.float32)

    @staticmethod
    def griffin_lim(mel):
        """inference.py:174-180: invert a mel spectrogram with Griffin-Lim (host, numpy/torch-CPU)"""
        from . import audio_host

        return audio_host.inv_mel_spectrogram(mel, hparams)

    @staticmethod
    def griffin_lim_many(mels, seeds=None):
        """Griffin-Lim of a list of mel spectrograms [80, T_b] in one sequence of launches on the H100 -> list of float64
        waveforms (synthesizer/audio.py inv_mel_spectrograms: seeds=None draws the phases from numpy's global state as the
        same sequence of griffin_lim calls would)"""
        from . import audio

        return audio.inv_mel_spectrograms(mels, hparams, seeds)

    def synthesize_from_sequences(self, inputs, embeddings, return_alignments=False, style_idx=0, min_stop_token=5,
                                  steps=2000, dropout_masks=None):
        """the part of synthesize_spectrograms after the text front-end (inference.py:104-142)"""
        if not isinstance(embeddings, list):
            embeddings = [embeddings]
        bs = hparams.synthesis_batch_size
        batched_inputs = [inputs[i:i + bs] for i in range(0, len(inputs), bs)]
        batched_embeds = [embeddings[i:i + bs] for i in range(0, len(embeddings), bs)]
        specs = []
        alignments = None
        for i, batch in enumerate(batched_inputs, 1):
            if self.verbose:
                print(f"\n| Generating {i}/{len(batched_inputs)}")
            max_text_len = max(len(text) for text in batch)
            chars = np.stack([pad1d(text, max_text_len) for text in batch])
            speaker_embeds = np.stack(batched_embeds[i - 1])
            chars = torch.tensor(chars).long()
            speaker_embeddings = torch.tensor(speaker_embeds).float()
            _, mels, alignments = self._model.generate(chars, speaker_embeddings, style_idx=style_idx,
                                                       min_stop_token=min_stop_token, steps=steps,
                                                       dropout_masks=dropout_masks)
            mels = mels.detach().cpu().numpy()
            for m in mels:
                # Trim silence from end of each spectrogram (inference.py:135-138)
                while m.shape[1] > 0 and np.max(m[:, -1]) < hparams.tts_stop_threshold:
                    m = m[:, :-1]
                specs.append(m)
        if self.verbose:
            print("\n\nDone.\n")
        return (specs, alignments) if return_alignments else specs
