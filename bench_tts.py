"""Text to speech through the library's entry point (mockingbird_b200.gen_voice, DESIGN §4p) on one GPU; prints one JSON line.

Stand-in seeded weights (synth_weights/ref_init.py): the Tacotron tacotron_state_dict(0, r=2), the speaker encoder
encoder_state_dict(0) and the 16 kHz HiFi-GAN HIFIGAN_CONFIG_16K in the drop-in default precision ("auto").  A seeded 4 s
speech-like reference clip (harvest_oracle.speechlike) and seeded documents of 4-16 sentences of 10-40 pinyin syllables,
read with gen_voice's Tacotron arguments (style_idx=-1, min_stop_token=4, steps=400).
  many     one synthesize_wavs call on all documents: ms, audio seconds per second, and the per-stage split (CUDA events
           recorded between the stages on the current stream)
  single   one synthesize_wav call per document: ms, and the speedup of many
  host     the route gen_voice.py takes with the package's drop-ins, document by document: synthesize_spectrograms (padded
           batches of 16), host np.concatenate, infer_waveform, then gen_one_wav's numpy cut, breaks, encoder.preprocess_wav
           and peak normalisation: ms, and the speedup of many
Every document of many is checked bitwise against its synthesize_wav.  The host route batches sentences by 16 and draws
dropout from torch's global RNG, so its audio differs from the other two (DESIGN §4p); its frames are reported beside.
The card name and power limit are read in the same run.
usage: python bench_tts.py [--iters N] [--warmup W] [--docs N]
"""
from __future__ import annotations

import argparse
import json
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "synth_weights"))
sys.path.insert(0, str(ROOT / "oracle"))

from bench_ppg2mel import card  # noqa: E402

SR = 16000
SYLLABLES = ["ni3", "hao3", "wo3", "men5", "zhong1", "guo2", "ren2", "shi4", "jie4", "da4", "jia1", "xie4", "peng2", "you3",
             "tian1", "qi4", "hen3", "hao3", "jin1", "tian1", "shuo1", "hua4", "xue2", "sheng1"]
TACOTRON_ARGS = dict(style_idx=-1, min_stop_token=4, steps=400)


def standin_models():
    """the stand-in synthesizer; installs the stand-in speaker encoder and 16 kHz vocoder as the module globals"""
    import ref_init as ri
    from mockingbird_b200.encoder import inference as enc
    from mockingbird_b200.encoder.model import SpeakerEncoder
    from mockingbird_b200.synthesizer.inference import Synthesizer
    from mockingbird_b200.vocoder.hifigan import inference as voc

    syn = Synthesizer("unused.pt", verbose=False)
    syn.load_state(ri.tacotron_state_dict(0, r=2, randomize_bn=True))
    m = SpeakerEncoder()
    m.load_state_dict(ri.encoder_state_dict(0))
    enc.set_model(m)
    voc.load_state(ri.hifigan_state_dict(ri.HIFIGAN_CONFIG_16K, 0), ri.HIFIGAN_CONFIG_16K)
    return syn


def documents(n, seed=5):
    import numpy as np

    rng = np.random.default_rng(seed)
    return [[" ".join(rng.choice(SYLLABLES, int(rng.integers(10, 41)))) for _ in range(int(rng.integers(4, 17)))]
            for _ in range(n)]


def host_route(syn, embed, texts):
    """gen_voice.py:15-42 with the package's drop-ins, one document"""
    import numpy as np

    from mockingbird_b200.encoder import inference as enc
    from mockingbird_b200.vocoder.hifigan import inference as voc

    specs = syn.synthesize_spectrograms(texts, [embed] * len(texts), **TACOTRON_ARGS)
    breaks = [spec.shape[1] for spec in specs]
    spec = np.concatenate(specs, axis=1)
    generated_wav, _ = voc.infer_waveform(spec)
    b_ends = np.cumsum(np.array(breaks) * syn.hparams.hop_size)
    b_starts = np.concatenate(([0], b_ends[:-1]))
    wavs = [generated_wav[start:end] for start, end, in zip(b_starts, b_ends)]
    breaks = [np.zeros(int(0.15 * syn.sample_rate))] * len(breaks)
    generated_wav = np.concatenate([i for w, b in zip(wavs, breaks) for i in (w, b)])
    generated_wav = enc.preprocess_wav(generated_wav)
    return generated_wav / np.abs(generated_wav).max() * 0.97, int(spec.shape[1])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=1)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--docs", type=int, default=64)
    a = ap.parse_args()
    import numpy as np
    import torch

    import harvest_oracle as ho
    from mockingbird_b200 import gen_voice
    from mockingbird_b200.vocoder.hifigan import inference as voc

    if not torch.cuda.is_available():
        raise SystemExit("bench_tts.py needs a CUDA device")
    torch.cuda.set_device(0)
    result = {"workload": f"gen_voice.synthesize_wavs: {a.docs} documents of 4-16 sentences of 10-40 pinyin syllables, one 4 s "
                          "reference, stand-in weights (Tacotron r=2 with a 400-frame cap, speaker encoder, 16 kHz HiFi-GAN)"}
    result["gpu"], result["power_limit"] = card()
    syn = standin_models()
    docs = documents(a.docs)
    ref = ho.speechlike(99, 4 * SR)

    def timed(fn, iters, warmup):
        for _ in range(warmup):
            fn()
        torch.cuda.synchronize()
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record()
        for _ in range(iters):
            out = fn()
        t1.record()
        t1.synchronize()
        return t0.elapsed_time(t1) / iters, out

    ms_many, (many, sr) = timed(lambda: gen_voice.synthesize_wavs(syn, docs, ref), a.iters, a.warmup)
    timeline = []
    gen_voice.synthesize_wavs(syn, docs, ref, timeline=timeline)
    timeline[-1][1].synchronize()
    stages, prev = {}, timeline[0]
    for name, ev in timeline[1:]:
        stages[name] = round(prev.elapsed_time(ev), 3)
        prev = ev
    ms_single, single = timed(lambda: [gen_voice.synthesize_wav(syn, d, ref)[0] for d in docs], 1, 0)
    assert all(np.array_equal(p, q, equal_nan=True) for p, q in zip(many, single)), \
        "a document of synthesize_wavs differs from its synthesize_wav"
    embed = gen_voice.reference_embedding(ref)
    torch.manual_seed(0)
    ms_host, host = timed(lambda: [host_route(syn, embed, d) for d in docs], 1, 0)
    sentences = sum(len(d) for d in docs)
    frames = [m.shape[1] for m in syn.synthesize_spectrograms_device(
        [s for d in docs for s in d], [embed] * sentences, seeds=[syn._model.seed + j for d in docs for j in range(len(d))],
        **TACOTRON_ARGS)]
    audio_out = sum(len(w) for w in many) / sr
    result["many"] = {"documents": a.docs, "sentences": sentences, "mel_frames": int(sum(frames)),
                      "audio_out_s": round(audio_out, 2), "ms": round(ms_many, 3),
                      "audio_s_per_s": round(audio_out / (ms_many / 1e3), 1), "stage_ms": stages,
                      "vocoder_mode": voc.generator.precision}
    result["single"] = {"calls": a.docs, "ms": round(ms_single, 3), "audio_s_per_s": round(audio_out / (ms_single / 1e3), 1),
                        "speedup_many": round(ms_single / ms_many, 2)}
    host_audio = sum(len(w) for w, _ in host) / sr
    result["host"] = {"calls": a.docs, "ms": round(ms_host, 3), "mel_frames": int(sum(f for _, f in host)),
                      "audio_out_s": round(host_audio, 2), "audio_s_per_s": round(host_audio / (ms_host / 1e3), 1),
                      "speedup_many": round(ms_host / ms_many, 2)}
    result["bitwise_many_vs_single"] = True
    print(json.dumps(result), flush=True)


if __name__ == "__main__":
    main()
