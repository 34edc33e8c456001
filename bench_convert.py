"""Voice conversion wav -> wav through the library's entry point (mockingbird_b200.run, DESIGN §4o) on one GPU; prints one
JSON line.

Stand-in seeded weights, as in bench_ppgx.py / bench_vc.py: the PPG extractor ref_init.PPGX_CONFIG, ppg2mel
ref_init.PPG2MEL_CONFIG with the stop bias lowered by 10 so that every clip runs to its step limit (the step counts do not
depend on the weights' stop decisions), the speaker encoder ref_init.encoder_state_dict(0) and the stand-in 24 kHz HiFi-GAN
in the drop-in default precision ("auto").  Seeded speech-like 16 kHz clips (harvest_oracle.speechlike: voiced glides,
silences, noise bursts), so that the F0 statistics of the conversion are those of voiced speech.
  many     convert_wavs on 64 source clips of 3-10 s to one 4 s reference: ms per call, converted audio seconds per second,
           and the per-stage split (CUDA events recorded between the stages on the current stream)
  single   the same 64 clips as 64 convert_wav calls (run.py's loop, one clip at a time): ms, and the speedup of many
Every clip of many is checked bitwise against its convert_wav.  The card name and power limit are read in the same run.
usage: python bench_convert.py [--iters N] [--warmup W] [--clips N]
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


def standin_models():
    """(extractor, convertor) with the stand-in weights; installs the stand-in speaker encoder and 24 kHz vocoder as the
    module globals convert_wavs uses"""
    import ref_init as ri
    from mockingbird_b200.encoder import inference as enc
    from mockingbird_b200.encoder.model import SpeakerEncoder
    from mockingbird_b200.ppg2mel import MelDecoderMOLv2
    from mockingbird_b200.ppg_extractor import build_model
    from mockingbird_b200.vocoder.hifigan import inference as voc

    ext = build_model(ri.PPGX_CONFIG)
    ext.load_state_dict(ri.ppg_extractor_state_dict(ri.PPGX_CONFIG, 0))
    ext.cuda().eval()
    psd = ri.ppg2mel_state_dict(0)
    psd["decoder.stop_layer.linear_layer.bias"] = psd["decoder.stop_layer.linear_layer.bias"] - 10.0  # run to the step limit
    conv = MelDecoderMOLv2(**ri.PPG2MEL_CONFIG).cuda()
    conv.load_state_dict(psd)
    conv.eval()
    m = SpeakerEncoder()
    m.load_state_dict(ri.encoder_state_dict(0))
    enc.set_model(m)
    voc.load_state(ri.hifigan_state_dict(ri.HIFIGAN_CONFIG_24K, 0), ri.HIFIGAN_CONFIG_24K)
    return ext, conv


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--clips", type=int, default=64)
    a = ap.parse_args()
    import numpy as np
    import torch

    import harvest_oracle as ho
    from mockingbird_b200 import run
    from mockingbird_b200.vocoder.hifigan import inference as voc

    if not torch.cuda.is_available():
        raise SystemExit("bench_convert.py needs a CUDA device")
    torch.cuda.set_device(0)
    result = {"workload": f"run.convert_wavs: {a.clips} source clips of 3-10 s (16 kHz) to one 4 s reference, stand-in "
                          "weights (PPGX_CONFIG, PPG2MEL_CONFIG run to its step limit, 24 kHz HiFi-GAN)"}
    result["gpu"], result["power_limit"] = card()
    ext, conv = standin_models()
    rng = np.random.default_rng(2)
    srcs = [ho.speechlike(10 + i, int(s * SR)) for i, s in enumerate(rng.uniform(3, 10, a.clips))]
    ref = ho.speechlike(99, 4 * SR)
    audio_in = sum(len(c) for c in srcs) / SR

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

    ms_many, (many, sr) = timed(lambda: run.convert_wavs(ext, conv, srcs, ref), a.iters, a.warmup)
    timeline = []
    run.convert_wavs(ext, conv, srcs, ref, timeline=timeline)
    timeline[-1][1].synchronize()
    stages, prev = {}, timeline[0]
    for name, ev in timeline[1:]:
        stages[name] = round(prev.elapsed_time(ev), 3)
        prev = ev
    ms_single, single = timed(lambda: [run.convert_wav(ext, conv, c, ref)[0] for c in srcs], 1, 0)
    assert all(np.array_equal(p, q) for p, q in zip(many, single)), "a clip of convert_wavs differs from its convert_wav"
    audio_out = sum(len(w) for w in many) / sr
    result["many"] = {"clips": a.clips, "audio_in_s": round(audio_in, 2), "audio_out_s": round(audio_out, 2),
                      "ms": round(ms_many, 3), "audio_s_per_s": round(audio_out / (ms_many / 1e3), 1),
                      "stage_ms": stages, "vocoder_mode": voc.generator.precision}
    result["single"] = {"calls": a.clips, "ms": round(ms_single, 3), "audio_s_per_s": round(audio_out / (ms_single / 1e3), 1),
                        "speedup_many": round(ms_single / ms_many, 2)}
    result["bitwise_many_vs_single"] = True
    print(json.dumps(result), flush=True)


if __name__ == "__main__":
    main()
