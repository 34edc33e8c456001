"""Harvest F0 tracking (mb_f0_*, DESIGN §4n) on one GPU, and the voice-conversion chain wav -> wav with real F0; prints one
JSON line.  Seeded synthetic speech-like 16 kHz clips (harvest_oracle.speechlike: harmonic series with F0 glides and
vibrato, digital silences, -60 dBFS noise and noise bursts):
  b1        one 10 s clip: ms per call, and the device time by kernel (torch.profiler in a run of its own)
  batch     64 clips of 3-10 s through compute_f0_many, against 64 single compute_f0 calls
  chain     the PPG extractor's extract_batch -> get_converted_lf0uv_many against one reference clip's statistics ->
            ppg2mel inference_batch -> 24 kHz HiFi-GAN, all with the stand-in seeded weights of bench_ppgx.py, for 16 clips
  cpu       the float64 restatement (oracle/harvest_oracle.py) on the 10 s clip on the host: the restatement, not pyworld
The card name and power limit are read in the same run.
usage: python bench_f0.py [--iters N] [--warmup W] [--no-cpu] [--no-chain]
"""
from __future__ import annotations

import argparse
import json
import re
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "synth_weights"))
sys.path.insert(0, str(ROOT / "oracle"))

from bench_ppg2mel import card  # noqa: E402
from bench_vc import cuda_timed, vocoder  # noqa: E402

SR = 16000


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--no-cpu", action="store_true")
    ap.add_argument("--no-chain", action="store_true")
    a = ap.parse_args()
    import numpy as np
    import torch

    import harvest_oracle as ho
    from mockingbird_b200 import f0_utils as fu

    if not torch.cuda.is_available():
        raise SystemExit("bench_f0.py needs a CUDA device")
    torch.cuda.set_device(0)
    result = {"workload": "Harvest F0 (16 kHz, 10 ms): B = 1 x 10 s; 64 x 3-10 s; VC chain with real F0"}
    result["gpu"], result["power_limit"] = card()
    # ---- one 10 s clip
    x10 = ho.speechlike(1, 10 * SR)
    ms, f0 = cuda_timed(lambda: fu.compute_f0(x10), a.iters, a.warmup)
    result["b1"] = {"audio_s": 10.0, "frames": len(f0), "voiced": int((f0 > 0).sum()), "ms": round(ms, 3),
                    "audio_s_per_s": round(10.0 / (ms / 1e3), 1)}
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fu.compute_f0(x10)
        torch.cuda.synchronize()
    by = {}
    for e in prof.key_averages():
        k = re.search(r"f0_\w+_kernel", e.key)
        if k and e.device_time_total > 0:
            by[k.group(0)] = by.get(k.group(0), 0.0) + e.device_time_total / 1e3
    result["b1"]["device_ms_by_kernel"] = {k: round(v, 3) for k, v in sorted(by.items(), key=lambda kv: -kv[1])}
    result["b1"]["device_ms"] = round(sum(by.values()), 3)
    # ---- 64 clips of 3-10 s
    rng = np.random.default_rng(2)
    clips = [ho.speechlike(10 + i, int(s * SR)) for i, s in enumerate(rng.uniform(3, 10, 64))]
    audio = sum(len(c) for c in clips) / SR
    ms_b, many = cuda_timed(lambda: fu.compute_f0_many(clips), a.iters, 1)
    ms_s, single = cuda_timed(lambda: [fu.compute_f0(c) for c in clips], max(1, a.iters // 2), 1)
    assert all(np.array_equal(p, q) for p, q in zip(many, single))
    result["batch"] = {"clips": 64, "audio_s": round(audio, 2), "ms_many": round(ms_b, 3), "ms_64_single": round(ms_s, 3),
                       "audio_s_per_s": round(audio / (ms_b / 1e3), 1), "speedup": round(ms_s / ms_b, 2)}
    # ---- chain with real F0
    if not a.no_chain:
        import ref_init as ri
        from mockingbird_b200.ppg2mel import MelDecoderMOLv2
        from mockingbird_b200.ppg_extractor import build_model
        from mockingbird_b200.vocoder._gan import infer_waveforms_batched

        m = build_model(ri.PPGX_CONFIG)
        m.load_state_dict(ri.ppg_extractor_state_dict(ri.PPGX_CONFIG, 0))
        m.cuda().eval()
        dec = MelDecoderMOLv2(**ri.PPG2MEL_CONFIG).cuda()
        dec.load_state_dict(ri.ppg2mel_state_dict(0))
        dec.eval()
        voc = vocoder(ri.HIFIGAN_CONFIG_24K, ri.hifigan_state_dict(ri.HIFIGAN_CONFIG_24K, 0), "auto")
        src = clips[:16]
        ref_m, ref_s = fu.compute_mean_std(fu.f02lf0(fu.compute_f0(ho.speechlike(99, 4 * SR))))
        spk = torch.randn(len(src), 256, generator=torch.Generator().manual_seed(4))

        def chain():
            feats = m.extract_batch([torch.from_numpy(c) for c in src])
            lf0s = fu.get_converted_lf0uv_many(src, [ref_m] * len(src), [ref_s] * len(src))
            utts = []
            for p, l in zip(feats, lf0s):
                n = min(p.shape[0], len(l))  # as run.py and the toolbox trim them
                utts.append((p[:n], torch.from_numpy(l[:n]).float().cuda()))
            outs = dec.inference_batch(utts, spk, seed=3)
            return infer_waveforms_batched(voc, "cuda", [o[1].t() for o in outs])

        with torch.no_grad():
            ms_c, wavs = cuda_timed(chain, 2, 1)
        assert all(torch.isfinite(w).all() for w in wavs)
        result["chain"] = {"clips": len(src), "audio_in_s": round(sum(len(c) for c in src) / SR, 2), "ms": round(ms_c, 3),
                           "audio_out_s": round(sum(w.numel() for w in wavs) / 24000, 2)}
    if not a.no_cpu:
        t0 = time.perf_counter()
        ho.harvest(x10)
        result["cpu_restatement"] = {"audio_s": 10.0, "s": round(time.perf_counter() - t0, 3),
                                     "what": "oracle/harvest_oracle.py (float64 numpy), not pyworld"}
    print(json.dumps(result), flush=True)


if __name__ == "__main__":
    main()
