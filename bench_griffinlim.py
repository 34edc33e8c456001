"""Griffin-Lim inversion of mel spectrograms (synthesizer/audio.py inv_mel_spectrograms) on one GPU; prints one JSON line.

Reference hparams (n_fft = win = 1024, hop 256, 80 mels, power 1.5, pre-emphasis 0.97) and 60 iterations, on seeded random
normalised mels in [-4, 4]:
  b1    one 5 s utterance (313 frames)
  b16   16 utterances of 3-10 s (lengths from numpy RandomState(16))
  b64   64 utterances of 3-10 s (lengths from numpy RandomState(64))
For each: device ms per call (CUDA events around the launch sequence on device-resident inputs, numpy uniforms and seeds);
the whole call with the numpy phase stream split into host draw, H2D (mels + uniforms), device and D2H; seconds of audio per
second of the whole call, with the numpy stream and with seeds; the bytes the iterations move per frame and iteration over
the device time, against the device-to-device copy bandwidth measured in the same run; and the host path
(audio_host.inv_mel_spectrogram, torch-CPU float64) for b1 and for the first two utterances of b16.
The card name and power limit are read in the same run.

usage: python bench_griffinlim.py [--iters N] [--warmup W] [--no-cpu]
"""
from __future__ import annotations

import argparse
import json
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "synth_weights"))

from bench_ppg2mel import card  # noqa: E402
from bench_vc import cuda_timed  # noqa: E402

SR, HOP, N_FFT, N_BINS, ITERS = 16000, 256, 1024, 513, 60


def frame_iteration_bytes():
    """bytes one frame moves per iteration: the frame kernel reads n_fft samples of y and n_bins magnitudes and writes
    n_fft windowed samples; the overlap-add reads those n_fft samples and writes hop samples (fp32)"""
    return 4 * (N_FFT + N_BINS + N_FFT + N_FFT + HOP)


def copy_bandwidth():
    import torch

    x = torch.empty(256 << 20, dtype=torch.float32, device="cuda")
    y = torch.empty_like(x)
    ms, _ = cuda_timed(lambda: y.copy_(x), 20, 3)
    return 2 * x.numel() * 4 / (ms * 1e-3)


def workload(lengths_frames, hp, args, gl):
    import numpy as np
    import torch

    mels = [(np.random.RandomState(1000 + i).rand(80, T) * 8 - 4).astype(np.float32) for i, T in enumerate(lengths_frames)]
    frames = list(lengths_frames)
    audio_s = sum(HOP * (T - 1) for T in frames) / SR
    flat = torch.from_numpy(np.concatenate([m.reshape(-1) for m in mels])).cuda()
    np.random.seed(0)
    u_dev = torch.from_numpy(np.concatenate([np.random.rand(N_BINS, T).reshape(-1) for T in frames])).cuda()
    seeds = list(range(len(frames)))
    dev_u, _ = cuda_timed(lambda: gl.forward_device(flat, frames, ITERS, uniforms=u_dev), args.iters, args.warmup)
    dev_s, _ = cuda_timed(lambda: gl.forward_device(flat, frames, ITERS, seeds=seeds), args.iters, args.warmup)

    def whole(use_seeds):
        split = {}
        t0 = time.perf_counter()
        us = None if use_seeds else [np.random.rand(N_BINS, T) for T in frames]
        t1 = time.perf_counter()
        fm = torch.from_numpy(np.concatenate([m.reshape(-1) for m in mels])).cuda()
        ud = None if use_seeds else torch.from_numpy(np.concatenate([u.reshape(-1) for u in us])).cuda()
        torch.cuda.synchronize()
        t2 = time.perf_counter()
        ys = gl.forward_device(fm, frames, ITERS, uniforms=ud, seeds=seeds if use_seeds else None)
        torch.cuda.synchronize()
        t3 = time.perf_counter()
        out = [y.cpu().numpy().astype(np.float64) for y in ys]
        t4 = time.perf_counter()
        split.update(host_draw_ms=(t1 - t0) * 1e3, h2d_ms=(t2 - t1) * 1e3, device_ms=(t3 - t2) * 1e3, d2h_ms=(t4 - t3) * 1e3,
                     total_ms=(t4 - t0) * 1e3)
        return split, out

    for _ in range(args.warmup):
        whole(False)
        whole(True)
    runs_u = [whole(False)[0] for _ in range(args.iters)]
    runs_s = [whole(True)[0] for _ in range(args.iters)]
    mean = lambda runs: {k: round(sum(r[k] for r in runs) / len(runs), 3) for k in runs[0]}  # noqa: E731
    wu, ws = mean(runs_u), mean(runs_s)
    F = sum(frames)
    res = dict(B=len(frames), frames=F, audio_s=round(audio_s, 3), device_ms_uniforms=round(dev_u, 3),
               device_ms_seeds=round(dev_s, 3), whole_call_numpy=wu, whole_call_seeds=ws,
               audio_s_per_s_numpy=round(audio_s / (wu["total_ms"] * 1e-3), 1),
               audio_s_per_s_seeds=round(audio_s / (ws["total_ms"] * 1e-3), 1),
               iteration_GBps=round(frame_iteration_bytes() * F * ITERS / (dev_s * 1e-3) / 1e9, 1))
    return res, mels


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--no-cpu", action="store_true")
    args = ap.parse_args()
    import numpy as np
    import torch

    from mockingbird_b200.synthesizer import audio, audio_host
    from mockingbird_b200.synthesizer.hparams import hparams

    torch.cuda.set_device(0)
    name, power = card()
    gl = audio._griffin_lim(hparams)
    bw = copy_bandwidth()
    out = dict(bench="griffinlim", gpu=name, power_limit=power, n_fft=N_FFT, hop=HOP, iterations=ITERS,
               bytes_per_frame_iteration=frame_iteration_bytes(), copy_GBps=round(bw / 1e9, 1))
    frames_of = lambda s: 1 + int(s * SR) // HOP  # noqa: E731
    loads = {"b1": [frames_of(5.0)],
             "b16": [frames_of(s) for s in np.random.RandomState(16).uniform(3, 10, 16)],
             "b64": [frames_of(s) for s in np.random.RandomState(64).uniform(3, 10, 64)]}
    for key, frames in loads.items():
        res, mels = workload(frames, hparams, args, gl)
        res["iteration_share_of_copy_bw"] = round(res["iteration_GBps"] * 1e9 / bw, 3)
        if not args.no_cpu and key in ("b1", "b16"):
            sub = mels[:1] if key == "b1" else mels[:2]
            t0 = time.perf_counter()
            for m in sub:
                audio_host.inv_mel_spectrogram(m, hparams)
            host_s = time.perf_counter() - t0
            res["host_path_s"] = round(host_s, 3)
            res["host_path_utterances"] = len(sub)
            res["host_path_audio_s_per_s"] = round(sum(HOP * (m.shape[1] - 1) for m in sub) / SR / host_s, 2)
        out[key] = res
    print(json.dumps(out))


if __name__ == "__main__":
    main()
