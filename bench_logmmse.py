"""Log-MMSE denoising (mockingbird_b200.logmmse) on one GPU; prints one JSON line.

16 kHz, the reference's parameters (window 320, hop 160, n_fft 640), eta 0.15, seeded speech-like clips
(oracle/logmmse_oracle.speechlike), each with the noise profile of its first and last 0.15 s:
  b1    one 10 s utterance
  b64   64 utterances of 3-10 s (lengths from numpy RandomState(64))
For each: device ms per call (CUDA events around the four launches on device-resident inputs); the whole call
(denoise_many: numpy in, numpy out); the scan kernel's device time (torch.profiler, a run of its own) and that time per frame
step of the longest utterance, the scan being serial in frames; the edge profiles' device ms; and a CPU baseline: the
per-frame numpy loop of oracle/logmmse_oracle.py (float64, the reference's algorithm) over the same clips, labelled as such.
The card name and power limit are read in the same run.

usage: python bench_logmmse.py [--iters N] [--warmup W] [--no-cpu]
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "oracle"))
sys.path.insert(0, str(ROOT / "synth_weights"))

from bench_ppg2mel import card  # noqa: E402
from bench_vc import cuda_timed  # noqa: E402

SR, EDGE = 16000, 2400


def workload(lengths, args):
    import numpy as np
    import torch

    import logmmse_oracle as lo
    from mockingbird_b200 import _lib, logmmse

    clips = [lo.speechlike(1000 + i, n) for i, n in enumerate(lengths)]
    edges = [np.concatenate([c[:EDGE], c[-EDGE:]]) for c in clips]
    profs = logmmse.profile_noise_many(edges, SR)
    p0 = profs[0]
    h = logmmse._handle(p0.window_size, p0.len1, p0.len2, p0.n_fft)
    L = _lib.lib()
    T, ws = h.workspace(lengths)
    x = torch.from_numpy(np.concatenate(clips)).cuda()
    win = torch.from_numpy(p0.win).cuda()
    mu2 = torch.from_numpy(np.stack([p.noise_mu2 for p in profs])).cuda()
    out = torch.empty_like(x)
    nz = torch.from_numpy(np.concatenate(edges)).cuda()
    mu2_out = torch.empty_like(mu2)
    TE = (C.c_int32 * len(edges))(*[len(e) for e in edges])
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)

    def denoise():
        _lib.check(L.mb_logmmse_denoise(h._handle, C.c_void_p(x.data_ptr()), T, len(lengths), C.c_void_p(win.data_ptr()),
                                        C.c_void_p(mu2.data_ptr()), 0.15, C.c_void_p(out.data_ptr()), None,
                                        C.c_void_p(ws.data_ptr()), ws.numel(), stream))

    def profile():
        _lib.check(L.mb_logmmse_profile(h._handle, C.c_void_p(nz.data_ptr()), TE, len(edges), C.c_void_p(win.data_ptr()),
                                        C.c_void_p(mu2_out.data_ptr()), C.c_void_p(ws.data_ptr()), ws.numel(), stream))

    dev_ms, _ = cuda_timed(denoise, args.iters, args.warmup)
    prof_ms, _ = cuda_timed(profile, args.iters, args.warmup)
    for _ in range(args.warmup):
        logmmse.denoise_many(clips, profs)
    t0 = time.perf_counter()
    for _ in range(args.iters):
        got = logmmse.denoise_many(clips, profs)
    whole_ms = (time.perf_counter() - t0) / args.iters * 1e3

    from torch.profiler import ProfilerActivity, profile as tprofile

    torch.cuda.synchronize()
    with tprofile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.iters):
            denoise()
        torch.cuda.synchronize()
    kern = {}
    for e in prof.key_averages():
        for name in ("lm_frame_kernel", "lm_scan_kernel", "lm_inverse_kernel", "lm_ola_kernel"):
            if name in e.key:
                kern[name] = round(e.device_time_total / args.iters / 1e3, 4)
    max_frames = max(n // 160 - 2 for n in lengths)
    audio_s = sum(lengths) / SR
    res = dict(B=len(lengths), audio_s=round(audio_s, 2), frames=sum(n // 160 - 2 for n in lengths), longest_frames=max_frames,
               device_ms=round(dev_ms, 3), whole_call_ms=round(whole_ms, 3), profile_device_ms=round(prof_ms, 4),
               kernel_ms=kern, audio_s_per_s_whole_call=round(audio_s / (whole_ms * 1e-3), 1))
    if "lm_scan_kernel" in kern:
        res["scan_us_per_frame_step"] = round(kern["lm_scan_kernel"] * 1e3 / max_frames, 3)
    if not args.no_cpu:
        t0 = time.perf_counter()
        for c, p in zip(clips, profs):
            lo.denoise_loop(c, p.win, p.n_fft, p.noise_mu2, 0.15)
        res["cpu_oracle_loop_ms"] = round((time.perf_counter() - t0) * 1e3, 1)
        res["cpu_oracle_loop_is"] = "oracle/logmmse_oracle.py per-frame numpy float64 loop on the host CPU"
    res["output_rms"] = float(np.sqrt(np.mean(np.concatenate(got).astype(np.float64) ** 2)))
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--no-cpu", action="store_true")
    args = ap.parse_args()
    import numpy as np
    import torch

    torch.cuda.set_device(0)
    name, power = card()
    out = dict(bench="logmmse", gpu=name, power_limit=power, sample_rate=SR, window=320, hop=160, n_fft=640, eta=0.15)
    loads = {"b1": [10 * SR], "b64": [int(s * SR) for s in np.random.RandomState(64).uniform(3, 10, 64)]}
    for key, lengths in loads.items():
        out[key] = workload(lengths, args)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
