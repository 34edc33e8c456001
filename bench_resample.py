"""Resampling and volume levelling (mockingbird_b200.resample, encoder.inference.preprocess_wavs) on one GPU; prints one
JSON line.

256 clips of 2-10 s (lengths from numpy RandomState(256)) of seeded speech-like int16 PCM, at 44.1 kHz and at 48 kHz, to the
encoder's 16 kHz:
  host_preprocess_ms     the host loop of audio_host.preprocess_wav (read, resample_poly, normalize_volume) over the
                         clips as WAV files
  kernel_ms              rs_resample_kernel alone on device-resident int16 clips (CUDA events); with bytes moved (int16 in,
                         float32 out), MACs counted per output sample from the shapes, and the achieved bandwidth
  device_ms              the device part of preprocess_wavs: rs_resample_kernel + rs_sumsq_kernel + rs_scale_kernel
                         (torch.profiler, a run of its own)
  whole_call_ms          preprocess_wavs from the WAV files to device-resident clips (host clock, synchronised)
  embed_*                preprocess_wavs then embed_utterances on the device-resident clips, against the host loop of
                         preprocess_wav then embed_utterances on the host arrays (speaker encoder with seeded weights)
The WAV files (16-bit mono PCM) are written to a temporary directory first; both routes read them.
The card name and power limit are read in the same run.

usage: python bench_resample.py [--iters N] [--warmup W] [--clips B]
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
sys.path.insert(0, str(ROOT / "synth_weights"))

from bench_ppg2mel import card  # noqa: E402
from bench_vc import cuda_timed  # noqa: E402

TARGET = 16000


def clips_at(sr, lengths_s, seed):
    import numpy as np

    rng = np.random.default_rng(seed)
    out = []
    for s in lengths_s:
        n = int(s * sr)
        t = np.arange(n) / sr
        x = np.sin(2 * np.pi * 180 * t) * (0.5 + 0.5 * np.sin(2 * np.pi * 3 * t)) + 0.3 * rng.standard_normal(n)
        out.append((x / np.abs(x).max() * 0.5 * 32767).astype(np.int16))
    return out


def macs(lengths, sr):
    """multiply-adds of the polyphase sums: per output sample, the taps whose input sample lies inside the clip"""
    import numpy as np

    from mockingbird_b200 import resample as rs

    up, down = rs.ratio(sr, TARGET)
    hl = 10 * max(up, down)
    total = 0
    for n in lengths:
        j = np.arange(rs.output_length(n, sr, TARGET), dtype=np.int64)
        cj = j * down + hl
        qmax = np.minimum((2 * hl - cj % up) // up, cj // up)
        qmin = np.maximum(0, cj // up - (n - 1))
        total += int((qmax - qmin + 1).sum())
    return total


def workload(sr, pcm, args, tmp):
    import numpy as np
    from scipy.io import wavfile
    import torch
    from torch.profiler import ProfilerActivity, profile as tprofile

    from mockingbird_b200 import _lib
    from mockingbird_b200 import resample as rs
    from mockingbird_b200.encoder import inference as enc
    from mockingbird_b200.synthesizer import audio_host

    lengths = [c.size for c in pcm]
    paths = []
    for i, c in enumerate(pcm):
        paths.append(Path(tmp) / f"{sr}_{i}.wav")
        wavfile.write(paths[-1], sr, c)
    res = dict(source_sr=sr, clips=len(pcm), audio_s=round(sum(lengths) / sr, 1))

    t0 = time.perf_counter()
    ref = [audio_host.preprocess_wav(p, None, True, False) for p in paths]
    res["host_preprocess_ms"] = round((time.perf_counter() - t0) * 1e3, 1)

    # the kernel alone on resident int16 input
    h = rs.resampler()
    up, down = rs.ratio(sr, TARGET)
    fi = h.filter_index(up, down)
    B = len(pcm)
    x = torch.from_numpy(np.concatenate(pcm)).cuda()
    n_out = [rs.output_length(n, sr, TARGET) for n in lengths]
    out = torch.empty(sum(n_out), dtype=torch.float32, device="cuda")
    L = _lib.lib()
    ws = h.workspace(int(L.mb_resample_workspace_bytes(h._handle, B)))
    lens, fis = (C.c_int32 * B)(*lengths), (C.c_int32 * B)(*[fi] * B)
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)

    def kernel():
        _lib.check(L.mb_resample_forward(h._handle, C.c_void_p(x.data_ptr()), 1, lens, fis, B, C.c_void_p(out.data_ptr()),
                                         C.c_void_p(ws.data_ptr()), ws.numel(), stream))

    k_ms, _ = cuda_timed(kernel, args.iters, args.warmup)
    nbytes = 2 * sum(lengths) + 4 * sum(n_out)
    mac = macs(lengths, sr)
    res.update(kernel_ms=round(k_ms, 4), bytes_moved=nbytes, macs=mac, achieved_GBps=round(nbytes / (k_ms * 1e-3) / 1e9, 1),
               achieved_GMACps=round(mac / (k_ms * 1e-3) / 1e9, 1), filter_in_smem=h.in_smem(up, down))

    def pre():
        return enc.preprocess_wavs(paths, trim_silence=False)

    for _ in range(args.warmup):
        pre()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(args.iters):
        dc = pre()
    torch.cuda.synchronize()
    res["whole_call_ms"] = round((time.perf_counter() - t0) / args.iters * 1e3, 3)
    got = dc.numpy()
    res["bitwise_equal_to_host"] = all(np.array_equal(a.view(np.int32), b.view(np.int32)) for a, b in zip(got, ref))

    with tprofile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.iters):
            pre()
        torch.cuda.synchronize()
    kern = {}
    for e in prof.key_averages():
        for name in ("rs_resample_kernel", "rs_sumsq_kernel", "rs_scale_kernel"):
            if name in e.key:
                kern[name] = kern.get(name, 0.0) + e.device_time_total / args.iters / 1e3
    res["device_ms"] = round(sum(kern.values()), 4)
    res["device_kernel_ms"] = {k: round(v, 4) for k, v in kern.items()}

    # feeding the speaker encoder: device-resident clips against the host route
    enc.embed_utterances(pre())
    enc.embed_utterances(ref[:4])
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    e_dev = enc.embed_utterances(pre())
    res["embed_device_route_ms"] = round((time.perf_counter() - t0) * 1e3, 1)
    t0 = time.perf_counter()
    e_host = enc.embed_utterances([audio_host.preprocess_wav(p, None, True, False) for p in paths])
    res["embed_host_route_ms"] = round((time.perf_counter() - t0) * 1e3, 1)
    res["embed_bitwise_equal"] = bool(np.array_equal(e_dev.view(np.int32), e_host.view(np.int32)))
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--clips", type=int, default=256)
    args = ap.parse_args()
    import numpy as np
    import torch

    import ref_init as ri
    from mockingbird_b200.encoder import inference as enc
    from mockingbird_b200.encoder.model import SpeakerEncoder

    torch.cuda.set_device(0)
    name, power = card()
    m = SpeakerEncoder()
    m.load_state_dict(ri.encoder_state_dict(0))
    m.eval()
    enc.set_model(m)
    secs = np.random.RandomState(256).uniform(2, 10, args.clips)
    out = dict(bench="resample", gpu=name, power_limit=power, target_sr=TARGET, input="int16 PCM")
    import tempfile

    with tempfile.TemporaryDirectory() as tmp:
        for sr in (44100, 48000):
            out[f"sr{sr}"] = workload(sr, clips_at(sr, secs, sr), args, tmp)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
