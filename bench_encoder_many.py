"""Many utterances through the speaker encoder (encoder.inference.embed_utterances) against one embed_utterance per
utterance; prints one JSON line.

Workload: U = 256 seeded speech-like signals of 2-10 s at 16 kHz (harmonics under a slow envelope plus noise), random-init
encoder weights (synth_weights/ref_init.py), partial windows of 160 frames with the default 50 % overlap.
  many     embed_utterances(wavs): length-sorted calls of at most 1024 partial rows, one mel launch and one
           mb_encoder_embed_rows per call, frames never leaving the device
  single   [embed_utterance(w) for w in wavs]: per utterance one mel launch, frames to the host, windows cut by numpy and
           copied back, the LSTM, and the mean / norm on the host
  U4096    embed_utterances on 4096 utterances of the same distribution (several calls)
  oracle   the CPU oracle restatement (oracle/melspec_oracle.encoder_mel + oracle/encoder_oracle.embed_utterance_partials,
           numpy float64 STFT and torch fp32 LSTM) on the first --oracle-utts utterances, in a child process with CUDA
           hidden; context for what the chain costs on the host, not the reference itself (librosa is absent here)
whole_call_ms: host clock around the call, which ends with its result on the host (median of --steps after --warmup).
device_busy_ms: the union of the call's GPU kernel and copy intervals in one further run under torch.profiler.
The card's name and power limit are read in the same run.

    python bench_encoder_many.py --steps 3 --warmup 1
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "synth_weights"))
sys.path.insert(0, str(ROOT / "oracle"))

from bench_wavernn_mol import _card  # noqa: E402

SR = 16000


def speech_like(n, seed):
    import numpy as np

    rng = np.random.default_rng(seed)
    t = np.arange(n) / SR
    f0 = 100 + 120 * rng.random()
    env = 0.5 + 0.5 * np.sin(2 * np.pi * (1 + 3 * rng.random()) * t + rng.random() * 6) ** 2
    y = sum(np.sin(2 * np.pi * f0 * k * t + rng.random() * 6) / k for k in range(1, 6))
    return (0.1 * env * y + 0.01 * rng.standard_normal(n)).astype(np.float32)


def inputs(u, seed):
    import numpy as np

    lengths = np.random.default_rng(seed).integers(2 * SR, 10 * SR + 1, u)
    return [speech_like(int(n), seed * 100003 + i) for i, n in enumerate(lengths)]


def _whole(fn, steps, warmup):
    import torch

    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ms = []
    for _ in range(steps):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ms.append((time.perf_counter() - t0) * 1e3)
    ms.sort()
    return ms[len(ms) // 2]


def _device_busy(fn):
    """the union of the call's GPU activity intervals (kernels and copies) in one run under torch.profiler, in ms"""
    import torch
    from torch.profiler import ProfilerActivity, profile

    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    spans = sorted((e.time_range.start, e.time_range.end) for e in prof.events()
                   if e.device_type == torch.autograd.DeviceType.CUDA)
    busy, end = 0.0, float("-inf")
    for a, b in spans:
        if b > end:
            busy += b - max(a, end)
            end = b
    return busy / 1e3


def _oracle_child(u_oracle):
    """runs in a child process with CUDA hidden: the oracle chain on the first u_oracle utterances"""
    import numpy as np
    import torch

    import encoder_oracle as eo
    import melspec_oracle as mo
    import ref_init as ri
    from mockingbird_b200.encoder.inference import compute_partial_slices

    sd = ri.encoder_state_dict(0)
    wavs = inputs(256, 1)[:u_oracle]
    t0 = time.perf_counter()
    for w in wavs:
        ws, ms = compute_partial_slices(len(w))
        frames = mo.encoder_mel(np.pad(w, (0, max(0, ws[-1].stop - len(w)))))
        eo.embed_utterance_partials(sd, torch.from_numpy(np.stack([frames[s] for s in ms])))
    dt = (time.perf_counter() - t0) * 1e3
    print(json.dumps({"utterances": u_oracle, "seconds_of_audio": round(sum(len(w) for w in wavs) / SR, 1),
                      "ms": round(dt, 1), "ms_per_utterance": round(dt / u_oracle, 1), "torch_threads": torch.get_num_threads()}))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--oracle-utts", type=int, default=8)
    ap.add_argument("--oracle-child", type=int, default=0, help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.oracle_child:
        _oracle_child(args.oracle_child)
        return
    import numpy as np
    import torch

    import ref_init as ri
    from mockingbird_b200.encoder import inference as enc
    from mockingbird_b200.encoder.model import SpeakerEncoder

    if not torch.cuda.is_available():
        raise SystemExit("bench_encoder_many.py measures on a CUDA device; none is visible")
    torch.cuda.set_device(0)
    m = SpeakerEncoder()
    m.load_state_dict(ri.encoder_state_dict(0))
    enc.set_model(m)
    result = {"workload": "speaker encoder, U utterances of 2-10 s at 16 kHz, partial windows of 160 frames, 50 % overlap, "
                          "ref_init weights", "card": _card(), "steps": args.steps, "warmup": args.warmup}
    wavs = inputs(256, 1)
    rows = sum(len(enc.compute_partial_slices(len(w))[1]) for w in wavs)
    entry = {"utterances": len(wavs), "seconds_of_audio": round(sum(len(w) for w in wavs) / SR, 1), "partial_rows": rows,
             "library_calls": len(enc.many_plan([enc.utterance_rows(len(w))[3] for w in wavs]))}
    many = lambda: enc.embed_utterances(wavs)  # noqa: E731
    single = lambda: [enc.embed_utterance(w) for w in wavs]  # noqa: E731
    got, ref = many(), np.stack(single())
    entry["max_abs_diff_many_vs_single"] = float(np.abs(got - ref).max())
    for name, fn in (("many", many), ("single", single)):
        entry[name] = {"whole_call_ms": round(_whole(fn, args.steps, args.warmup), 1),
                       "device_busy_ms": round(_device_busy(fn), 1)}
    entry["whole_call_speedup"] = round(entry["single"]["whole_call_ms"] / entry["many"]["whole_call_ms"], 2)
    result["U256"] = entry
    big = inputs(4096, 2)
    fn = lambda: enc.embed_utterances(big)  # noqa: E731
    result["U4096"] = {"seconds_of_audio": round(sum(len(w) for w in big) / SR, 1),
                       "partial_rows": sum(len(enc.compute_partial_slices(len(w))[1]) for w in big),
                       "library_calls": len(enc.many_plan([enc.utterance_rows(len(w))[3] for w in big])),
                       "whole_call_ms": round(_whole(fn, max(1, args.steps // 2), min(1, args.warmup)), 1),
                       "device_busy_ms": round(_device_busy(fn), 1)}
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    proc = subprocess.run([sys.executable, __file__, "--oracle-child", str(args.oracle_utts)], env=env, capture_output=True,
                          text=True, timeout=3600)
    if proc.returncode == 0:
        o = json.loads(proc.stdout.strip().splitlines()[-1])
    else:
        o = {"error": proc.stderr.strip().splitlines()[-1] if proc.stderr.strip() else f"exit {proc.returncode}"}
    result["oracle_restatement_cpu"] = o
    print(json.dumps(result))


if __name__ == "__main__":
    main()
