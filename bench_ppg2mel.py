"""Voice-conversion mel decoder (ppg2mel MelDecoderMOLv2.inference) on one GPU; prints one JSON line.

Two configurations, seeded random-init weights (ref_init.ppg2mel_state_dict(0)) and random PPG / pitch inputs:
  b1     one 10 s utterance (1000 PPG frames, 250 encoder frames, <= 500 decoder steps), the reference's calling
         pattern (MelDecoderMOLv2.inference, B = 1)
  batch  64 utterances of 3-10 s (300-1000 frames) through inference_batch (one padded call)
For each: ms per call, ms per decoder step (call time over the longest row's steps), mel frames/s, real-time factor
(audio seconds per second at 100 mel frames/s, the 10 ms hop of the PPG front-end), kernel launches per decoder step
(the slope of the library's launch counter over step count), and for b1 the torch-CPU oracle's time on the same input.
The card name and power limit are read in the same run.  Algorithmic work per decoder step and row: 4.77 MMAC of
weights plus 256 * T_enc for the context; the postnet is 4.34 MMAC per mel frame.

usage: python bench_ppg2mel.py [--iters N] [--warmup W] [--no-cpu]
"""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "synth_weights"))

FRAMES_PER_S = 100.0  # mel frames per second of audio (16 kHz, hop 160: the PPG front-end's frame rate)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, power = [s.strip() for s in out.split(",")]
        return name, power
    except Exception:
        import torch

        return torch.cuda.get_device_name(0), "unknown"


def inputs(lengths, seed):
    import torch

    g = torch.Generator().manual_seed(seed)
    utts = [(torch.randn(T, 144, generator=g),
             torch.stack([torch.randn(T, generator=g), (torch.rand(T, generator=g) < 0.7).float()], 1)) for T in lengths]
    return utts, torch.randn(len(lengths), 256, generator=g)


def timed(fn, iters, warmup):
    import torch

    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(iters):
        out = fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / iters, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--no-cpu", action="store_true")
    a = ap.parse_args()
    import torch

    import ref_init as ri
    from mockingbird_b200 import _lib
    from mockingbird_b200.ppg2mel import MelDecoderMOLv2

    if not torch.cuda.is_available():
        raise SystemExit("bench_ppg2mel.py needs a CUDA device")
    torch.cuda.set_device(0)
    sd = ri.ppg2mel_state_dict(0)
    sd["decoder.stop_layer.linear_layer.bias"] = sd["decoder.stop_layer.linear_layer.bias"] - 10.0  # run to max steps
    model = MelDecoderMOLv2(**ri.PPG2MEL_CONFIG).cuda()
    model.load_state_dict(sd)
    model.eval()
    L = _lib.lib()
    result = {"workload": "ppg2mel MelDecoderMOLv2.inference: b1 = 1 x 1000 PPG frames; batch = 64 x 300-1000 frames"}
    name, power = card()
    result["gpu"], result["power_limit"] = name, power

    def launches_per_step(run, steps_a, steps_b, run_b):
        c0 = L.mb_launch_count()
        run()
        torch.cuda.synchronize()
        c1 = L.mb_launch_count()
        run_b()
        torch.cuda.synchronize()
        c2 = L.mb_launch_count()
        ga, gb = -(-steps_a // 16) * 16, -(-steps_b // 16) * 16  # steps issued: whole graph groups of 16
        return ((c1 - c0) - (c2 - c1)) / (ga - gb)

    # ---- B = 1, 10 s
    utts, spk = inputs([1000], 1)
    ppg, lf0 = utts[0]
    args = (ppg[None].cuda(), lf0[None].cuda(), spk[:1].cuda())
    dt, out = timed(lambda: model.inference(*args, seed=3), a.iters, a.warmup)
    n = out[2].shape[0]
    short = (ppg[None, :200].cuda(), lf0[None, :200].cuda(), spk[:1].cuda())
    lps = launches_per_step(lambda: model.inference(*args, seed=3), n, 100, lambda: model.inference(*short, seed=3))
    b1 = {"ms_per_call": round(dt * 1e3, 3), "steps": n, "ms_per_step": round(dt * 1e3 / n, 4),
          "mel_frames_per_s": round(2 * n / dt, 1), "rtf": round(dt / (2 * n / FRAMES_PER_S), 5),
          "launches_per_step": round(lps, 2)}
    if not a.no_cpu:
        sys.path.insert(0, str(ROOT / "oracle"))
        import ppg2mel_oracle as po

        t0 = time.perf_counter()
        r = po.inference(sd, ppg, lf0, spk[0], generator=torch.Generator().manual_seed(3))
        cpu = time.perf_counter() - t0
        b1["cpu_oracle_s"] = round(cpu, 3)
        b1["cpu_oracle_steps"] = r["steps"]
        b1["cpu_threads"] = torch.get_num_threads()
    result["b1"] = b1

    # ---- batch of 64, 3-10 s
    lengths = torch.randint(300, 1001, (64,), generator=torch.Generator().manual_seed(2)).tolist()
    utts, spk = inputs(lengths, 4)
    dt, outs = timed(lambda: model.inference_batch(utts, spk, seed=3), a.iters, a.warmup)
    steps = [o[2].shape[0] for o in outs]
    frames = 2 * sum(steps)
    result["batch"] = {"rows": 64, "ms_per_call": round(dt * 1e3, 3), "max_steps": max(steps),
                       "ms_per_step": round(dt * 1e3 / max(steps), 4), "mel_frames_per_s": round(frames / dt, 1),
                       "rtf": round(dt / (frames / FRAMES_PER_S), 6)}
    print(json.dumps(result), flush=True)


if __name__ == "__main__":
    main()
