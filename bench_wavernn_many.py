"""Many utterances in one WaveRNN sample loop (WaveRNN.generate_many_device) on one GPU; prints one JSON line.

  uniform  U in {1, 8, 32, 64, 128, 256} unbatched utterances of 80 frames (the cfg-1 shape of bench_wavernn.py: 16 000
           sequential steps each), RAW and MOL sampler, noise from rng "torch" with per-utterance seeds (one MT19937 stream
           per utterance, drawn by host threads) and from rng "device" (the built-in generator: no host work).  Beside
           each: U times the single generate_*_device call of one such utterance, timed in the same run.
  ragged   64 unbatched utterances of randint(40, 400) frames (seeded): the live-row schedule against the same loop with
           every utterance padded to the longest (what a fixed-length batch would cost).  RAW, rng "device".
  folded   16 utterances of 3 to 10 s, batched (target 8000, overlap 400): all their folds in one loop against the 16
           single calls.  RAW, rng "device".
The device part is timed with CUDA events around the whole call (conditioning, every chunk, the host noise producer where
there is one), mels resident on the device, every shape warmed up, median of --steps runs.  samples_per_s counts delivered
samples (rows x their own steps); us_per_step is the time over the longest row's steps; GFLOP/s uses the algorithmic work
per sample of bench_wavernn.py.  The card name and its enforced power limit are read in the same run.

    python bench_wavernn_many.py --steps 3 --warmup 1
"""
from __future__ import annotations

import argparse
import json
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "synth_weights"))

from bench_wavernn import FLOP_PER_DRAW  # noqa: E402
from bench_wavernn_mol import _card, _model, _time  # noqa: E402

TARGET, OVERLAP = 8000, 400
UNIFORM_U = (1, 8, 32, 64, 128, 256)


def _mels(lengths, seed):
    import torch

    g = torch.Generator().manual_seed(seed)
    return [(torch.rand(1, 80, int(T), generator=g) * 2 - 1).cuda() for T in lengths]


def _report(ms, samples, max_steps):
    return {"ms": round(ms, 2), "samples_per_s": round(samples / (ms * 1e-3), 1), "us_per_step": round(ms * 1e3 / max_steps, 3),
            "gflops": round(samples * FLOP_PER_DRAW / (ms * 1e-3) / 1e9, 1)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--max-u", type=int, default=256, help="largest uniform batch to run")
    args = ap.parse_args()
    import numpy as np
    import torch

    from mockingbird_b200.vocoder.wavernn.models.fatchord_version import RowPlan

    if not torch.cuda.is_available():
        raise SystemExit("bench_wavernn_many.py measures on a CUDA device; none is visible")
    torch.cuda.set_device(0)
    result = {"workload": "WaveRNN generate_many_device: many utterances in one sample loop", "card": _card(),
              "steps": args.steps, "warmup": args.warmup,
              "unit": "samples_per_s = delivered rows x steps / s; us_per_step = call time / steps of the longest row"}
    models = {mode: _model(mode) for mode in ("RAW", "MOL")}

    def single(m, mel, batched):
        run = m.generate_samples_device if m.mode == "MOL" else m.generate_indices_device
        return lambda: run(mel, batched, TARGET, OVERLAP, None)

    uniform = {}
    for mode, m in models.items():
        for rng in ("torch", "device"):
            m.rng = rng
            mels = _mels([80] * max(UNIFORM_U), seed=1)
            torch.manual_seed(1234)
            one_ms = _time(single(m, mels[0], False), args.steps, args.warmup)
            entry = {"single_call": _report(one_ms, 16000, 16000)}
            for U in UNIFORM_U:
                if U > args.max_u:
                    continue
                seeds = list(range(U))
                ms = _time(lambda: m.generate_many_device(mels[:U], False, TARGET, OVERLAP, seeds=seeds), args.steps, args.warmup)
                r = _report(ms, U * 16000, 16000)
                r["sequential_ms"] = round(U * one_ms, 1)  # U single calls, from the single call timed above
                r["speedup"] = round(U * one_ms / ms, 2)
                entry[f"U{U}"] = r
            uniform[f"{mode}_{rng}"] = entry
            m.rng = "torch"
    result["uniform_80_frames"] = uniform

    m = models["RAW"]
    m.rng = "device"
    lengths = np.random.default_rng(0).integers(40, 400, 64)
    mels = _mels(lengths, seed=2)
    padded = _mels([int(lengths.max())] * 64, seed=2)
    seeds = list(range(64))
    delivered = int(lengths.sum()) * 200
    ms = _time(lambda: m.generate_many_device(mels, False, TARGET, OVERLAP, seeds=seeds), args.steps, args.warmup)
    ms_pad = _time(lambda: m.generate_many_device(padded, False, TARGET, OVERLAP, seeds=seeds), args.steps, args.warmup)
    plan = RowPlan([int(T) for T in lengths], False, TARGET, OVERLAP)
    result["ragged_64"] = {"frames_min_mean_max": [int(lengths.min()), round(float(lengths.mean()), 1), int(lengths.max())],
                           "live_rows": _report(ms, delivered, plan.max_steps),
                           "padded_to_longest": _report(ms_pad, delivered, plan.max_steps),
                           "saved": round(1.0 - ms / ms_pad, 4)}

    lengths = np.random.default_rng(1).integers(240, 801, 16)  # 3 to 10 s at 80 frames / s
    mels = _mels(lengths, seed=3)
    plan = RowPlan([int(T) for T in lengths], True, TARGET, OVERLAP)
    seeds = list(range(16))
    ms = _time(lambda: m.generate_many_device(mels, True, TARGET, OVERLAP, seeds=seeds), args.steps, args.warmup)
    seq = 0.0
    for u, mel in enumerate(mels):
        m.seed = u
        seq += _time(single(m, mel, True), args.steps, args.warmup)
    m.rng, m.seed = "torch", 0
    r = _report(ms, plan.rows * plan.max_steps, plan.max_steps)
    r.update({"rows": plan.rows, "utterances": 16, "sequential_ms": round(seq, 1), "speedup": round(seq / ms, 2)})
    result["folded_16"] = r
    print(json.dumps(result))


if __name__ == "__main__":
    main()
