"""WaveRNN workloads of bench.py.

wavernn_cfg1  BASELINE.json configs[0]: WaveRNN.generate on one 80-frame x 80-bin random mel, batched=False
              (16 000 strictly sequential draws of ONE row) - the reference's CPU-runnable case; GPU side + CPU leg.
wavernn_cfg3  configs[2]: batched generate (target 8000, overlap 400) on a 30 s random mel -> 58 folds x 8800 steps.
              A "step" is one whole generate() of that utterance.  value = delivered audio samples/s (487 600 per step;
              the 510 400 raw draws/s beside it) with the mel resident in HBM; reported for BOTH noise sources:
                rng="torch"   the reference-identical stream (MT19937 continuation of the torch generator,
                              csrc/mt_stream.cu) - the integer samples equal the reference's (tests/test_fullsize.py)
                rng="device"  the built-in counter-based generator
              e2e = wavernn.inference.infer_waveform(host numpy mel) -> host float64 waveform, post-processing included.
              Under torchrun every rank vocodes its own utterance (weak scaling); `measure_cfg3_sharded` deals the 58
              folds of ONE utterance across the ranks (SURVEY.md 8e row 2) and gathers the int16 rows on rank 0.
CPU leg: oracle/wavernn_torch_oracle.py, the torch-CPU restatement of the reference loop (pinned to the reference's
integer samples), all host threads, bounded number of steps.
"""
from __future__ import annotations

import json
import os
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parent
FRAMES, TARGET, OVERLAP = 2400, 8000, 400
FLOP_PER_DRAW = 8.14e6  # SURVEY.md 8d


def _geometry(frames=FRAMES):
    total = frames * 200
    folds = (total - OVERLAP) // (TARGET + OVERLAP)
    if total - (folds * (TARGET + OVERLAP) + OVERLAP) != 0:
        folds += 1
    steps = TARGET + 2 * OVERLAP
    delivered = folds * (TARGET + OVERLAP) + OVERLAP  # unfolded length; wave_len = (T-1)*hop_length(256) is longer: no trim (SURVEY fact 8)
    return folds, steps, delivered


def cpu_torch_oracle(workload: str, nsteps: int, threads: int):
    """the torch-CPU port of the reference loop on `nsteps` steps of the config; returns (draws/s, seconds)"""
    sys.path.insert(0, str(ROOT / "oracle"))
    sys.path.insert(0, str(ROOT / "synth_weights"))
    import torch
    import ref_init as ri
    import wavernn_torch_oracle as wt

    torch.set_num_threads(threads)
    sd = ri.wavernn_state_dict(0, randomize_bn=True)
    torch.manual_seed(1234)
    if workload == "wavernn_cfg1":
        mel = torch.rand(1, 80, 80, generator=torch.Generator().manual_seed(1)) * 2 - 1
        idx, dt = wt.generate_indices(sd, mel, False, TARGET, OVERLAP, max_steps=nsteps)
    else:
        mel = torch.rand(1, 80, FRAMES, generator=torch.Generator().manual_seed(3)) * 2 - 1
        idx, dt = wt.generate_indices(sd, mel, True, TARGET, OVERLAP, max_steps=nsteps)
    return idx.size / dt, dt


def run_reference(args, threads):
    """--impl reference: the torch-CPU port on a bounded number of steps per bench step"""
    cfg1 = args.workload == "wavernn_cfg1"
    folds, steps, delivered = (1, 16000, 16000) if cfg1 else _geometry()
    n = 2000 if cfg1 else 300
    per = []
    for s in range(args.warmup + args.steps):
        v, dt = cpu_torch_oracle(args.workload, n, threads)
        if s >= args.warmup:
            per.append(dt)
    secs = sum(per)
    draws_per_s = folds * n * args.steps / secs
    value = draws_per_s * delivered / (folds * steps)
    print(json.dumps({
        "impl": "reference", "metric": "vocoder audio samples/sec", "value": value, "unit": "samples/s",
        "n_gpus": args.gpus, "steps": args.steps, "warmup": args.warmup, "ms_per_step": 1e3 * delivered / value,
        "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "f32", "data": "synthetic",
        "config": {"workload": _workload_name(cfg1)},
        "cpu_baseline": {"value": value, "unit": "samples/s", "cores": threads, "kind": "port",
                         "sample": f"{n} of {steps} steps x {folds} fold rows per step, torch-CPU port of the reference loop "
                                   "(oracle/wavernn_torch_oracle.py, integer samples pinned to the reference)"},
        "e2e": {"value": value, "unit": "samples/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
        "gpu_launches": 0}))


def _workload_name(cfg1: bool) -> str:
    if cfg1:
        return "wavernn_cfg1: WaveRNN.generate, one 80-frame x 80-bin mel, batched=False (16000 sequential draws)"
    return ("wavernn_cfg3: batched generate, 30 s mel (2400 frames), target 8000 / overlap 400 -> 58 folds x 8800 "
            "sequential steps per GPU")


def _model(ctx):
    sys.path.insert(0, str(ROOT / "synth_weights"))
    import ref_init as ri
    from mockingbird_b200.vocoder.wavernn import inference as rnn_vocoder

    model = rnn_vocoder.load_state(ri.wavernn_state_dict(0, randomize_bn=True), rng="torch", seed=1234 + ctx.rank)
    if ctx.world > 1:
        ctx.dist.broadcast(model.packed_arena(), src=0)
    return model, rnn_vocoder


def _cpu_leg(workload, nsteps, folds, steps, delivered):
    from bench_common import cpu_child, host_threads

    threads = host_threads()
    r = cpu_child(workload, nsteps, threads, 240.0)
    if not r:
        return None
    return {"value": r["value"] * delivered / (folds * steps), "unit": "samples/s", "raw_draws_per_s": r["value"], "cores": threads,
            "kind": "port", "sample": f"{nsteps} of {steps} steps x {folds} rows ({r['seconds']:.1f} s), torch-CPU port of the "
                                      "reference loop (oracle/wavernn_torch_oracle.py; integer samples pinned to the reference)"}


def measure_cfg1(ctx, args, cpu: bool, steps: int = 3):
    """configs[0]: latency-bound single row; the reference measures this on CPU (8.5 s here on 8 cores)"""
    import torch

    model, rnn_vocoder = _model(ctx)
    mel = torch.rand(1, 80, 80, generator=torch.Generator().manual_seed(1)) * 2 - 1
    mel_np = (mel[0] * 4.0).numpy()
    delivered, draws = 16000, 16000

    def step_e2e():
        torch.manual_seed(1234)
        rnn_vocoder.infer_waveform(mel_np, batched=False, target=TARGET, overlap=OVERLAP, progress_callback=lambda *a: None)

    mel_dev = mel.to(ctx.dev)

    def step_resident():
        torch.manual_seed(1234)
        ctx.outputs = {"indices": model.generate_indices(mel_dev, False, TARGET, OVERLAP, None)}

    r = ctx.timed(step_resident, steps, 1, 1.0, host_clock=True)
    e = ctx.timed(step_e2e, steps, 1, 0.0, host_clock=True)
    if ctx.rank != 0:
        return None
    ms = r["ms"] / steps
    return {
        "metric": "vocoder audio samples/sec", "value": ctx.world * delivered / (ms * 1e-3), "unit": "samples/s", "n_gpus": ctx.world,
        "steps": steps, "ms_per_step": ms, "us_per_sample_step": ms * 1e3 / draws, "raw_draws_per_s": ctx.world * draws / (ms * 1e-3),
        "scaling": "weak", "dtype": "f32", "config": {"workload": _workload_name(True), "rng": "torch (reference-identical stream)"},
        "burst": {"value": ctx.world * delivered * steps / (r["ms_burst"] * 1e-3)},
        "e2e": {"value": ctx.world * delivered * steps / (e["ms"] * 1e-3), "unit": "samples/s", "h2d_bytes_per_step": int(mel_np.nbytes) + draws * 512 * 8,
                "d2h_bytes_per_step": draws * 2, "ms_per_step": e["ms"] / steps,
                "surface": "vocoder.wavernn.inference.infer_waveform(host mel, batched=False) -> host float64 waveform"},
        "roofline": {"bound": "latency", "kernel": "k_sample_loop", "achieved": FLOP_PER_DRAW * draws / (ms * 1e-3) / 1e12, "peak": 72.0,
                     "unit": "TFLOP/s", "frac": FLOP_PER_DRAW * draws / (ms * 1e-3) / 1e12 / 72.0, "traffic": None,
                     "note": "ONE row: 16 000 dependent steps x 6 grid barriers; nothing to batch - the config is the reference's CPU case"},
        "cpu_baseline": _cpu_leg("wavernn_cfg1", 4000, 1, 16000, delivered) if cpu else None}


def measure_cfg3(ctx, args, cpu: bool, steps: int = 3):
    import torch

    from mockingbird_b200 import _lib

    model, rnn_vocoder = _model(ctx)
    folds, nsteps, delivered = _geometry()
    mel = torch.rand(1, 80, FRAMES, generator=torch.Generator().manual_seed(3 + ctx.rank)) * 2 - 1
    mel_dev = mel.to(ctx.dev)
    mel_np = (mel[0] * 4.0).numpy()
    lib = _lib.lib()
    out = {}

    def step_resident():
        ctx.outputs = {f"indices_{model.rng}": model.generate_indices(mel_dev, True, TARGET, OVERLAP, None)}

    def step_e2e():
        wav, _ = rnn_vocoder.infer_waveform(mel_np, batched=True, target=TARGET, overlap=OVERLAP, progress_callback=lambda *a: None)
        out["n"] = len(wav)

    res, outputs = {}, {}
    for mode in ("torch", "device"):
        model.rng = mode
        torch.manual_seed(1234)
        l0 = lib.mb_launch_count()
        r = ctx.timed(step_resident, steps, 1, 0.0, host_clock=True)
        launches = int(lib.mb_launch_count() - l0) * steps // (2 * steps + 1)
        outputs.update(ctx.outputs)
        e = ctx.timed(step_e2e, steps, 1, 0.0, host_clock=True)
        res[mode] = (r, e, launches)
    ctx.outputs = outputs
    model.rng = "torch"
    if ctx.rank != 0:
        return None
    assert out["n"] == delivered, (out["n"], delivered)
    w = ctx.world

    def v(ms_total):
        return w * delivered * steps / (ms_total * 1e-3)

    r, e, launches = res["torch"]
    rd, ed, _ = res["device"]
    ms = r["ms"] / steps
    flops = FLOP_PER_DRAW * folds * nsteps
    return {
        "metric": "vocoder audio samples/sec", "value": v(r["ms"]), "unit": "samples/s", "n_gpus": w, "steps": steps,
        "ms_per_step": ms, "rtf": (ms * 1e-3) / (delivered / 16000.0), "raw_draws_per_s": w * folds * nsteps / (ms * 1e-3),
        "us_per_sample_step": ms * 1e3 / nsteps, "scaling": "weak", "dtype": "f32",
        "config": {"workload": _workload_name(False), "rng": "torch: MT19937 continuation of the global torch generator + device "
                   "-log1p(-u) (reference-identical integer samples, tests/test_fullsize.py::test_gpu_wavernn_cfg3_identical)",
                   "parallelism": f"dp{w}", "l2": "weights shared-memory resident, exchange buffers L2 resident by design (no flush applicable)"},
        "burst": {"value": v(r["ms_burst"])},
        "e2e": {"value": v(e["ms"]), "unit": "samples/s", "h2d_bytes_per_step": int(mel_np.nbytes) + folds * nsteps * 512 * 8,
                "d2h_bytes_per_step": folds * nsteps * 2, "ms_per_step": e["ms"] / steps,
                "surface": "vocoder.wavernn.inference.infer_waveform(host mel) -> host float64 waveform (xfade/unfold, mu-law, "
                           "de-emphasis, fade on the host in float64 like the reference)"},
        "value_device_rng": v(rd["ms"]), "e2e_device_rng": {"value": v(ed["ms"]), "unit": "samples/s", "ms_per_step": ed["ms"] / steps,
                                                          "h2d_bytes_per_step": int(mel_np.nbytes), "d2h_bytes_per_step": folds * nsteps * 2},
        "gpu_launches": launches, "clocks": r["clocks"],
        "roofline": {"bound": "latency", "kernel": "k_sample_loop (persistent cooperative, weights smem-stationary)",
                     "achieved": flops / (ms * 1e-3) / 1e12, "peak": 72.0, "unit": "TFLOP/s", "frac": flops / (ms * 1e-3) / 1e12 / 72.0,
                     "traffic": None, "note": "FP32 FFMA (integer-exact samples rule out tensor-core operand rounding); 8800 dependent "
                                              "steps x 6 grid barriers bound the time, not HBM (4 B of conditioning per draw); north-star "
                                              "target is absolute: >= 1e6 samples/s"},
        "cpu_baseline": _cpu_leg("wavernn_cfg3", 600, folds, nsteps, delivered) if cpu else None}


def measure_cfg3_sharded(ctx, args, steps: int = 3):
    """SURVEY.md 8e row 2: the 58 folds of ONE 30 s utterance dealt contiguously across the ranks (8/7 per GPU at N=8),
    int16 rows gathered on rank 0 which cross-fades / unfolds; strong scaling of a single utterance's latency."""
    import torch

    model, _ = _model(ctx)
    folds, nsteps, delivered = _geometry()
    mel = torch.rand(1, 80, FRAMES, generator=torch.Generator().manual_seed(3)) * 2 - 1  # the SAME utterance on every rank
    out = {}

    def step():
        torch.manual_seed(1234)
        wav = model.generate_sharded(mel, TARGET, OVERLAP, True, progress_callback=None)
        if wav is not None:
            out["n"] = len(wav)

    r = ctx.timed(step, steps, 1, 0.0, host_clock=True)
    if ctx.rank != 0:
        return None
    ms = r["ms"] / steps
    return {"metric": "vocoder audio samples/sec", "value": delivered / (ms * 1e-3), "unit": "samples/s", "n_gpus": ctx.world,
            "steps": steps, "ms_per_step": ms, "scaling": "strong", "dtype": "f32",
            "rows_per_gpu": [int(-(-folds // ctx.world)), int(folds // ctx.world)],
            "config": {"workload": "wavernn_cfg3 fold-sharded: ONE 30 s utterance, 58 folds dealt contiguously over the ranks, int16 "
                                   "gather on rank 0 + host unfold (host numpy mel -> host float64 waveform)",
                       "rng": "torch (every rank continues the same MT19937 stream and reads its own rows)"},
            "e2e": {"value": delivered / (ms * 1e-3), "unit": "samples/s", "h2d_bytes_per_step": 80 * FRAMES * 4 + folds * nsteps * 512 * 8,
                    "d2h_bytes_per_step": folds * nsteps * 2, "ms_per_step": ms},
            "note": "fewer rows per GPU do not shorten the 8800 dependent steps: per-GPU efficiency drops with N as SURVEY.md 8e predicts; "
                    "the >= 58-rows-per-GPU case is wavernn_cfg3 (one utterance per GPU)"}
