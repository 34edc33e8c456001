"""Tacotron workload of bench.py (tacotron_cfg4): BASELINE.json configs[3],
Tacotron generate + postnet, batch 64 random token sequences of length <= 120, steps=400, r=2,
min_stop_token=10 (early stop disabled, SURVEY.md fact 7), style_idx=-1.

A "step" is one whole generate() of the batch (25,600 mel frames).  value is reported in the bench
metric's unit (audio samples/s at the vocoders' 200 samples per frame); mel frames/s is given beside it.
e2e: host token ids / embeddings in, host numpy spectrograms out (Synthesizer surface after the
text front-end).  Under torchrun every rank synthesises its own batch (weak scaling)."""
from __future__ import annotations

import json
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parent
B, TC, STEPS, R = 64, 120, 400, 2
WORKLOAD = ("tacotron_cfg4: Tacotron generate + postnet, B=64, len<=120, steps=400, r=2, min_stop_token=10, "
            "style_idx=-1 per GPU")


def make_inputs(rank=0):
    import torch

    g = torch.Generator().manual_seed(4 + rank)
    chars = torch.randint(2, 75, (B, TC), generator=g)
    lens = torch.randint(20, TC + 1, (B,), generator=g)
    lens[0] = TC
    for b in range(B):
        chars[b, lens[b]:] = 0
    emb = torch.rand(B, 256, generator=torch.Generator().manual_seed(5 + rank))
    emb = emb / emb.norm(dim=1, keepdim=True)
    return chars, emb, lens


def cpu_oracle(steps: int, threads: int):
    """torch-CPU oracle (matches the reference to 1 ulp) on the cfg-4 batch with `steps` decoder frames"""
    sys.path.insert(0, str(ROOT / "oracle"))
    sys.path.insert(0, str(ROOT / "synth_weights"))
    import torch
    import ref_init as ri
    import tacotron_oracle as to

    torch.set_num_threads(threads)
    sd = ri.tacotron_state_dict(0, r=R, randomize_bn=True)
    chars, emb, _ = make_inputs()
    g = torch.Generator().manual_seed(9)
    nst = steps // R
    masks = [torch.rand(B, TC, 256, generator=g) < 0.5 for _ in range(2)] + \
            [torch.rand(B, 256, generator=g) < 0.5 for _ in range(2 * nst)]
    t0 = time.perf_counter()
    mel, lin, _ = to.generate(sd, chars, emb, steps, -1, 10, masks, r=R)
    dt = time.perf_counter() - t0
    return B * mel.shape[2] / dt, dt


def run_reference(args, threads):
    per = []
    n = 80
    for s in range(args.warmup + args.steps):
        v, dt = cpu_oracle(n, threads)
        if s >= args.warmup:
            per.append(dt)
    secs = sum(per)
    fps = B * n * args.steps / secs
    print(json.dumps({
        "impl": "reference", "metric": "vocoder audio samples/sec", "value": fps * 200, "unit": "samples/s",
        "mel_frames_per_s": fps, "n_gpus": args.gpus, "steps": args.steps, "warmup": args.warmup,
        "ms_per_step": 1e3 * B * STEPS / fps, "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
        "dtype": "f32", "data": "synthetic", "config": {"workload": WORKLOAD},
        "cpu_baseline": {"value": fps * 200, "unit": "samples/s", "cores": threads, "kind": "port",
                         "sample": "80 of 400 decoder frames per step, torch-CPU oracle (1 ulp from the reference); ms_per_step scaled to 400"},
        "e2e": {"value": fps * 200, "unit": "samples/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
        "gpu_launches": 0}))


def measure(ctx, args, cpu: bool, steps: int = 3):
    import torch

    sys.path.insert(0, str(ROOT / "synth_weights"))
    import ref_init as ri
    from bench_common import cpu_child, host_threads, peaks
    from mockingbird_b200 import _lib
    from mockingbird_b200.synthesizer.hparams import hparams as shp
    from mockingbird_b200.synthesizer.inference import Synthesizer

    rank, world, dev = ctx.rank, ctx.world, ctx.dev
    syn = Synthesizer("unused.pt", verbose=False)
    model = syn.load_state(ri.tacotron_state_dict(0, r=R, randomize_bn=True))
    if world > 1:
        ctx.dist.broadcast(model.packed_arena(), src=0)
    chars, emb, lens = make_inputs(rank)
    chars_dev, emb_dev = chars.to(dev), emb.to(dev)
    seqs = [chars[b, : int(lens[b])].tolist() for b in range(B)]
    embs = [emb[b].numpy() for b in range(B)]
    lib = _lib.lib()
    old_bs = shp.synthesis_batch_size
    shp.synthesis_batch_size = B  # one padded batch of 64 like the config (the reference default is 16)

    def step_resident():
        mel, linear, attn = model.generate(chars_dev, emb_dev, steps=STEPS, style_idx=-1, min_stop_token=10)
        ctx.outputs = {"mel": mel, "linear": linear, "attn": attn}

    def step_e2e():
        syn.synthesize_from_sequences(seqs, embs, False, -1, 10, STEPS)

    try:
        l0 = lib.mb_launch_count()
        r = ctx.timed(step_resident, steps, 2, min(args.soak_seconds, 1.0), host_clock=True)
        launches = int(lib.mb_launch_count() - l0) * steps // (2 + 2 * steps + max(r["soak_steps"], 0))
        e = ctx.timed(step_e2e, steps, 1, 0.0, host_clock=True)
    finally:
        shp.synthesis_batch_size = old_bs
    if rank != 0:
        return None
    frames = B * STEPS
    ms = r["ms"] / steps
    fps = world * frames / (ms * 1e-3)
    cpu_d = None
    if cpu:
        threads = host_threads()
        rc = cpu_child("tacotron_cfg4", 80, threads, 240.0)
        if rc:
            cpu_d = {"value": rc["value"] * 200, "unit": "samples/s", "mel_frames_per_s": rc["value"], "cores": threads,
                     "kind": "port", "sample": f"80 of 400 decoder frames, B=64 ({rc['seconds']:.1f} s), torch-CPU oracle"}
    flops = 2.0 * (20.99e6 * 200 * B + 8.03e6 * STEPS * B + 3.2e6 * TC * B)
    pk = peaks()
    return {
        "metric": "vocoder audio samples/sec", "value": fps * 200, "unit": "samples/s", "mel_frames_per_s": fps,
        "n_gpus": world, "steps": steps, "ms_per_step": ms, "higher_is_better": True, "scaling": "weak", "dtype": "f32 (3-term f16 split on tensor cores, FP32-equivalent)",
        "config": {"workload": WORKLOAD, "parallelism": f"dp{world}",
                   "l2": "decoder weights (162 MB of hi/lo fp16 images) stream from L2/HBM every step; no flush applicable"},
        "burst": {"value": world * frames * steps / (r["ms_burst"] * 1e-3) * 200},
        "e2e": {"value": world * frames * steps / (e["ms"] * 1e-3) * 200, "unit": "samples/s",
                "h2d_bytes_per_step": int(B * TC * 8 + B * 256 * 4), "d2h_bytes_per_step": int(frames * 80 * 4),
                "ms_per_step": e["ms"] / steps, "surface": "Synthesizer.synthesize_from_sequences (host ids / embeds -> host numpy mels)"},
        "gpu_launches": launches, "clocks": r["clocks"],
        "roofline": {"bound": "tensor", "kernel": "tc_skinny / tc_gru / tc_big (wgmma GEMMs, 3-term fp16 split = 3 MMA flops per "
                                                   "useful flop, FP32-equivalent)",
                     "achieved": flops / (ms * 1e-3) / 1e12, "peak": pk["tflops_sustained"], "unit": "TFLOP/s",
                     "frac": 3.0 * flops / (ms * 1e-3) / 1e12 / pk["tflops_sustained"], "traffic": None,
                     "peak_source": pk["source"] + ", bf16 sustained (fp16 same rate)",
                     "note": "achieved = useful (FP32-equivalent) FLOPs of the whole generate / time; frac counts the 3 MMA passes. "
                             "The path is bound by 200 dependent decoder steps, not by the tensor pipe"},
        "cpu_baseline": cpu_d}
