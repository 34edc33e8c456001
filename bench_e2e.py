"""End-to-end workload of bench.py (--workload e2e_cfg5): BASELINE.json configs[4], speaker encoder ->
Tacotron -> HiFi-GAN on synthetic utterances sharded across the GPUs, 128 utterances per GPU
(1024 on 8 GPUs; weak scaling).

Per utterance (SURVEY.md 8d cfg 5): 6 synthetic partial windows rand(6,160,40) -> speaker embedding;
token sequence of random length 20..120; Tacotron steps=400, r=2, min_stop_token=10 (no early stop),
style_idx=-1 -> 400-frame mel; HiFi-GAN -> 80 000 audio samples.  The global utterance list is
length-sorted and dealt round-robin to ranks (distributed.shard_utterances); no collective on the data path.

A "step" is the whole pipeline over the rank's 128 utterances.  `value`: device-resident (inputs in
HBM, model-level calls).  `e2e`: through the drop-in module surfaces with host numpy in and out
(encoder.inference.embed_utterances_frames -> Synthesizer.synthesize_from_sequences ->
hifigan.inference.infer_waveforms), host<->device copies inside the timed region."""
from __future__ import annotations

import json
import os
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parent
UTT_PER_GPU, PARTIALS, PFRAMES, STEPS, R, VBATCH = 128, 6, 160, 400, 2, 32
# Tacotron batch of the pipeline: the decoder step is latency-bound and its tensor-core GEMMs use 128-row tiles, so 128 rows cost
# about what 64 do (cfg 4 itself is DEFINED as batch 64 and stays so in bench_tacotron.py)
TBATCH = int(os.environ.get("MB_BENCH_TBATCH", "128"))


def make_utterances(n_total: int):
    """global synthetic utterance list: (token lengths, token ids, partial mel windows seed)"""
    import torch

    g = torch.Generator().manual_seed(6)
    lens = torch.randint(20, 121, (n_total,), generator=g)
    chars = torch.randint(2, 75, (n_total, 120), generator=g)
    return lens, chars


def cpu_oracle(n_utt: int, threads: int, frames: int = 200):
    """CPU oracles chained the same way on `n_utt` utterances with `frames` decoder frames each"""
    sys.path.insert(0, str(ROOT / "oracle"))
    sys.path.insert(0, str(ROOT / "synth_weights"))
    import torch
    import encoder_oracle as eo
    import gan_oracle as go
    import ref_init as ri
    import tacotron_oracle as to

    torch.set_num_threads(threads)
    lens, chars = make_utterances(n_utt)
    tsd = ri.tacotron_state_dict(0, r=R, randomize_bn=True)
    esd = ri.encoder_state_dict(0)
    cfg = ri.HIFIGAN_CONFIG_16K
    gsd = go.fold_weight_norm(ri.hifigan_state_dict(cfg, 0))
    parts = torch.rand(n_utt * PARTIALS, PFRAMES, 40, generator=torch.Generator().manual_seed(7)) * 0.2
    tc = int(lens.max())
    ch = chars[:, :tc].clone()
    for b in range(n_utt):
        ch[b, lens[b]:] = 0
    g = torch.Generator().manual_seed(9)
    nst = frames // R
    masks = [torch.rand(n_utt, tc, 256, generator=g) < 0.5 for _ in range(2)] + \
            [torch.rand(n_utt, 256, generator=g) < 0.5 for _ in range(2 * nst)]
    t0 = time.perf_counter()
    with torch.no_grad():
        pe = eo.embed_frames(esd, parts).view(n_utt, PARTIALS, -1).mean(1)
        emb = pe / pe.norm(dim=1, keepdim=True)
        mel, lin, _ = to.generate(tsd, ch, emb, frames, -1, 10, masks, r=R)
        n = 0
        for b in range(n_utt):  # batch-1 vocoder calls like hifigan/inference.py:66-70
            n += go.hifigan_forward(gsd, cfg, lin[b:b + 1]).numel()
    dt = time.perf_counter() - t0
    return n / dt, dt


def run_reference(args, threads):
    per = []
    n_utt, frames = 8, 200  # bounded sample per step
    for s in range(args.warmup + args.steps):
        v, dt = cpu_oracle(n_utt, threads, frames)
        if s >= args.warmup:
            per.append(dt)
    secs = sum(per)
    v = n_utt * frames * 200 * args.steps / secs
    print(json.dumps({
        "impl": "reference", "metric": "vocoder audio samples/sec", "value": v, "unit": "samples/s",
        "utterances_per_s": v / 80000.0, "n_gpus": args.gpus, "steps": args.steps, "warmup": args.warmup,
        "ms_per_step": 1e3 * secs / args.steps, "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
        "dtype": "f32", "data": "synthetic",
        "config": {"workload": "e2e_cfg5: encoder -> Tacotron(steps=400, r=2) -> HiFi-GAN, 128 utterances per GPU"},
        "cpu_baseline": {"value": v, "unit": "samples/s", "cores": threads, "kind": "port",
                         "sample": "8 utterances x 200 of 400 decoder frames per step, torch-CPU oracles chained"},
        "e2e": {"value": v, "unit": "samples/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
        "gpu_launches": 0}))


def measure(ctx, args, cpu: bool, steps: int = 2, strong_total: int = 0):
    """weak scaling (default): 128 utterances per GPU.  strong_total=1024: the FIXED 1024-utterance job of BASELINE.json
    configs[4] dealt over however many GPUs there are (N = 1 holds all 1024) - the driver's N = 1,2,4,8 runs give
    the strong-scaling curve."""
    import numpy as np
    import torch

    sys.path.insert(0, str(ROOT / "synth_weights"))  # seeded random-init weights (no checkpoints exist)
    import ref_init as ri
    from bench_common import cpu_child, host_threads, log
    from mockingbird_b200 import _lib
    from mockingbird_b200.distributed import shard_utterances
    from mockingbird_b200.encoder import inference as enc_inf
    from mockingbird_b200.encoder.model import SpeakerEncoder
    from mockingbird_b200.synthesizer.hparams import hparams as shp
    from mockingbird_b200.synthesizer.inference import Synthesizer
    from mockingbird_b200.vocoder.hifigan import inference as gan_vocoder

    rank, world, dev = ctx.rank, ctx.world, ctx.dev
    # models: every rank builds the objects, rank 0's packed weights are broadcast over NCCL
    enc = SpeakerEncoder(dev)
    enc.load_state_dict(ri.encoder_state_dict(0))
    enc.eval()
    enc_inf.set_model(enc, dev)
    syn = Synthesizer("unused.pt", verbose=False)
    taco = syn.load_state(ri.tacotron_state_dict(0, r=R, randomize_bn=True))
    taco.to(dev)
    cfg = ri.HIFIGAN_CONFIG_16K
    gen = gan_vocoder.load_state(ri.hifigan_state_dict(cfg, 0), cfg)
    if world > 1:
        for m in (enc, taco, gen):
            ctx.dist.broadcast(m.packed_arena(), src=0)
    old_bs = shp.synthesis_batch_size
    shp.synthesis_batch_size = TBATCH

    n_total = strong_total if strong_total else UTT_PER_GPU * world
    lens, chars = make_utterances(n_total)
    mine = shard_utterances(lens.tolist(), rank, world)
    n_mine = len(mine)
    seqs = [chars[i, : int(lens[i])].tolist() for i in mine]  # sorted longest first -> little padding per batch
    parts = [(torch.rand(PARTIALS, PFRAMES, 40, generator=torch.Generator().manual_seed(1000 + i)) * 0.2).numpy() for i in mine]
    parts_dev = torch.from_numpy(np.concatenate(parts)).to(dev)
    offsets = list(range(0, n_mine * PARTIALS + 1, PARTIALS))
    chars_dev = []
    for s0 in range(0, n_mine, TBATCH):
        tc = max(len(q) for q in seqs[s0:s0 + TBATCH])
        c = torch.zeros(min(TBATCH, n_mine - s0), tc, dtype=torch.int32)
        for b, q in enumerate(seqs[s0:s0 + TBATCH]):
            c[b, : len(q)] = torch.tensor(q, dtype=torch.int32)
        chars_dev.append(c.to(dev))
    lib = _lib.lib()
    produced = {"samples": 0}

    def step_resident():
        emb = enc.reduce_partials(enc.forward(parts_dev), offsets)
        n = 0
        wavs = []
        for bi, c in enumerate(chars_dev):
            _, lin, _ = taco.generate(c, emb[bi * TBATCH: bi * TBATCH + c.shape[0]], steps=STEPS, style_idx=-1, min_stop_token=10)
            for v in range(0, lin.shape[0], VBATCH):
                wavs.append(gen(lin[v:v + VBATCH].contiguous()))
                n += wavs[-1].numel()
        produced["samples"] = n
        ctx.outputs = {"wav": torch.cat([w.reshape(w.shape[0], -1) for w in wavs])}

    def step_e2e():
        embeds = enc_inf.embed_utterances_frames(parts)
        specs = syn.synthesize_from_sequences(seqs, list(embeds), False, -1, 10, STEPS)
        wavs = gan_vocoder.infer_waveforms(specs, batch_size=VBATCH)
        produced["samples"] = sum(len(w) for w in wavs)

    try:
        l0 = lib.mb_launch_count()
        r = ctx.timed(step_resident, steps, 1, 0.0, host_clock=True)
        launches = int(lib.mb_launch_count() - l0) * steps // (1 + 2 * steps)
        n_res = produced["samples"]
        # stage split of one resident step (events between stages)
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
        torch.cuda.synchronize()
        ev[0].record()
        emb = enc.reduce_partials(enc.forward(parts_dev), offsets)
        ev[1].record()
        lins = [taco.generate(c, emb[bi * TBATCH: bi * TBATCH + c.shape[0]], steps=STEPS, style_idx=-1, min_stop_token=10)[1]
                for bi, c in enumerate(chars_dev)]
        ev[2].record()
        for lin in lins:
            for v in range(0, lin.shape[0], VBATCH):
                gen(lin[v:v + VBATCH].contiguous())
        ev[3].record()
        torch.cuda.synchronize()
        split = {"encoder_ms": ev[0].elapsed_time(ev[1]), "tacotron_ms": ev[1].elapsed_time(ev[2]),
                 "hifigan_ms": ev[2].elapsed_time(ev[3])}
        del lins
        e = ctx.timed(step_e2e, steps, 1, 0.0, host_clock=True)
        n_e2e = produced["samples"]
    finally:
        shp.synthesis_batch_size = old_bs
    # totals over ranks (shards differ by at most one utterance)
    tot = torch.tensor([float(n_res), float(n_e2e)], device=dev)
    if world > 1:
        ctx.dist.all_reduce(tot)
    if rank != 0:
        return None
    ms = r["ms"] / steps
    cpu_d = None
    if cpu:
        threads = host_threads()
        rc = cpu_child("e2e_cfg5", 16, threads, 300.0)
        if rc:
            cpu_d = {"value": rc["value"], "unit": "samples/s", "cores": threads, "kind": "port",
                     "sample": f"16 utterances x 200 of 400 decoder frames ({rc['seconds']:.1f} s), torch-CPU oracles chained"}
    value = float(tot[0]) / (ms * 1e-3)
    h2d = sum(p.nbytes for p in parts) + sum(len(q) for q in seqs) * 8 + n_mine * 256 * 4 + n_mine * 80 * STEPS * 4
    d2h = n_mine * 256 * 4 + n_mine * 80 * STEPS * 4 + n_e2e * 4
    flops = 2.0 * n_mine * (20.99e6 * (STEPS // R) + 8.03e6 * STEPS + 3.2e6 * 70)
    taco_s = split["tacotron_ms"] * 1e-3
    name = (f"e2e_cfg5 strong: encoder -> Tacotron(steps=400, r=2) -> HiFi-GAN on a FIXED {n_total} utterances dealt over {world} GPU(s)"
            if strong_total else
            f"e2e_cfg5: encoder -> Tacotron(steps=400, r=2) -> HiFi-GAN, 128 utterances per GPU ({n_total} total), length-sorted round-robin shards")
    return {
        "metric": "vocoder audio samples/sec", "value": value, "unit": "samples/s",
        "utterances_per_s": value / (STEPS * 200), "n_gpus": world, "steps": steps,
        "ms_per_step": ms, "rtf": (ms * 1e-3) / (float(tot[0]) / world / 16000.0), "higher_is_better": True,
        "scaling": "strong" if strong_total else "weak",
        "dtype": "f32-equivalent (encoder, Tacotron: 3-term f16 split) / f16 operands + f32 accumulate (HiFi-GAN)",
        "config": {"workload": name, "utterances_total": n_total, "utterances_this_rank": n_mine, "parallelism": f"dp{world}",
                   "l2": "per-step working set (activations of >= 128 utterances) exceeds L2"},
        "stage_split_ms": split,
        "burst": {"value": float(tot[0]) * steps / (r["ms_burst"] * 1e-3)},
        "e2e": {"value": float(tot[1]) * steps / (e["ms"] * 1e-3), "unit": "samples/s", "h2d_bytes_per_step": int(h2d),
                "d2h_bytes_per_step": int(d2h), "ms_per_step": e["ms"] / steps,
                "surface": "encoder.inference.embed_utterances_frames -> Synthesizer.synthesize_from_sequences -> "
                           "hifigan.inference.infer_waveforms (host numpy between the stages, like the reference's callers)"},
        "gpu_launches": launches, "clocks": r["clocks"],
        "roofline": {"bound": "latency", "kernel": "Tacotron stage (200 dependent decoder steps per batch of 64)",
                     "achieved": flops / taco_s / 1e12, "peak": 72.0, "unit": "TFLOP/s",
                     "frac": flops / taco_s / 1e12 / 72.0, "traffic": None,
                     "note": "pipeline of three models; per-stage times in stage_split_ms; the HiFi-GAN stage has its own roofline in the headline"},
        "cpu_baseline": cpu_d}
