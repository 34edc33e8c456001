"""Tacotron.generate_stream against generate_many on the same texts, in the same process, alternated; prints one JSON line.

Workloads (random-init weights from synth_weights/ref_init.py, r = 2, style_idx = -1, seeded texts of 20-150 characters as in
bench_tacotron_many.py):
  N256     bench_tacotron_many.py's 256-text list, caps of 5 frames per character, min_stop_token = 10: every text runs to its cap
  N1024    the same generator at 1024 texts
  shared   256 texts with one cap of 750 frames for all and min_stop_token = 4, so the stop rule ends rows at steps the caps
           do not predict (generate_many sorts by characters, not by the steps the texts will take)
For each arm: ms (median of --steps runs after --warmup, host clock around the call with device synchronises), frames_per_s (each
text's own frames over that time), decoder_steps (generate_many: the steps its loop ran per chunk, replayed from its polling
rule and the texts' done steps; generate_stream: the steps its loop counted), first_result_ms (generate_many returns everything at once) and whether every
text's mel, linear and attention are bitwise equal between the arms.  The card's name and power limit are read in the same run.

    python bench_tacotron_stream.py --steps 3 --warmup 1
"""
from __future__ import annotations

import argparse
import json
import statistics
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "synth_weights"))

from bench_tacotron_many import _inputs  # noqa: E402
from bench_wavernn_mol import _card  # noqa: E402

R = 2


def _loop_steps(nst, last):
    """decoder steps generate_many's loop runs for a chunk of nst steps whose last row ends at step `last`: it replays 8-step
    graphs while 8 more steps fit (nst >= 16), polling after every 16 steps and after the last replay, then launches the
    remaining steps directly, polling at every 16th step and at the end; it stops at the first poll that sees every row done
    (tacotron.cu, generate_impl)"""
    si, found = 0, False
    if nst >= 16:
        while si + 8 <= nst and not found:
            si += 8
            if si % 16 == 0 or si + 8 > nst:
                found = last <= si - 1
    while si < nst and not found:
        if si % 16 == 15 or si == nst - 1:
            found = last <= si
        si += 1
    return si


def _many_steps(lengths, frames, caps, chunk_rows):
    """decoder steps generate_many ran over all its chunks, from each text's frames (its done step) and cap"""
    from mockingbird_b200.synthesizer.models.tacotron import many_plan

    total = 0
    for chunk in many_plan(lengths, chunk_rows):
        nst = max(-(-caps[i] // R) for i in chunk)
        total += _loop_steps(nst, max(frames[i] // R for i in chunk) - 1)
    return total


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    args = ap.parse_args()
    import torch

    import ref_init as ri
    from mockingbird_b200.synthesizer.inference import Synthesizer
    from mockingbird_b200.synthesizer.models.tacotron import MANY_CHUNK_ROWS

    if not torch.cuda.is_available():
        raise SystemExit("bench_tacotron_stream.py measures on a CUDA device; none is visible")
    torch.cuda.set_device(0)
    model = Synthesizer("unused.pt", verbose=False).load_state(ri.tacotron_state_dict(0, r=R, randomize_bn=True))
    result = {"workload": "Tacotron generate_stream vs generate_many: texts of 20-150 chars, r=2, style_idx=-1",
              "card": _card(), "steps": args.steps, "warmup": args.warmup, "slots": MANY_CHUNK_ROWS,
              "unit": "frames_per_s = sum of each text's own frames / s of the whole call"}

    def many(seqs, emb, caps, mst, seeds):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = model.generate_many(seqs, emb, steps=caps, style_idx=-1, min_stop_token=mst, seeds=seeds)
        torch.cuda.synchronize()
        ms = (time.perf_counter() - t0) * 1e3
        return out, ms, ms

    def stream(seqs, emb, caps, mst, seeds):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out, first = [None] * len(seqs), None
        for i, mel, lin, attn in model.generate_stream(seqs, emb, steps=caps, style_idx=-1, min_stop_token=mst, seeds=seeds):
            if first is None:
                first = (time.perf_counter() - t0) * 1e3
            out[i] = (mel, lin, attn)
        torch.cuda.synchronize()
        return out, (time.perf_counter() - t0) * 1e3, first

    cases = {"N256": (_inputs(256, 356), 10, False), "N1024": (_inputs(1024, 1124), 10, False),
             "shared": (_inputs(256, 356), 4, True)}
    for name, ((seqs, emb, caps), mst, shared) in cases.items():
        if shared:
            caps = [max(caps)] * len(seqs)
        seeds = list(range(len(seqs)))
        arms = {"many": many, "stream": stream}
        times = {k: [] for k in arms}
        firsts = {k: [] for k in arms}
        outs = {}
        for rep in range(args.warmup + args.steps):
            for k, fn in arms.items():  # alternated in each repetition
                out, ms, first = fn(seqs, emb, caps, mst, seeds)
                outs[k] = out
                if rep >= args.warmup:
                    times[k].append(ms)
                    firsts[k].append(first)
        frames = [o[0].shape[1] for o in outs["many"]]
        useful = sum(frames)
        equal = all(all(a.shape == b.shape and torch.equal(a, b) for a, b in zip(x, y)) for x, y in zip(outs["many"], outs["stream"]))
        steps_many = _many_steps([len(s) for s in seqs], frames, caps, MANY_CHUNK_ROWS)
        entry = {"texts": len(seqs), "min_stop_token": mst, "cap_frames": "shared 750" if shared else "5 per char",
                 "frames_total": useful, "texts_stopped_before_cap": sum(f < -(-c // R) * R for f, c in zip(frames, caps)),
                 "bitwise_equal": equal}
        for k in arms:
            ms = statistics.median(times[k])
            entry[k] = {"ms": round(ms, 1), "frames_per_s": round(useful / (ms * 1e-3), 1),
                        "first_result_ms": round(statistics.median(firsts[k]), 1),
                        "decoder_steps": steps_many if k == "many" else int(model.stream_steps)}
        entry["stream_speedup"] = round(entry["many"]["ms"] / entry["stream"]["ms"], 3)
        result[name] = entry
    print(json.dumps(result))


if __name__ == "__main__":
    main()
