"""Many texts through Tacotron, each computed as its own B = 1 generate (Tacotron.generate_many); prints one JSON line.

Workload: N in {64, 256} seeded token sequences of 20-150 characters, random-init weights (synth_weights/ref_init.py, r = 2),
style_idx = -1, min_stop_token = 10.  The random weights never pass that stop threshold, so every utterance runs to its own
cap of 5 frames per character (100-750 frames), and all three arms compute the same utterance lengths:
  many     generate_many: length-sorted ragged batches of at most MANY_CHUNK_ROWS rows, every row stopping at its own cap
           (also at chunk sizes 32 and 64 for N = 256: the measurement behind the default)
  padded   the reference's batching: batches of 16 in input order, each run to its longest cap, which is what a batch-wide
           stop costs (generate on the padded batch)
  single   one B = 1 generate per text
useful_frames_per_s counts each utterance's own frames; row_step_ratio = computed row-steps / useful row-steps, with a chunk's
computed steps taken as its longest cap (the stop is polled every 16 steps, so at most 15 more run).  Every call is timed with
CUDA events around the whole call, median of --steps runs after --warmup; the card's name and power limit are read in the same run.

    python bench_tacotron_many.py --steps 3 --warmup 1
"""
from __future__ import annotations

import argparse
import json
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "synth_weights"))

from bench_wavernn_mol import _card, _time  # noqa: E402

R, FRAMES_PER_CHAR, MIN_STOP, PAD_BATCH = 2, 5, 10, 16


def _inputs(n, seed):
    import torch

    g = torch.Generator().manual_seed(seed)
    lengths = torch.randint(20, 151, (n,), generator=g).tolist()
    seqs = [torch.randint(2, 75, (t,), generator=g) for t in lengths]
    emb = torch.rand(n, 256, generator=g)
    return seqs, emb / emb.norm(dim=1, keepdim=True), [FRAMES_PER_CHAR * t for t in lengths]


def _steps(frames):
    return -(-frames // R)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    args = ap.parse_args()
    import torch

    import ref_init as ri
    from mockingbird_b200.synthesizer.inference import Synthesizer
    from mockingbird_b200.synthesizer.models.tacotron import MANY_CHUNK_ROWS, many_plan

    if not torch.cuda.is_available():
        raise SystemExit("bench_tacotron_many.py measures on a CUDA device; none is visible")
    torch.cuda.set_device(0)
    model = Synthesizer("unused.pt", verbose=False).load_state(ri.tacotron_state_dict(0, r=R, randomize_bn=True))
    result = {"workload": "Tacotron generate_many: texts of 20-150 chars, caps of 5 frames per char, r=2, min_stop_token=10, "
                          "style_idx=-1", "card": _card(), "steps": args.steps, "warmup": args.warmup,
              "default_chunk_rows": MANY_CHUNK_ROWS,
              "unit": "useful_frames_per_s = sum of each utterance's own frames / s of the whole call"}

    def report(ms, useful_frames, computed, useful):
        return {"ms": round(ms, 1), "useful_frames_per_s": round(useful_frames / (ms * 1e-3), 1),
                "row_step_ratio": round(computed / useful, 3)}

    for n in (64, 256):
        seqs, emb, caps = _inputs(n, 100 + n)
        useful_frames = sum(_steps(c) * R for c in caps)
        useful = sum(_steps(c) for c in caps)
        entry = {"chars_min_mean_max": [min(len(s) for s in seqs), round(sum(len(s) for s in seqs) / n, 1),
                                        max(len(s) for s in seqs)]}
        seeds = list(range(n))
        got = model.generate_many(seqs, emb, steps=caps, style_idx=-1, min_stop_token=MIN_STOP, seeds=seeds)
        assert [o[0].shape[1] for o in got] == [_steps(c) * R for c in caps], "an utterance stopped before its cap"
        for rows in sorted({MANY_CHUNK_ROWS, 32, 64} if n == 256 else {MANY_CHUNK_ROWS}):
            plan = many_plan([len(s) for s in seqs], rows)
            computed = sum(len(c) * max(_steps(caps[i]) for i in c) for c in plan)
            ms = _time(lambda: model.generate_many(seqs, emb, steps=caps, style_idx=-1, min_stop_token=MIN_STOP, seeds=seeds,
                                                   chunk_rows=rows), args.steps, args.warmup)
            entry[f"many_chunk{rows}"] = report(ms, useful_frames, computed, useful)
        batches = []
        for k in range(0, n, PAD_BATCH):
            idx = list(range(k, min(n, k + PAD_BATCH)))
            tc = max(len(seqs[i]) for i in idx)
            chars = torch.zeros(len(idx), tc, dtype=torch.long)
            for b, i in enumerate(idx):
                chars[b, : len(seqs[i])] = seqs[i]
            batches.append((chars.cuda(), emb[idx].cuda(), max(caps[i] for i in idx)))

        def padded():
            for chars, e, cap in batches:
                model.generate(chars, e, steps=cap, style_idx=-1, min_stop_token=MIN_STOP)

        computed = sum(c.shape[0] * _steps(cap) for c, _, cap in batches)
        entry["padded16"] = report(_time(padded, args.steps, args.warmup), useful_frames, computed, useful)
        singles = [(s[None].cuda(), emb[i:i + 1].cuda(), caps[i]) for i, s in enumerate(seqs)]

        def single():
            for chars, e, cap in singles:
                model.generate(chars, e, steps=cap, style_idx=-1, min_stop_token=MIN_STOP)

        entry["single"] = report(_time(single, args.steps, args.warmup), useful_frames, useful, useful)
        best = entry[f"many_chunk{MANY_CHUNK_ROWS}"]["ms"]
        entry["speedup_vs_padded16"] = round(entry["padded16"]["ms"] / best, 2)
        entry["speedup_vs_single"] = round(entry["single"]["ms"] / best, 2)
        result[f"N{n}"] = entry
    print(json.dumps(result))


if __name__ == "__main__":
    main()
