"""VITS on the GPU, one JSON line: one ~10 s utterance (device time and the whole infer call), 64 texts of 20-150 tokens
through infer_many against one infer per text, and the reference's Vits.infer on the CPU for context (child process, only
where the reference tree and its harness exist; absent otherwise).  Usual VITS shape (synth_weights/ref_init.VITS_CONFIG),
seeded weights; the decoder in `--precision`.  Writes nothing to the tree."""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "synth_weights"))


def _cpu_reference(tokens: int, length_scale: float):
    """Vits.infer of the live reference on the host cores, in a child process (None where the reference is absent)"""
    code = f"""
import sys, time, json, torch
sys.path.insert(0, {str(ROOT / 'oracle')!r}); sys.path.insert(0, {str(ROOT / 'synth_weights')!r})
import ref_harness
if not ref_harness.reference_available(): print('null'); raise SystemExit
import ref_init as ri, make_golden_vits as mg
m = mg.build_vits(ri.VITS_CONFIG, ri.vits_state_dict(ri.VITS_CONFIG, 0))
x = torch.randint(0, 80, (1, {tokens}), generator=torch.Generator().manual_seed(1)); emo = torch.randn(1, 1024)
torch.manual_seed(0)
with torch.no_grad():
    t = time.perf_counter(); o = m.infer(x, torch.tensor([{tokens}]), sid=torch.tensor([0]), emo=emo, noise_scale=.667,
                                         noise_scale_w=.8, length_scale={length_scale})[0]; dt = time.perf_counter() - t
print(json.dumps({{"ms": dt * 1e3, "samples": o.shape[-1], "threads": torch.get_num_threads()}}))
"""
    try:
        out = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=1200)
        line = out.stdout.strip().splitlines()[-1] if out.stdout.strip() else "null"
        return json.loads(line)
    except Exception:
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--precision", default="f16x3")
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--no-cpu", action="store_true")
    args = ap.parse_args()
    import ref_init as ri
    from mockingbird_b200 import _lib
    from mockingbird_b200.synthesizer.models.vits import Vits

    dev = _lib.require_cuda()
    cfg = ri.VITS_CONFIG
    m = Vits(**cfg, precision=args.precision)
    m.load_state_dict(ri.vits_state_dict(cfg, 0))
    m.cuda().eval()
    m.remove_weight_norm()
    g = torch.Generator().manual_seed(1)
    tokens = 200
    x = torch.randint(0, cfg["n_vocab"], (1, tokens), generator=g)
    emo = torch.randn(1, 1024, generator=g)
    sid = torch.tensor([0])
    # length_scale so that the utterance lasts about 10 s at 22.05 kHz
    torch.manual_seed(0)
    o = m.infer(x, torch.tensor([tokens]), sid=sid, emo=emo, noise_scale=.667, noise_scale_w=.8)[0]
    ls = 1.0
    for _ in range(3):  # ceil and the SDP make the length only roughly proportional to length_scale
        ls *= 10 * 22050 / o.shape[-1]
        torch.manual_seed(0)
        o = m.infer(x, torch.tensor([tokens]), sid=sid, emo=emo, noise_scale=.667, noise_scale_w=.8, length_scale=ls)[0]
    def run():
        torch.manual_seed(0)  # the same noise, so the same length, in every repetition
        return m.infer(x, torch.tensor([tokens]), sid=sid, emo=emo, noise_scale=.667, noise_scale_w=.8, length_scale=ls)

    for _ in range(3):
        o = run()[0]
    torch.cuda.synchronize()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    wall, dev_ms = [], []
    for _ in range(args.reps):
        t = time.perf_counter()
        ev[0].record()
        run()
        ev[1].record()
        torch.cuda.synchronize()
        wall.append((time.perf_counter() - t) * 1e3)
        dev_ms.append(ev[0].elapsed_time(ev[1]))
    samples = int(o.shape[-1])
    # 64 texts of 20-150 tokens
    lens = torch.randint(20, 151, (64,), generator=g).tolist()
    seqs = [torch.randint(0, cfg["n_vocab"], (n,), generator=g) for n in lens]
    emos = torch.randn(64, 1024, generator=g)
    sids = [i % cfg["n_speakers"] for i in range(64)]
    seeds = list(range(64))
    m.infer_many(seqs, sids, emos, seeds)
    torch.cuda.synchronize()
    t = time.perf_counter()
    wavs = m.infer_many(seqs, sids, emos, seeds)
    many_ms = (time.perf_counter() - t) * 1e3
    t = time.perf_counter()
    for i in range(64):
        m.infer_many([seqs[i]], [sids[i]], emos[i:i + 1], [seeds[i]])
    single_ms = (time.perf_counter() - t) * 1e3
    total = sum(w.size for w in wavs)
    props = torch.cuda.get_device_properties(dev)
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                               timeout=30).stdout.strip().splitlines()[0]
    except Exception:
        power = None
    res = {"metric": "vits", "gpu": props.name, "power_limit": power, "precision": args.precision, "config": "ref_init.VITS_CONFIG",
           "utterance": {"tokens": tokens, "samples": samples, "seconds_audio": samples / 22050,
                         "device_ms": sorted(dev_ms)[len(dev_ms) // 2], "call_ms": sorted(wall)[len(wall) // 2],
                         "realtime_factor": samples / 22050 / (sorted(wall)[len(wall) // 2] / 1e3)},
           "many": {"texts": 64, "tokens": [min(lens), max(lens)], "samples": int(total), "infer_many_ms": many_ms,
                    "one_call_per_text_ms": single_ms, "speedup": single_ms / many_ms}}
    if not args.no_cpu:
        ref = _cpu_reference(tokens, ls)
        if ref is not None:
            res["cpu_reference"] = ref
    print(json.dumps(res))


if __name__ == "__main__":
    main()
