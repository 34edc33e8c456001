"""Achieved HBM bandwidth of every launch of the HiFi-GAN tensor-core forward, per launch and per stage.

usage: python tools/gan_stage_bandwidth.py [--batch 32] [--frames 256] [--reps 10] [--out file.json]

Times each op with CUDA events (mb_gan_forward_profiled; a fused resblock pair is one launch, timed at its first conv) and
divides by the bytes the launch moves, counted from the plan (layer_info / tc_plan_info) with the plane rules of tc_forward
(gan_tc.cu) for the f16tc precision:
  * operand: the fp16 input plane once (C x 2 B per input row; a 3-term-split layer reads its hi/lo plane, 2 C x 2 B); re-reads
    of halo rows and of the phases of a transposed conv are L2 hits and not counted;
  * residual (convs2 / fused pair): fp32 (C x 4 B) in the full-rate stage, the activated fp16 plane (C x 2 B) elsewhere;
  * outputs: the fp16 plane where a tensor-core conv reads it (hi/lo, 2 C x 2 B, when that conv is a 3-term-split layer),
    the fp32 plane where a residual or the fp32 conv_post reads it;
  * the MRF running sum S of a resblock's last pair: written (store), read and written (add, by L2 reductions), or read
    (add_div, before the output planes of the stage).
This is the traffic the launches cannot avoid; 'layer_work' (bench.py roofline) is a different, layer-granular fp32 figure.
The HiFi-GAN 16 kHz config only (ResBlock1, the cfg-2 benchmark shape by default)."""
import argparse
import json
import re
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "synth_weights"))

import torch  # noqa: E402

import ref_init as ri  # noqa: E402
from mockingbird_b200.vocoder.hifigan.models import Generator  # noqa: E402

HBM_GBS = 3350.0  # H100 SXM data sheet


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "power limit unknown"
    return f"{name}, {q}"


def layers(g):
    out = []
    for i in range(g.num_layers()):
        info = g.layer_info(i)
        kind, name = info.split()[:2]
        d = {k: int(v) for k, v in (t.split("=") for t in info.split()[2:])}
        p = g.tc_plan_info(i) if kind == "conv" else {}
        out.append((kind, name, d, p))
    return out


def launch_bytes(ops, i, B, T):
    """(label, bytes) of the launch that op i starts, or None when op i belongs to the previous op's fused pair"""
    kind, name, d, p = ops[i]
    if kind != "conv":
        return "add", 3 * 4 * B * T * d["rate_in"] * d["cout"]
    if p.get("fused_prev"):
        return None
    full_rate = max(o[2]["rate_in"] * (o[2]["stride"] if o[0] == "conv" else 1) for o in ops)
    rate_out = d["rate_in"] * d["stride"]
    rows_in, rows_out = B * T * d["rate_in"], B * T * rate_out
    nxt = next((o for o in ops[i + 1 + (1 if p.get("fuse_next") else 0):] if o[0] == "conv"), None)
    out16 = 0 if nxt is None or not nxt[3]["use_tc"] else (4 if nxt[3]["x3"] else 2)  # bytes per output channel
    if p.get("split3"):  # conv_pre: mel -> split plane (256 ch), then Cout / 256 launches over it
        n_half = d["cout"] // 256
        return "conv_pre", rows_in * (d["cin"] * 4 + 512 + n_half * 512) + rows_out * d["cout"] * out16
    if not p.get("use_tc"):  # conv_post (fp32 kernel): S in, wav out
        return name, rows_in * d["cin"] * 4 + rows_out * d["cout"] * 4
    C = d["cout"]
    operand = rows_in * d["cin"] * (4 if p["x3"] else 2)
    if name.startswith("ups."):
        return "ups", operand + rows_out * C * (2 + (4 if rate_out == full_rate else 0))
    m = re.match(r"resblocks\.(\d+)\.convs([12])\.(\d+)$", name)
    last_name = ops[i + 1][1] if p.get("fuse_next") else name
    m2 = re.match(r"resblocks\.(\d+)\.convs2\.(\d+)$", last_name)
    if m and m.group(2) == "1" and not m2:  # unfused c1: intermediate fp16 plane for c2
        return "convs1", operand + rows_out * C * 2
    label = "pair" if p.get("fuse_next") else "convs2"
    ld = ops[i + 1][2] if p.get("fuse_next") else d
    res = rows_out * C * (4 if rate_out == full_rate else 2)
    rb = m2.group(1)
    k_last = max(int(o[1].split(".")[-1]) for o in ops if o[1].startswith(f"resblocks.{rb}.convs2."))
    if int(m2.group(2)) < k_last:  # x of the next pair: its operand, and its residual
        out = rows_out * C * (2 + (4 if rate_out == full_rate else 0))
    elif ld["mode"] == 0:  # S = v
        out = rows_out * C * 4
    elif ld["mode"] == 1:  # S += v in L2
        out = rows_out * C * 8
    else:  # S = (S + v) / 3 -> the next stage's planes
        out = rows_out * C * 4 + rows_out * C * (out16 if out16 else 4)
    return label, operand + res + out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--frames", type=int, default=256)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default=None, help="also write the table as JSON")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("gan_stage_bandwidth: needs a CUDA device")
    cfg = ri.HIFIGAN_CONFIG_16K
    g = Generator(cfg, precision="f16tc").cuda()
    g.load_state_dict(ri.hifigan_state_dict(cfg, 0))
    g.eval()
    g.remove_weight_norm()
    mel = (torch.rand(a.batch, 80, a.frames, generator=torch.Generator().manual_seed(2)) * 8 - 4).cuda()
    for _ in range(3):
        g(mel)
        g.forward_profiled(mel)
    n = g.num_layers()
    ms = [0.0] * n
    for _ in range(a.reps):
        _, t = g.forward_profiled(mel)
        for i in range(n):
            ms[i] += t[i] / a.reps
    ops = layers(g)
    rows = []
    for i in range(n):
        lb = launch_bytes(ops, i, a.batch, a.frames)
        if lb is None:
            rows[-1]["ms"] += ms[i]  # the fused pair's second event window (nothing launched in it)
            continue
        kind, name, d, p = ops[i]
        rate_out = d["rate_in"] * (d.get("stride", 1) if kind == "conv" else 1)
        rows.append({"idx": i, "name": name, "kind": lb[0], "C": d["cout"], "rate_out": rate_out,
                     "kernel": list(p.get("kernel", ())), "ms": ms[i], "bytes": lb[1]})
    hdr = f"{'idx':>3} {'launch':<24} {'kind':<8} {'C':>4} {'kernel':<14} {'ms':>8} {'MB':>8} {'GB/s':>7} {'%HBM':>5}"
    print(f"card: {card()}")
    print(f"HiFi-GAN 16 kHz f16tc, batch {a.batch} x {a.frames} frames, mean of {a.reps} profiled forwards; HBM {HBM_GBS:.0f} GB/s "
          "(data sheet)")
    print(hdr)
    for r in rows:
        gbs = r["bytes"] / (r["ms"] * 1e-3) / 1e9 if r["ms"] > 0 else 0.0
        r["gbs"] = gbs
        print(f"{r['idx']:>3} {r['name']:<24} {r['kind']:<8} {r['C']:>4} {','.join(map(str, r['kernel'])):<14} {r['ms']:>8.4f} "
              f"{r['bytes'] / 1e6:>8.1f} {gbs:>7.0f} {100 * gbs / HBM_GBS:>5.1f}")
    print("\nper stage (C, kind)")
    stages = {}
    for r in rows:
        s = stages.setdefault((r["C"], r["kind"]), [0, 0.0, 0])
        s[0] += 1
        s[1] += r["ms"]
        s[2] += r["bytes"]
    summary = []
    for (c, kind), (cnt, t, b) in sorted(stages.items(), key=lambda kv: (-kv[0][0], kv[0][1])):
        gbs = b / (t * 1e-3) / 1e9
        summary.append({"C": c, "kind": kind, "launches": cnt, "ms": t, "bytes": b, "gbs": gbs})
        print(f"  C={c:<4} {kind:<8} launches={cnt:<3} ms={t:8.3f}  GB={b / 1e9:7.3f}  {gbs:6.0f} GB/s  {100 * gbs / HBM_GBS:5.1f} %")
    tot_ms, tot_b = sum(r["ms"] for r in rows), sum(r["bytes"] for r in rows)
    print(f"  total   ms={tot_ms:.3f}  GB={tot_b / 1e9:.3f}  {tot_b / (tot_ms * 1e-3) / 1e9:.0f} GB/s")
    if a.out:
        Path(a.out).parent.mkdir(parents=True, exist_ok=True)
        Path(a.out).write_text(json.dumps({"card": card(), "launches": rows, "stages": summary}, indent=1) + "\n")


if __name__ == "__main__":
    main()
