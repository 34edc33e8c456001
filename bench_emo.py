"""Emotion-vector extraction (the wav2vec2 model of extract_emo, stand-in config of ref_init) on one GPU.  Prints one JSON
line: the card and its power limit, one 10 s clip (device time and whole call), 64 clips of 3-10 s through extract_emos
against 64 extract_emo calls, algorithmic GMAC and TFLOP/s (the tensor-core GEMMs issue 3x that as a 3-term fp16 split),
and the float32 torch restatement of one 3 s clip on the host threads.  --profile adds a torch.profiler kernel breakdown
of the 10 s clip in a separate run."""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "oracle"))
sys.path.insert(0, str(ROOT / "synth_weights"))

import ref_init as ri  # noqa: E402


def gmac(cfg: dict, n: int) -> float:
    """multiply-accumulates of one n-sample clip"""
    import wav2emo_oracle as wo

    t, c_in, mac = n, 1, 0
    for c, k, s in zip(cfg["conv_dim"], cfg["conv_kernel"], cfg["conv_stride"]):
        t = (t - k) // s + 1
        mac += t * c * c_in * k
        c_in = c
    D, U, L = cfg["hidden_size"], cfg["intermediate_size"], cfg["num_hidden_layers"]
    T = wo.num_frames(cfg, n)
    mac += T * D * c_in  # projection
    mac += T * D * (D // cfg["num_conv_pos_embedding_groups"]) * cfg["num_conv_pos_embeddings"]
    mac += L * T * (4 * D * D + 2 * D * U)  # q k v o, ff1 ff2
    mac += L * 2 * T * T * D  # scores and context
    return mac / 1e9


def card() -> dict:
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()
    name, power = (out[0].split(", ") + ["?"])[:2] if out else (torch.cuda.get_device_name(0), "?")
    return {"gpu": name, "power_limit": power}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--profile", action="store_true")
    args = ap.parse_args()
    from mockingbird_b200.synthesizer import preprocess_audio as pa
    from mockingbird_b200.synthesizer.models.wav2emo import EmotionExtractorModel

    cfg = ri.WAV2EMO_CONFIG
    sd = ri.wav2emo_state_dict(cfg, 0)
    m = EmotionExtractorModel(cfg)
    m.load_state_dict(sd)
    pa.load_model(m)
    rng = np.random.default_rng(0)
    clip10 = (0.2 * rng.standard_normal(160000)).astype(np.float32)
    clips = [(0.2 * rng.standard_normal(int(n))).astype(np.float32) for n in rng.integers(48000, 160001, 64)]
    if args.profile:
        from torch.profiler import ProfilerActivity, profile

        pa.extract_emo(clip10, 16000, True)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(3):
                pa.extract_emo(clip10, 16000, True)
            torch.cuda.synchronize()
        groups = {"attention": ("attn_tc_kernel",), "gemm": ("tc_big", "im2col"), "pos_conv": ("posconv",),
                  "feature_encoder": ("conv0", "ln_act_rows", "norm_kernel")}
        tot, by = 0.0, {k: 0.0 for k in groups}
        by["other"] = 0.0
        for e in prof.key_averages():
            us = e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total
            if us <= 0:
                continue
            tot += us
            g = next((k for k, keys in groups.items() if any(s in e.key for s in keys)), "other")
            by[g] += us
        print(json.dumps({"workload": "wav2emo_profile_10s", **card(),
                          "share": {k: round(v / tot, 4) for k, v in by.items()}, "device_ms_per_call": tot / 3 / 1e3}))
        return
    for _ in range(2):
        pa.extract_emo(clip10, 16000, True)
    torch.cuda.synchronize()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    wav = torch.from_numpy(clip10).cuda()
    m._forward(wav, [clip10.size], True, False, False)
    ev[0].record()
    for _ in range(args.reps):
        m._forward(wav, [clip10.size], True, False, False)
    ev[1].record()
    torch.cuda.synchronize()
    dev_ms = ev[0].elapsed_time(ev[1]) / args.reps
    t0 = time.perf_counter()
    for _ in range(args.reps):
        pa.extract_emo(clip10, 16000, True)
    call_ms = (time.perf_counter() - t0) * 1e3 / args.reps
    pa.extract_emos(clips)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    pa.extract_emos(clips)
    torch.cuda.synchronize()
    many_ms = (time.perf_counter() - t0) * 1e3
    t0 = time.perf_counter()
    for c in clips:
        pa.extract_emo(c, 16000, True)
    singles_ms = (time.perf_counter() - t0) * 1e3
    g10 = gmac(cfg, clip10.size)
    g64 = sum(gmac(cfg, c.size) for c in clips)
    import wav2emo_oracle as wo  # float32 torch restatement on the host threads, for context

    sd32 = {k: v.float() for k, v in sd.items()}
    x3 = wo.normalize(clip10[:48000])
    torch.set_num_threads(torch.get_num_threads())
    t0 = time.perf_counter()
    with torch.no_grad():
        wo.forward(sd32, cfg, x3, dtype=torch.float32)
    cpu_ms = (time.perf_counter() - t0) * 1e3
    print(json.dumps({
        "workload": "wav2emo", **card(), "config": "stand-in (hidden 1024, 12 layers, 16 heads, 4096 units)",
        "clip10s": {"device_ms": round(dev_ms, 3), "call_ms": round(call_ms, 3), "gmac": round(g10, 2),
                    "tflops": round(2 * g10 / dev_ms, 2)},
        "clips64_3_10s": {"extract_emos_ms": round(many_ms, 2), "extract_emo_x64_ms": round(singles_ms, 2),
                          "gmac": round(g64, 1), "tflops_batched": round(2 * g64 / many_ms, 2)},
        "note": "TFLOP/s are algorithmic (2 x MAC); the tensor-core GEMMs issue 3x their share as a 3-term fp16 split",
        "host_fp32_torch_3s_ms": round(cpu_ms, 1), "host_threads": torch.get_num_threads(),
    }))


if __name__ == "__main__":
    main()
