"""PPG extractor (Conformer ASR encoder, stand-in config ref_init.PPGX_CONFIG: D = 144, 4 heads, 16 blocks, Conv2d input
layer without subsampling) on one GPU, and the whole voice-conversion chain wav -> wav; prints one JSON line.
Seeded random-init weights (ref_init.ppg_extractor_state_dict(PPGX_CONFIG, 0)), synthetic 16 kHz wavs (tones + noise):
  b1        one 10 s utterance (B = 1): ms per call, audio seconds per second
  batch     64 utterances of 3-10 s through extract_batch (length-sorted padded calls): ms, audio seconds per second
  b1_device the B = 1 10 s call's device time by kernel family (torch.profiler in a run of its own)
  conv2     device time of embed.conv.2 (conv2d_tc_kernel) in that call, and the achieved TFLOP/s on its algorithmic MACs
            (T x n_mels x D x D x 25)
  chain     extractor -> ppg2mel inference_batch (synthetic lf0_uv of the same length, pyworld is not available; stop bias
            lowered so every row runs to its step limit) -> 24 kHz HiFi-GAN, all on the device, for the 64 utterances
  cpu       the torch-CPU oracle (oracle/ppgx_oracle.py) on one 3 s utterance, for context
The card name and power limit are read in the same run.
usage: python bench_ppgx.py [--iters N] [--warmup W] [--no-cpu]
"""
from __future__ import annotations

import argparse
import json
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "synth_weights"))

from bench_ppg2mel import card  # noqa: E402
from bench_vc import cuda_timed, vocode_on_device, vocoder  # noqa: E402

SR = 16000


def synth(n: int, seed: int):
    import numpy as np

    g = np.random.RandomState(seed)
    t = np.arange(n) / SR
    f = 150 + 100 * g.rand()
    x = 0.3 * np.sin(2 * np.pi * f * t) + 0.2 * np.sin(2 * np.pi * 7.3 * f * t) + 0.05 * g.randn(n)
    return x.astype(np.float32)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--no-cpu", action="store_true")
    a = ap.parse_args()
    import torch

    import ref_init as ri
    from mockingbird_b200.ppg2mel import MelDecoderMOLv2
    from mockingbird_b200.ppg_extractor import build_model

    if not torch.cuda.is_available():
        raise SystemExit("bench_ppgx.py needs a CUDA device")
    torch.cuda.set_device(0)
    cfg = ri.PPGX_CONFIG
    sd = ri.ppg_extractor_state_dict(cfg, 0)
    m = build_model(cfg)
    m.load_state_dict(sd)
    m.cuda().eval()
    result = {"workload": "PPG extractor (stand-in PPGX_CONFIG, D 144, 16 blocks): B = 1 x 10 s; 64 x 3-10 s; "
                          "chain = extractor + ppg2mel + 24 kHz HiFi-GAN"}
    result["gpu"], result["power_limit"] = card()
    # ---- B = 1, 10 s
    w10 = torch.from_numpy(synth(10 * SR, 1))
    lens10 = torch.LongTensor([w10.numel()])
    with torch.no_grad():
        ms, out = cuda_timed(lambda: m(w10[None], lens10), a.iters, a.warmup)
    T = out.shape[1]
    result["b1"] = {"audio_s": 10.0, "frames": T, "ms": round(ms, 3), "audio_s_per_s": round(10.0 / (ms / 1e3), 1)}
    # ---- 64 utterances of 3-10 s
    g = torch.Generator().manual_seed(2)
    secs = (3 + 7 * torch.rand(64, generator=g)).tolist()
    wavs = [synth(int(s * SR), 10 + i) for i, s in enumerate(secs)]
    audio = sum(len(w) for w in wavs) / SR
    with torch.no_grad():
        ms_b, ppgs = cuda_timed(lambda: m.extract_batch(wavs), max(1, a.iters // 2), 1)
    result["batch"] = {"utterances": 64, "audio_s": round(audio, 2), "ms": round(ms_b, 3),
                       "audio_s_per_s": round(audio / (ms_b / 1e3), 1)}
    # ---- embed.conv.2 device time (profiled run of its own)
    from torch.profiler import ProfilerActivity, profile

    with torch.no_grad(), profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(3):
            m(w10[None], lens10)
        torch.cuda.synchronize()
    calls = 3
    groups = {}  # kernel family -> device us per call
    fam = (("conv2d_tc_kernel", "conv2d_tc"), ("tc_big_kernel", "tc_big"), ("attn_kernel", "attn"), ("dw_kernel", "dw"),
           ("ln_tiles_kernel", "layernorm"), ("ln_rows_kernel", "layernorm"), ("act_tiles_kernel", "act_tiles"),
           ("frontend_kernel", "frontend"), ("mvn_kernel", "frontend"), ("conv0_kernel", "conv0"))
    all_us = 0.0
    n_kernels = 0
    for e in prof.events():
        if e.device_type.name != "CUDA" or e.device_time <= 0:
            continue
        name = next((g for k, g in fam if k in e.name), "other")
        groups[name] = groups.get(name, 0.0) + e.device_time / calls
        all_us += e.device_time / calls
        n_kernels += 1
    result["b1_device"] = {"ms": round(all_us / 1e3, 3), "kernels_per_call": n_kernels // calls,
                           "by_kernel_ms": {k: round(v / 1e3, 3) for k, v in sorted(groups.items(), key=lambda kv: -kv[1])}}
    if "conv2d_tc" in groups:
        us = groups["conv2d_tc"]
        macs = T * cfg["frontend_conf"]["n_mels"] * 144 * 144 * 25
        result["conv2"] = {"ms": round(us / 1e3, 4), "gmac": round(macs / 1e9, 2),
                           "tflops": round(2 * macs / (us / 1e6) / 1e12, 1), "share_of_device_time": round(us / all_us, 3)}
    # ---- chain: extractor -> ppg2mel -> 24 kHz vocoder
    psd = ri.ppg2mel_state_dict(0)
    psd["decoder.stop_layer.linear_layer.bias"] = psd["decoder.stop_layer.linear_layer.bias"] - 10.0
    dec = MelDecoderMOLv2(**ri.PPG2MEL_CONFIG).cuda()
    dec.load_state_dict(psd)
    dec.eval()
    voc = vocoder(ri.HIFIGAN_CONFIG_24K, ri.hifigan_state_dict(ri.HIFIGAN_CONFIG_24K, 0), "auto")
    spk = torch.randn(64, 256, generator=torch.Generator().manual_seed(4))

    def chain():
        feats = m.extract_batch(wavs)
        utts = []
        for p in feats:
            n = p.shape[0]
            lf0 = torch.stack([torch.linspace(4.5, 5.5, n, device="cuda"), (torch.arange(n, device="cuda") % 7 > 1).float()], -1)
            utts.append((p, lf0))
        outs = dec.inference_batch(utts, spk, seed=3)
        mels = [o[1].t() for o in outs]
        return feats, vocode_on_device(voc, mels)

    with torch.no_grad():
        ms_c, (feats, outw) = cuda_timed(chain, max(1, a.iters // 2), 1)
    assert all(torch.isfinite(w).all() for w in outw)
    result["chain"] = {"utterances": 64, "audio_in_s": round(audio, 2), "ppg_frames": sum(p.shape[0] for p in feats),
                       "audio_out_s": round(sum(w.numel() for w in outw) / 24000, 2), "ms": round(ms_c, 3),
                       "audio_in_s_per_s": round(audio / (ms_c / 1e3), 1), "vocoder_mode": voc.precision}
    # ---- torch-CPU oracle, one 3 s utterance
    if not a.no_cpu:
        sys.path.insert(0, str(ROOT / "oracle"))
        import ppgx_oracle as po

        w3 = torch.from_numpy(synth(3 * SR, 3))
        t0 = time.perf_counter()
        with torch.no_grad():
            po.forward(sd, cfg, w3)
        cpu = time.perf_counter() - t0
        result["cpu_oracle"] = {"audio_s": 3.0, "s": round(cpu, 3), "threads": torch.get_num_threads()}
    print(json.dumps(result), flush=True)


if __name__ == "__main__":
    main()
