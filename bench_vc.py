"""Voice-conversion back half on one GPU: the 24 kHz HiFi-GAN vocoder, and ppg2mel followed by that vocoder; prints one JSON line.

Seeded random-init weights (ref_init.hifigan_state_dict(HIFIGAN_CONFIG_24K, 0), the stand-in 24 kHz config: rates [5,4,3,2,2],
kernels [11,9,7,5,5], 512 channels, hop 240; ref_init.ppg2mel_state_dict(0)) and random inputs:
  vocoder   B = 32 x 256 mel frames (61 440 samples per row) in the drop-in default precision ("auto", the mode it picked is
            reported) and in f16x3: ms per batch, samples/s, real-time factor (compute time over audio time); for the auto mode,
            the per-layer device times of the folded upsampling layers ups.{i}.1 (forward_profiled) with their folded MACs and the
            achieved TFLOP/s
  vc        ppg2mel inference_batch on 64 utterances of 3-10 s (300-1000 PPG frames, stop bias lowered so that every row runs to
            its step limit, as in bench_ppg2mel.py), then the vocoder on the postnet mels while they stay on the device
            (length-sorted padded batches of 32 with per-row lengths): total ms and audio seconds per second
  cpu       the torch-CPU oracle vocoding one 3 s utterance, for context
The card name and power limit are read in the same run.

usage: python bench_vc.py [--iters N] [--warmup W] [--no-cpu]
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

from bench_ppg2mel import card, inputs  # noqa: E402

SR = 24000
HOP = 240
FRAME_S = HOP / SR  # 10 ms mel frames


def cuda_timed(fn, iters, warmup):
    """mean ms per call over `iters` calls (CUDA events around the whole loop) and the last output"""
    import torch

    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(iters):
        out = fn()
    t1.record()
    t1.synchronize()
    return t0.elapsed_time(t1) / iters, out


def vocoder(cfg, sd, precision):
    from mockingbird_b200.vocoder.hifigan.models import Generator

    g = Generator(cfg, precision=precision).cuda()
    g.load_state_dict(sd)
    g.eval()
    g.remove_weight_norm()
    return g


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--no-cpu", action="store_true")
    a = ap.parse_args()
    import torch

    import ref_init as ri
    from mockingbird_b200.ppg2mel import MelDecoderMOLv2
    from mockingbird_b200.vocoder._gan import infer_waveforms_batched

    if not torch.cuda.is_available():
        raise SystemExit("bench_vc.py needs a CUDA device")
    torch.cuda.set_device(0)
    cfg = ri.HIFIGAN_CONFIG_24K
    sd = ri.hifigan_state_dict(cfg, 0)
    result = {"workload": "24 kHz HiFi-GAN (stand-in config) B = 32 x 256 frames; vc = ppg2mel 64 x 3-10 s + 24 kHz vocoder"}
    name, power = card()
    result["gpu"], result["power_limit"] = name, power

    # ---- vocoder, B = 32 x 256 frames
    B, T = 32, 256
    mel = (torch.rand(B, 80, T, generator=torch.Generator().manual_seed(2)) * 8 - 4).cuda()
    audio_s = B * T * FRAME_S
    voc = {"batch": B, "frames": T, "samples_per_row": T * HOP}
    g_auto = None
    for precision in ("auto", "f16x3"):
        g = vocoder(cfg, sd, precision)
        with torch.no_grad():
            ms, _ = cuda_timed(lambda: g(mel), a.iters, a.warmup)
        key = "auto" if precision == "auto" else "f16x3"
        voc[key] = {"mode": g.precision, "ms_per_batch": round(ms, 3), "samples_per_s": round(B * T * HOP / (ms / 1e3), 1),
                    "rtf": round(ms / 1e3 / audio_s, 6)}
        if precision == "auto":
            voc[key]["calibration"] = {k: (round(v, 7) if isinstance(v, float) else v) for k, v in g.calibration.items()}
            g_auto = g
    # per-layer device times of the folded upsampling layers (auto mode)
    g_auto.forward_profiled(mel)
    _, per_layer = g_auto.forward_profiled(mel)
    layers = []
    for i in range(g_auto.num_layers()):
        lname = g_auto.layer_info(i).split()[1]
        if lname.startswith("ups."):
            macs, _ = g_auto.layer_work(i, B, T)
            ms = per_layer[i]
            layers.append({"layer": lname, "ms": round(ms, 4), "folded_gmac": round(macs / 1e9, 3),
                           "tflops": round(2 * macs / (ms / 1e3) / 1e12, 2) if ms > 0 else None,
                           "x3": g_auto.tc_plan_info(i)["x3"]})
    voc["ups_layers_auto"] = layers
    voc["forward_profiled_total_ms"] = round(sum(per_layer), 3)
    result["vocoder"] = voc

    # ---- voice-conversion back half: ppg2mel (64 x 3-10 s) -> 24 kHz vocoder, mels kept on the device
    psd = ri.ppg2mel_state_dict(0)
    psd["decoder.stop_layer.linear_layer.bias"] = psd["decoder.stop_layer.linear_layer.bias"] - 10.0  # run to the step limit
    model = MelDecoderMOLv2(**ri.PPG2MEL_CONFIG).cuda()
    model.load_state_dict(psd)
    model.eval()
    lengths = torch.randint(300, 1001, (64,), generator=torch.Generator().manual_seed(2)).tolist()
    utts, spk = inputs(lengths, 4)

    def vc():
        outs = model.inference_batch(utts, spk, seed=3)
        mels = [o[1].t() if o[1].shape[-1] == 80 else o[1] for o in outs]  # postnet mel as [80, T]
        return mels, infer_waveforms_batched(g_auto, "cuda", mels)

    with torch.no_grad():
        ms, (mels, wavs) = cuda_timed(vc, max(1, a.iters // 2), 1)
        t_mel, _ = cuda_timed(lambda: model.inference_batch(utts, spk, seed=3), max(1, a.iters // 2), 1)
    frames = sum(m.shape[1] for m in mels)
    assert all(w.numel() == m.shape[1] * HOP for w, m in zip(wavs, mels))
    result["vc"] = {"utterances": 64, "mel_frames": frames, "audio_s": round(frames * FRAME_S, 2), "ms_total": round(ms, 3),
                    "ms_ppg2mel": round(t_mel, 3), "ms_vocoder": round(ms - t_mel, 3),
                    "audio_s_per_s": round(frames * FRAME_S / (ms / 1e3), 1), "vocoder_mode": g_auto.precision}

    # ---- torch-CPU oracle, one 3 s utterance
    if not a.no_cpu:
        sys.path.insert(0, str(ROOT / "oracle"))
        import hifigan24k_oracle as o24

        m3 = torch.rand(1, 80, 300, generator=torch.Generator().manual_seed(3)) * 8 - 4
        t0 = time.perf_counter()
        with torch.no_grad():
            o24.hifigan24k_forward(sd, cfg, m3)
        cpu = time.perf_counter() - t0
        result["cpu_oracle"] = {"frames": 300, "audio_s": 3.0, "s": round(cpu, 3), "rtf": round(cpu / 3.0, 3),
                                "threads": torch.get_num_threads()}
    print(json.dumps(result), flush=True)


if __name__ == "__main__":
    main()
