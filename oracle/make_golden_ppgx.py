"""Record tests/golden/ppgx_seed0.npz from the LIVE reference PPG extractor (TEST INFRASTRUCTURE).

Run in the build container only (needs the reference tree):

    CUDA_VISIBLE_DEVICES="" python oracle/make_golden_ppgx.py

The unmodified ``models.ppg_extractor.build_model`` runs on the CPU through ``ppgx_harness`` with the stand-in configs of
``ref_init`` (the released extractor's yaml is not in the reference tree), seeded like ``torch.manual_seed(seed);
build_model(args)``, eval.  The conv-module BatchNorm statistics are replaced by ``ref_init``'s seeded draws (identity in a
fresh module); the other weights are not stored: tests rebuild them with ``ref_init.ppg_extractor_state_dict``, which
tests/test_ppgx_cpu.py proves bit-identical to this constructor.  melmat is the current librosa meaning of ``norm=1``
(per-filter L1), routed by the harness.

Cases (wavs from ``synthetic_wav``: tones + noise with a run of exact zeros):
  a      PPGX_CONFIG, 3 s: the output, and the embed / block 0 / block 7 / last block taps
  b      PPGX_CONFIG, 1.37 s: the output (a second length for the batch tests)
  v_*    PPGX_CONFIG_SMALL and each variant of ref_init.PPGX_SMALL_VARIANTS on one ~1 s wav `v_wav` (STFT frames a
         multiple of 4, which the reference's subsampling masks need); `fe_defaults` leaves the STFT keys out of
         frontend_conf, so DefaultFrontend's defaults (n_fft 1024, win_length 800, hop 160) apply
  long   PPGX_CONFIG_SMALL, 5010 * 160 samples (5011 frames > the 5000-row table: pe_len rebuilt), rows [0, 64) and
         [T - 64, T) of the output; then `short` (0.5 s) on the SAME module instance, whose table keeps 5011 rows
"""
from __future__ import annotations

import os
import sys
from pathlib import Path

os.environ.setdefault("CUDA_VISIBLE_DEVICES", "")
HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE))
sys.path.insert(0, str(HERE.parent))
sys.path.insert(0, str(HERE.parent / "synth_weights"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import ppgx_harness as ph  # noqa: E402
import ref_init as ri  # noqa: E402
from make_golden import GOLDEN, meta  # noqa: E402

TAPS_A = (0, 1, 8, 16)  # tap index: 0 = embed output, 1 + i = block i output


def synthetic_wav(n: int, seed: int) -> np.ndarray:
    """three tones, a chirp and white noise at 16 kHz, with exact zeros over [0.40 n, 0.45 n)"""
    g = np.random.RandomState(seed)
    t = np.arange(n) / 16000.0
    x = 0.3 * np.sin(2 * np.pi * 220 * t) + 0.2 * np.sin(2 * np.pi * 1250 * t + 0.3) + 0.1 * np.sin(2 * np.pi * 3100 * t)
    x += 0.1 * np.sin(2 * np.pi * (300 + 800 * t) * t) + 0.05 * g.randn(n)
    x[int(0.40 * n):int(0.45 * n)] = 0.0
    return x.astype(np.float32)


def build(cfg, seed=0):
    m = ph.build_ppg_extractor(cfg, seed)
    m.load_state_dict(ri.ppg_extractor_state_dict(cfg, seed, randomize_bn=True))
    return m.eval()


def run(m, wav, taps=False):
    got, hooks = [], []
    if taps:
        def keep(mod, inp, o):  # ((x, pos_emb) or x, mask)
            got.append((o[0][0] if isinstance(o[0], tuple) else o[0])[0].clone())

        hooks = [m.encoder.embed.register_forward_hook(keep)] + [b.register_forward_hook(keep) for b in m.encoder.encoders]
    with torch.no_grad():
        out = m(torch.from_numpy(wav)[None], torch.LongTensor([len(wav)]))[0]
    for h in hooks:
        h.remove()
    return out.numpy(), [t.numpy() for t in got]


def main():
    GOLDEN.mkdir(parents=True, exist_ok=True)
    torch.set_num_threads(len(os.sched_getaffinity(0)))
    z = {}
    m = build(ri.PPGX_CONFIG)
    for case, n, seed in (("a", 48000, 1), ("b", 21920, 2)):
        wav = synthetic_wav(n, seed)
        out, taps = run(m, wav, taps=case == "a")
        z[case + "_wav"], z[case + "_out"] = wav, out
        if case == "a":
            z["a_tap_index"] = np.array(TAPS_A)
            z["a_taps"] = np.stack([taps[i] for i in TAPS_A])
    variants = dict(small=ri.PPGX_CONFIG_SMALL, **ri.PPGX_SMALL_VARIANTS)
    z["v_wav"] = wav = synthetic_wav(15840 + 37, 3)  # one wav for every variant
    for name, cfg in variants.items():
        z[f"v_{name}_out"] = run(build(cfg), wav)[0]
    m = build(ri.PPGX_CONFIG_SMALL)
    wav = synthetic_wav(5010 * 160, 4)
    out = run(m, wav)[0]
    z["long_wav_seed"], z["long_n"] = np.array(4), np.array(5010 * 160)
    z["long_head"], z["long_tail"] = out[:64], out[-64:]
    z["long_pe_len"] = np.array(m.encoder.embed.out[1].pe.shape[1])
    wav = synthetic_wav(8000, 5)
    z["short_wav"], z["short_out"] = wav, run(m, wav)[0]
    z["short_pe_len"] = np.array(m.encoder.embed.out[1].pe.shape[1])
    taps = {k: z.pop(k) for k in ("a_tap_index", "a_taps")}
    np.savez_compressed(GOLDEN / "ppgx_seed0.1.npz", **taps)  # golden_io.load joins the parts
    path = GOLDEN / "ppgx_seed0.npz"
    np.savez_compressed(path, **z, meta=meta(weights_seed=0, config="ref_init.PPGX_CONFIG / PPGX_CONFIG_SMALL (+ variants), stand-ins",
                                             melmat="librosa.filters.mel(norm=1) as per-filter L1 (librosa >= 0.8 meaning)",
                                             bn="ref_init.ppg_extractor_state_dict(randomize_bn=True)",
                                             wavs="make_golden_ppgx.synthetic_wav(n, seed)"))
    print(path.name, path.stat().st_size, {k: v.shape for k, v in z.items()})


if __name__ == "__main__":
    main()
