"""Full-size golden fixtures at the BASELINE.json configuration sizes, from the LIVE reference
(TEST INFRASTRUCTURE; build container only: needs /root/reference).

    CUDA_VISIBLE_DEVICES="" python oracle/make_golden_full.py [cfg1] [cfg3] [cfg4] [fregan]

  cfg1   WaveRNN.generate(mel rand(1,80,80;seed 1)*2-1, batched=False, 8000, 400, True), seed 1234
         (fatchord_version.py:153-257) -> 16 000 draws as int16 class ids + float64 waveform
  cfg3   WaveRNN.generate(mel rand(1,80,2400;seed 3)*2-1, batched=True, 8000, 400, True), seed 1234
         -> 58 folds x 8 800 draws as int16 [58,8800] (~1 MB) + a strided view of the float64 waveform
  cfg4   Tacotron.generate(chars [64,120] len in [20,120], embeds [64,256], steps=400, style_idx=-1,
         min_stop_token=10), r=2, dropout masks captured bit-packed (tacotron.py:199-298); stored:
         4 full rows of mel / postnet / attention + float64 row sums of every row
  fregan FreGAN.forward on the cfg-2 shape (mel rand(32,80,256;seed 2)*8-4), rows 0 and 31

SURVEY.md section 8(d) names these inputs.  Weights: synth_weights/ref_init.py seeded state dicts (pinned
bit-identical to the reference constructors by tests/test_oracle_pinned.py).
"""
from __future__ import annotations

import os
import sys
import time
from pathlib import Path

os.environ.setdefault("CUDA_VISIBLE_DEVICES", "")
HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE))
sys.path.insert(0, str(HERE.parent / "synth_weights"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import ref_harness as rh  # noqa: E402
import ref_init as ri  # noqa: E402
from make_golden import GOLDEN, meta  # noqa: E402

WAV_STRIDE = 16  # cfg3 waveform stored as wav[::16] + head + tail (the integers carry the parity)


def _wavernn_run(model, fv, mel, batched, target, overlap, seed):
    cap = {}
    orig_x = model.xfade_and_unfold
    orig_d = fv.decode_mu_law

    def wrap_x(y, t, o):
        cap["folds"] = np.array(y, copy=True)
        return orig_x(y, t, o)

    def wrap_d(y, mu, from_labels=True):
        cap["y"] = np.array(y, copy=True)
        return orig_d(y, mu, from_labels)

    model.xfade_and_unfold = wrap_x
    fv.decode_mu_law = wrap_d
    try:
        torch.manual_seed(seed)
        t0 = time.perf_counter()
        wav = model.generate(mel, batched, target, overlap, True, progress_callback=lambda *a: None)
        dt = time.perf_counter() - t0
    finally:
        fv.decode_mu_law = orig_d
        model.xfade_and_unfold = orig_x
    return wav, cap, dt


def _wavernn_model():
    import models.vocoder.wavernn.models.fatchord_version as fv

    model = rh.build_wavernn(seed=0)
    model.load_state_dict(ri.wavernn_state_dict(0, randomize_bn=True))
    return model, fv


def golden_cfg1():
    model, fv = _wavernn_model()
    mel = torch.rand(1, 80, 80, generator=torch.Generator().manual_seed(1)) * 2 - 1
    wav, cap, dt = _wavernn_run(model, fv, mel, False, 8000, 400, 1234)
    idx = np.rint((cap["y"] + 1) * 511 / 2).astype(np.int16)[None]
    assert idx.shape == (1, 16000), idx.shape
    np.savez_compressed(GOLDEN / "wavernn_cfg1.npz", idx=idx, wav=wav,
                        meta=meta(weights="ref_init.wavernn_state_dict(0, randomize_bn=True)", gen_seed=1234,
                                  mel="rand(1,80,80;seed 1)*2-1", call="generate(mel, False, 8000, 400, True)",
                                  reference_cpu_seconds=round(dt, 2)))
    print("cfg1", idx.shape, wav.shape, f"{dt:.1f}s")


def golden_cfg3():
    model, fv = _wavernn_model()
    mel = torch.rand(1, 80, 2400, generator=torch.Generator().manual_seed(3)) * 2 - 1
    wav, cap, dt = _wavernn_run(model, fv, mel, True, 8000, 400, 1234)
    idx = np.rint((cap["folds"] + 1) * 511 / 2).astype(np.int16)
    assert idx.shape == (58, 8800), idx.shape
    np.savez_compressed(GOLDEN / "wavernn_cfg3.idx.npz", idx=idx)  # split: no golden file above 1 MB (oracle/golden_io.py)
    np.savez_compressed(GOLDEN / "wavernn_cfg3.npz", wav_len=np.array(len(wav)),
                        wav_strided=wav[::WAV_STRIDE], wav_head=wav[:4096], wav_tail=wav[-8192:],
                        wav_sum=np.array([wav.sum(), np.abs(wav).sum()]),
                        meta=meta(weights="ref_init.wavernn_state_dict(0, randomize_bn=True)", gen_seed=1234,
                                  mel="rand(1,80,2400;seed 3)*2-1", call="generate(mel, True, 8000, 400, True)",
                                  wav_stride=WAV_STRIDE, reference_cpu_seconds=round(dt, 2)))
    print("cfg3", idx.shape, wav.shape, f"{dt:.1f}s")


def cfg4_inputs():
    """SURVEY.md 8(d) cfg 4: chars randint(2,75,(64,120);seed 4), per-row length randint(20,121), tail 0;
    embeds = L2-normalised rand(64,256;seed 5)"""
    g = torch.Generator().manual_seed(4)
    chars = torch.randint(2, 75, (64, 120), generator=g)
    lens = torch.randint(20, 121, (64,), generator=g)
    lens[0] = 120
    for b in range(64):
        chars[b, lens[b]:] = 0
    emb = torch.rand(64, 256, generator=torch.Generator().manual_seed(5))
    emb = emb / emb.norm(dim=1, keepdim=True)
    return chars, emb


CFG4_ROWS = [0, 21, 42, 63]


def golden_cfg4():
    import make_golden_tacotron as mgt

    model = rh.build_tacotron(seed=0)
    model.load_state_dict(ri.tacotron_state_dict(0, r=2, randomize_bn=True), strict=True)
    model.eval()
    chars, emb = cfg4_inputs()
    torch.manual_seed(77)
    t0 = time.perf_counter()
    mel, linear, attn, masks = mgt.capture_generate(model, chars, emb, 400, -1, 10)
    dt = time.perf_counter() - t0
    assert mel.shape == (64, 80, 400), mel.shape
    enc_m, dec_m = mgt.pack_masks(masks)
    rows = CFG4_ROWS
    # split: no golden file above 1 MB (oracle/golden_io.py)
    np.savez_compressed(GOLDEN / "tacotron_cfg4.enc_masks.npz", enc_masks=enc_m)
    np.savez_compressed(GOLDEN / "tacotron_cfg4.dec_masks.npz", dec_masks=dec_m)
    np.savez_compressed(GOLDEN / "tacotron_cfg4.outputs.npz", linear=linear[rows].numpy(), attn=attn[rows].numpy())
    np.savez_compressed(
        GOLDEN / "tacotron_cfg4.npz", chars=chars.numpy().astype(np.int16), emb=emb.numpy(),
        rows=np.array(rows), mel=mel[rows].numpy(),
        mel_rowsum=mel.double().sum(dim=(1, 2)).numpy(), mel_rowabs=mel.double().abs().sum(dim=(1, 2)).numpy(),
        linear_rowsum=linear.double().sum(dim=(1, 2)).numpy(), linear_rowabs=linear.double().abs().sum(dim=(1, 2)).numpy(),
        mel_absmax=np.array(float(mel.abs().max())), linear_absmax=np.array(float(linear.abs().max())),
        attn_argmax=attn.argmax(dim=2).numpy().astype(np.int16), cfg=np.array([400, -1, 10, 2]),
        meta=meta(weights="ref_init.tacotron_state_dict(0, r=2, randomize_bn=True)", gen_seed=77,
                  inputs="make_golden_full.cfg4_inputs()", reference_cpu_seconds=round(dt, 2)))
    print("cfg4", mel.shape, attn.shape, f"{dt:.1f}s")


def golden_fregan_cfg2():
    g = rh.build_fregan(seed=0)
    with torch.no_grad():
        mel = torch.rand(32, 80, 256, generator=torch.Generator().manual_seed(2)) * 8 - 4
        pick = [0, 31]
        wav = torch.cat([g(mel[i:i + 1]) for i in pick])
    np.savez_compressed(GOLDEN / "fregan_cfg2.npz", full_pick=np.array(pick), wav_full=wav.numpy(),
                        meta=meta(weights_seed=0, mel_full="rand(32,80,256;seed 2)*8-4 rows 0 and 31"))
    print("fregan", wav.shape)


def main():
    GOLDEN.mkdir(parents=True, exist_ok=True)
    rh.install()
    torch.set_num_threads(len(os.sched_getaffinity(0)))
    which = sys.argv[1:] or ["cfg1", "cfg3", "cfg4", "fregan"]
    jobs = {"cfg1": golden_cfg1, "cfg3": golden_cfg3, "cfg4": golden_cfg4, "fregan": golden_fregan_cfg2}
    for w in which:
        jobs[w]()
    for p in sorted(GOLDEN.glob("*.npz")):
        print(p.name, p.stat().st_size)


if __name__ == "__main__":
    main()
