"""ppg2mel golden vectors from the LIVE reference: ``python oracle/make_golden_ppg2mel.py`` writes
tests/golden/ppg2mel_seed0.npz (split into parts by size, see golden_io.py).

The reference model is ``MelDecoderMOLv2(**ref_init.PPG2MEL_CONFIG)`` (unmodified, imported through ref_harness) with
the weights of ``ref_init.ppg2mel_state_dict(0, randomize_bn=True)``.  Its PreNet dropout is always on
(rnn_decoder_mol.py:20): the keep masks are captured by wrapping torch.nn.functional.dropout (only the training=True
calls: MOLAttention's and the Postnet's dropout are off in eval), and the per-step stop logits with a forward hook on
``decoder.stop_layer``.  Reference files are untouched.

The stop layer of the seeded weights gives logits within ~0.1 of zero, so each case sets the stop layer (weight
scale s, bias b, stored in the fixture) to reach one termination path with |logit| >= 0.05 at every decisive step
(n >= min_decoder_step), so that the step count can be required exactly:
  a  T = 103 (T % 4 = 3): runs to max_decoder_step
  b  T = 400: stops at exactly min_decoder_step
  c  T = 262 (T % 4 = 2): stops by the sigmoid rule after min_decoder_step
"""
from __future__ import annotations

import sys
from pathlib import Path

import numpy as np
import torch
import torch.nn.functional as F

HERE = Path(__file__).resolve().parent
sys.path[:0] = [str(HERE), str(HERE.parent / "synth_weights")]

import ref_harness as rh  # noqa: E402
import ref_init as ri  # noqa: E402

MARGIN = 0.05
MASK_SEED = 77


def make_inputs(T: int, seed: int):
    g = torch.Generator().manual_seed(seed)
    ppg = torch.randn(T, 144, generator=g)
    lf0_uv = torch.stack([torch.randn(T, generator=g), (torch.rand(T, generator=g) < 0.7).float()], 1)
    spk = torch.randn(256, generator=g)
    return ppg, lf0_uv, spk


def run_reference(model, ppg, lf0_uv, spk):
    masks, stops = [], []
    orig = F.dropout

    def wrapped(x, p=0.5, training=True, inplace=False):
        out = orig(x, p, training, inplace)
        if training:
            masks.append(((out != 0) | (x == 0)).reshape(-1))  # where x == 0 the mask is irrelevant; record "keep"
        return out

    hook = model.decoder.stop_layer.register_forward_hook(lambda m, i, o: stops.append(float(o.reshape(()))))
    F.dropout = wrapped
    try:
        torch.manual_seed(MASK_SEED)
        with torch.no_grad():
            mel, post, align = model.inference(ppg[None], lf0_uv[None], spk[None])
    finally:
        F.dropout = orig
        hook.remove()
    return mel, post, align, masks, np.array(stops, np.float32)


def pick_stop_layer(z: np.ndarray, T_enc: int, kind: str):
    """(scale, center) such that s * (z - center) meets the case's termination with the margin; z are the raw
    logits of the steps a run to max_decoder_step produces"""
    mx = 2 * T_enc
    mn = mx - 5
    if kind == "max":
        return 1.0, float(z[mn - 1:mx].max()) + 0.2
    if kind == "min":
        return 1.0, float(z[mn - 1]) - 0.2
    # sigmoid rule at the first step k > min_step where z rises past a level between z[k-1] and z[k]
    for k in range(mn, mx - 1):
        lo, hi = float(z[mn - 1:k].max()), float(z[k])
        if hi > lo:
            c = 0.5 * (lo + hi)
            return MARGIN * 2.4 / (hi - lo), c
    raise RuntimeError("no rising stop logit after min_decoder_step")


def main():
    rh.install()
    from models.ppg2mel import MelDecoderMOLv2

    torch.manual_seed(0)
    model = MelDecoderMOLv2(**ri.PPG2MEL_CONFIG)
    base = ri.ppg2mel_state_dict(0, randomize_bn=True)
    model.load_state_dict(base, strict=True)
    model.eval()
    w0 = base["decoder.stop_layer.linear_layer.weight"].clone()
    b0 = base["decoder.stop_layer.linear_layer.bias"].clone()
    out, meta = {}, []
    for name, T, kind in (("a", 103, "max"), ("b", 400, "min"), ("c", 262, "sigmoid")):
        ppg, lf0_uv, spk = make_inputs(T, seed=500 + T)
        T_enc = (T // 2) // 2
        # the raw logit trajectory to max_decoder_step (stop layer pushed far negative; the mel path does not read it)
        model.decoder.stop_layer.linear_layer.bias.data = b0 - 1e3
        *_, z = run_reference(model, ppg, lf0_uv, spk)
        z = z + 1e3
        s, c = pick_stop_layer(z, T_enc, kind)
        w, b = w0 * s, (b0 - c) * s
        model.decoder.stop_layer.linear_layer.weight.data = w
        model.decoder.stop_layer.linear_layer.bias.data = b
        mel, post, align, masks, stops = run_reference(model, ppg, lf0_uv, spk)
        n = align.shape[0]
        mx, mn = 2 * T_enc, 2 * T_enc - 5
        assert len(stops) == n and len(masks) == 2 * n, (len(stops), len(masks), n)
        want = {"max": mx, "min": mn}.get(kind)
        assert (want is None and mn < n < mx) or n == want, (name, kind, n, mn, mx)
        dec = stops[max(mn, 1) - 1:n]
        assert (np.abs(dec) >= MARGIN).all(), (name, dec)
        m1 = np.packbits(torch.stack(masks[0::2]).numpy().astype(np.uint8), axis=-1)
        m2 = np.packbits(torch.stack(masks[1::2]).numpy().astype(np.uint8), axis=-1)
        out.update({f"{name}_ppg": ppg.numpy(), f"{name}_lf0_uv": lf0_uv.numpy(), f"{name}_spk": spk.numpy(),
                    f"{name}_stop_w": w.numpy(), f"{name}_stop_b": b.numpy(), f"{name}_mask1": m1, f"{name}_mask2": m2,
                    f"{name}_mel": mel.numpy(), f"{name}_mel_postnet": post.numpy(), f"{name}_alignments": align.numpy(),
                    f"{name}_stop": stops})
        meta.append(f"{name}: T={T} T_enc={T_enc} steps={n} ({kind}) min={mn} max={mx} stop scale={s:.4g}")
        print(meta[-1], "decisive |logit| min", float(np.abs(dec).min()))
    out["meta"] = np.array("weights ref_init.ppg2mel_state_dict(0, randomize_bn=True) with a per-case stop layer; "
                           f"masks torch.manual_seed({MASK_SEED}); " + "; ".join(meta))
    dst = HERE.parent / "tests" / "golden"
    part1 = {k: v for k, v in out.items() if not k.startswith("b_")}
    part2 = {k: v for k, v in out.items() if k.startswith("b_")}
    np.savez_compressed(dst / "ppg2mel_seed0.npz", **part1)
    np.savez_compressed(dst / "ppg2mel_seed0.1.npz", **part2)
    for p in sorted(dst.glob("ppg2mel_seed0*.npz")):
        print(p.name, p.stat().st_size)


if __name__ == "__main__":
    main()
