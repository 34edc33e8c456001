"""Golden vectors of the VITS synthesizer from the live, unmodified reference (models/synthesizer/models/vits.py).

    python oracle/make_golden_vits.py      -> tests/golden/vits_{toy,full_sdp,full_dp}.npz

No VITS config or checkpoint ships with the reference, so two stand-in configs are used (synth_weights/ref_init.py): a
toy one and the usual VITS shape, the latter with and without the stochastic duration predictor.  Weights are
ref_init.vits_state_dict.  Each case is one padded batch run through ``Vits.infer`` under ``torch.manual_seed``, so the
noise tensors are the reference's own draws; they are stored with the inputs and every output the tests compare.
``ceil`` is discontinuous: the maker asserts every duration w lies at least MARGIN from an integer and records the
smallest distance, so that no tolerance can flip a frame.
"""
from __future__ import annotations

import sys
import types
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "oracle"))
sys.path.insert(0, str(ROOT / "synth_weights"))

import ref_harness  # noqa: E402
import ref_init as ri  # noqa: E402

MARGIN = 1e-3
TOY_CASE = dict(cfg="toy", seed=11, lengths=[9, 5, 3], sid=[2, 0, 1], noise_scale=0.667, noise_scale_w=0.8, length_scale=1.3,
                max_len=None)
FULL_CASE = dict(seed=12, lengths=[23, 14], sid=[3, 1], noise_scale=0.667, noise_scale_w=0.8, length_scale=1.0, max_len=None)
CASES = {
    "toy": dict(TOY_CASE, cfg=ri.VITS_TOY),
    "full_sdp": dict(FULL_CASE, cfg=ri.VITS_CONFIG),
    "full_dp": dict(FULL_CASE, cfg=dict(ri.VITS_CONFIG, use_sdp=False), seed=14, max_len=40),
    "toy_1spk": dict(TOY_CASE, cfg=ri.VITS_TOY_1SPK, seed=16, sid=None, max_len=11),
}


def build_vits(cfg: dict, sd: dict):
    """the reference's Vits(**cfg) in eval mode with `sd` loaded (weight norm removed first, so that `sd`'s folded
    "weight" tensors load as they are)"""
    ref_harness.install()
    if "monotonic_align" not in sys.modules:  # imported at vits.py's module scope, used by training only
        sys.modules["monotonic_align"] = types.ModuleType("monotonic_align")
    from models.synthesizer.models.vits import Vits

    torch.manual_seed(0)
    m = Vits(**cfg)
    for f in m.flow.flows[0::2]:
        f.enc.remove_weight_norm()
    m.dec.remove_weight_norm()
    missing, unexpected = m.load_state_dict(sd, strict=False)
    assert not unexpected, unexpected
    assert all(k.startswith("enc_q.") or k.startswith("dp.post_") for k in missing), [k for k in missing if not k.startswith("enc_q.")]
    return m.eval()


def make_case(name: str, c: dict) -> dict:
    cfg = c["cfg"]
    sd = ri.vits_state_dict(cfg, seed=c["seed"])
    model = build_vits(cfg, sd)
    g = torch.Generator().manual_seed(c["seed"] + 100)
    lens = c["lengths"]
    B, T = len(lens), max(lens)
    x = torch.randint(0, cfg["n_vocab"], (B, T), generator=g)
    for r, n in enumerate(lens):
        x[r, n:] = 0
    x_lengths = torch.tensor(lens, dtype=torch.long)
    emo = torch.randn(B, 1024, generator=g)
    sid = torch.tensor(c["sid"], dtype=torch.long) if c["sid"] is not None else None
    rec = {}
    # the durations before ceil, to check the margin: the same modules infer calls, same noise draw
    torch.manual_seed(c["seed"])
    with torch.no_grad():
        xe, m_p, logs_p, x_mask = model.enc_p(x, x_lengths, emo)
        gg = model.emb_g(sid).unsqueeze(-1) if sid is not None else None
        if cfg["use_sdp"]:
            noise_state = torch.get_rng_state()
            logw = model.dp(xe, x_mask, g=gg, reverse=True, noise_scale=c["noise_scale_w"])
            torch.set_rng_state(noise_state)
            sdp_noise = torch.randn(B, 2, T)
        else:
            logw = model.dp(xe, x_mask, g=gg)
            sdp_noise = torch.zeros(B, 2, T)
        w = (torch.exp(logw) * x_mask * c["length_scale"]).double()
    valid = x_mask.bool().expand_as(w)
    frac = (w - torch.round(w)).abs()[valid]
    margin = float(frac.min())
    assert c["max_len"] is None or c["max_len"] < int(y_max := torch.ceil(w).sum((1, 2)).max()), (name, "max_len must cut", y_max)
    assert margin >= MARGIN, f"{name}: a duration lies {margin:.2e} from an integer (< {MARGIN}); pick another seed"
    torch.manual_seed(c["seed"])
    with torch.no_grad():
        o, attn, y_mask, (z, z_p, m_p_y, logs_p_y) = model.infer(x, x_lengths, sid=sid, emo=emo, noise_scale=c["noise_scale"],
                                                                 length_scale=c["length_scale"], noise_scale_w=c["noise_scale_w"],
                                                                 max_len=c["max_len"])
    # the prior noise: the draw after the SDP's, same state
    torch.manual_seed(c["seed"])
    if cfg["use_sdp"]:
        torch.randn(B, 2, T)
    eps = torch.randn_like(m_p_y)
    w_ceil = torch.ceil(w).to(torch.int32)[:, 0]
    rec.update(x=x.numpy().astype(np.int32), x_lengths=np.array(lens, np.int32),
               sid=sid.numpy().astype(np.int32) if sid is not None else np.zeros(0, np.int32),
               emo=emo.numpy(), seed=np.int64(c["seed"]), sdp_noise=sdp_noise.numpy(), eps=eps.numpy(),
               noise_scale=np.float32(c["noise_scale"]), noise_scale_w=np.float32(c["noise_scale_w"]),
               length_scale=np.float32(c["length_scale"]), max_len=np.int32(c["max_len"] or 0), w_ceil=w_ceil.numpy(),
               y_lengths=y_mask.sum([1, 2]).numpy().astype(np.int32), attn=attn.numpy(), m_p=m_p.numpy(), logs_p=logs_p.numpy(),
               m_p_y=m_p_y.numpy(), logs_p_y=logs_p_y.numpy(), z_p=z_p.numpy(), z=z.numpy(), o=o.numpy(),
               duration_margin=np.float64(margin))
    return rec


def main() -> None:
    out = ROOT / "tests" / "golden"
    torch.set_num_threads(1)
    for name, c in CASES.items():
        rec = make_case(name, c)
        np.savez_compressed(out / f"vits_{name}.npz", **rec)
        print(name, {k: v.shape for k, v in rec.items() if hasattr(v, "shape") and v.ndim}, "margin", rec["duration_margin"])


if __name__ == "__main__":
    main()
