"""How sensitive is the ppg2mel MoL attention to 1-ulp differences in sigmoid?  (DESIGN.md section 4g)

The discretised MoL weights alpha = phi[j+1] - phi[j] have a discontinuity (alpha == 0 -> 1e-5): at the edge of a
saturated region one ulp of sigmoid decides between alpha ~ 6e-8 and alpha = 1e-5.  This runs the torch-CPU oracle on
the golden cases with the keep masks the reference drew, once with torch.sigmoid and once each with its result moved by
+1 / -1 ulp (every element, in the MoL attention only), and reports the relative errors against the unperturbed run,
how many alignment entries flip across the eps rule, and whether the step count changes.

usage: python tools/ppg2mel_precision_study.py
"""
import sys
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path[:0] = [str(ROOT / "oracle"), str(ROOT / "synth_weights")]

import golden_io  # noqa: E402
import ppg2mel_oracle as po  # noqa: E402
import ref_init as ri  # noqa: E402


def main():
    z = golden_io.load(ROOT / "tests" / "golden" / "ppg2mel_seed0.npz")
    for c in "abc":
        sd = ri.ppg2mel_state_dict(0)
        sd["decoder.stop_layer.linear_layer.weight"] = torch.from_numpy(z[c + "_stop_w"])
        sd["decoder.stop_layer.linear_layer.bias"] = torch.from_numpy(z[c + "_stop_b"])
        m1 = torch.from_numpy(np.unpackbits(z[c + "_mask1"], axis=-1)).bool()
        m2 = torch.from_numpy(np.unpackbits(z[c + "_mask2"], axis=-1)).bool()
        args = (torch.from_numpy(z[c + "_ppg"]), torch.from_numpy(z[c + "_lf0_uv"]), torch.from_numpy(z[c + "_spk"]))
        base = po.inference(sd, *args, masks=list(zip(m1, m2)))
        eps_base = int((base["alignments"] == 1e-5).sum())
        print(f"case {c}: T={args[0].shape[0]} steps={base['steps']} alignment entries == 1e-5: {eps_base} of "
              f"{base['alignments'].numel()}")
        for d, name in ((float("inf"), "+1 ulp"), (float("-inf"), "-1 ulp")):
            sig = lambda x, d=d: torch.nextafter(torch.sigmoid(x), torch.full_like(x, d))  # noqa: E731
            r = po.inference(sd, *args, masks=list(zip(m1, m2)), sigmoid=sig)
            n = min(r["steps"], base["steps"])
            a, b = r["alignments"][:n], base["alignments"][:n]
            flips = int(((a == 1e-5) != (b == 1e-5)).sum())
            e = {k: po.rel_errors(r[k][:2 * n if k != "alignments" else n], base[k][:2 * n if k != "alignments" else n])
                 for k in ("mel", "mel_postnet", "alignments")}
            print(f"  sigmoid {name}: steps {r['steps']}, eps-rule flips {flips}, "
                  + ", ".join(f"{k} max_rel {v['max_rel']:.2e} rms_rel {v['rms_rel']:.2e}" for k, v in e.items()))


if __name__ == "__main__":
    main()
