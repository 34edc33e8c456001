"""F0 post-processing golden vectors from the LIVE reference (TEST INFRASTRUCTURE; needs the reference tree):

    python oracle/make_golden_f0.py

writes tests/golden/f0_seed0.npz.  The unmodified utils/f0_utils.py is imported through ref_harness with a `pyworld` stub
whose `harvest` is oracle/harvest_oracle.py (pyworld itself cannot be installed here), so the file pins every line of the
reference's own post-processing on the restatement's F0.  Four seeded speech-like clips of 1, 1.5, 2.2 and 3 s:
  clip_i                 the input (float32)
  f0_i                   utils/f0_utils.compute_f0(clip)
  mean_i, std_i          compute_mean_std(f02lf0(f0_i))
  conv_i, raw_i          get_converted_lf0uv(clip, mean_0, std_0, convert=True / False)
and hand-made contours for the branches the clips may not reach, each with get_cont_lf0's (uv, cont_lf0) and the argument
after the call (convert_continuos_f0 edits it in place):
  zero      all unvoiced (float32)
  edges     voiced at the first and the last frame, gaps between (float32)
  two       voiced on exactly two frames (float64)
"""
from __future__ import annotations

import sys
import types
from pathlib import Path

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE))

import numpy as np  # noqa: E402

import harvest_oracle as ho  # noqa: E402
import ref_harness as rh  # noqa: E402

SEED = 0
LENGTHS = [16000, 24000, 35200, 48000]
OUT = HERE.parent / "tests" / "golden" / "f0_seed0.npz"


def clips():
    return [ho.speechlike(SEED * 100 + i, n) for i, n in enumerate(LENGTHS)]


def contours():
    zero = np.zeros(40, dtype=np.float32)
    edges = np.zeros(40, dtype=np.float32)
    edges[[0, 1, 2, 10, 11, 25, 39]] = [120.0, 121.5, 123.0, 140.0, 141.0, 180.0, 95.0]
    two = np.zeros(30)
    two[[7, 19]] = [210.0, 190.0]
    return dict(zero=zero, edges=edges, two=two)


def main():
    rh.install()
    stub = types.ModuleType("pyworld")
    stub.harvest = ho.harvest
    sys.modules["pyworld"] = stub
    from utils import f0_utils as ref

    z = {}
    cs = clips()
    for i, x in enumerate(cs):
        f0 = ref.compute_f0(x)
        z[f"clip_{i}"] = x
        z[f"f0_{i}"] = f0
        z[f"mean_{i}"], z[f"std_{i}"] = ref.compute_mean_std(ref.f02lf0(f0))
    for i, x in enumerate(cs):
        z[f"conv_{i}"] = ref.get_converted_lf0uv(x, z["mean_0"], z["std_0"], convert=True)
        z[f"raw_{i}"] = ref.get_converted_lf0uv(x, z["mean_0"], z["std_0"], convert=False)
    for name, f0 in contours().items():
        arg = f0.copy()
        uv, cont = ref.get_cont_lf0(arg)
        z[f"{name}_f0"], z[f"{name}_uv"], z[f"{name}_cont"], z[f"{name}_after"] = f0, uv, cont, arg
    OUT.parent.mkdir(parents=True, exist_ok=True)
    np.savez_compressed(OUT, **z)
    print(f"wrote {OUT} ({OUT.stat().st_size} bytes)")


if __name__ == "__main__":
    main()
