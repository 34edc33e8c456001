"""Log-MMSE golden vectors from the LIVE reference (TEST INFRASTRUCTURE; needs the reference tree):

    python oracle/make_golden_logmmse.py

writes tests/golden/logmmse_seed0.npz.  Six seeded speech-like fp32 clips (logmmse_oracle.speechlike) of lengths
320 (the shortest the reference accepts; no frame), 479 and 480 (no frame / one frame), 6401 (just over the 0.4 s at
which load_preprocess_wav starts denoising), 9600 and 28000 samples: 2.8 s in all at 16 kHz, which keeps the file under
700 KB.  The GPU tests add a seeded 10 s clip against logmmse_oracle.  For each clip i:
  clip_i          the input
  mu2_i           utils/logmmse.profile_noise(first and last 0.15 s of the clip).noise_mu2 (float64 [640])
  out015_i        utils/logmmse.denoise(clip, profile, eta=0.15)
  out0_i          the same with eta = 0
  pre_i           models/synthesizer/inference.py Synthesizer.load_preprocess_wav on the clip: the reference function
                  itself, with its librosa.load returning the clip (rescale, edge profile, denoise over 0.4 s)
"""
from __future__ import annotations

import sys
from pathlib import Path

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE))

import numpy as np  # noqa: E402

import logmmse_oracle as lo  # noqa: E402
import ref_harness as rh  # noqa: E402

SEED = 0
SR = 16000
LENGTHS = [320, 479, 480, 6401, 9600, 28000]
OUT = HERE.parent / "tests" / "golden" / "logmmse_seed0.npz"


def clips():
    return [lo.speechlike(SEED * 100 + i, n, SR) for i, n in enumerate(LENGTHS)]


def edges(wav):
    e = int(SR * 0.15)
    return np.concatenate([wav[:e], wav[-e:]])


def main():
    rh.install()
    import scipy

    from utils import logmmse as ref
    import models.synthesizer.inference as si

    z = {}
    for i, x in enumerate(clips()):
        p = ref.profile_noise(edges(x).copy(), SR)
        z[f"clip_{i}"] = x
        z[f"mu2_{i}"] = p.noise_mu2
        z[f"out015_{i}"] = ref.denoise(x, p, eta=0.15)
        z[f"out0_{i}"] = ref.denoise(x, p, eta=0.0)
        si.librosa.load = lambda path, sr, _x=x: (_x.copy(), sr)
        z[f"pre_{i}"] = si.Synthesizer.load_preprocess_wav("clip.wav")
        assert z[f"pre_{i}"].dtype == np.float32
    z["meta"] = np.array([f"numpy {np.__version__}", f"scipy {scipy.__version__}", f"seed {SEED}", f"sr {SR}",
                          "lengths " + " ".join(map(str, LENGTHS))])
    np.savez_compressed(OUT, **z)
    print(f"wrote {OUT} ({OUT.stat().st_size} bytes)")


if __name__ == "__main__":
    main()
