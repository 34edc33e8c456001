"""Record tests/golden/hifigan24k_seed0.npz from the LIVE reference (TEST INFRASTRUCTURE).

Run in the build container only (needs the reference tree):

    CUDA_VISIBLE_DEVICES="" python oracle/make_golden_hifigan24k.py

The unmodified reference ``Generator`` (models/vocoder/hifigan/models.py) is built at ``sampling_rate == 24000`` with the
stand-in config ``ref_init.HIFIGAN_CONFIG_24K`` (the released 24 kHz checkpoint's json is not in the reference tree), seeded
like hifigan/inference.py builds it, eval, weight norm removed.  Weights are not stored: tests rebuild them with
``ref_init.hifigan_state_dict``, which tests/test_hifigan24k_cpu.py proves bit-identical to this constructor.

Cases: a small batch (B = 2, T = 24) and rows 0 and 31 of the B = 32 x 256-frame batch (mel rand * 8 - 4, seed 2, as for
hifigan_seed0.npz), each row vocoded on its own.
"""
from __future__ import annotations

import os
import sys
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


def build_reference_24k(cfg: dict, seed: int = 0):
    """reference Generator for a 24 kHz config, eval, weight-norm folded (hifigan/inference.py:47-53)"""
    rh.install()
    from utils.util import AttrDict
    from models.vocoder.hifigan.models import Generator

    torch.manual_seed(seed)
    g = Generator(AttrDict(cfg))
    g.eval()
    g.remove_weight_norm()
    return g


def main():
    GOLDEN.mkdir(parents=True, exist_ok=True)
    torch.set_num_threads(len(os.sched_getaffinity(0)))
    g = build_reference_24k(ri.HIFIGAN_CONFIG_24K, seed=0)
    with torch.no_grad():
        mel_small = torch.rand(2, 80, 24, generator=torch.Generator().manual_seed(2)) * 8 - 4
        wav_small = g(mel_small)
        mel_full = torch.rand(32, 80, 256, generator=torch.Generator().manual_seed(2)) * 8 - 4
        pick = [0, 31]
        wav_full = torch.cat([g(mel_full[i:i + 1]) for i in pick])
    out = GOLDEN / "hifigan24k_seed0.npz"
    np.savez_compressed(out, mel_small=mel_small.numpy(), wav_small=wav_small.numpy(), full_pick=np.array(pick),
                        wav_full=wav_full.numpy(),
                        meta=meta(weights_seed=0, config="ref_init.HIFIGAN_CONFIG_24K (stand-in)",
                                  mel_small="rand(2,80,24;seed 2)*8-4", mel_full="rand(32,80,256;seed 2)*8-4 rows 0 and 31"))
    print(out.name, out.stat().st_size)


if __name__ == "__main__":
    main()
