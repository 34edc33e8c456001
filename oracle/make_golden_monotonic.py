"""Golden paths of the reference's own compiled monotonic_align core (oracle/_ref, built by build_oracle.build_ref() where the
reference tree exists) for the cases of tests/test_monotonic.py -> tests/golden/monotonic_ref.npz, so that the tests compare
against the reference without it."""
import sys
from pathlib import Path

import numpy as np

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE))
import monotonic_oracle as mo  # noqa: E402

RESTATEMENT_SHAPES = [(3, 37, 11), (2, 1, 1), (4, 64, 64), (2, 300, 75)]
CUDA_SHAPES = [(3, 37, 11), (2, 1, 1), (4, 64, 64), (16, 1000, 200), (2, 300, 75)]


def case(seed, b, ty, tx):
    rng = np.random.RandomState(seed)
    v = (rng.randn(b, ty, tx) * 3).astype(np.float32)
    t_ys = rng.randint(max(1, ty // 2), ty + 1, size=b).astype(np.int32)
    t_xs = np.minimum(rng.randint(1, tx + 1, size=b), t_ys).astype(np.int32)  # a monotonic path needs t_x <= t_y
    t_ys[0], t_xs[0] = ty, min(tx, ty)
    return v, t_ys, t_xs


def key(seed, shape):
    return f"s{seed}_" + "x".join(map(str, shape))


def main():
    core = mo.reference_core()
    assert core is not None, "oracle/_ref not built"
    out = {}
    for seed, shapes in ((1, RESTATEMENT_SHAPES), (2, CUDA_SHAPES)):
        for shape in shapes:
            v, t_ys, t_xs = case(seed, *shape)
            p, vv = np.zeros(v.shape, np.int32), v.copy()
            core.maximum_path_c(p, vv, t_ys, t_xs)
            out[key(seed, shape) + "_path"] = np.packbits(p.astype(np.uint8), axis=-1)
            if seed == 1:
                out[key(seed, shape) + "_value"] = vv
    np.savez_compressed(HERE.parent / "tests" / "golden" / "monotonic_ref.npz", **out)


if __name__ == "__main__":
    main()
