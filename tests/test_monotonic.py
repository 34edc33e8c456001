"""monotonic_align.maximum_path (SURVEY.md 8f row N4): numpy restatement == the reference's own compiled core.pyx == the CUDA
wavefront DP.  The reference's paths are stored in tests/golden/monotonic_ref.npz (oracle/make_golden_monotonic.py); where the
compiled reference exists (oracle/_ref, oracle/build_oracle.build_ref()) the stored paths are checked against it as well."""
import numpy as np
import pytest
import torch

import make_golden_monotonic as mgm
import monotonic_oracle as mo

_case = mgm.case


def _reference(golden_dir, seed, shape, v, t_ys, t_xs):
    """the compiled reference's (path, value) for one case: from the golden file, cross-checked against the live module if built"""
    z = np.load(golden_dir / "monotonic_ref.npz")
    k = mgm.key(seed, shape)
    p_ref = np.unpackbits(z[k + "_path"], axis=-1, count=shape[-1]).astype(np.int32)
    v_ref = z[k + "_value"] if k + "_value" in z.files else None
    core = mo.reference_core()
    if core is not None:
        p_live, v_live = np.zeros(v.shape, np.int32), v.copy()
        core.maximum_path_c(p_live, v_live, t_ys, t_xs)
        assert np.array_equal(p_live, p_ref) and (v_ref is None or np.array_equal(v_live, v_ref))
    return p_ref, v_ref


@pytest.mark.parametrize("shape", mgm.RESTATEMENT_SHAPES)
def test_restatement_equals_compiled_reference(shape, golden_dir):
    v, t_ys, t_xs = _case(1, *shape)
    p_ref, v_ref = _reference(golden_dir, 1, shape, v, t_ys, t_xs)
    p, vv = mo.maximum_path_numpy(v, t_ys, t_xs)
    assert np.array_equal(p, p_ref) and np.array_equal(vv, v_ref)
    assert np.array_equal(p.sum(axis=(1, 2)), t_ys)  # one cell per frame


@pytest.mark.gpu
@pytest.mark.parametrize("shape", mgm.CUDA_SHAPES)
def test_cuda_equals_reference(shape, golden_dir):
    from mockingbird_b200.monotonic_align import maximum_path

    v, t_ys, t_xs = _case(2, *shape)
    b, ty, tx = shape
    mask = np.zeros((b, ty, tx), np.float32)
    for i in range(b):
        mask[i, : t_ys[i], : t_xs[i]] = 1
    got = maximum_path(torch.from_numpy(v).cuda(), torch.from_numpy(mask).cuda())
    assert got.dtype == torch.float32 and got.shape == (b, ty, tx)
    p_ref, _ = _reference(golden_dir, 2, shape, v, t_ys, t_xs)
    assert np.array_equal(got.cpu().numpy().astype(np.int32), p_ref)
    # size-independent properties: exactly one cell per valid frame, monotone non-decreasing column, ends at the corners
    g = got.cpu().numpy()
    for i in range(b):
        cols = g[i, : t_ys[i]].argmax(axis=1)
        assert g[i].sum() == t_ys[i] and cols[0] == 0 and cols[-1] == t_xs[i] - 1
        assert np.all(np.diff(cols) >= 0) and np.all(np.diff(cols) <= 1)
