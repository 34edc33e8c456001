"""The workspace contract of the handle-free compute calls (include/mockingbird_b200.h, Conventions): a NULL workspace is
MB_ERR_INVALID, one byte short of *_workspace_bytes is MB_ERR_WORKSPACE, and neither queues anything.  Every pointer
but the workspace is a placeholder: the calls must refuse before they touch the device."""
import ctypes as C

import pytest

from mockingbird_b200 import _lib

MB_ERR_INVALID, MB_ERR_WORKSPACE = 1, 4  # include/mockingbird_b200.h
DEV = C.c_void_p(0x10000)  # never dereferenced


def _refusals(call, need):
    """call(workspace, bytes) -> status, for NULL and for need - 1 bytes; the launch counter must not move"""
    lib = _lib.lib()
    assert need > 0
    n0 = lib.mb_launch_count()
    assert call(None, need) == MB_ERR_INVALID
    assert call(DEV, need - 1) == MB_ERR_WORKSPACE
    assert lib.mb_launch_count() == n0


@pytest.mark.parametrize("name", ["mb_resample_sumsq", "mb_resample_scale", "mb_resample_rescale"])
def test_resample_levelling(name):
    lib = _lib.lib()
    lengths = (C.c_int32 * 3)(100, 7, 4000)
    need = lib.mb_resample_level_workspace_bytes(3)
    if name == "mb_resample_sumsq":
        _refusals(lambda ws, n: lib.mb_resample_sumsq(DEV, lengths, 3, DEV, ws, n, None), need)
    elif name == "mb_resample_scale":
        _refusals(lambda ws, n: lib.mb_resample_scale(DEV, lengths, 3, DEV, DEV, ws, n, None), need)
    else:
        _refusals(lambda ws, n: lib.mb_resample_rescale(DEV, lengths, 3, C.c_float(0.9), DEV, ws, n, None), need)


@pytest.mark.parametrize("batched", [0, 1])
def test_wavernn_postprocess(batched):
    lib = _lib.lib()
    folds, target, overlap = (3, 100, 20) if batched else (1, 0, 0)
    steps = target + 2 * overlap if batched else 500
    need = lib.mb_wavernn_postprocess_workspace_bytes(folds, steps, batched, target, overlap)
    n_out = C.c_int64(0)
    _refusals(lambda ws, n: lib.mb_wavernn_postprocess(DEV, folds, steps, batched, target, overlap, 512, 1, C.c_double(0.97),
                                                       300, 0, DEV, C.byref(n_out), ws, n, None), need)
    _refusals(lambda ws, n: lib.mb_wavernn_postprocess_f32(DEV, folds, steps, batched, target, overlap, C.c_double(0.97), 300,
                                                           0, DEV, C.byref(n_out), ws, n, None), need)


def test_taco_debug():
    lib = _lib.lib()
    s = _lib.TacoDebugSpec()
    s.kind, s.nseg, s.M, s.N, s.W, s.y = 0, 1, 4, 8, DEV.value, DEV.value  # kind 0: MB_TACO_DBG_GEMM
    s.x[0], s.K[0] = DEV.value, 16
    need = lib.mb_taco_debug_workspace_bytes(C.byref(s))
    _refusals(lambda ws, n: lib.mb_taco_debug(C.byref(s), ws, n, None, None, 0), need)


def test_taco_tc_debug():
    lib = _lib.lib()
    s = _lib.TacoTcDebugSpec()
    s.kind, s.M, s.N, s.K0 = _lib.MB_TACO_TC_SKINNY_PLAIN, 4, 64, 128
    s.w[0], s.x[0] = DEV.value, DEV.value
    need = lib.mb_taco_tc_debug_workspace_bytes(C.byref(s))
    _refusals(lambda ws, n: lib.mb_taco_tc_debug(C.byref(s), ws, n, None, None, 0), need)


@pytest.mark.parametrize("kind", [_lib.MB_PPGX_DBG_MVN, _lib.MB_PPGX_DBG_CONV2D_TC])
def test_ppgx_debug(kind):
    lib = _lib.lib()
    s = _lib.PpgxDebugSpec()
    s.kind, s.B, s.T, s.F, s.C, s.N, s.k, s.stride, s.pad, s.rows_total = kind, 2, 16, 20, 32, 64, 3, 2, 1, 128
    s.len, s.x_hi, s.x_lo, s.w, s.y_hi, s.y_lo = (DEV.value,) * 6
    need = lib.mb_ppgx_debug_workspace_bytes(C.byref(s))
    _refusals(lambda ws, n: lib.mb_ppgx_debug(C.byref(s), ws, n, None, None, 0), need)
