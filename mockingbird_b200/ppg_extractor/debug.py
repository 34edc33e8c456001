"""Test hook: one launch of a PPG-extractor kernel (mb_ppgx_debug) on torch CUDA tensors, through the launch helpers the
forward uses (conv2d_tc also packs its weight as finalize does)."""
from __future__ import annotations

import ctypes as C
from typing import Optional, Sequence

import torch

from .. import _lib

KINDS = {"frontend": _lib.MB_PPGX_DBG_FRONTEND, "mvn": _lib.MB_PPGX_DBG_MVN, "conv0": _lib.MB_PPGX_DBG_CONV0,
         "conv2d_tc": _lib.MB_PPGX_DBG_CONV2D_TC, "ln_tiles": _lib.MB_PPGX_DBG_LN_TILES,
         "act_tiles": _lib.MB_PPGX_DBG_ACT_TILES, "ln_rows": _lib.MB_PPGX_DBG_LN_ROWS, "dw": _lib.MB_PPGX_DBG_DW,
         "attn": _lib.MB_PPGX_DBG_ATTN}
_INTS = ("B", "T", "n_max", "n_fft", "win_length", "hop_length", "F", "C", "N", "k", "stride", "pad", "M", "D", "ld",
         "rows_total", "act", "flags", "H", "dk", "ldp", "rel")
_PTRS = ("len", "len2", "x", "x_hi", "x_lo", "w", "bias", "P", "pu", "pv", "y", "y_hi", "y_lo")


def _p(t: Optional[torch.Tensor]):
    if t is None:
        return None
    assert t.is_cuda, "device tensors expected"
    return t.data_ptr()


def ppgx_debug(kind: str, *, bn: Sequence[Optional[torch.Tensor]] = (), stream=None, **kw) -> str:
    """Runs one launch (synchronising the stream) and returns the report line.  Keyword arguments are the fields of
    mb_ppgx_debug_spec: integers by value, tensors (or None) for the pointers."""
    s = _lib.PpgxDebugSpec()
    s.kind = KINDS[kind]
    for k, v in kw.items():
        if k in _INTS:
            setattr(s, k, int(v))
        elif k in _PTRS:
            setattr(s, k, _p(v))
        else:
            raise TypeError(f"ppgx_debug: unknown field {k}")
    for i, t in enumerate(bn):
        s.bn[i] = _p(t)
    lib = _lib.lib()
    need = lib.mb_ppgx_debug_workspace_bytes(C.byref(s))
    ws = torch.empty(max(need, 1), dtype=torch.uint8, device="cuda")
    rep = C.create_string_buffer(256)
    st = stream if stream is not None else torch.cuda.current_stream().cuda_stream
    _lib.check(lib.mb_ppgx_debug(C.byref(s), C.c_void_p(ws.data_ptr()), need, C.c_void_p(st), rep, 256))
    torch.cuda.synchronize()
    return rep.value.decode()


def parse_report(line: str) -> dict:
    return dict(kv.split("=", 1) for kv in line.split())
