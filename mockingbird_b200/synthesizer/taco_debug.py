"""Test hook: one launch of an FP32 kernel of the Tacotron path (mb_taco_debug) on torch CUDA tensors, through the launcher the
forward uses.  Argument meanings per kind are listed with MB_TACO_DBG_* in include/mockingbird_b200.h."""
from __future__ import annotations

import ctypes as C
from typing import Optional, Sequence

import torch

from .. import _lib


def _p(t: Optional[torch.Tensor]):
    if t is None:
        return None
    assert t.is_cuda, "device tensors expected"
    return t.data_ptr()


def taco_debug(kind: str, *, segs: Sequence[dict] = (), W=None, ldw: int = 0, bias=None, M: int = 0, N: int = 0, T: int = 1,
               act: int = 0, bn_scale=None, bn_shift=None, mask=None, res=None, ldres: int = 0, y=None, ldy: int = 0,
               step_mode: int = 0, step_ptr=None, step_j: int = 0, x_step: int = 0, x_first=None, mask_step: int = 0,
               ins: Sequence = (), outs: Sequence = (), n: Sequence[int] = (), fval: float = 0.0, seed: int = 0,
               row_len=None, row_done=None, row_caps=None, row_seeds=None, fma_chain: int = 0, row_start=None, ring: int = 0,
               stream=None) -> str:
    """Enqueues one launch, synchronises and returns the report line.  `segs`: GemmArgs segments as dicts with keys
    x, K, ld, shift, w_off, w_stride (x may be an int device address, e.g. a pointer offset by one float).  row_len,
    row_done, row_caps (int32) and row_seeds (int64 holding the uint64 seeds) are the per-row arrays of ragged batches;
    row_start (int32) and ring the per-row step origin of streamed decoding."""
    s = _lib.TacoDebugSpec()
    s.kind = _lib.MB_TACO_DBG[kind]
    s.nseg = len(segs)
    for j, g in enumerate(segs):
        s.x[j] = g["x"] if isinstance(g["x"], int) else _p(g["x"])
        s.K[j], s.ld[j] = g["K"], g["ld"]
        s.shift[j], s.w_off[j], s.w_stride[j] = g.get("shift", 0), g.get("w_off", 0), g.get("w_stride", 1)
    s.W, s.ldw, s.bias, s.M, s.N, s.T, s.act = _p(W), ldw, _p(bias), M, N, T, act
    s.bn_scale, s.bn_shift, s.mask, s.res, s.ldres = _p(bn_scale), _p(bn_shift), _p(mask), _p(res), ldres
    s.y, s.ldy = _p(y), ldy
    s.step_mode, s.step_ptr, s.step_j, s.x_step, s.x_first, s.mask_step = step_mode, _p(step_ptr), step_j, x_step, _p(x_first), mask_step
    for i, t in enumerate(ins):
        s.in_[i] = _p(t)
    for i, t in enumerate(outs):
        s.out[i] = _p(t)
    for i, v in enumerate(n):
        s.n[i] = int(v)
    s.fval, s.seed = fval, seed
    s.row_len, s.row_done, s.row_caps, s.row_seeds = _p(row_len), _p(row_done), _p(row_caps), _p(row_seeds)
    s.fma_chain = fma_chain
    s.row_start, s.ring = _p(row_start), ring
    lib = _lib.lib()
    need = lib.mb_taco_debug_workspace_bytes(C.byref(s))
    if need == 0:
        _lib.check(lib.mb_taco_debug(C.byref(s), None, 0, None, None, 0))
    ws = torch.empty(need, dtype=torch.uint8, device="cuda")
    rep = C.create_string_buffer(256)
    st = stream if stream is not None else torch.cuda.current_stream().cuda_stream
    _lib.check(lib.mb_taco_debug(C.byref(s), C.c_void_p(ws.data_ptr()), need, C.c_void_p(st), rep, 256))
    torch.cuda.synchronize()
    return rep.value.decode()


def parse_report(line: str) -> dict:
    return dict(kv.split("=", 1) for kv in line.split())
