"""Test hook: one launch of a 3-term-split tensor-core GEMM of the Tacotron / speaker-encoder family (mb_taco_tc_debug) on torch
CUDA tensors, prepared by the same absmax -> scale -> pack -> split functions the forward uses."""
from __future__ import annotations

import ctypes as C
from typing import Optional, Sequence

import torch

from .. import _lib

KINDS = {"plain": _lib.MB_TACO_TC_SKINNY_PLAIN, "lstm": _lib.MB_TACO_TC_SKINNY_LSTM, "gru": _lib.MB_TACO_TC_GRU,
         "lstm_seq": _lib.MB_TACO_TC_LSTM_SEQ, "big": _lib.MB_TACO_TC_BIG}


def _p(t: Optional[torch.Tensor]):
    if t is None:
        return None
    assert t.is_cuda, "device tensors expected"
    return t.data_ptr()


def tc_debug(kind: str, *, M: int, N: int = 0, H: int = 0, K0: int = 0, K1: int = 0,
             w: Sequence[Optional[torch.Tensor]] = (), b: Sequence[Optional[torch.Tensor]] = (), ldw: int = 0,
             x: Sequence[Optional[torch.Tensor]] = (), ldx: Sequence[int] = (), nseg: int = 1, T: int = 1,
             shift: Sequence[int] = (), w_off: Sequence[int] = (), w_stride: Sequence[int] = (), kb0: int = 0, kb_count: int = 0,
             pre: Optional[torch.Tensor] = None, ldpre: int = 0, step_ptr: Optional[torch.Tensor] = None, step_j: int = 0,
             y_step: int = 0, y: Optional[torch.Tensor] = None, ldy: int = 0, c=None, h=None, xres=None,
             gi: Sequence[Optional[torch.Tensor]] = (), ldgi: int = 0, hst: Sequence = (), out: Sequence = (), ldout: int = 0,
             ndir: int = 1, s_hi: Sequence = (), s_lo: Sequence = (), s_k0: Sequence[int] = (), nxt_hi: Sequence = (),
             nxt_lo: Sequence = (), act: int = 0, bn_scale=None, bn_shift=None, res=None, ldres: int = 0, compact: int = -1,
             cluster: int = 0, pdl: int = -1, a_tiles=None, w_tiles=None, len=None, t1: int = 0, row_start=None, ring: int = 0,
             stream=None) -> str:
    """Runs one launch (synchronising the stream) and returns the report line.  Pointers are taken as given: sub-views such as
    strided gi / out slices pass their base pointer with the row stride in ld*.  `len` (int32, device): valid length of each
    sequence (big) or row (gru, with `t1` the backward direction's time index) of a ragged batch."""
    s = _lib.TacoTcDebugSpec()
    s.kind = KINDS[kind]
    s.M, s.N, s.H, s.K0, s.K1 = M, N, H, K0, K1
    for i, t in enumerate(w):
        s.w[i] = _p(t)
    for i, t in enumerate(b):
        s.b[i] = _p(t)
    s.ldw, s.nseg, s.T = ldw, nseg, T
    for i, t in enumerate(x):
        s.x[i] = _p(t)
    for arr, vals in ((s.ldx, ldx), (s.shift, shift), (s.w_off, w_off), (s.w_stride, w_stride), (s.s_k0, s_k0)):
        for i, v in enumerate(vals):
            arr[i] = int(v)
    s.kb0, s.kb_count, s.pre, s.ldpre = kb0, kb_count, _p(pre), ldpre
    s.step_ptr, s.step_j, s.y_step = _p(step_ptr), step_j, y_step
    s.y, s.ldy, s.c, s.h, s.xres = _p(y), ldy, _p(c), _p(h), _p(xres)
    for arr, vals in ((s.gi, gi), (s.hst, hst), (s.out, out), (s.s_hi, s_hi), (s.s_lo, s_lo), (s.nxt_hi, nxt_hi),
                      (s.nxt_lo, nxt_lo)):
        for i, t in enumerate(vals):
            arr[i] = _p(t)
    s.ldgi, s.ldout, s.ndir = ldgi, ldout, ndir
    s.act, s.bn_scale, s.bn_shift, s.res, s.ldres = act, _p(bn_scale), _p(bn_shift), _p(res), ldres
    s.compact, s.cluster, s.pdl = compact, cluster, pdl
    s.a_tiles, s.w_tiles = _p(a_tiles), _p(w_tiles)
    s.len, s.t1 = _p(len), t1
    s.row_start, s.ring = _p(row_start), ring  # PLAIN: per-row step origin (int32 device [M])
    lib = _lib.lib()
    need = lib.mb_taco_tc_debug_workspace_bytes(C.byref(s))
    if need == 0:
        _lib.check(lib.mb_taco_tc_debug(C.byref(s), None, 0, None, None, 0))
    ws = torch.empty(need, dtype=torch.uint8, device="cuda")
    rep = C.create_string_buffer(512)
    st = stream if stream is not None else torch.cuda.current_stream().cuda_stream
    _lib.check(lib.mb_taco_tc_debug(C.byref(s), C.c_void_p(ws.data_ptr()), need, C.c_void_p(st), rep, 512))
    torch.cuda.synchronize()
    return rep.value.decode()


def parse_report(line: str) -> dict:
    out = {}
    for kv in line.split():
        k, v = kv.split("=", 1)
        out[k] = v
    return out
