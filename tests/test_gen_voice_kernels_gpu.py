"""The text-to-speech chain's kernels launch by launch against numpy, bitwise: the trailing-silence trim of Tacotron rows
(mb_tacotron_trim_frames), the break assembly (mb_tts_join) and the float64 levelling entries (mb_resample_*_f64), and the
float32 levelling entries' old bits next to them."""
import ctypes as C

import numpy as np
import pytest
import torch

from mockingbird_b200 import _lib
from mockingbird_b200 import resample as rs
from mockingbird_b200.synthesizer import audio_host

pytestmark = pytest.mark.gpu

THRESHOLD = -3.4


def _same(got, want, what):
    """same dtype and shape, NaN where numpy has NaN, every other element bit for bit"""
    got, want = np.asarray(got), np.asarray(want)
    assert got.dtype == want.dtype and got.shape == want.shape, (what, got.dtype, want.dtype, got.shape, want.shape)
    nan = np.isnan(want)
    assert np.array_equal(np.isnan(got), nan), what
    iv = np.int64 if got.dtype == np.float64 else np.int32
    assert np.array_equal(got[~nan].view(iv), want[~nan].view(iv)), what


def _trim(lin, row_frames):
    L = _lib.lib()
    B, n_mels, F = lin.shape
    d = torch.from_numpy(lin).cuda().contiguous()
    out = torch.full((B,), -7, dtype=torch.int32, device="cuda")
    ws = _lib.workspace(int(L.mb_tacotron_trim_workspace_bytes(B)), "cuda")
    n0 = L.mb_launch_count()
    _lib.check(L.mb_tacotron_trim_frames(C.c_void_p(d.data_ptr()), B, n_mels, F, (C.c_int32 * B)(*row_frames),
                                         C.c_float(THRESHOLD), C.c_void_p(out.data_ptr()), C.c_void_p(ws.data_ptr()),
                                         ws.numel(), C.c_void_p(torch.cuda.current_stream().cuda_stream)))
    assert L.mb_launch_count() == n0 + 1
    return out.cpu().tolist()


def _numpy_trim(m):
    """synthesizer/inference.py:135-138 on one row"""
    while m.shape[1] > 0 and np.max(m[:, -1]) < THRESHOLD:
        m = m[:, :-1]
    return m.shape[1]


@pytest.mark.parametrize("F", [1, 2, 37, 400, 1001])
def test_trim_frames_is_the_numpy_loop(F):
    rng = np.random.default_rng(F)
    B = 12
    lin = rng.uniform(-4.0, -3.5, (B, 80, F)).astype(np.float32)  # silent everywhere ...
    row_frames = [F, 0, 1, F, F, max(F - 1, 0), F // 2, F, F, F, F, F]
    for b in (0, 3, 5, 6, 7, 8, 9, 10):  # ... but a loud frame somewhere
        t = int(rng.integers(0, F))
        lin[b, int(rng.integers(0, 80)), t] = rng.uniform(-3.4, 2.0)
    lin[3, 5, F - 1] = np.float32(THRESHOLD)  # exactly at the threshold: not below it, not silent
    lin[7, 79, F // 3] = np.nan  # a NaN frame counts as not silent
    lin[8, :, :] = np.float32(THRESHOLD) - np.float32(1e-6)  # all-silent row, just below
    lin[9, :, F - 1] = np.nan
    lin[10, 0, 0] = 0.0  # only the first frame is loud
    lin[11, :, :] = 5.0  # nothing to trim
    got = _trim(lin, row_frames)
    want = [_numpy_trim(lin[b, :, :row_frames[b]]) for b in range(B)]
    assert got == want
    assert got[1] == 0 and got[8] == 0 and got[11] == row_frames[11]
    assert got[3] == row_frames[3] and got[9] == row_frames[9]


def test_trim_frames_per_row_alone():
    """a row's trim does not depend on the other rows of the launch"""
    rng = np.random.default_rng(5)
    lin = rng.uniform(-3.6, -3.3, (9, 80, 64)).astype(np.float32)
    rows = [64, 10, 0, 1, 64, 33, 2, 64, 50]
    full = _trim(lin, rows)
    for b in range(9):
        assert _trim(np.ascontiguousarray(lin[b:b + 1]), [rows[b]]) == [full[b]]


def _join(rows, frames, hop_size, zeros):
    """mb_tts_join over float32 device rows -> the float64 documents (host), one launch"""
    L = _lib.lib()
    dev = [torch.from_numpy(r).cuda() for r in rows]
    pieces = []
    for w, fr in zip(dev, frames):
        ends = np.cumsum(np.array(fr, np.int64) * hop_size)
        starts = np.concatenate(([0], ends[:-1]))
        for a, b in zip(starts.tolist(), ends.tolist()):
            pieces.append(_lib.TtsPiece(w.data_ptr() if w.numel() else None, w.numel(), a, b, zeros, 0))
    n = len(pieces)
    table = (_lib.TtsPiece * n)(*pieces)
    off = (C.c_int64 * (n + 1))()
    _lib.check(L.mb_tts_join_plan(table, n, off))
    out = torch.full((off[n],), 7.0, dtype=torch.float64, device="cuda")
    ws = _lib.workspace(int(L.mb_tts_join_workspace_bytes(n)), "cuda")
    n0 = L.mb_launch_count()
    _lib.check(L.mb_tts_join(table, n, C.c_void_p(out.data_ptr()), C.c_void_p(ws.data_ptr()), ws.numel(),
                             C.c_void_p(torch.cuda.current_stream().cuda_stream)))
    assert L.mb_launch_count() == n0 + (1 if off[n] else 0)
    flat = out.cpu().numpy()
    first = np.concatenate(([0], np.cumsum([len(f) for f in frames]))).tolist()
    return [flat[off[first[d]]:off[first[d + 1]]] for d in range(len(frames))]


def _numpy_breaks(generated_wav, breaks, hop_size, sample_rate):
    """gen_voice.py:30-34 verbatim"""
    b_ends = np.cumsum(np.array(breaks) * hop_size)
    b_starts = np.concatenate(([0], b_ends[:-1]))
    wavs = [generated_wav[start:end] for start, end, in zip(b_starts, b_ends)]
    breaks = [np.zeros(int(0.15 * sample_rate))] * len(breaks)
    return np.concatenate([i for w, b in zip(wavs, breaks) for i in (w, b)])


@pytest.mark.parametrize("voc_hop", [200, 256, 300])
def test_join_is_gen_voice_s_breaks(voc_hop):
    rng = np.random.default_rng(voc_hop)
    frames = [list(rng.integers(0, 60, int(rng.integers(1, 12)))) for _ in range(17)]
    frames.append([0, 0, 0])  # every sentence trimmed away
    frames.append([1])
    frames.append([700] * 4)
    rows = [rng.standard_normal(int(sum(f)) * voc_hop).astype(np.float32) for f in frames]
    rows[3][5] = np.nan
    got = _join(rows, frames, 256, int(0.15 * 16000))
    for d, (row, fr) in enumerate(zip(rows, frames)):
        _same(got[d], _numpy_breaks(row, fr, 256, 16000), f"document {d}")


def test_join_one_long_piece_and_odd_zeros():
    rng = np.random.default_rng(9)
    row = rng.standard_normal(1_000_003).astype(np.float32)
    got = _join([row], [[1_000_003]], 1, 3)
    _same(got[0], np.concatenate([row.astype(np.float64), np.zeros(3)]), "1e6 samples")


LENGTHS = [1, 2, 3, 4, 5, 6, 7, 8, 127, 128, 129, 1024, 2400, 16001, 1_000_003]


def _docs(dtype, seed=0):
    rng = np.random.default_rng(seed)
    out = []
    for k, n in enumerate(LENGTHS):
        x = rng.standard_normal(n) * 10.0 ** rng.uniform(-4, 0)
        if k % 3 == 0:
            x[:n // 2] = 0.0  # a leading silence as the breaks leave one
        out.append(x.astype(dtype))
    return out


def _clips(docs):
    return rs.DeviceClips(torch.from_numpy(np.concatenate(docs)).cuda(), [len(d) for d in docs], 16000)


def test_float64_levelling_is_numpy():
    docs = _docs(np.float64)
    docs.append(np.zeros(2400 * 3))  # an all-zero document: numpy's levelling gives all NaN
    nan_doc = _docs(np.float64, 1)[12].copy()
    nan_doc[100] = np.nan
    docs.append(nan_doc)
    dc = _clips(docs)
    ms = rs.mean_squares(dc)
    assert ms.dtype == np.float64
    for i, d in enumerate(docs):
        _same(np.float64(ms[i]), np.float64(np.mean(d ** 2)), f"mean square {i}")
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        for kw in ({"increase_only": True}, {}, {"decrease_only": True}):
            got = rs.normalize_volume_device(dc, -30, **kw).numpy()
            for i, d in enumerate(docs):
                _same(got[i], audio_host.normalize_volume(d, -30, **kw), f"normalize_volume {kw} document {i}")
        got = rs.rescale_device(dc, 0.97).numpy()
        for i, d in enumerate(docs):
            _same(got[i], d / np.abs(d).max() * 0.97, f"rescale document {i}")
        # the chain's order: levelling, then the peak normalisation
        lev = rs.rescale_device(rs.normalize_volume_device(dc, -30, increase_only=True), 0.97).numpy()
        for i, d in enumerate(docs):
            w = audio_host.normalize_volume(d, -30, increase_only=True)
            _same(lev[i], w / np.abs(w).max() * 0.97, f"levelled document {i}")
    assert np.isnan(lev[-2]).all() and np.isnan(lev[-1]).all()


def test_float32_levelling_keeps_its_bits():
    docs = _docs(np.float32, 2)
    docs.append(np.zeros(300, np.float32))
    dc = _clips(docs)
    ms = rs.mean_squares(dc)
    assert ms.dtype == np.float32
    for i, d in enumerate(docs):
        assert ms[i] == np.mean(d ** 2), i
    with np.errstate(divide="ignore", invalid="ignore"):
        for kw in ({"increase_only": True}, {}, {"decrease_only": True}):
            got = rs.normalize_volume_device(dc, -30, **kw).numpy()
            for i, d in enumerate(docs):
                _same(got[i], audio_host.normalize_volume(d, -30, **kw), f"float32 normalize_volume {kw} clip {i}")
        got = rs.rescale_device(dc, 0.9).numpy()
        for i, d in enumerate(docs):
            _same(got[i], d / np.abs(d).max() * 0.9, f"float32 rescale clip {i}")
