"""CPU tests of the resampling and levelling contract (mockingbird_b200.resample, csrc/resample.cu; DESIGN.md section 4k).

The numpy restatements below follow the kernels' arithmetic step by step: the polyphase table [up][taps] visited in
descending tap index with one rounded float32 multiply and one rounded float32 add per tap, and the sum of squares split
into the kernel's subtrees of numpy's pairwise tree.  Each is held bitwise to scipy / numpy, which is what makes the device
results bitwise the host's.  The work-item table and the refusals need no device."""
import ctypes as C

import numpy as np
import pytest
from scipy.signal import resample_poly

from mockingbird_b200 import _lib
from mockingbird_b200 import resample as rs

# (source, target): the rates a user hands in, the reverse direction, the identity, and a ratio whose filter (2000 phases,
# 110 141 taps) is far larger than shared memory
RATIOS = [(44100, 16000), (48000, 16000), (22050, 16000), (24000, 16000), (11025, 16000), (8000, 16000), (16000, 24000),
          (16000, 16000), (44056, 16000)]


def polyphase_table(up, down):
    h = rs.design_filter(up, down)
    taps = -(-h.size // up)
    t = np.zeros((up, taps), np.float32)
    for p in range(up):
        col = h[p::up]
        t[p, :col.size] = col
    return t, 10 * max(up, down)


def resample_restated(x, source_sr, target_sr):
    """rs_resample_kernel in numpy: output j reads phase (j down + half_len) mod up of the table from q = qmax down to qmin"""
    up, down = rs.ratio(source_sr, target_sr)
    if up == down:
        return x.astype(np.float32)
    table, hl = polyphase_table(up, down)
    n = x.size
    j = np.arange(-(-n * up // down), dtype=np.int64)
    cj = j * down + hl
    phase, ntop = cj % up, cj // up
    qmax = np.minimum((2 * hl - phase) // up, ntop)
    qmin = np.maximum(0, ntop - (n - 1))
    acc = np.zeros(j.size, np.float32)
    for step in range(int((qmax - qmin).max()) + 1):
        q = qmax - step
        live = q >= qmin
        qc = np.where(live, q, 0)
        prod = table[phase, qc] * x[np.where(live, ntop - qc, 0)]
        acc = np.where(live, acc + prod, acc)
    return acc


def pairwise(a):
    """numpy's pairwise_sum of float32 (the leaf: 8 running lanes, combined ((0+1)+(2+3))+((4+5)+(6+7)), then the rest)"""
    n = a.size
    if n < 8:
        r = np.float32(-0.0)
        for v in a:
            r = np.float32(r + v)
        return r
    if n <= 128:
        r = a[:8].copy()
        m = n - n % 8
        for i in range(8, m, 8):
            r = r + a[i:i + 8]
        res = np.float32(np.float32(np.float32(r[0] + r[1]) + np.float32(r[2] + r[3]))
                         + np.float32(np.float32(r[4] + r[5]) + np.float32(r[6] + r[7])))
        for v in a[m:]:
            res = np.float32(res + v)
        return res
    n2 = n // 2
    n2 -= n2 % 8
    return np.float32(pairwise(a[:n2]) + pairwise(a[n2:]))


def split(n):
    n2 = n // 2
    return n2 - n2 % 8


def pairwise_depth(n):
    """the kernel's subtree depth: <= 8, every node above it internal (> 128 elements)"""
    sizes, d = {n}, 0
    while d < 8 and min(sizes) > 128:
        sizes = {c for s in sizes for c in (split(s), s - split(s))}
        d += 1
    return d


def sumsq_restated(x):
    """rs_sumsq_kernel in numpy: 2^depth subtrees (one per thread), then the levels above them bottom up"""
    sq = x * x
    d = pairwise_depth(sq.size)
    parts = []
    for t in range(1 << d):
        off, n = 0, sq.size
        for b in range(d - 1, -1, -1):
            n2 = split(n)
            if (t >> b) & 1:
                off, n = off + n2, n - n2
            else:
                n = n2
        parts.append(pairwise(sq[off:off + n]))
    while len(parts) > 1:
        parts = [np.float32(parts[i] + parts[i + 1]) for i in range(0, len(parts), 2)]
    return parts[0]


def _bits_equal(a, b):
    return a.dtype == b.dtype and a.shape == b.shape and np.array_equal(a.view(np.int32), b.view(np.int32))


@pytest.mark.parametrize("src,dst", RATIOS)
def test_restated_tap_order_is_resample_poly(src, dst):
    rng = np.random.default_rng(src + dst)
    up, down = rs.ratio(src, dst)
    per_phase = -(-(20 * max(up, down) + 1) // up)
    for n in (1, 2, 3, per_phase // 2, per_phase - 1, 5000):
        n = max(1, n)
        x = rng.uniform(-1, 1, n).astype(np.float32)
        assert _bits_equal(resample_restated(x, src, dst), resample_poly(x, up, down)), (src, dst, n)


@pytest.mark.parametrize("src", [44100, 48000, 44056])
def test_restated_tap_order_60_seconds(src):
    x = (np.random.default_rng(src).standard_normal(60 * src) * 0.1).astype(np.float32)
    up, down = rs.ratio(src, 16000)
    assert _bits_equal(resample_restated(x, src, 16000), resample_poly(x, up, down))


def test_ascending_tap_order_is_not_resample_poly():
    """the order is the contract: visiting the taps the other way round changes most samples"""
    x = np.random.default_rng(3).uniform(-1, 1, 4000).astype(np.float32)
    up, down = rs.ratio(44100, 16000)
    table, hl = polyphase_table(up, down)
    ref = resample_poly(x, up, down)
    out = np.empty_like(ref)
    for j in range(ref.size):
        cj = j * down + hl
        p, ntop = cj % up, cj // up
        acc = np.float32(0)
        for q in range(max(0, ntop - (x.size - 1)), min((2 * hl - p) // up, ntop) + 1):
            acc = np.float32(acc + table[p, q] * x[ntop - q])
        out[j] = acc
    assert np.mean(out != ref) > 0.1


@pytest.mark.parametrize("n", [1, 2, 7, 8, 9, 127, 128, 129, 130, 255, 256, 1000, 8191, 8192, 8193, 32768 + 5, 100_003,
                               960_000])
def test_restated_pairwise_sum_is_numpy(n):
    x = (np.random.default_rng(n).standard_normal(n) * 0.3).astype(np.float32)
    s = sumsq_restated(x)
    assert s == np.add.reduce(x ** 2) and pairwise(x * x) == s
    m = np.mean(x ** 2)
    assert type(m) is np.float32 and m == np.float32(np.float64(s) / n)


def test_work_item_table():
    L = _lib.lib()
    h = C.c_void_p()
    _lib.check(L.mb_resample_create(-1, C.byref(h)))
    try:
        idx = {}
        for src, dst in RATIOS:
            up, down = rs.ratio(src, dst)
            if up == down:
                idx[(src, dst)] = -1
                continue
            f = rs.design_filter(up, down)
            i = C.c_int32()
            _lib.check(L.mb_resample_add_filter(h, up, down, f.ctypes.data_as(C.c_void_p), f.size, C.byref(i)))
            idx[(src, dst)] = i.value
            assert L.mb_resample_filter_in_smem(h, i.value) == (1 if up * -(-f.size // up) * 4 <= 64 * 1024 else 0)
        assert L.mb_resample_filter_in_smem(h, idx[(44056, 16000)]) == 0
        assert L.mb_resample_filter_in_smem(h, idx[(11025, 16000)]) == 1
        clips = [(44100, 16000, 1), (48000, 16000, 160_000), (16000, 16000, 513), (44056, 16000, 7), (8000, 16000, 512),
                 (11025, 16000, 44_100), (16000, 24000, 2)]
        B = len(clips)
        lens = (C.c_int32 * B)(*[n for _, _, n in clips])
        fis = (C.c_int32 * B)(*[idx[(s, d)] for s, d, _ in clips])
        tile0 = (C.c_int32 * (B + 1))()
        offs = (C.c_int64 * (B + 1))()
        _lib.check(L.mb_resample_work_items(h, lens, fis, B, tile0, offs))
        outs = [resample_poly(np.zeros(n, np.float32), *rs.ratio(s, d)).size for s, d, n in clips]
        assert outs == [rs.output_length(n, s, d) for s, d, n in clips]
        assert list(offs) == np.concatenate([[0], np.cumsum(outs)]).tolist()
        assert list(tile0) == np.concatenate([[0], np.cumsum([-(-m // 512) for m in outs])]).tolist()
        lens[3] = 0
        assert L.mb_resample_work_items(h, lens, fis, B, tile0, offs) != 0 and b"clip 3" in L.mb_last_error()
        lens[3] = 7
        fis[5] = 99
        assert L.mb_resample_work_items(h, lens, fis, B, tile0, offs) != 0 and b"clip 5" in L.mb_last_error()
        # the same ratio twice gives the same filter; a ratio that is not reduced or a wrong tap count is refused
        f = rs.design_filter(160, 441)
        i = C.c_int32()
        _lib.check(L.mb_resample_add_filter(h, 160, 441, f.ctypes.data_as(C.c_void_p), f.size, C.byref(i)))
        assert i.value == idx[(44100, 16000)]
        assert L.mb_resample_add_filter(h, 320, 882, f.ctypes.data_as(C.c_void_p), f.size, C.byref(i)) != 0
        assert L.mb_resample_add_filter(h, 160, 441, f.ctypes.data_as(C.c_void_p), f.size - 1, C.byref(i)) != 0
        assert L.mb_resample_add_filter(h, 1, 1, f.ctypes.data_as(C.c_void_p), 21, C.byref(i)) != 0
        assert L.mb_resample_output_length(160, 441, 44100) == 16000 and L.mb_resample_output_length(0, 1, 5) == -1
    finally:
        L.mb_resample_destroy(h)


@pytest.mark.parametrize("wavs,srs,match", [
    ([np.zeros(0, np.float32)], 44100, "clip 0 is empty"),
    ([np.zeros(5, np.float32), np.zeros((2, 5), np.float32)], 44100, "clip 1 must be one-dimensional"),
    ([np.zeros(5, np.float64)], 44100, "clip 0 is float64"),
    ([np.zeros(5, np.float32), np.zeros(5, np.int32)], 44100, "clip 1 has dtype int32"),
    ([np.zeros(5, np.float32)], 0, "clip 0: sample rate 0"),
    ([np.zeros(5, np.float32)], -16000, "clip 0: sample rate -16000"),
    ([np.zeros(5, np.float32)], 44100.5, "clip 0: sample rate 44100.5"),
    ([np.zeros(5, np.float32)], "44100", "clip 0: sample rate '44100'"),
    ([np.zeros(5, np.float32)] * 2, [44100, None], "clip 1: sample rate None"),
    ([np.zeros(5, np.float32)] * 2, [44100], "1 source rates for 2 clips"),
])
def test_refusals_before_anything_is_queued(wavs, srs, match):
    with pytest.raises(ValueError, match=match):
        rs.resample_device(wavs, srs, 16000)


def test_refusals_of_the_loaders():
    with pytest.raises(ValueError, match="target: sample rate 0"):
        rs.resample_device([np.zeros(5, np.float32)], 16000, 0)
    with pytest.raises(ValueError, match="clip 1 has dtype int16"):
        rs.load_clips([np.zeros(5, np.float32), np.zeros(5, np.int16)], None, 16000)
    with pytest.raises(ValueError, match="clip 0 is float64"):
        rs.load_clips([np.zeros(5)], 44100, 16000)
    clips, rates = rs.load_clips([np.zeros(5, np.float32), np.ones(3, np.float32)], [None, 22050], 16000)
    assert rates == [16000, 22050] and [c.size for c in clips] == [5, 3]


def test_read_native_keeps_int16_pcm(tmp_path):
    from scipy.io import wavfile

    from mockingbird_b200.synthesizer import audio_host

    pcm = (np.random.default_rng(0).standard_normal(1000) * 3000).astype(np.int16)
    wavfile.write(tmp_path / "m.wav", 44100, pcm)
    wavfile.write(tmp_path / "s.wav", 48000, np.stack([pcm, pcm[::-1]], axis=1))
    x, sr = rs.read_native(tmp_path / "m.wav")
    assert sr == 44100 and x.dtype == np.int16 and np.array_equal(x, pcm)
    assert np.array_equal(x.astype(np.float32) / np.float32(32768), audio_host.load_wav(tmp_path / "m.wav", None)[0])
    y, sr = rs.read_native(tmp_path / "s.wav")
    assert sr == 48000 and _bits_equal(y, audio_host.load_wav(tmp_path / "s.wav", None)[0])
