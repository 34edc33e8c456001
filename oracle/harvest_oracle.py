"""Harvest F0 tracker, restated in float64 numpy (TEST INFRASTRUCTURE): the spec `csrc/f0.cu` is held to (DESIGN §4n).

Harvest is M. Morise, "Harvest: A high-performance fundamental frequency estimator from speech signals", Interspeech 2017,
as implemented in WORLD.  This module restates it at the one configuration any caller of `utils/f0_utils.py` uses:
16 kHz input, f0_floor = 80, f0_ceil = 600, a 1 ms internal frame period, and output frames every 10 ms.

Stages (`harvest(x)` runs them in order; `harvest_stages(x)` also returns what the device's debug outputs hold):
  1. decimate      by 2 with WORLD's third-order IIR (the Chebyshev type I design of 0.05 dB ripple at 0.4 of Nyquist),
                   forward and backward over the signal with 9 odd-reflected samples at each end; keep every 2nd sample
                   ending on the last one; one zero appended (y_length = 1 + len // 2); subtract the mean
  2. channels      128 band-pass channels at 72 * 2 ** ((i + 1) / 40) Hz, Nuttall window times a cosine, applied directly
                   in time: f[i] = sum_k h[k] y[i + L + 1 - k] (WORLD's delay compensation), summed over k ascending
  3. raw           per channel, four event sequences (negative / positive zero crossings, peaks, dips), each as intervals
                   fs / (e_{j+1} - e_j) at (e_j + e_{j+1}) / 2 / fs; each linearly interpolated (and extrapolated) at the
                   1 ms frames, averaged, kept inside [bf / 1.1, bf * 1.1] and [80, 600]; a channel with fewer than 3
                   intervals of some kind is 0 everywhere
  4. official      per frame, every run of >= 10 voiced channels (channel 0 and 127 forced unvoiced) gives its mean; nc
                   is the largest count over the clip's frames; each frame then holds 7 nc slots: its own candidates and
                   those of the frames 1, 2, 3 before and 1, 2, 3 after (zeros where a frame has fewer or none)
  5. refine        each slot: Blackman window of 2 int(1.5 fs / f0 + 1) + 1 samples and its central-difference derivative,
                   DFT at the first min(6, int(fs / 2 / f0)) harmonic bins of an N = 2 ** (2 + floor(log2 length)) point
                   transform, instantaneous frequencies weighted by amplitude; dropped outside [80, 600] or below score 2.5
  6. unreliable    a slot of frame 1 .. T-2 is dropped when no slot of the frame before or after is within 5 %
  7. contour       best score per frame, FixStep1 (0.008), FixStep2 (erosion over +-2 frames), FixStep3 (extension by
                   candidates within 18 %, merge), FixStep4 (linear fill of gaps shorter than 9 frames)
  8. smoothing     each voiced run alone, zero-phase second-order low-pass with the run's edge values held for 300 frames
                   on each side
  9. output        frame i of the 10 ms contour is the 1 ms contour at frame 10 i

Substitutes where WORLD's exact rule is not restated with confidence (named in DESIGN §4n as well):
  * FixStep3's merge orders the kept runs by their extended start (a stable sort) and starts from the first of them.
  * FixStep4 fills a gap between a run ending at e and one starting at s with a + (b - a) (j - e) / (s - e).
  * Smoothing runs the filter over the run plus 300 held frames on each side, not over the whole padded contour; the
    state the longer run-in would add is below 0.875 ** 300 (~4e-18) of the held value.
  * A clip shorter than 10 samples reflects its edge padding with clamped indices.
Everything else (ExtendSub's running mean carried from run to run included) follows WORLD's code as restated.

All arithmetic is float64 and written in the order the device evaluates it (the device is compiled without FMA
contraction), so the decimated signal, the filter bank, the events and the raw and official candidates are bitwise
equal; the window tables use libm's cos (`math.cos`), as the device's host-computed tables do.  Refinement uses the
device's own cos on its side, so refined values differ in the last bits.
"""
from __future__ import annotations

import math

import numpy as np

FS = 16000
FRAME_PERIOD = 10.0
F0_FLOOR = 80.0
F0_CEIL = 600.0
RATIO = 2
FSD = FS / RATIO  # 8000.0
CHANNELS_IN_OCTAVE = 40
N_FACT = 9
DEC_A = (0.041156734567757189, -0.42599112459189636, 0.041037215479961225)  # wt = x + a0 w0 + a1 w1 + a2 w2
DEC_B = (0.16797464681802227, 0.50392394045406674)  # y = b0 wt + b1 w0 + b1 w1 + b0 w2
SMOOTH_B = (0.0078202080334971724, 0.015640416066994345)
SMOOTH_A = (1.7347257688092754, -0.76600660094326412)
SMOOTH_LAG = 300
MEAN_CHUNK = 256
TWIDDLE_N = 1024


def channel_count():
    return 1 + int(math.log(F0_CEIL * 1.1 / (F0_FLOOR * 0.9)) / math.log(2.0) * CHANNELS_IN_OCTAVE)


NCH = channel_count()  # 128
MAX_OWN = int(NCH / 10.0 + 0.5)  # 13 official candidates per frame at most
MAX_SLOTS = MAX_OWN * 7  # 91


def boundary_f0(i):
    return F0_FLOOR * 0.9 * 2.0 ** ((i + 1) / CHANNELS_IN_OCTAVE)


def mround(x):
    return int(x - 0.5) if x < 0 else int(x + 0.5)


def frames_1ms(n):
    return int(1000.0 * n / FS / 1.0) + 1


def frames_out(n, frame_period=FRAME_PERIOD):
    return int(1000.0 * n / FS / frame_period) + 1


def band_pass(c):
    """taps of channel c: Nuttall window of 2 L + 1 samples times cos(2 pi bf (k - L) / fs), L = round(2 fs / bf)"""
    bf = boundary_f0(c)
    L = mround(FSD / bf * 2.0)
    n = 2 * L + 1
    h = np.empty(n)
    for k in range(n):
        t = k / (n - 1.0)
        w = 0.355768 - 0.487396 * math.cos(2.0 * math.pi * t) + 0.144232 * math.cos(4.0 * math.pi * t) - \
            0.012604 * math.cos(6.0 * math.pi * t)
        h[k] = w * math.cos(2.0 * math.pi * bf * (k - L) / FSD)
    return L, h


def twiddles():
    q = range(TWIDDLE_N)
    return (np.array([math.cos(2.0 * math.pi * k / TWIDDLE_N) for k in q]),
            np.array([math.sin(2.0 * math.pi * k / TWIDDLE_N) for k in q]))


# ---------------------------------------------------------------------------------------------------------- 1. decimation
def _iir3(v):
    a0, a1, a2 = DEC_A
    b0, b1 = DEC_B
    w0 = w1 = w2 = 0.0
    out = [0.0] * len(v)
    for i, x in enumerate(v):
        wt = x + a0 * w0 + a1 * w1 + a2 * w2
        out[i] = b0 * wt + b1 * w0 + b1 * w1 + b0 * w2
        w2, w1, w0 = w1, w0, wt
    return out


def decimate(x):
    """stage 1: the decimated, mean-removed signal of 1 + len(x) // 2 samples"""
    x = [float(v) for v in np.asarray(x, dtype=np.float64)]
    L = len(x)
    cl = lambda i: x[min(max(i, 0), L - 1)]  # noqa: E731
    pad = [2 * x[0] - cl(N_FACT - i) for i in range(N_FACT)] + x + \
          [2 * x[L - 1] - cl(L - 2 - i) for i in range(N_FACT)]
    p = _iir3(pad)[::-1]
    p = _iir3(p)[::-1]
    nout = (L - 1) // RATIO + 1
    nbeg = RATIO - RATIO * nout + L
    n = 1 + L // RATIO
    y = np.zeros(n)
    y[:nout] = [p[nbeg - 1 + k * RATIO + N_FACT] for k in range(nout)]
    return y - mean_chunked(y)


def mean_chunked(y):
    """the mean as the device sums it: each 256-sample chunk left to right, then the chunk sums left to right"""
    total = 0.0
    for i in range(0, len(y), MEAN_CHUNK):
        total += float(np.cumsum(y[i:i + MEAN_CHUNK])[-1])
    return total / len(y)


# ------------------------------------------------------------------------------------------------ 2-3. channels and events
def filtered(y, L, h):
    n = len(y)
    P = 2 * L + 2
    yp = np.concatenate([np.zeros(P), y, np.zeros(P)])
    acc = np.zeros(n)
    for k in range(2 * L + 1):
        s = P + L + 1 - k
        acc = acc + h[k] * yp[s:s + n]
    return acc


def zero_crossing_intervals(f):
    """WORLD's ZeroCrossingEngine: (locations, intervals) of the negative-going crossings of f"""
    i = np.nonzero((f[:-1] > 0.0) & (f[1:] <= 0.0))[0]
    e = i + 1
    fine = e.astype(np.float64) - f[e - 1] / (f[e] - f[e - 1])
    return (fine[:-1] + fine[1:]) / 2.0 / FSD, FSD / (fine[1:] - fine[:-1])


def four_events(f):
    g = -f
    d = g[:-1] - g[1:]
    return [zero_crossing_intervals(f), zero_crossing_intervals(g), zero_crossing_intervals(d), zero_crossing_intervals(-d)]


def interp_at(loc, val, t):
    """WORLD's interp1 (histc): linear inside, the first / last interval extended outside"""
    k = np.clip(np.searchsorted(loc, t, side="right"), 1, len(loc) - 1)
    s = (t - loc[k - 1]) / (loc[k] - loc[k - 1])
    return val[k - 1] + s * (val[k] - val[k - 1])


def raw_candidates(y, T):
    """stage 3: [channels][T] raw candidates, and the [channels][4] interval counts"""
    t = np.arange(T) / 1000.0
    raw = np.zeros((NCH, T))
    counts = np.zeros((NCH, 4), dtype=np.int64)
    for c in range(NCH):
        L, h = band_pass(c)
        ev = four_events(filtered(y, L, h))
        counts[c] = [len(v) for _, v in ev]
        if (counts[c] < 3).any():
            continue
        v = [interp_at(loc, val, t) for loc, val in ev]
        avg = (((v[0] + v[1]) + v[2]) + v[3]) / 4.0
        bf = boundary_f0(c)
        bad = (avg > bf * 1.1) | (avg < bf / 1.1) | (avg > F0_CEIL) | (avg < F0_FLOOR)
        raw[c] = np.where(bad, 0.0, avg)
    return raw, counts


# ------------------------------------------------------------------------------------------------ 4. official candidates
def official_candidates(raw):
    """[T][MAX_OWN] own candidates and their counts per frame"""
    T = raw.shape[1]
    own = np.zeros((T, MAX_OWN))
    cnt = np.zeros(T, dtype=np.int64)
    vuv = raw > 0
    vuv[0] = vuv[-1] = False
    for i in range(T):
        col = vuv[:, i]
        d = np.diff(col.astype(np.int8))
        st = np.nonzero(d == 1)[0] + 1
        ed = np.nonzero(d == -1)[0] + 1
        for s, e in zip(st, ed):
            if e - s < 10:
                continue
            acc = 0.0
            for c in range(s, e):
                acc += float(raw[c, i])
            own[i, cnt[i]] = acc / (e - s)
            cnt[i] += 1
    return own, cnt


def overlap(own, cnt):
    T = own.shape[0]
    nc = int(cnt.max()) if T else 0
    S = 7 * nc
    cand = np.zeros((T, S))
    if nc == 0:
        return cand, nc
    o = own[:, :nc]
    cand[:, :nc] = o
    for b in range(1, 4):
        cand[b:, b * nc:(b + 1) * nc] = o[:-b] if b < T else o[:0]
        cand[:T - b, (b + 3) * nc:(b + 4) * nc] = o[b:] if b < T else o[:0]
    return cand, nc


# ----------------------------------------------------------------------------------------------------------- 5. refinement
def refine(y, cand, chunk=4096):
    """stage 5: refined candidates and scores, the shape of cand"""
    T, S = cand.shape
    n = len(y)
    C, Sn = twiddles()
    f_out = np.zeros((T, S))
    s_out = np.zeros((T, S))
    fi, si = np.nonzero(cand > 0.0)
    for c0 in range(0, len(fi), chunk):
        fr, sl = fi[c0:c0 + chunk], si[c0:c0 + chunk]
        f0 = cand[fr, sl]
        K = len(f0)
        hw = (1.5 * FSD / f0 + 1.0).astype(np.int64)
        nw = 2 * hw + 1
        wl = (2.0 * hw + 1.0) / FSD
        N = 1 << (2 + np.array([int(v).bit_length() - 1 for v in nw]))
        pos = fr / 1000.0
        bt0 = (-hw).astype(np.float64) / FSD
        v = (pos + bt0) * FSD + 0.001
        basic = np.where(v < 0, (v - 0.5).astype(np.int64), (v + 0.5).astype(np.int64))
        J = int(nw.max())
        j = np.arange(J)
        idx = basic[:, None] + j[None, :]
        tmp = (idx - 1.0) / FSD - pos[:, None]
        w = 0.42 + 0.5 * np.cos(2.0 * math.pi * tmp / wl[:, None]) + 0.08 * np.cos(4.0 * math.pi * tmp / wl[:, None])
        live = j[None, :] < nw[:, None]
        w = np.where(live, w, 0.0)
        wn = np.concatenate([w[:, 1:], np.zeros((K, 1))], axis=1)
        wp = np.concatenate([np.zeros((K, 1)), w[:, :-1]], axis=1)
        dw = -(wn - wp) / 2.0
        dw[:, 0] = -w[:, 1] / 2.0
        last = nw - 1
        dw[np.arange(K), last] = w[np.arange(K), last - 1] / 2.0
        dw = np.where(live, dw, 0.0)
        xs = y[np.clip(idx - 1, 0, n - 1)]
        xw, xd = xs * w, xs * dw
        nh = np.minimum((FSD / 2.0 / f0).astype(np.int64), 6)
        h1 = np.arange(6) + 1.0
        m = f0[:, None] * N[:, None] / FSD * h1[None, :]
        m = np.where(m < 0, (m - 0.5).astype(np.int64), (m + 0.5).astype(np.int64))
        stride = (TWIDDLE_N // N)[:, None]
        mr = np.zeros((K, 6)); mi = np.zeros((K, 6)); dr = np.zeros((K, 6)); di = np.zeros((K, 6))
        for jj in range(J):
            q = (jj * m) % N[:, None] * stride
            c, s = C[q], Sn[q]
            a, b = xw[:, jj:jj + 1], xd[:, jj:jj + 1]
            mr = mr + a * c; mi = mi - a * s
            dr = dr + b * c; di = di - b * s
        num_i = mr * di - mi * dr
        pw = mr * mr + mi * mi
        with np.errstate(divide="ignore", invalid="ignore"):
            inst = np.where(pw == 0.0, 0.0, m * FSD / N[:, None] + num_i / pw * FSD / 2.0 / math.pi)
        amp = np.sqrt(pw)
        num = np.zeros(K); den = np.zeros(K); sc = np.zeros(K)
        for h in range(6):
            on = h < nh
            num = np.where(on, num + amp[:, h] * inst[:, h], num)
            den = np.where(on, den + amp[:, h] * (h + 1.0), den)
            sc = np.where(on, sc + np.abs((inst[:, h] / (h + 1.0) - f0) / f0), sc)
        rf = num / (den + 1e-12)
        rs = 1.0 / (sc / nh + 1e-12)
        bad = (rf < F0_FLOOR) | (rf > F0_CEIL) | (rs < 2.5)
        f_out[fr, sl] = np.where(bad, 0.0, rf)
        s_out[fr, sl] = np.where(bad, 0.0, rs)
    return f_out, s_out


# --------------------------------------------------------------------------------------- 6-7. unreliable removal, contour
def remove_unreliable(cand, score):
    cand, score = cand.copy(), score.copy()
    T, S = cand.shape
    if T < 3 or S == 0:
        return cand, score
    ref = cand[1:-1]

    def best_err(nb):
        with np.errstate(divide="ignore", invalid="ignore"):
            e = np.abs(ref[:, :, None] - nb[:, None, :]) / ref[:, :, None]
        return np.minimum(e.min(axis=2), 1.0)

    e1, e2 = best_err(cand[2:]), best_err(cand[:-2])
    drop = (ref != 0.0) & (e1 > 0.05) & (e2 > 0.05)
    cand[1:-1][drop] = 0.0
    score[1:-1][drop] = 0.0
    return cand, score


def select_best(ref, cands, allowed):
    best_f0, best = 0.0, allowed
    for c in cands:
        t = abs(ref - c) / ref
        if t > best:
            continue
        best_f0, best = c, t
    return best_f0


def search_base(cand, score):
    T = cand.shape[0]
    base = np.zeros(T)
    for i in range(T):
        bs = 0.0
        for j in range(cand.shape[1]):
            if score[i, j] > bs:
                base[i], bs = cand[i, j], score[i, j]
    return base


def fix_step1(b, allowed=0.008):
    out = np.zeros(len(b))
    with np.errstate(divide="ignore", invalid="ignore"):
        for i in range(2, len(b)):
            if b[i] == 0.0:
                continue
            r = b[i - 1] * 2 - b[i - 2]
            out[i] = 0.0 if (abs((b[i] - r) / r) > allowed and abs(b[i] - b[i - 1]) / b[i - 1] > allowed) else b[i]
    return out


def fix_step2(s1, voice_range_minimum=6):
    out = s1.copy()
    c = (voice_range_minimum - 1) // 2
    for i in range(c, len(s1) - c):
        if (s1[i - c:i + c + 1] == 0).any():
            out[i] = 0.0
    return out


def boundaries(f):
    """WORLD's GetBoundaryList: (start, end) inclusive of every voiced run, the first and last frame counted unvoiced"""
    v = (f > 0).astype(np.int8)
    if len(v):
        v[0] = v[-1] = 0
    d = np.diff(v)
    return list(zip((np.nonzero(d == 1)[0] + 1).tolist(), np.nonzero(d == -1)[0].tolist()))


def _extend(ch, origin, last, shift, cand, allowed):
    tmp, new_origin, count = ch[origin], origin, 0
    for i in range(abs(last - origin) + 1):
        k = origin + shift * i + shift
        v = select_best(tmp, cand[k], allowed)
        ch[k] = v
        if v == 0.0:
            count += 1
        else:
            tmp, count, new_origin = v, 0, k
        if count == 4:
            break
    return new_origin


def search_score(f0, cands, scores):
    s = 0.0
    for c, sc in zip(cands, scores):
        if f0 == c and s < sc:
            s = sc
    return s


def fix_step3(s2, cand, score, allowed=0.18):
    T = len(s2)
    secs = boundaries(s2)
    chans, bnd = [], []
    for st, ed in secs:
        ch = np.zeros(T)
        ch[st:ed + 1] = s2[st:ed + 1]
        ned = _extend(ch, ed, min(T - 2, ed + 100), 1, cand, allowed)
        nst = _extend(ch, st, max(1, st - 100), -1, cand, allowed)
        chans.append(ch)
        bnd.append((nst, ned))
    kept = []
    mean = np.float64(0.0)
    with np.errstate(divide="ignore", invalid="ignore"):
        for k, (st, ed) in enumerate(bnd):
            for j in range(st, ed):
                mean = mean + chans[k][j]
            mean = mean / np.float64(ed - st)
            if np.float64(2200.0) / mean < ed - st:
                kept.append(k)
    if not kept:
        return s2.copy()
    order = sorted(kept, key=lambda k: bnd[k][0])
    merged = chans[order[0]].copy()
    cst, ced = bnd[order[0]]
    for k in order[1:]:
        st2, ed2 = bnd[k]
        ch = chans[k]
        if st2 - ced > 0:
            merged[st2:ed2 + 1] = ch[st2:ed2 + 1]
            cst, ced = st2, ed2
        elif cst <= st2 and ced >= ed2:
            continue
        else:
            sc1 = sc2 = 0.0
            for i in range(st2, ced + 1):
                sc1 += search_score(merged[i], cand[i], score[i])
                sc2 += search_score(ch[i], cand[i], score[i])
            lo = ced if sc1 > sc2 else st2
            merged[lo:ed2 + 1] = ch[lo:ed2 + 1]
            ced = ed2
    return merged


def fix_step4(s3, threshold=9):
    out = s3.copy()
    secs = boundaries(s3)
    for (_, e), (s, _) in zip(secs[:-1], secs[1:]):
        if s - e - 1 >= threshold:
            continue
        a, b = s3[e], s3[s]
        for j in range(e + 1, s):
            out[j] = a + (b - a) * float(j - e) / float(s - e)
    return out


# ------------------------------------------------------------------------------------------------------------ 8. smoothing
def runs(f):
    v = np.concatenate([[0], (f > 0).astype(np.int8), [0]])
    d = np.diff(v)
    return list(zip(np.nonzero(d == 1)[0].tolist(), (np.nonzero(d == -1)[0] - 1).tolist()))


def smooth(c):
    a0, a1 = SMOOTH_A
    b0, b1 = SMOOTH_B
    out = np.zeros(len(c))
    for st, ed in runs(c):
        lo, hi = st - SMOOTH_LAG, ed + SMOOTH_LAG
        xs = [float(c[min(max(j, st), ed)]) for j in range(lo, hi + 1)]
        w0 = w1 = 0.0
        f = [0.0] * len(xs)
        for j, x in enumerate(xs):
            wt = x + a0 * w0 + a1 * w1
            f[j] = b0 * wt + b1 * w0 + b0 * w1
            w1, w0 = w0, wt
        w0 = w1 = 0.0
        yv = [0.0] * len(xs)
        for j in range(len(xs) - 1, -1, -1):
            wt = f[j] + a0 * w0 + a1 * w1
            yv[j] = b0 * wt + b1 * w0 + b0 * w1
            w1, w0 = w0, wt
        out[st:ed + 1] = yv[SMOOTH_LAG:SMOOTH_LAG + ed - st + 1]
    return out


# ------------------------------------------------------------------------------------------------------------------ entry
def harvest_stages(x):
    """every stage of one clip: a dict of the intermediate results (the names of the device's debug outputs)"""
    x = np.asarray(x, dtype=np.float64)
    if x.ndim != 1 or len(x) == 0:
        raise ValueError("harvest_oracle: a non-empty one-dimensional signal is required")
    T = frames_1ms(len(x))
    y = decimate(x)
    raw, counts = raw_candidates(y, T)
    own, cnt = official_candidates(raw)
    cand, nc = overlap(own, cnt)
    rc, rs = refine(y, cand)
    cc, cs = remove_unreliable(rc, rs)
    base = search_base(cc, cs)
    s1 = fix_step1(base)
    s2 = fix_step2(s1)
    s3 = fix_step3(s2, cc, cs)
    s4 = fix_step4(s3)
    sm = smooth(s4)
    n_out = frames_out(len(x))
    f0 = sm[np.minimum(T - 1, np.arange(n_out) * 10)]
    return dict(y=y, raw=raw, interval_counts=counts, raw_count=(raw > 0).sum(axis=0), own=own, official_count=cnt, nc=nc,
                refined=rc, scores=rs, reliable=cc, reliable_scores=cs, base=base, step1=s1, step2=s2, step3=s3,
                contour=s4, smoothed=sm, f0=f0)


def harvest(x, fs=FS, frame_period=FRAME_PERIOD, f0_floor=F0_FLOOR, f0_ceil=F0_CEIL):
    """(f0, temporal_positions) as pyworld.harvest returns them, for the one supported configuration"""
    if (fs, frame_period, f0_floor, f0_ceil) != (FS, FRAME_PERIOD, F0_FLOOR, F0_CEIL):
        raise ValueError("harvest_oracle restates fs = 16000, frame_period = 10, f0_floor = 80, f0_ceil = 600 only")
    f0 = harvest_stages(x)["f0"]
    return f0, np.arange(len(f0)) * frame_period / 1000.0


# ----------------------------------------------------------------------------------------------- synthetic test signals
def voiced(f0_track, sr=FS, seed=0, harmonics=12):
    """a harmonic series following the per-sample F0 track, with a gentle spectral tilt"""
    rng = np.random.default_rng(seed)
    ph = 2 * np.pi * np.cumsum(f0_track) / sr
    out = np.zeros(len(f0_track))
    for k in range(1, harmonics + 1):
        amp = 1.0 / k ** 0.8
        live = k * f0_track < 0.45 * sr
        out += np.where(live, amp * np.sin(k * ph + rng.uniform(0, 2 * np.pi)), 0.0)
    return out / np.max(np.abs(out)) * 0.5


def speechlike(seed, n, sr=FS):
    """seeded speech-like clip: voiced segments with F0 glides and vibrato, digital silences, -60 dBFS noise and noise
    bursts (float32)"""
    rng = np.random.default_rng(seed)
    out = np.zeros(n)
    i = 0
    while i < n:
        kind = rng.choice(3, p=[0.6, 0.25, 0.15])
        m = min(n - i, int(rng.uniform(0.15, 0.6) * sr))
        t = np.arange(m) / sr
        if kind == 0:
            f_a, f_b = rng.uniform(90, 320, size=2)
            track = f_a + (f_b - f_a) * t / max(t[-1], 1e-9) + rng.uniform(0, 8) * np.sin(2 * np.pi * rng.uniform(4, 7) * t)
            seg = voiced(track, sr, int(rng.integers(1 << 30))) * rng.uniform(0.3, 1.0)
            seg *= np.minimum(1.0, np.minimum(t, t[-1] - t) / 0.02)
        elif kind == 1:
            seg = rng.standard_normal(m) * 1e-3
        else:
            seg = rng.standard_normal(m) * rng.uniform(0.01, 0.2)
        out[i:i + m] = seg
        i += m
    return out.astype(np.float32)
