// Harvest F0 tracking on H100 (mb_f0_*): DESIGN.md section 4n.
//
//   replaces  pyworld.harvest(wav, 16000, frame_period=10, f0_floor=80, f0_ceil=600), as utils/f0_utils.py:14-20
//             (compute_f0) calls it
//
// float64 throughout, compiled without FMA contraction (build.py) so that every stage up to the official candidates is
// evaluated in the order oracle/harvest_oracle.py writes it.  B clips of different lengths run in one sequence of five
// launches; nothing a clip computes reads another clip's data, so each clip's result does not depend on its batch.
//   f0_decimate_kernel  one CTA per clip: the forward-backward third-order IIR over the padded clip (one thread; the
//                       recurrence is sequential), every 2nd sample, the chunked mean subtracted
//   f0_bank_kernel      one CTA per (channel, clip): the band-pass filter in time over 1024-sample tiles staged in shared
//                       memory, the four event kinds of each tile compacted in order, each new interval resolving the 1 ms
//                       frames it brackets -> ev [frame][channel][4]
//   f0_official_kernel  one thread per (clip, 1 ms frame): average, range check, runs of >= 10 voiced channels -> <= 13
//                       own candidates; atomicMax of the clip's largest count nc
//   f0_refine_kernel    one thread per (clip, frame, slot < 91): the slot's candidate (own or of a frame within +-3),
//                       Blackman window and derivative, direct DFT at <= 6 harmonic bins -> refined f0 and score
//   f0_fix_kernel       one CTA per clip: unreliable-candidate removal, base contour, FixStep1-4, smoothing per voiced run,
//                       subsampling to 10 ms
#include <cmath>
#include <cstring>
#include <vector>

#include "mb_common.h"

using namespace mb;

namespace {

constexpr int kNch = 128;        // 1 + int(log2(660 / 72) * 40)
constexpr int kMaxOwn = 13;      // round(128 / 10)
constexpr int kSlots = 91;       // 7 * kMaxOwn
constexpr int kNFact = 9;
constexpr int kMeanChunk = 256;
constexpr int kTwN = 1024;       // twiddle table; every refinement transform (128 .. 1024 points) indexes it with a stride
constexpr int kTile = 1024;
constexpr int kBankThreads = 256;
constexpr int kFixThreads = 256;
constexpr int kExt = 101;        // frames one extension can write on each side of a run
constexpr int kLag = 300;        // smoothing: held frames on each side of a run
constexpr int kMaxL = 222;       // round(2 * 8000 / 72.0...) for channel 0
constexpr double kFs = 8000.0;   // 16 kHz decimated by 2
constexpr double kFloor = 80.0, kCeil = 600.0;
constexpr double kPi = 3.14159265358979323846;

__constant__ double kDecA[3] = {0.041156734567757189, -0.42599112459189636, 0.041037215479961225};
__constant__ double kDecB[2] = {0.16797464681802227, 0.50392394045406674};

struct F0Clip {
  int64_t x;    // first input sample
  int64_t y;    // first decimated sample
  int64_t pad;  // first sample of the padded decimation buffers
  int64_t f;    // first 1 ms frame
  int64_t sec;  // first run slot
  int64_t out;  // first 10 ms output frame
  int32_t L, n, T, n_out;
};

struct F0Params {
  const F0Clip* clips;
  const double* x;
  const double* bf;      // [128] channel frequencies
  const double* chL;     // [128] half filter lengths
  const double* choff;   // [128] first tap of each channel in taps
  const double* taps;
  const double* twc;     // [1024] cos(2 pi q / 1024)
  const double* tws;     // [1024] sin
  double* y;             // decimated signals
  double* p1;            // padded decimation buffers
  double* p2;
  double* ev;            // [frames][128][4] per-kind interpolated intervals
  int32_t* icount;       // [clip][128][4] intervals per kind
  double* own;           // [frames][13]
  int32_t* ocount;       // [frames]
  int32_t* rcount;       // [frames] channels with a raw candidate
  int32_t* nc;           // [clip]
  double* rf;            // [frames][91] refined candidates
  double* rs;            // scores
  double* cf;            // after the unreliable-candidate removal
  double* cs;
  double* base;          // [frames] contour stages
  double* s1;
  double* s2;
  double* s3;
  double* s4;
  double* sm;
  int32_t* sec;          // [run slots][4]: start, end, extended start, extended end
  int32_t* ord;          // [run slots]
  double* ext;           // [run slots][2][101] extension values after the end and before the start
  double* tail;          // [clip][kFixThreads][300]
  double* f0;            // [output frames]
};

__device__ __forceinline__ int mround(double x) { return x < 0 ? (int)(x - 0.5) : (int)(x + 0.5); }

// ------------------------------------------------------------------------------------------------------------- decimate
__device__ __forceinline__ double pad_at(const double* __restrict__ x, int L, int i) {
  if (i < kNFact) return 2 * x[0] - x[min(max(kNFact - i, 0), L - 1)];
  if (i < kNFact + L) return x[i - kNFact];
  return 2 * x[L - 1] - x[min(max(L - 2 - (i - kNFact - L), 0), L - 1)];
}

__global__ void __launch_bounds__(256) f0_decimate_kernel(const F0Params p) {
  __shared__ double part[256];
  __shared__ double mean_s;
  const F0Clip u = p.clips[blockIdx.x];
  const double* __restrict__ x = p.x + u.x;
  double* __restrict__ a = p.p1 + u.pad;
  double* __restrict__ b = p.p2 + u.pad;
  double* __restrict__ y = p.y + u.y;
  const int np = u.L + 2 * kNFact;
  if (threadIdx.x == 0) {
    // inputs are loaded kDecBlock at a time into registers so that their latency is not on the recurrence
    constexpr int kDecBlock = 32;
    const double a0 = kDecA[0], a1 = kDecA[1], a2 = kDecA[2], b0 = kDecB[0], b1 = kDecB[1];
    double w0 = 0.0, w1 = 0.0, w2 = 0.0, v[kDecBlock];
    for (int i0 = 0; i0 < np; i0 += kDecBlock) {
#pragma unroll
      for (int j = 0; j < kDecBlock; ++j) v[j] = i0 + j < np ? pad_at(x, u.L, i0 + j) : 0.0;
#pragma unroll
      for (int j = 0; j < kDecBlock; ++j) {
        if (i0 + j >= np) break;
        const double wt = v[j] + a0 * w0 + a1 * w1 + a2 * w2;
        a[i0 + j] = b0 * wt + b1 * w0 + b1 * w1 + b0 * w2;
        w2 = w1, w1 = w0, w0 = wt;
      }
    }
    w0 = w1 = w2 = 0.0;
    for (int i0 = np - 1; i0 >= 0; i0 -= kDecBlock) {
#pragma unroll
      for (int j = 0; j < kDecBlock; ++j) v[j] = i0 - j >= 0 ? a[i0 - j] : 0.0;
#pragma unroll
      for (int j = 0; j < kDecBlock; ++j) {
        if (i0 - j < 0) break;
        const double wt = v[j] + a0 * w0 + a1 * w1 + a2 * w2;
        b[i0 - j] = b0 * wt + b1 * w0 + b1 * w1 + b0 * w2;
        w2 = w1, w1 = w0, w0 = wt;
      }
    }
  }
  __syncthreads();
  const int nout = (u.L - 1) / 2 + 1;
  const int nbeg = 2 - 2 * nout + u.L;
  for (int k = threadIdx.x; k < u.n; k += blockDim.x) y[k] = k < nout ? b[nbeg - 1 + 2 * k + kNFact] : 0.0;
  __syncthreads();
  // mean: each 256-sample chunk left to right (a thread per chunk), then the chunk sums left to right
  const int nch = (u.n + kMeanChunk - 1) / kMeanChunk;
  double total = 0.0;
  for (int c0 = 0; c0 < nch; c0 += blockDim.x) {
    const int c = c0 + threadIdx.x;
    if (c < nch) {
      const int e = min(u.n, (c + 1) * kMeanChunk);
      double s = y[c * kMeanChunk];
      for (int i = c * kMeanChunk + 1; i < e; ++i) s += y[i];
      part[threadIdx.x] = s;
    }
    __syncthreads();
    if (threadIdx.x == 0)
      for (int i = 0; i < min((int)blockDim.x, nch - c0); ++i) total += part[i];
    __syncthreads();
  }
  if (threadIdx.x == 0) mean_s = total / u.n;
  __syncthreads();
  const double m = mean_s;
  for (int k = threadIdx.x; k < u.n; k += blockDim.x) y[k] = y[k] - m;
}

// ------------------------------------------------------------------------------------------------------ filter bank
struct KindCarry {
  double c;         // last crossing
  double loc0, v0;  // the interval before the last
  double loc1, v1;  // the last interval
  int has_c, nint;
};

// the frames interval gi (>= 1; (pl, pv) before it, (l, v) itself) resolves: gi == 1 from frame 0, otherwise from the
// first frame at or after pl; up to the last frame before l
__device__ void resolve(double* __restrict__ ev, int T, int kind, int gi, double pl, double pv, double l, double v) {
  int f = 0;
  if (gi > 1) {
    f = max(0, (int)ceil(pl * 1000.0) - 1);
    while (f < T && f / 1000.0 < pl) ++f;
  }
  for (; f < T && f / 1000.0 < l; ++f) {
    const double s = (f / 1000.0 - pl) / (l - pl);
    ev[(size_t)f * (kNch * 4) + kind] = pv + s * (v - pv);
  }
}

// whether sample i (fs[2 + ii]) ends an event of `kind` and, if so, its fine position: kinds 0 / 1 are the negative-going
// crossings of f / g = -f at the pair (i - 1, i); kinds 2 / 3 those of d / -d, d[j] = g[j] - g[j + 1], at the pair
// (i - 2, i - 1).  WORLD's ZeroCrossingEngine: the crossing ending at sample e is e - s[e - 1] / (s[e] - s[e - 1]).
__device__ __forceinline__ bool event_at(const double* fs, int ii, int i, int kind, double& pos) {
  double a, b;
  int e;
  if (kind < 2) {
    if (i < 1) return false;
    a = fs[1 + ii], b = fs[2 + ii], e = i;
    if (kind == 1) a = -a, b = -b;
  } else {
    if (i < 2) return false;
    const double g0 = -fs[ii], g1 = -fs[1 + ii], g2 = -fs[2 + ii];
    a = g0 - g1, b = g1 - g2, e = i - 1;
    if (kind == 3) a = -a, b = -b;
  }
  if (!(0.0 < a && b <= 0.0)) return false;
  pos = e - a / (b - a);
  return true;
}

// an exclusive scan over the block of four 16-bit counters packed in one word
__device__ __forceinline__ uint64_t block_scan4(uint64_t v, uint64_t* warp_tot, uint64_t& total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  uint64_t inc = v;
  for (int o = 1; o < 32; o <<= 1) {
    const uint64_t t = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += t;
  }
  if (lane == 31) warp_tot[warp] = inc;
  __syncthreads();
  uint64_t before = 0, all = 0;
  for (int w = 0; w < kBankThreads / 32; ++w) {
    if (w < warp) before += warp_tot[w];
    all += warp_tot[w];
  }
  total = all;
  return before + inc - v;
}

__global__ void __launch_bounds__(kBankThreads) f0_bank_kernel(const F0Params p) {
  __shared__ double h[2 * kMaxL + 1];
  __shared__ double ys[kTile + 2 * kMaxL];
  __shared__ double fs[kTile + 2];  // fs[2 + i] = f[i0 + i]; fs[0], fs[1] carry f[i0 - 2], f[i0 - 1]
  __shared__ double cross[4][kTile / 2 + 2];
  __shared__ uint64_t warp_tot[kBankThreads / 32];
  __shared__ KindCarry carry[4];
  __shared__ int cnt[4];
  const int ch = blockIdx.x;
  const F0Clip u = p.clips[blockIdx.y];
  const int n = u.n, T = u.T;
  const int L = (int)p.chL[ch], K = 2 * L + 1;
  const double* taps = p.taps + (int64_t)p.choff[ch];
  const double* __restrict__ y = p.y + u.y;
  double* __restrict__ ev = p.ev + (size_t)u.f * (kNch * 4) + (size_t)ch * 4;
  for (int k = threadIdx.x; k < K; k += blockDim.x) h[k] = taps[k];
  if (threadIdx.x < 4) carry[threadIdx.x] = KindCarry{0.0, 0.0, 0.0, 0.0, 0.0, 0, 0};
  if (threadIdx.x < 2) fs[threadIdx.x] = 0.0;
  for (int i0 = 0; i0 < n; i0 += kTile) {
    const int m = min(kTile, n - i0);
    for (int j = threadIdx.x; j < m + 2 * L; j += blockDim.x) {
      const int yi = i0 - L + 1 + j;
      ys[j] = yi >= 0 && yi < n ? y[yi] : 0.0;
    }
    __syncthreads();
    for (int ii = threadIdx.x; ii < m; ii += blockDim.x) {
      double acc = 0.0;
      for (int k = 0; k < K; ++k) acc = acc + h[k] * ys[ii + 2 * L - k];
      fs[2 + ii] = acc;
    }
    __syncthreads();
    // events of positions i0 + 4 t .. i0 + 4 t + 3: counted, scanned, then written in order
    unsigned flags = 0;  // bit 4 q + kind
    for (int q = 0; q < 4; ++q) {
      const int ii = 4 * threadIdx.x + q;
      if (ii >= m) break;
      double pos;
      for (int t = 0; t < 4; ++t)
        if (event_at(fs, ii, i0 + ii, t, pos)) flags |= 1u << (4 * q + t);
    }
    uint64_t tot, packed = 0;
    for (int t = 0; t < 4; ++t) packed |= (uint64_t)__popc(flags & (0x1111u << t)) << (16 * t);
    const uint64_t ex = block_scan4(packed, warp_tot, tot);
    for (int t = 0; t < 4; ++t) {
      int o = (int)((ex >> (16 * t)) & 0xffff);
      for (int q = 0; q < 4; ++q) {
        double pos;
        if ((flags >> (4 * q + t)) & 1u) {
          event_at(fs, 4 * threadIdx.x + q, i0 + 4 * threadIdx.x + q, t, pos);
          cross[t][o++] = pos;
        }
      }
    }
    if (threadIdx.x < 4) cnt[threadIdx.x] = (int)((tot >> (16 * threadIdx.x)) & 0xffff);
    __syncthreads();
    // each crossing q closes an interval with the crossing before it (the carried one for q = 0); interval gi >= 1
    // resolves the frames it brackets with the interval before it
    const int c0 = cnt[0], c1 = c0 + cnt[1], c2 = c1 + cnt[2], c3 = c2 + cnt[3];
    for (int it = threadIdx.x; it < c3; it += blockDim.x) {
      const int t = it < c0 ? 0 : it < c1 ? 1 : it < c2 ? 2 : 3;
      const int q = it - (t == 0 ? 0 : t == 1 ? c0 : t == 2 ? c1 : c2);
      const KindCarry& cr = carry[t];
      const double* cl = cross[t];
      if (q == 0 && !cr.has_c) continue;
      const double prev = q > 0 ? cl[q - 1] : cr.c;
      const double loc = (prev + cl[q]) / 2.0 / kFs, val = kFs / (cl[q] - prev);
      const int gi = cr.nint + q - (cr.has_c ? 0 : 1);
      if (gi < 1) continue;
      double pl, pv;
      if (q == 0) {
        pl = cr.loc1, pv = cr.v1;
      } else {
        const double pp = q > 1 ? cl[q - 2] : cr.c;
        pl = (pp + prev) / 2.0 / kFs, pv = kFs / (prev - pp);
      }
      resolve(ev, T, t, gi, pl, pv, loc, val);
    }
    __syncthreads();
    if (threadIdx.x < 4) {
      KindCarry& cr = carry[threadIdx.x];
      const double* cl = cross[threadIdx.x];
      for (int q = 0; q < cnt[threadIdx.x]; ++q) {  // in order: at most kTile / 2 + 1 steps
        if (cr.has_c) {
          cr.loc0 = cr.loc1, cr.v0 = cr.v1;
          cr.loc1 = (cr.c + cl[q]) / 2.0 / kFs, cr.v1 = kFs / (cl[q] - cr.c);
          ++cr.nint;
        }
        cr.c = cl[q], cr.has_c = 1;
      }
      if (threadIdx.x < 2) fs[threadIdx.x] = fs[m + threadIdx.x];  // f[i0 + m - 2], f[i0 + m - 1]
    }
    __syncthreads();
  }
  // frames at or after the last interval: the last two intervals, extended
  for (int t = 0; t < 4; ++t) {
    const KindCarry cr = carry[t];
    if (cr.nint < 2) continue;
    int f = max(0, (int)ceil(cr.loc1 * 1000.0) - 1);
    while (f < T && f / 1000.0 < cr.loc1) ++f;
    for (f += threadIdx.x; f < T; f += blockDim.x) {
      const double s = (f / 1000.0 - cr.loc0) / (cr.loc1 - cr.loc0);
      ev[(size_t)f * (kNch * 4) + t] = cr.v0 + s * (cr.v1 - cr.v0);
    }
  }
  if (threadIdx.x < 4) p.icount[((size_t)blockIdx.y * kNch + ch) * 4 + threadIdx.x] = carry[threadIdx.x].nint;
}

// ------------------------------------------------------------------------------------------------ official candidates
__global__ void __launch_bounds__(128) f0_official_kernel(const F0Params p) {
  __shared__ int ok[kNch];
  const F0Clip u = p.clips[blockIdx.y];
  for (int c = threadIdx.x; c < kNch; c += blockDim.x) {
    const int32_t* ic = p.icount + ((size_t)blockIdx.y * kNch + c) * 4;
    ok[c] = ic[0] >= 3 && ic[1] >= 3 && ic[2] >= 3 && ic[3] >= 3;
  }
  __syncthreads();
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= u.T) return;
  const double* e = p.ev + (size_t)(u.f + f) * (kNch * 4);
  double* own = p.own + (size_t)(u.f + f) * kMaxOwn;
  int nraw = 0, k = 0, st = -1;
  double acc = 0.0;
  for (int c = 0; c < kNch; ++c) {
    double r = 0.0;
    if (ok[c]) {
      const double avg = (((e[4 * c] + e[4 * c + 1]) + e[4 * c + 2]) + e[4 * c + 3]) / 4.0;
      const double bf = p.bf[c];
      r = (avg > bf * 1.1 || avg < bf / 1.1 || avg > kCeil || avg < kFloor) ? 0.0 : avg;
    }
    nraw += r > 0.0;
    const bool v = r > 0.0 && c != 0 && c != kNch - 1;
    if (v) {
      if (st < 0) st = c, acc = 0.0;
      acc += r;
    } else if (st >= 0) {
      if (c - st >= 10 && k < kMaxOwn) own[k++] = acc / (c - st);
      st = -1;
    }
  }
  for (int j = k; j < kMaxOwn; ++j) own[j] = 0.0;
  p.ocount[u.f + f] = k;
  p.rcount[u.f + f] = nraw;
  atomicMax(p.nc + blockIdx.y, k);
}

// --------------------------------------------------------------------------------------------------------- refinement
__global__ void __launch_bounds__(128) f0_refine_kernel(const F0Params p) {
  const F0Clip u = p.clips[blockIdx.y];
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int f = (int)(idx / kSlots), s = (int)(idx % kSlots);
  if (f >= u.T) return;
  const int nc = p.nc[blockIdx.y];
  const size_t o = (size_t)(u.f + f) * kSlots + s;
  double f0 = 0.0;
  if (s < 7 * nc) {
    const int b = s / nc, j = s % nc;
    const int src = b == 0 ? f : b <= 3 ? f - b : f + (b - 3);
    if (src >= 0 && src < u.T) f0 = p.own[(size_t)(u.f + src) * kMaxOwn + j];
  }
  if (!(f0 > 0.0)) {
    p.rf[o] = 0.0, p.rs[o] = 0.0;
    return;
  }
  const double* __restrict__ y = p.y + u.y;
  const int hw = (int)(1.5 * kFs / f0 + 1.0);
  const int nw = 2 * hw + 1;
  const double wl = (2.0 * hw + 1.0) / kFs;
  const int N = 1 << (2 + (31 - __clz(nw)));
  const int stride = kTwN / N;
  const double pos = f / 1000.0;
  const int basic = mround((pos + (double)(-hw) / kFs) * kFs + 0.001);
  const int nh = min((int)(kFs / 2.0 / f0), 6);
  int m[6];
  double mr[6], mi[6], dr[6], di[6];
#pragma unroll
  for (int k = 0; k < 6; ++k) {
    m[k] = mround(f0 * N / kFs * (k + 1.0));
    mr[k] = mi[k] = dr[k] = di[k] = 0.0;
  }
  auto win = [&](int j) {
    const double tmp = (basic + j - 1.0) / kFs - pos;
    return 0.42 + 0.5 * cos(2.0 * kPi * tmp / wl) + 0.08 * cos(4.0 * kPi * tmp / wl);
  };
  double wp = 0.0, wc = win(0), wn = win(1);
  for (int j = 0; j < nw; ++j) {
    const double dw = j == 0 ? -wn / 2.0 : j == nw - 1 ? wp / 2.0 : -(wn - wp) / 2.0;
    const double xs = y[min(max(basic + j - 1, 0), u.n - 1)];
    const double xw = xs * wc, xd = xs * dw;
#pragma unroll
    for (int k = 0; k < 6; ++k) {
      const int q = (int)(((int64_t)j * m[k]) % N) * stride;
      const double c = p.twc[q], sn = p.tws[q];
      mr[k] = mr[k] + xw * c;
      mi[k] = mi[k] - xw * sn;
      dr[k] = dr[k] + xd * c;
      di[k] = di[k] - xd * sn;
    }
    wp = wc, wc = wn;
    wn = j + 2 < nw ? win(j + 2) : 0.0;
  }
  double num = 0.0, den = 0.0, sc = 0.0;
#pragma unroll
  for (int k = 0; k < 6; ++k) {
    if (k >= nh) continue;
    const double ni = mr[k] * di[k] - mi[k] * dr[k];
    const double pw = mr[k] * mr[k] + mi[k] * mi[k];
    const double inst = pw == 0.0 ? 0.0 : m[k] * kFs / N + ni / pw * kFs / 2.0 / kPi;
    const double amp = sqrt(pw);
    num = num + amp * inst;
    den = den + amp * (k + 1.0);
    sc = sc + fabs((inst / (k + 1.0) - f0) / f0);
  }
  const double rf = num / (den + 1e-12);
  const double rs = 1.0 / (sc / nh + 1e-12);
  const bool bad = rf < kFloor || rf > kCeil || rs < 2.5;
  p.rf[o] = bad ? 0.0 : rf;
  p.rs[o] = bad ? 0.0 : rs;
}

// ----------------------------------------------------------------------------------------------------- fixing, smoothing
__device__ __forceinline__ double select_best(double ref, const double* c, int S, double allowed) {
  double best_f0 = 0.0, best = allowed;
  for (int i = 0; i < S; ++i) {
    const double t = fabs(ref - c[i]) / ref;
    if (t > best) continue;
    best_f0 = c[i], best = t;
  }
  return best_f0;
}

__device__ __forceinline__ double search_score(double f0, const double* c, const double* s, int S) {
  double r = 0.0;
  for (int i = 0; i < S; ++i)
    if (f0 == c[i] && r < s[i]) r = s[i];
  return r;
}

// (start, end) of every run of nonzero frames into sec[k * 4 + 0 / 1]; with `forced`, frames 0 and T - 1 count as zero
__device__ __forceinline__ int list_runs(const double* f, int T, bool forced, int32_t* sec) {
  int k = 0, st = -1;
  for (int i = 0; i <= T; ++i) {
    const bool v = i < T && f[i] > 0 && !(forced && (i == 0 || i == T - 1));
    if (v && st < 0) st = i;
    if (!v && st >= 0) {
      sec[4 * k] = st, sec[4 * k + 1] = i - 1;
      ++k, st = -1;
    }
  }
  return k;
}

// run k's channel after the extensions: s2 inside the run, the extension values within kExt frames of it, 0 elsewhere
__device__ __forceinline__ double chan(const double* s2, const int32_t* sec, const double* ext, int k, int j) {
  const int st = sec[4 * k], ed = sec[4 * k + 1];
  if (j >= st && j <= ed) return s2[j];
  if (j > ed && j - ed - 1 < kExt) return ext[(size_t)k * 2 * kExt + (j - ed - 1)];
  if (j < st && st - 1 - j < kExt) return ext[(size_t)k * 2 * kExt + kExt + (st - 1 - j)];
  return 0.0;
}

__global__ void __launch_bounds__(kFixThreads) f0_fix_kernel(const F0Params p) {
  __shared__ int nsec_s, nkeep_s;
  const F0Clip u = p.clips[blockIdx.x];
  const int T = u.T, S = 7 * p.nc[blockIdx.x];
  const size_t F = u.f;
  const double* rf = p.rf + F * kSlots;
  const double* rs = p.rs + F * kSlots;
  double* cf = p.cf + F * kSlots;
  double* cs = p.cs + F * kSlots;
  double *base = p.base + F, *s1 = p.s1 + F, *s2 = p.s2 + F, *s3 = p.s3 + F, *s4 = p.s4 + F, *sm = p.sm + F;
  int32_t* sec = p.sec + u.sec * 4;
  int32_t* ord = p.ord + u.sec;
  double* ext = p.ext + u.sec * 2 * kExt;
  // 6. unreliable candidates, against the slots before the removal
  for (int64_t it = threadIdx.x; it < (int64_t)T * kSlots; it += blockDim.x) {
    const int i = (int)(it / kSlots), j = (int)(it % kSlots);
    double v = rf[it], sc = rs[it];
    if (j < S && i > 0 && i < T - 1 && v != 0.0) {
      double e1 = 1.0, e2 = 1.0;
      for (int k = 0; k < S; ++k) {
        e1 = fmin(e1, fabs(v - rf[(int64_t)(i + 1) * kSlots + k]) / v);
        e2 = fmin(e2, fabs(v - rf[(int64_t)(i - 1) * kSlots + k]) / v);
      }
      if (e1 > 0.05 && e2 > 0.05) v = 0.0, sc = 0.0;
    }
    cf[it] = v, cs[it] = sc;
  }
  __syncthreads();
  // 7. base contour, FixStep1, FixStep2
  for (int i = threadIdx.x; i < T; i += blockDim.x) {
    double b = 0.0, bs = 0.0;
    for (int j = 0; j < S; ++j)
      if (cs[(int64_t)i * kSlots + j] > bs) b = cf[(int64_t)i * kSlots + j], bs = cs[(int64_t)i * kSlots + j];
    base[i] = b;
  }
  __syncthreads();
  for (int i = threadIdx.x; i < T; i += blockDim.x) {
    double o = 0.0;
    if (i >= 2 && base[i] != 0.0) {
      const double r = base[i - 1] * 2 - base[i - 2];
      o = (fabs((base[i] - r) / r) > 0.008 && fabs(base[i] - base[i - 1]) / base[i - 1] > 0.008) ? 0.0 : base[i];
    }
    s1[i] = o;
  }
  __syncthreads();
  for (int i = threadIdx.x; i < T; i += blockDim.x) {
    double o = s1[i];
    if (i >= 2 && i < T - 2)
      for (int j = -2; j <= 2; ++j)
        if (s1[i + j] == 0) o = 0.0;
    s2[i] = o;
  }
  __syncthreads();
  // FixStep3: runs of s2, each extended both ways through the candidates within 18 %
  if (threadIdx.x == 0) nsec_s = list_runs(s2, T, true, sec);
  __syncthreads();
  const int nsec = nsec_s;
  for (int k = threadIdx.x; k < nsec; k += blockDim.x) {
    const int st = sec[4 * k], ed = sec[4 * k + 1];
    double* fwd = ext + (size_t)k * 2 * kExt;
    double* bwd = fwd + kExt;
    for (int i = 0; i < 2 * kExt; ++i) fwd[i] = 0.0;
    int last = min(T - 2, ed + 100), org = ed, cnt = 0;
    double tmp = s2[ed];
    for (int i = 0; i <= last - ed; ++i) {
      const int j = ed + i + 1;
      const double v = select_best(tmp, cf + (int64_t)j * kSlots, S, 0.18);
      fwd[i] = v;
      if (v == 0.0) ++cnt;
      else tmp = v, cnt = 0, org = j;
      if (cnt == 4) break;
    }
    sec[4 * k + 3] = org;
    last = max(1, st - 100), org = st, cnt = 0;
    tmp = s2[st];
    for (int i = 0; i <= st - last; ++i) {
      const int j = st - i - 1;
      const double v = select_best(tmp, cf + (int64_t)j * kSlots, S, 0.18);
      bwd[i] = v;
      if (v == 0.0) ++cnt;
      else tmp = v, cnt = 0, org = j;
      if (cnt == 4) break;
    }
    sec[4 * k + 2] = org;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    // ExtendSub: the running mean carries over from run to run; a run is kept when 2200 / mean < its length
    double mean = 0.0;
    int nk = 0;
    for (int k = 0; k < nsec; ++k) {
      const int st = sec[4 * k + 2], ed = sec[4 * k + 3];
      for (int j = st; j < ed; ++j) mean += chan(s2, sec, ext, k, j);
      mean /= (double)(ed - st);
      if (2200.0 / mean < ed - st) ord[nk++] = k;
    }
    for (int a = 1; a < nk; ++a) {  // stable insertion sort by extended start
      const int v = ord[a];
      int b = a - 1;
      while (b >= 0 && sec[4 * ord[b] + 2] > sec[4 * v + 2]) ord[b + 1] = ord[b], --b;
      ord[b + 1] = v;
    }
    nkeep_s = nk;
  }
  __syncthreads();
  const int nk = nkeep_s;
  for (int i = threadIdx.x; i < T; i += blockDim.x) s3[i] = nk == 0 ? s2[i] : chan(s2, sec, ext, ord[0], i);
  __syncthreads();
  if (threadIdx.x == 0 && nk > 1) {
    int cst = sec[4 * ord[0] + 2], ced = sec[4 * ord[0] + 3];
    for (int a = 1; a < nk; ++a) {
      const int k = ord[a], st2 = sec[4 * k + 2], ed2 = sec[4 * k + 3];
      if (st2 - ced > 0) {
        for (int j = st2; j <= ed2; ++j) s3[j] = chan(s2, sec, ext, k, j);
        cst = st2, ced = ed2;
      } else if (cst <= st2 && ced >= ed2) {
        continue;
      } else {
        double sc1 = 0.0, sc2 = 0.0;
        for (int i = st2; i <= ced; ++i) {
          sc1 += search_score(s3[i], cf + (int64_t)i * kSlots, cs + (int64_t)i * kSlots, S);
          sc2 += search_score(chan(s2, sec, ext, k, i), cf + (int64_t)i * kSlots, cs + (int64_t)i * kSlots, S);
        }
        for (int j = sc1 > sc2 ? ced : st2; j <= ed2; ++j) s3[j] = chan(s2, sec, ext, k, j);
        ced = ed2;
      }
    }
  }
  __syncthreads();
  // FixStep4: gaps shorter than 9 frames between runs of s3, filled linearly
  for (int i = threadIdx.x; i < T; i += blockDim.x) s4[i] = s3[i];
  if (threadIdx.x == 0) nsec_s = list_runs(s3, T, true, sec);
  __syncthreads();
  for (int k = threadIdx.x; k + 1 < nsec_s; k += blockDim.x) {
    const int e = sec[4 * k + 1], s = sec[4 * (k + 1)];
    if (s - e - 1 >= 9) continue;
    const double a = s3[e], b = s3[s];
    for (int j = e + 1; j < s; ++j) s4[j] = a + (b - a) * (double)(j - e) / (double)(s - e);
  }
  __syncthreads();
  // 8. smoothing of each run of s4 with its edge values held kLag frames on each side
  for (int i = threadIdx.x; i < T; i += blockDim.x) sm[i] = 0.0;
  if (threadIdx.x == 0) nsec_s = list_runs(s4, T, false, sec);
  __syncthreads();
  {
    const double A0 = 1.7347257688092754, A1 = -0.76600660094326412;
    const double B0 = 0.0078202080334971724, B1 = 0.015640416066994345;
    double* tail = p.tail + ((size_t)blockIdx.x * kFixThreads + threadIdx.x) * kLag;
    for (int k = threadIdx.x; k < nsec_s; k += blockDim.x) {
      const int st = sec[4 * k], ed = sec[4 * k + 1];
      double w0 = 0.0, w1 = 0.0;
      for (int j = st - kLag; j <= ed + kLag; ++j) {
        const double x = s4[min(max(j, st), ed)];
        const double wt = x + A0 * w0 + A1 * w1;
        const double o = B0 * wt + B1 * w0 + B0 * w1;
        w1 = w0, w0 = wt;
        if (j > ed) tail[j - ed - 1] = o;
        else if (j >= st) sm[j] = o;
      }
      w0 = w1 = 0.0;
      for (int j = ed + kLag; j >= st; --j) {
        const double x = j > ed ? tail[j - ed - 1] : sm[j];
        const double wt = x + A0 * w0 + A1 * w1;
        const double o = B0 * wt + B1 * w0 + B0 * w1;
        w1 = w0, w0 = wt;
        if (j <= ed) sm[j] = o;
      }
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < u.n_out; i += blockDim.x) p.f0[u.out + i] = sm[min(T - 1, 10 * i)];
}

int64_t frames_1ms(int32_t L) { return (int64_t)(1000.0 * L / 16000 / 1.0) + 1; }
int64_t frames_out(int32_t L) { return (int64_t)(1000.0 * L / 16000 / 10.0) + 1; }

struct Layout {
  size_t clips, y, p1, p2, ev, icount, own, ocount, rcount, nc, rf, rs, cf, cs, base, s1, s2, s3, s4, sm, sec, ord, ext, tail;
  size_t total;
  int64_t Y, P, F, R, O;
  int Tmax;
};

Layout layout(int32_t batch, const int32_t* lengths) {
  Layout l{};
  for (int b = 0; b < batch; ++b) {
    const int64_t T = frames_1ms(lengths[b]);
    l.Y += 1 + lengths[b] / 2;
    l.P += lengths[b] + 2 * kNFact;
    l.F += T;
    l.R += T / 2 + 2;
    l.O += frames_out(lengths[b]);
    l.Tmax = (int)std::max<int64_t>(l.Tmax, T);
  }
  WsLayout ws;
  l.clips = ws.take(sizeof(F0Clip) * (size_t)batch);
  l.y = ws.take<double>(l.Y) * 8;
  l.p1 = ws.take<double>(l.P) * 8;
  l.p2 = ws.take<double>(l.P) * 8;
  l.ev = ws.take<double>((size_t)l.F * kNch * 4) * 8;
  l.icount = ws.take<int32_t>((size_t)batch * kNch * 4) * 4;
  l.own = ws.take<double>((size_t)l.F * kMaxOwn) * 8;
  l.ocount = ws.take<int32_t>(l.F) * 4;
  l.rcount = ws.take<int32_t>(l.F) * 4;
  l.nc = ws.take<int32_t>(batch) * 4;
  l.rf = ws.take<double>((size_t)l.F * kSlots) * 8;
  l.rs = ws.take<double>((size_t)l.F * kSlots) * 8;
  l.cf = ws.take<double>((size_t)l.F * kSlots) * 8;
  l.cs = ws.take<double>((size_t)l.F * kSlots) * 8;
  l.base = ws.take<double>(l.F) * 8;
  l.s1 = ws.take<double>(l.F) * 8;
  l.s2 = ws.take<double>(l.F) * 8;
  l.s3 = ws.take<double>(l.F) * 8;
  l.s4 = ws.take<double>(l.F) * 8;
  l.sm = ws.take<double>(l.F) * 8;
  l.sec = ws.take<int32_t>((size_t)l.R * 4) * 4;
  l.ord = ws.take<int32_t>(l.R) * 4;
  l.ext = ws.take<double>((size_t)l.R * 2 * kExt) * 8;
  l.tail = ws.take<double>((size_t)batch * kFixThreads * kLag) * 8;
  l.total = ws.total();
  return l;
}

constexpr int32_t kMaxLength = 1 << 28;  // samples per clip: 4.6 hours at 16 kHz

int check_lengths(const char* fn, int32_t batch, const int32_t* lengths) {
  if (batch <= 0) return fail(MB_ERR_INVALID, "%s: batch = %d", fn, batch);
  for (int b = 0; b < batch; ++b)
    if (lengths[b] <= 0 || lengths[b] > kMaxLength)
      return fail(MB_ERR_INVALID, "%s: clip %d has %d samples; 1 .. %d are supported", fn, b, (int)lengths[b], kMaxLength);
  return MB_OK;
}

}  // namespace

struct mb_f0 {
  WeightTable w;
  std::vector<double> table;  // bf [128], L [128], first tap [128], taps, twiddle cos [1024], sin [1024]
  size_t taps_off = 0, tw_off = 0;
  bool finalized = false;
};

extern "C" {

int mb_f0_create(mb_f0** out) {
  if (!out) return fail(MB_ERR_INVALID, "mb_f0_create: null argument");
  mb_f0* h = new mb_f0();
  std::vector<double> bf(kNch), Ls(kNch), offs(kNch), taps;
  for (int c = 0; c < kNch; ++c) {
    bf[c] = 80.0 * 0.9 * std::pow(2.0, (c + 1) / 40.0);
    const double v = kFs / bf[c] * 2.0;
    const int L = (int)(v + 0.5);
    if (L > kMaxL) {  // the bank kernel's shared-memory tile is sized for kMaxL
      delete h;
      return fail(MB_ERR_INVALID, "mb_f0_create: channel %d needs %d taps per side, more than %d", c, L, kMaxL);
    }
    Ls[c] = L;
    offs[c] = (double)taps.size();
    const int n = 2 * L + 1;
    for (int k = 0; k < n; ++k) {
      const double t = k / (n - 1.0);
      const double w = 0.355768 - 0.487396 * std::cos(2.0 * kPi * t) + 0.144232 * std::cos(4.0 * kPi * t) -
                       0.012604 * std::cos(6.0 * kPi * t);
      taps.push_back(w * std::cos(2.0 * kPi * bf[c] * (k - L) / kFs));
    }
  }
  h->table.insert(h->table.end(), bf.begin(), bf.end());
  h->table.insert(h->table.end(), Ls.begin(), Ls.end());
  h->table.insert(h->table.end(), offs.begin(), offs.end());
  h->taps_off = h->table.size();
  h->table.insert(h->table.end(), taps.begin(), taps.end());
  h->tw_off = h->table.size();
  for (int q = 0; q < kTwN; ++q) h->table.push_back(std::cos(2.0 * kPi * q / kTwN));
  for (int q = 0; q < kTwN; ++q) h->table.push_back(std::sin(2.0 * kPi * q / kTwN));
  h->w.add_derived("tables", 2 * h->table.size());
  *out = h;
  return MB_OK;
}

void mb_f0_destroy(mb_f0* h) { delete h; }

size_t mb_f0_arena_bytes(const mb_f0* h) { return h ? h->w.floats() * sizeof(float) : 0; }

int mb_f0_set_arena(mb_f0* h, void* arena, size_t bytes) {
  if (int rc = check_arena("mb_f0_set_arena", h, arena, bytes, mb_f0_arena_bytes(h), 256)) return rc;
  h->w.attach((float*)arena);
  h->finalized = false;
  return MB_OK;
}

int mb_f0_finalize(mb_f0* h, void* stream) {
  if (!h || !h->w.ptr("tables")) return fail(MB_ERR_STATE, "mb_f0_finalize: no arena");
  cudaStream_t st = (cudaStream_t)stream;
  MB_CUDA_CHECK(cudaMemcpyAsync(h->w.ptr("tables"), h->table.data(), sizeof(double) * h->table.size(), cudaMemcpyHostToDevice, st));
  MB_CUDA_CHECK(cudaStreamSynchronize(st));  // the source is pageable host memory owned by the handle
  h->finalized = true;
  return MB_OK;
}

size_t mb_f0_workspace_bytes(const mb_f0* h, int32_t batch, const int32_t* lengths_host) {
  if (!h || batch <= 0 || !lengths_host) return 0;
  for (int b = 0; b < batch; ++b)
    if (lengths_host[b] <= 0 || lengths_host[b] > kMaxLength) return 0;
  return layout(batch, lengths_host).total;
}

int mb_f0_harvest(mb_f0* h, const double* x, const int32_t* lengths_host, int32_t batch, double* f0_out,
                  const mb_f0_debug* debug, void* workspace, size_t workspace_bytes, void* stream) {
  if (!h || !x || !lengths_host || !f0_out) return fail(MB_ERR_INVALID, "mb_f0_harvest: null argument");
  if (!h->finalized) return fail(MB_ERR_STATE, "mb_f0_harvest: tables not finalized");
  if (int rc = check_lengths("mb_f0_harvest", batch, lengths_host)) return rc;
  const Layout l = layout(batch, lengths_host);
  char* ws;
  if (int rc = bind("mb_f0_harvest", workspace, workspace_bytes, l.total, &ws)) return rc;
  std::vector<F0Clip> clips(batch);
  int64_t xo = 0, yo = 0, po = 0, fo = 0, ro = 0, oo = 0;
  for (int b = 0; b < batch; ++b) {
    const int32_t L = lengths_host[b];
    const int64_t T = frames_1ms(L);
    clips[b] = F0Clip{xo, yo, po, fo, ro, oo, L, 1 + L / 2, (int32_t)T, (int32_t)frames_out(L)};
    xo += L, yo += 1 + L / 2, po += L + 2 * kNFact, fo += T, ro += T / 2 + 2, oo += frames_out(L);
  }
  cudaStream_t st = (cudaStream_t)stream;
  MB_CUDA_CHECK(cudaMemcpyAsync(ws + l.clips, clips.data(), sizeof(F0Clip) * batch, cudaMemcpyHostToDevice, st));
  MB_CUDA_CHECK(cudaMemsetAsync(ws + l.nc, 0, sizeof(int32_t) * batch, st));
  const double* tab = (const double*)h->w.ptr("tables");
  F0Params p;
  memset(&p, 0, sizeof(p));
  p.clips = (const F0Clip*)(ws + l.clips);
  p.x = x;
  p.bf = tab, p.chL = tab + kNch, p.choff = tab + 2 * kNch;
  p.taps = tab + h->taps_off;
  p.twc = tab + h->tw_off, p.tws = tab + h->tw_off + kTwN;
  p.y = (double*)(ws + l.y), p.p1 = (double*)(ws + l.p1), p.p2 = (double*)(ws + l.p2);
  p.ev = (double*)(ws + l.ev), p.icount = (int32_t*)(ws + l.icount), p.own = (double*)(ws + l.own);
  p.ocount = (int32_t*)(ws + l.ocount), p.rcount = (int32_t*)(ws + l.rcount), p.nc = (int32_t*)(ws + l.nc);
  p.rf = (double*)(ws + l.rf), p.rs = (double*)(ws + l.rs), p.cf = (double*)(ws + l.cf), p.cs = (double*)(ws + l.cs);
  p.base = (double*)(ws + l.base), p.s1 = (double*)(ws + l.s1), p.s2 = (double*)(ws + l.s2), p.s3 = (double*)(ws + l.s3);
  p.s4 = (double*)(ws + l.s4), p.sm = (double*)(ws + l.sm);
  p.sec = (int32_t*)(ws + l.sec), p.ord = (int32_t*)(ws + l.ord), p.ext = (double*)(ws + l.ext), p.tail = (double*)(ws + l.tail);
  p.f0 = f0_out;
  f0_decimate_kernel<<<batch, 256, 0, st>>>(p);
  MB_LAUNCH_CHECK("f0_decimate_kernel");
  f0_bank_kernel<<<dim3(kNch, batch), kBankThreads, 0, st>>>(p);
  MB_LAUNCH_CHECK("f0_bank_kernel");
  f0_official_kernel<<<dim3((l.Tmax + 127) / 128, batch), 128, 0, st>>>(p);
  MB_LAUNCH_CHECK("f0_official_kernel");
  f0_refine_kernel<<<dim3((unsigned)(((int64_t)l.Tmax * kSlots + 127) / 128), batch), 128, 0, st>>>(p);
  MB_LAUNCH_CHECK("f0_refine_kernel");
  f0_fix_kernel<<<batch, kFixThreads, 0, st>>>(p);
  MB_LAUNCH_CHECK("f0_fix_kernel");
  if (debug) {
    const size_t F = (size_t)l.F;
    if (debug->raw_count) MB_CUDA_CHECK(cudaMemcpyAsync(debug->raw_count, p.rcount, 4 * F, cudaMemcpyDeviceToDevice, st));
    if (debug->official_count) MB_CUDA_CHECK(cudaMemcpyAsync(debug->official_count, p.ocount, 4 * F, cudaMemcpyDeviceToDevice, st));
    if (debug->refined) MB_CUDA_CHECK(cudaMemcpyAsync(debug->refined, p.rf, 8 * F * kSlots, cudaMemcpyDeviceToDevice, st));
    if (debug->scores) MB_CUDA_CHECK(cudaMemcpyAsync(debug->scores, p.rs, 8 * F * kSlots, cudaMemcpyDeviceToDevice, st));
    if (debug->contour) MB_CUDA_CHECK(cudaMemcpyAsync(debug->contour, p.s4, 8 * F, cudaMemcpyDeviceToDevice, st));
  }
  return MB_OK;
}

}  // extern "C"
