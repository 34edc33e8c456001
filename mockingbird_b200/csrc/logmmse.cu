// Log-MMSE speech enhancement on H100 (mb_logmmse_*): DESIGN.md section 4j.
//
//   replaces  utils/logmmse.py:36-69 (profile_noise), :72-133 (denoise), as called by
//             models/synthesizer/inference.py:145-159 (load_preprocess_wav)
//
// Everything is float64 until the one rounding of the output to fp32.  B utterances of different lengths run in one
// sequence of four launches whatever B is:
//   lm_frame_kernel    window (x + DBL_EPSILON), n_fft-point FFT, |X_f[k]| for k = 0 .. n_fft / 2 -> sg [F][stride]
//   lm_scan_kernel     one CTA per utterance, one thread per bin (two above 704 bins): the frame recursion of gammak,
//                      ksi, the VAD statistic (one block reduction, which also carries "some xk_prev bin is 0"), the
//                      noise_mu2 update, E1 and the gain hw_f[k], written over |X_f[k]| in sg
//   lm_inverse_kernel  the same forward FFT again (bitwise the one above), times hw_f, inverse FFT -> first W samples
//   lm_ola_kernel      out[f hop + i] = y_{f-1}[hop + i] + y_f[i] rounded once to fp32; zeros past nframes * hop
// and the noise profile is one more kernel (lm_profile_kernel, one CTA per utterance): sum_j |X_j[k]| over the
// non-overlapping frames in frame order, / n_frames, squared.
//
// The FFT kernels take two real frames of ONE utterance as the real and imaginary parts of one complex transform (mb_fft.cuh,
// radix 4 / 2 / 5 over host float64 twiddles), so an utterance's output does not depend on the rest of the batch.  The
// half spectrum stands for the whole: the mirror bins enter the VAD sum with weight 2.
#include <cfloat>
#include <cmath>
#include <cstring>
#include <vector>

#include "mb_common.h"
#include "mb_fft.cuh"

using namespace mb;

namespace {

constexpr int kFftThreads = 128;
constexpr int kScanMaxThreads = 704;  // one bin per thread up to 704 bins (n_fft <= 1280), two above (544 threads at 2048)
constexpr int kPrefetch = 8;          // values of |X| each scan thread holds in registers ahead of use (8 frames of one bin
                                      // or 4 frames of two)

// utils/logmmse.py's constants: aa = mu = 0.98, ksi_min = 10 ** (-25 / 10)
constexpr double kAa = 0.98, kMu = 0.98;
constexpr double kKsiMin = 0x1.9e7c6e43390b7p-9;

struct LmUtt {
  int32_t f0;       // first frame of the utterance in the batch
  int32_t nframes;  // L // hop - W // hop (denoise) or L // W (profile)
  int64_t o;        // first input / output sample
  int32_t L;
  int32_t pad;
};

struct LmParams {
  int n_fft, W, hop, nb, stride;
  double eta;
  const double* window;     // [W]
  const double2* tw;        // [n_fft] exp(-2 pi i m / n_fft)
  const int2* pairs;        // [P] (utterance, first local frame)
  const LmUtt* utt;         // [B]
  const float* x;           // the utterances back to back
  const double* noise_mu2;  // [B][n_fft] (bins 0 .. n_fft / 2 are read)
  double* sg;               // [F][stride] |X_f[k]|, then hw_f[k]
  double* frames;           // [F][W]
  double* vad;              // [F] or null
  double* mu2_out;          // [B][n_fft] (profile)
  float* out;
};

// E1(x) for x > 0.  x <= 1: the power series -gamma - ln x + sum_{k=1..19} (-1)^(k+1) x^k / (k k!) by Horner's rule (the
// 20th term is below 2^-60), Euler's constant as a double-double.  x > 1: the continued fraction
// e^-x / (x + 1 - 1^2 / (x + 3 - 2^2 / (x + 5 - ...))) evaluated backwards from depth 120 / x + 12, which converges to
// double precision on (1, 60] and, unlike the forward (Lentz) product, does not accumulate one rounding per term.  Within 5
// ulp of E1 computed to 40 digits over [1e-8, 60].
__device__ double lm_exp1(double x) {
  if (x <= 1.0) {
    constexpr double c[19] = {
      1.0, 0.25, 0.05555555555555555, 0.010416666666666666, 0.0016666666666666668, 0.0002314814814814815,
      2.834467120181406e-05, 3.1001984126984127e-06, 3.0619243582206544e-07, 2.755731922398589e-08,
      2.27746439867652e-09, 1.7397297489890083e-10, 1.2353110643708935e-11, 8.193389712664089e-13,
      5.0981091545465446e-14, 2.9871733327421158e-15, 1.6537983849091297e-16, 8.677337204770125e-18,
      4.326650129802279e-19};
    double p = c[18];
#pragma unroll
    for (int k = 17; k >= 0; --k) p = c[k] - x * p;
    return ((x * p - 0.57721566490153286061) + 4.942915152430645e-18) - log(x);  // gamma = 0.577... - 4.94e-18
  }
  const int n = (int)(120.0 / x) + 12;
  double t = 0.0;
  for (int i = n; i > 0; --i) t = ((double)i * i) / (x + (2.0 * i + 1.0) - t);
  return exp(-x) / (x + 1.0 - t);
}

// window * (x + DBL_EPSILON) of the frames starting at samples s0 and s1 (s1 < 0: a zero frame), zero-padded to n_fft, as
// the real and imaginary parts of a[0 .. n_fft)
__device__ __forceinline__ void load_pair(const LmParams& p, const float* __restrict__ x, int64_t s0, int64_t s1, double2* a) {
  for (int j = threadIdx.x; j < p.n_fft; j += blockDim.x) {
    double va = 0.0, vb = 0.0;
    if (j < p.W) {
      const double w = p.window[j];
      va = w * ((double)x[s0 + j] + DBL_EPSILON);
      if (s1 >= 0) vb = w * ((double)x[s1 + j] + DBL_EPSILON);
    }
    a[j] = make_double2(va, vb);
  }
}

// the spectra of the real and imaginary input of Z at bin k: (Z[k] + conj Z[N-k]) / 2, (Z[k] - conj Z[N-k]) / 2i
__device__ __forceinline__ void untangle(const double2* Z, int k, int N, double2& A, double2& B) {
  const double2 zk = Z[k], zn = Z[k == 0 ? 0 : N - k];
  A = make_double2(0.5 * (zk.x + zn.x), 0.5 * (zk.y - zn.y));
  B = make_double2(0.5 * (zk.y + zn.y), -0.5 * (zk.x - zn.x));
}

__global__ void __launch_bounds__(kFftThreads) lm_frame_kernel(const LmParams p) {
  extern __shared__ double2 sm[];
  const int2 pr = p.pairs[blockIdx.x];
  const LmUtt u = p.utt[pr.x];
  const int t0 = pr.y;
  if (t0 >= u.nframes) return;  // the placeholder pair of an utterance without frames (it only zeroes the output)
  const bool two = t0 + 1 < u.nframes;
  load_pair(p, p.x + u.o, (int64_t)t0 * p.hop, two ? (int64_t)(t0 + 1) * p.hop : -1, sm);
  __syncthreads();
  const double2* X = stockham<false>(sm, sm + p.n_fft, p.tw, p.n_fft);
  double* row = p.sg + (size_t)(u.f0 + t0) * p.stride;
  for (int k = threadIdx.x; k < p.nb; k += blockDim.x) {
    double2 A, B;
    untangle(X, k, p.n_fft, A, B);
    row[k] = hypot(A.x, A.y);
    if (two) row[p.stride + k] = hypot(B.x, B.y);
  }
}

// sum over the block of v (fixed order: warp shuffles, then warp 0 over the warp partials) and OR of z; every thread
// gets both
__device__ __forceinline__ double block_sum_or(double v, int z, double* red_s, int* red_z, int& z_out) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  for (int o = 16; o > 0; o >>= 1) {
    v += __shfl_down_sync(0xffffffffu, v, o);
    z |= __shfl_down_sync(0xffffffffu, z, o);
  }
  if (lane == 0) red_s[warp] = v, red_z[warp] = z;
  __syncthreads();
  if (warp == 0) {
    v = lane < nw ? red_s[lane] : 0.0;
    z = lane < nw ? red_z[lane] : 0;
    for (int o = 16; o > 0; o >>= 1) {
      v += __shfl_down_sync(0xffffffffu, v, o);
      z |= __shfl_down_sync(0xffffffffu, z, o);
    }
    if (lane == 0) red_s[32] = v, red_z[32] = z;
  }
  __syncthreads();
  z_out = red_z[32];
  return red_s[32];
}

template <int BPT>
__global__ void __launch_bounds__(BPT == 1 ? kScanMaxThreads : 544) lm_scan_kernel(const LmParams p) {
  constexpr int D = kPrefetch / BPT;  // the same registers for the prefetch whatever BPT is
  __shared__ double red_s[33];
  __shared__ int red_z[33];
  const LmUtt u = p.utt[blockIdx.x];
  const int nf = u.nframes;
  double* rows = p.sg + (size_t)u.f0 * p.stride;
  const double* mu2_in = p.noise_mu2 + (size_t)blockIdx.x * p.n_fft;
  int kk[BPT];
  bool live[BPT];
  double nm[BPT], xk[BPT], wgt[BPT], pre[BPT][D];
#pragma unroll
  for (int i = 0; i < BPT; ++i) {
    kk[i] = threadIdx.x + i * blockDim.x;
    live[i] = kk[i] < p.nb;
    nm[i] = live[i] ? mu2_in[kk[i]] : 1.0;
    xk[i] = 0.0;
    wgt[i] = (kk[i] == 0 || 2 * kk[i] == p.n_fft) ? 1.0 : 2.0;  // bins 1 .. n_fft / 2 - 1 stand for their mirrors too
#pragma unroll
    for (int d = 0; d < D; ++d) pre[i][d] = live[i] && d < nf ? rows[(size_t)d * p.stride + kk[i]] : 0.0;
  }
  bool prior = true;  // xk_prev starts as zeros: the first frame takes the prior branch
  for (int f0 = 0; f0 < nf; f0 += D) {
#pragma unroll
    for (int d = 0; d < D; ++d) {
      const int f = f0 + d;
      if (f >= nf) break;  // uniform across the block
      double ls = 0.0, s2[BPT], xn[BPT];
      int zero = 0;
#pragma unroll
      for (int i = 0; i < BPT; ++i) {
        const double s = pre[i][d];
        const int nx = f + D;
        pre[i][d] = live[i] && nx < nf ? rows[(size_t)nx * p.stride + kk[i]] : 0.0;
        s2[i] = s * s;
        const double g = fmin(s2[i] / nm[i], 40.0);
        const double gm1 = fmax(g - 1.0, 0.0);
        const double ksi = prior ? kAa + (1.0 - kAa) * gm1 : fmax(kKsiMin, kAa * xk[i] / nm[i] + (1.0 - kAa) * gm1);
        const double a = ksi / (1.0 + ksi);
        const double lsk = g * ksi / (1.0 + ksi) - log(1.0 + ksi);
        const double hw = a * exp(0.5 * lm_exp1(fmax(a * g, 1e-8)));
        const double sh = s * hw;
        xn[i] = sh * sh;
        if (live[i]) {
          ls += wgt[i] * lsk;
          zero |= xn[i] == 0.0;
          rows[(size_t)f * p.stride + kk[i]] = hw;
        }
      }
      int any_zero;
      const double vad = block_sum_or(ls, zero, red_s, red_z, any_zero) / p.W;
      if (p.vad && threadIdx.x == 0) p.vad[u.f0 + f] = vad;
      const bool update = vad < p.eta;
#pragma unroll
      for (int i = 0; i < BPT; ++i) {
        if (update) nm[i] = kMu * nm[i] + (1.0 - kMu) * s2[i];
        xk[i] = xn[i];
      }
      prior = any_zero != 0;
    }
  }
}

__global__ void __launch_bounds__(kFftThreads) lm_inverse_kernel(const LmParams p) {
  extern __shared__ double2 sm[];
  const int N = p.n_fft;
  const int2 pr = p.pairs[blockIdx.x];
  const LmUtt u = p.utt[pr.x];
  const int t0 = pr.y;
  if (t0 >= u.nframes) return;
  const bool two = t0 + 1 < u.nframes;
  double2* a = sm;
  double2* b = sm + N;
  load_pair(p, p.x + u.o, (int64_t)t0 * p.hop, two ? (int64_t)(t0 + 1) * p.hop : -1, a);
  __syncthreads();
  const double2* X = stockham<false>(a, b, p.tw, N);
  double2* C = X == a ? b : a;
  const double* ha = p.sg + (size_t)(u.f0 + t0) * p.stride;
  for (int k = threadIdx.x; k < p.nb; k += blockDim.x) {
    double2 A, B;
    untangle(X, k, N, A, B);
    const double hb = two ? ha[p.stride + k] : 0.0;
    const double2 ya = cscale(A, ha[k]), yb = cscale(B, hb);
    C[k] = make_double2(ya.x - yb.y, ya.y + yb.x);  // Ya + i Yb
    if (k != 0 && 2 * k != N) C[N - k] = make_double2(ya.x + yb.y, yb.x - ya.y);  // conj(Ya) + i conj(Yb)
  }
  __syncthreads();
  const double2* z = stockham<true>(C, C == a ? b : a, p.tw, N);
  const double inv_n = 1.0 / N;
  double* fa = p.frames + (size_t)(u.f0 + t0) * p.W;
  for (int j = threadIdx.x; j < p.W; j += blockDim.x) {
    fa[j] = z[j].x * inv_n;
    if (two) fa[p.W + j] = z[j].y * inv_n;
  }
}

// output hop blocks t0, t0 + 1 of a pair; the last pair of an utterance also zeroes the samples past nframes * hop
__global__ void __launch_bounds__(256) lm_ola_kernel(const LmParams p) {
  const int H = p.hop;
  const int2 pr = p.pairs[blockIdx.x];
  const LmUtt u = p.utt[pr.x];
  const int t0 = pr.y;
  const double* fr = p.frames + (size_t)u.f0 * p.W;
  float* out = p.out + u.o;
  for (int i = threadIdx.x; i < 2 * H; i += blockDim.x) {
    const int f = t0 + i / H, j = i - (i / H) * H;
    if (f >= u.nframes) break;
    const double tail = f > 0 ? fr[(size_t)(f - 1) * p.W + H + j] : 0.0;
    out[(int64_t)f * H + j] = (float)(tail + fr[(size_t)f * p.W + j]);
  }
  if (t0 + 2 >= u.nframes)
    for (int64_t n = (int64_t)u.nframes * H + threadIdx.x; n < u.L; n += blockDim.x) out[n] = 0.f;
}

// noise_mu2 of one utterance: (sum_j |X_j[k]| / n_frames)^2 over the frames x[j W .. (j + 1) W), summed in frame order
__global__ void __launch_bounds__(kFftThreads) lm_profile_kernel(const LmParams p) {
  extern __shared__ double2 sm[];
  const int N = p.n_fft;
  double* acc = (double*)(sm + 2 * N);  // [nb]
  const LmUtt u = p.utt[blockIdx.x];
  for (int k = threadIdx.x; k < p.nb; k += blockDim.x) acc[k] = 0.0;
  for (int t0 = 0; t0 < u.nframes; t0 += 2) {
    const bool two = t0 + 1 < u.nframes;
    __syncthreads();  // the previous pair's spectrum has been read
    load_pair(p, p.x + u.o, (int64_t)t0 * p.W, two ? (int64_t)(t0 + 1) * p.W : -1, sm);
    __syncthreads();
    const double2* X = stockham<false>(sm, sm + N, p.tw, N);
    for (int k = threadIdx.x; k < p.nb; k += blockDim.x) {
      double2 A, B;
      untangle(X, k, N, A, B);
      double s = acc[k] + hypot(A.x, A.y);
      if (two) s += hypot(B.x, B.y);
      acc[k] = s;
    }
  }
  double* mu2 = p.mu2_out + (size_t)blockIdx.x * N;
  for (int k = threadIdx.x; k < p.nb; k += blockDim.x) {
    const double m = acc[k] / u.nframes;
    mu2[k] = m * m;
    if (k != 0 && 2 * k != N) mu2[N - k] = m * m;
  }
}

__global__ void lm_exp1_kernel(const double* __restrict__ x, double* __restrict__ y, int64_t n) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) y[i] = lm_exp1(x[i]);
}

struct Layout {
  size_t pairs, utt, sg, frames, total;
  int64_t n_pairs, F;
};

Layout layout(const mb_logmmse_config& c, int stride, int32_t batch, const int32_t* lengths) {
  Layout l{};
  for (int b = 0; b < batch; ++b) {
    const int64_t nf = lengths[b] / c.len2 - c.window_size / c.len2;
    l.n_pairs += nf > 0 ? (nf + 1) / 2 : 1;
    l.F += nf > 0 ? nf : 0;
  }
  WsLayout ws;  // byte offsets
  l.pairs = ws.take(sizeof(int2) * (size_t)l.n_pairs);
  l.utt = ws.take(sizeof(LmUtt) * (size_t)batch);
  l.sg = ws.take(sizeof(double) * (size_t)l.F * stride);
  l.frames = ws.take(sizeof(double) * (size_t)l.F * c.window_size);
  l.total = ws.total();
  return l;
}

}  // namespace

struct mb_logmmse {
  mb_logmmse_config cfg{};
  int nb = 0, stride = 0;
  WeightTable w;
  std::vector<double> tw;  // [n_fft][2], written into the arena at finalize
  bool finalized = false;
};

extern "C" {

int mb_logmmse_create(const mb_logmmse_config* cfg, mb_logmmse** out) {
  if (!cfg || !out) return fail(MB_ERR_INVALID, "mb_logmmse_create: null argument");
  const mb_logmmse_config& c = *cfg;
  const int N = c.n_fft;
  if (!fft_supported(N))
    return fail(MB_ERR_INVALID, "mb_logmmse_create: n_fft = %d is not 2^a or 5 * 2^a in [64, 2048]", N);
  if (c.window_size <= 0 || c.window_size % 2 != 0 || c.window_size > N)
    return fail(MB_ERR_INVALID, "mb_logmmse_create: window_size = %d must be even and in [2, n_fft = %d]", c.window_size, N);
  if (c.len1 != c.window_size / 2 || c.len2 != c.window_size / 2)
    return fail(MB_ERR_INVALID, "mb_logmmse_create: len1 = %d and len2 = %d must both be window_size / 2 = %d", c.len1, c.len2,
                c.window_size / 2);
  mb_logmmse* h = new mb_logmmse();
  h->cfg = c;
  h->nb = N / 2 + 1;
  h->stride = (h->nb + 1) & ~1;  // rows of a multiple of 16 bytes
  h->w.add_derived("twiddles", 4 * (size_t)N);
  h->tw.resize(2 * (size_t)N);
  fft_twiddles(N, h->tw.data());
  *out = h;
  return MB_OK;
}

void mb_logmmse_destroy(mb_logmmse* h) { delete h; }

size_t mb_logmmse_arena_bytes(const mb_logmmse* h) { return h ? h->w.floats() * sizeof(float) : 0; }

int mb_logmmse_set_arena(mb_logmmse* h, void* arena, size_t bytes) {
  if (int rc = check_arena("mb_logmmse_set_arena", h, arena, bytes, mb_logmmse_arena_bytes(h), 256)) return rc;
  h->w.attach((float*)arena);
  h->finalized = false;
  return MB_OK;
}

int mb_logmmse_finalize(mb_logmmse* h, void* stream) {
  if (!h || !h->w.ptr("twiddles") || mb_logmmse_arena_bytes(h) == 0) return fail(MB_ERR_STATE, "mb_logmmse_finalize: no arena");
  cudaStream_t st = (cudaStream_t)stream;
  MB_CUDA_CHECK(cudaMemcpyAsync(h->w.ptr("twiddles"), h->tw.data(), sizeof(double) * h->tw.size(), cudaMemcpyHostToDevice, st));
  MB_CUDA_CHECK(cudaStreamSynchronize(st));  // the source is pageable host memory owned by the handle
  h->finalized = true;
  return MB_OK;
}

size_t mb_logmmse_workspace_bytes(const mb_logmmse* h, int32_t batch, const int32_t* lengths_host) {
  if (!h || batch <= 0 || !lengths_host) return 0;
  for (int b = 0; b < batch; ++b)
    if (lengths_host[b] < 2 * h->cfg.len2) return 0;
  return layout(h->cfg, h->stride, batch, lengths_host).total;
}

// dynamic shared memory above the 48 KB default (two n_fft-point double2 buffers are 64 KB at n_fft = 2048)
static int allow_smem(const void* kernel, size_t bytes) {
  if (bytes > 48 * 1024) MB_CUDA_CHECK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
  return MB_OK;
}

static int fill_params(mb_logmmse* h, const char* fn, int32_t batch, const double* window, LmParams& p) {
  if (!h->finalized) return fail(MB_ERR_STATE, "%s: twiddles not finalized", fn);
  if (batch <= 0) return fail(MB_ERR_INVALID, "%s: batch = %d", fn, batch);
  memset(&p, 0, sizeof(p));
  p.n_fft = h->cfg.n_fft;
  p.W = h->cfg.window_size;
  p.hop = h->cfg.len2;
  p.nb = h->nb;
  p.stride = h->stride;
  p.window = window;
  p.tw = (const double2*)h->w.ptr("twiddles");
  return MB_OK;
}

int mb_logmmse_profile(mb_logmmse* h, const float* noise, const int32_t* lengths_host, int32_t batch, const double* window,
                       double* noise_mu2, void* workspace, size_t workspace_bytes, void* stream) {
  if (!h || !noise || !lengths_host || !window || !noise_mu2) return fail(MB_ERR_INVALID, "mb_logmmse_profile: null argument");
  LmParams p;
  if (int rc = fill_params(h, "mb_logmmse_profile", batch, window, p)) return rc;
  const int W = h->cfg.window_size;
  for (int b = 0; b < batch; ++b)
    if (lengths_host[b] < W)
      return fail(MB_ERR_INVALID, "mb_logmmse_profile: noise %d has %d samples, fewer than window_size = %d", b,
                  (int)lengths_host[b], W);
  // the utterance table at the start of the workspace mb_logmmse_workspace_bytes sizes for these lengths
  char* ws;
  if (int rc = bind("mb_logmmse_profile", workspace, workspace_bytes, mb_logmmse_workspace_bytes(h, batch, lengths_host), &ws))
    return rc;
  std::vector<LmUtt> utt(batch);
  int64_t o = 0;
  for (int b = 0; b < batch; ++b) {
    utt[b] = LmUtt{0, lengths_host[b] / W, o, lengths_host[b], 0};
    o += lengths_host[b];
  }
  cudaStream_t st = (cudaStream_t)stream;
  MB_CUDA_CHECK(cudaMemcpyAsync(ws, utt.data(), sizeof(LmUtt) * utt.size(), cudaMemcpyHostToDevice, st));
  p.utt = (const LmUtt*)ws;
  p.x = noise;
  p.mu2_out = noise_mu2;
  const size_t smem = 2 * sizeof(double2) * p.n_fft + sizeof(double) * p.nb;
  if (int rc = allow_smem((const void*)lm_profile_kernel, smem)) return rc;
  lm_profile_kernel<<<batch, kFftThreads, smem, st>>>(p);
  MB_LAUNCH_CHECK("lm_profile_kernel");
  return MB_OK;
}

int mb_logmmse_denoise(mb_logmmse* h, const float* x, const int32_t* lengths_host, int32_t batch, const double* window,
                       const double* noise_mu2, double eta, float* out, double* vad_out, void* workspace,
                       size_t workspace_bytes, void* stream) {
  if (!h || !x || !lengths_host || !window || !noise_mu2 || !out) return fail(MB_ERR_INVALID, "mb_logmmse_denoise: null argument");
  LmParams p;
  if (int rc = fill_params(h, "mb_logmmse_denoise", batch, window, p)) return rc;
  const mb_logmmse_config& c = h->cfg;
  int64_t F = 0;
  for (int b = 0; b < batch; ++b) {
    if (lengths_host[b] < 2 * c.len2)
      return fail(MB_ERR_INVALID, "mb_logmmse_denoise: utterance %d has %d samples; at least 2 * len2 = %d are needed", b,
                  (int)lengths_host[b], 2 * c.len2);
    F += lengths_host[b] / c.len2 - c.window_size / c.len2;
  }
  if (F > ((int64_t)1 << 28))
    return fail(MB_ERR_INVALID, "mb_logmmse_denoise: %lld frames are too many for one call", (long long)F);
  const Layout l = layout(c, h->stride, batch, lengths_host);
  char* ws;
  if (int rc = bind("mb_logmmse_denoise", workspace, workspace_bytes, l.total, &ws)) return rc;
  // host tables: pair -> (utterance, first local frame), one placeholder pair for an utterance without frames;
  // utterance -> first frame, frame count, first sample, length
  std::vector<char> host(l.sg - l.pairs);
  int2* pairs = (int2*)host.data();
  LmUtt* utt = (LmUtt*)(host.data() + (l.utt - l.pairs));
  int64_t f0 = 0, o = 0, np = 0;
  for (int b = 0; b < batch; ++b) {
    const int nf = lengths_host[b] / c.len2 - c.window_size / c.len2;
    utt[b] = LmUtt{(int32_t)f0, nf, o, lengths_host[b], 0};
    pairs[np++] = make_int2(b, 0);
    for (int t = 2; t < nf; t += 2) pairs[np++] = make_int2(b, t);
    f0 += nf;
    o += lengths_host[b];
  }
  cudaStream_t st = (cudaStream_t)stream;
  MB_CUDA_CHECK(cudaMemcpyAsync(ws + l.pairs, host.data(), host.size(), cudaMemcpyHostToDevice, st));
  p.eta = eta;
  p.pairs = (const int2*)(ws + l.pairs);
  p.utt = (const LmUtt*)(ws + l.utt);
  p.x = x;
  p.noise_mu2 = noise_mu2;
  p.sg = (double*)(ws + l.sg);
  p.frames = (double*)(ws + l.frames);
  p.vad = vad_out;
  p.out = out;
  const unsigned P = (unsigned)l.n_pairs;
  const size_t fsmem = 2 * sizeof(double2) * p.n_fft;
  if (int rc = allow_smem((const void*)lm_frame_kernel, fsmem)) return rc;
  if (int rc = allow_smem((const void*)lm_inverse_kernel, fsmem)) return rc;
  lm_frame_kernel<<<P, kFftThreads, fsmem, st>>>(p);
  MB_LAUNCH_CHECK("lm_frame_kernel");
  if (h->nb <= kScanMaxThreads) lm_scan_kernel<1><<<batch, (h->nb + 31) / 32 * 32, 0, st>>>(p);
  else lm_scan_kernel<2><<<batch, ((h->nb + 1) / 2 + 31) / 32 * 32, 0, st>>>(p);
  MB_LAUNCH_CHECK("lm_scan_kernel");
  lm_inverse_kernel<<<P, kFftThreads, fsmem, st>>>(p);
  MB_LAUNCH_CHECK("lm_inverse_kernel");
  lm_ola_kernel<<<P, 256, 0, st>>>(p);
  MB_LAUNCH_CHECK("lm_ola_kernel");
  return MB_OK;
}

int mb_logmmse_exp1(const double* x, double* y, int64_t n, void* stream) {
  if (!x || !y || n < 0) return fail(MB_ERR_INVALID, "mb_logmmse_exp1: bad argument");
  if (n == 0) return MB_OK;
  lm_exp1_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(x, y, n);
  MB_LAUNCH_CHECK("lm_exp1_kernel");
  return MB_OK;
}

}  // extern "C"
