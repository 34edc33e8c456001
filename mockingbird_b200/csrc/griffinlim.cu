// Griffin-Lim inversion of normalised dB mel spectrograms on H100 (mb_griffinlim_*): DESIGN.md section 4i.
//
//   replaces  models/synthesizer/audio.py:84-99 (inv_mel_spectrogram), :105-124 (_griffin_lim, librosa.stft / istft),
//             :162-166 (_mel_to_linear), :177-206 (_db_to_amp, _denormalize), :25-28 (inv_preemphasis)
//
// B utterances of different lengths run in one sequence of launches whose count depends on n_iters only:
//   gl_mag_kernel         denormalise, 10^(dB/20), max(1e-10, inv_mel_basis @ .) ** power -> S [F][n_bins] (double, one
//                         rounding to fp32 at the end)
//   gl_frame_kernel<0|1>  S * exp(2 pi i u) (uniforms uploaded as float64, or Philox keyed by (seed, bin, frame)) -> inverse
//                         FFT -> windowed frame [F][n_fft]
//   gl_ola_kernel         overlap-add, divided by the window sum-square where it exceeds FLT_MIN, trimmed by n_fft / 2
//   n_iters x { gl_frame_kernel<2>: gather the frame from y (centred, reflect or zero padding), window, forward FFT,
//               S * X / |X| (angle(0) = 0), inverse FFT, window;  gl_ola_kernel }
//   gl_deemph_kernel      lfilter([1], [1, -k], y) in chunks of two hops, each warmed up over the preceding W samples
//
// One CTA per pair of consecutive frames of ONE utterance (local frames 2p, 2p + 1; an odd last frame is paired with
// zeros): the two real frames are the real and imaginary parts of one complex transform.  The pairing depends on the
// utterance alone, so each utterance's output is bitwise what a B = 1 call gives.  The FFT is the shared-memory Stockham of
// mb_fft.cuh (radix 4, radix-2 last stage for odd log2 n_fft) over twiddles computed on the host in float64.
#include <cfloat>
#include <cmath>
#include <cstring>
#include <vector>

#include "../../include/mb_wavernn_math.h"
#include "mb_common.h"
#include "mb_fft.cuh"

using namespace mb;

namespace {

constexpr int kThreads = 256;
constexpr int kMaxWarm = 4096;  // largest inverse pre-emphasis warm-up accepted at create

struct GlUtt {
  int32_t f0;    // first frame of the utterance in the batch (S, frames, mels, uniforms are frame-major by utterance)
  int32_t T;     // frames
  int64_t o;     // first output sample
  uint64_t seed;
};

struct GlParams {
  int n_fft, hop, n_bins, n_mels, pad_mode, warm;
  int signal_normalization, allow_clipping, symmetric;
  double power, preemphasis, max_abs_value, min_level_db, ref_level_db;
  const float* basis;   // [n_bins][n_mels]
  const float* window;  // [n_fft]
  const float2* tw;     // [n_fft] exp(-2 pi i k / n_fft)
  const int2* pairs;    // [P] (utterance, first local frame)
  const GlUtt* utt;     // [B]
  const float* mels;    // per utterance [n_mels][T]
  const double* uniforms;
  float* S;             // [F][n_bins]
  float* frames;        // [F][n_fft]
  float* y;             // [sum hop (T - 1)]
  float* out;
};

// sample i of the centred signal (i in padded coordinates minus n_fft / 2): reflect (numpy "reflect") or zero outside [0, L)
__device__ __forceinline__ float sample_at(const float* __restrict__ y, int L, int i, int pad_mode) {
  if (i < 0) {
    if (pad_mode != 0) return 0.f;
    i = -i;
  } else if (i >= L) {
    if (pad_mode != 0) return 0.f;
    i = 2 * (L - 1) - i;
  }
  return y[i];
}

__device__ __forceinline__ float2 unit(float2 x) {  // X / |X|, and 1 where X = 0 (np.angle(0) = 0)
  const float m = hypotf(x.x, x.y);
  return m > 0.f ? make_float2(x.x / m, x.y / m) : make_float2(1.f, 0.f);
}

// initial phasor exp(2 pi i u) of bin k, local frame t: sincospi in double, rounded once
__device__ __forceinline__ float2 initial_phasor(const GlParams& p, const GlUtt& u, int k, int t, bool seeded) {
  double uu;
  if (seeded) {
    uint32_t o[4];
    mb_philox4x32((uint32_t)k, (uint32_t)t, 0u, 0x676c696du, (uint32_t)u.seed, (uint32_t)(u.seed >> 32), o);
    uu = (double)((((uint64_t)o[0] << 32) | o[1]) >> 11) * 0x1.0p-53;
  } else {
    uu = p.uniforms[(size_t)p.n_bins * u.f0 + (size_t)k * u.T + t];
  }
  double s, c;
  sincospi(2.0 * uu, &s, &c);
  return make_float2((float)c, (float)s);
}

// magnitudes of the frames of one pair: S[k] = max(1e-10, sum_m inv_mel_basis[k][m] 10^((D[m] + ref) / 20)) ** power
__global__ void __launch_bounds__(kThreads) gl_mag_kernel(const GlParams p) {
  extern __shared__ double amp[];  // [2][n_mels]
  const int2 pr = p.pairs[blockIdx.x];
  const GlUtt u = p.utt[pr.x];
  const int nf = pr.y + 1 < u.T ? 2 : 1;
  const float* mel = p.mels + (size_t)p.n_mels * u.f0;
  for (int i = threadIdx.x; i < nf * p.n_mels; i += blockDim.x) {
    const int f = i / p.n_mels, m = i - f * p.n_mels;
    double D = mel[(size_t)m * u.T + pr.y + f];
    if (p.signal_normalization) {  // _denormalize
      const double A = p.max_abs_value, lo = p.min_level_db;
      if (p.symmetric) {
        if (p.allow_clipping) D = fmin(fmax(D, -A), A);
        D = ((D + A) * -lo / (2.0 * A)) + lo;
      } else {
        if (p.allow_clipping) D = fmin(fmax(D, 0.0), A);
        D = (D * -lo / A) + lo;
      }
    }
    amp[i] = pow(10.0, (D + p.ref_level_db) * 0.05);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < nf * p.n_bins; i += blockDim.x) {
    const int f = i / p.n_bins, k = i - f * p.n_bins;
    const float* b = p.basis + (size_t)k * p.n_mels;
    const double* a = amp + f * p.n_mels;
    double s = 0.0;
    for (int m = 0; m < p.n_mels; ++m) s = fma((double)__ldg(b + m), a[m], s);
    p.S[(size_t)(u.f0 + pr.y + f) * p.n_bins + k] = (float)pow(fmax(1e-10, s), p.power);
  }
}

// MODE 0: initial phases from uniforms, 1: from seeds, 2: phases of stft(y)
template <int MODE>
__global__ void __launch_bounds__(kThreads) gl_frame_kernel(const GlParams p) {
  extern __shared__ float2 sm[];
  const int N = p.n_fft, half = N / 2;
  float2* a = sm;
  float2* b = sm + N;
  const int2 pr = p.pairs[blockIdx.x];
  const GlUtt u = p.utt[pr.x];
  const int t0 = pr.y;
  const bool two = t0 + 1 < u.T;
  const float* Sa = p.S + (size_t)(u.f0 + t0) * p.n_bins;
  const float* Sb = Sa + p.n_bins;
  float2* C;  // Hermitian-completed spectrum of frame t0 + i frame t0 + 1, input of the inverse transform
  if (MODE == 2) {
    const int L = p.hop * (u.T - 1);
    const float* y = p.y + u.o;
    for (int j = threadIdx.x; j < N; j += blockDim.x) {
      const float w = p.window[j];
      const float va = sample_at(y, L, t0 * p.hop + j - half, p.pad_mode) * w;
      const float vb = two ? sample_at(y, L, (t0 + 1) * p.hop + j - half, p.pad_mode) * w : 0.f;
      a[j] = make_float2(va, vb);
    }
    __syncthreads();
    const float2* X = stockham<false>(a, b, p.tw, N);
    C = X == a ? b : a;
    for (int k = threadIdx.x; k <= half; k += blockDim.x) {
      const float2 zk = X[k], zn = X[(N - k) & (N - 1)];
      const float2 A = make_float2(0.5f * (zk.x + zn.x), 0.5f * (zk.y - zn.y));    // (Z[k] + conj Z[N-k]) / 2
      const float2 Bv = make_float2(0.5f * (zk.y + zn.y), -0.5f * (zk.x - zn.x));  // (Z[k] - conj Z[N-k]) / 2i
      float2 ca = unit(A), cb = unit(Bv);
      const float sa = Sa[k], sb = two ? Sb[k] : 0.f;
      ca = make_float2(sa * ca.x, sa * ca.y);
      cb = make_float2(sb * cb.x, sb * cb.y);
      if (k == 0 || k == half) ca.y = cb.y = 0.f;  // irfft ignores the imaginary parts of DC and Nyquist
      C[k] = make_float2(ca.x - cb.y, ca.y + cb.x);
      if (k != 0 && k != half) C[N - k] = make_float2(ca.x + cb.y, cb.x - ca.y);
    }
  } else {
    C = a;
    for (int k = threadIdx.x; k <= half; k += blockDim.x) {
      float2 ca = initial_phasor(p, u, k, t0, MODE == 1);
      float2 cb = two ? initial_phasor(p, u, k, t0 + 1, MODE == 1) : make_float2(0.f, 0.f);
      const float sa = Sa[k], sb = two ? Sb[k] : 0.f;
      ca = make_float2(sa * ca.x, sa * ca.y);
      cb = make_float2(sb * cb.x, sb * cb.y);
      if (k == 0 || k == half) ca.y = cb.y = 0.f;
      C[k] = make_float2(ca.x - cb.y, ca.y + cb.x);
      if (k != 0 && k != half) C[N - k] = make_float2(ca.x + cb.y, cb.x - ca.y);
    }
  }
  __syncthreads();
  const float2* z = stockham<true>(C, C == a ? b : a, p.tw, N);
  const float inv_n = 1.0f / (float)N;  // exact
  float* fa = p.frames + (size_t)(u.f0 + t0) * N;
  for (int j = threadIdx.x; j < N; j += blockDim.x) {
    const float w = p.window[j];
    fa[j] = w * (z[j].x * inv_n);
    if (two) fa[N + j] = w * (z[j].y * inv_n);
  }
}

// overlap-add of the hop blocks t0, t0 + 1 of a pair (those below T - 1): output sample n = t hop + i of the utterance is
// padded sample q = n + n_fft / 2, the sum over the frames s with s hop <= q < s hop + n_fft
__global__ void __launch_bounds__(kThreads) gl_ola_kernel(const GlParams p) {
  const int N = p.n_fft, H = p.hop;
  const int2 pr = p.pairs[blockIdx.x];
  const GlUtt u = p.utt[pr.x];
  for (int i = threadIdx.x; i < 2 * H; i += blockDim.x) {
    const int t = pr.y + i / H;
    if (t >= u.T - 1) break;
    const int n = t * H + (i - (i / H) * H), q = n + N / 2;
    const int lo = q - N + 1 <= 0 ? 0 : (q - N + H) / H;
    const int hi = min(q / H, u.T - 1);
    float acc = 0.f, wss = 0.f;
    for (int s = lo; s <= hi; ++s) {
      const int j = q - s * H;
      const float w = p.window[j];
      acc += p.frames[(size_t)(u.f0 + s) * N + j];
      wss = fmaf(w, w, wss);
    }
    p.y[u.o + n] = wss > FLT_MIN ? acc / wss : acc;
  }
}

// out = lfilter([1], [1, -k], y) per utterance: thread = pair, outputs of hop blocks t0, t0 + 1; the recursion restarts W
// samples earlier (or at the utterance start), which changes the result by less than k^W < 2^-30 of the state
__global__ void __launch_bounds__(128) gl_deemph_kernel(const GlParams p, int n_pairs) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_pairs) return;
  const int2 pr = p.pairs[i];
  const GlUtt u = p.utt[pr.x];
  const int L = p.hop * (u.T - 1);
  const int n0 = pr.y * p.hop, n1 = min(n0 + 2 * p.hop, L);
  const float* x = p.y + u.o;
  float* o = p.out + u.o;
  double acc = 0.0;
  for (int n = max(0, n0 - p.warm); n < n0; ++n) acc = fma(p.preemphasis, acc, (double)x[n]);
  for (int n = n0; n < n1; ++n) {
    acc = fma(p.preemphasis, acc, (double)x[n]);
    o[n] = (float)acc;
  }
}

struct Layout {
  size_t pairs, utt, S, frames, y, total;
  int64_t n_pairs, F, samples;
};

Layout layout(int n_fft, int n_bins, int hop, int32_t batch, const int32_t* frames_host) {
  Layout l{};
  for (int b = 0; b < batch; ++b) {
    const int64_t T = frames_host[b] > 0 ? frames_host[b] : 0;
    l.n_pairs += (T + 1) / 2;
    l.F += T;
    l.samples += T > 0 ? (int64_t)hop * (T - 1) : 0;
  }
  WsLayout ws;  // byte offsets
  l.pairs = ws.take(sizeof(int2) * (size_t)l.n_pairs);
  l.utt = ws.take(sizeof(GlUtt) * (size_t)batch);
  l.S = ws.take(sizeof(float) * (size_t)l.F * n_bins);
  l.frames = ws.take(sizeof(float) * (size_t)l.F * n_fft);
  l.y = ws.take(sizeof(float) * (size_t)l.samples);
  l.total = ws.total();
  return l;
}

}  // namespace

struct mb_griffinlim {
  mb_griffinlim_config cfg{};
  int n_bins = 0, warm = 0;
  WeightTable w;
  std::vector<float> tables;  // window [n_fft] | twiddles [n_fft][2], written into the arena at finalize
  float* arena = nullptr;
  bool finalized = false;
};

extern "C" {

int mb_griffinlim_create(const mb_griffinlim_config* cfg, mb_griffinlim** out) {
  if (!cfg || !out) return fail(MB_ERR_INVALID, "mb_griffinlim_create: null argument");
  const mb_griffinlim_config& c = *cfg;
  const int N = c.n_fft;
  if (N != 256 && N != 512 && N != 1024 && N != 2048)
    return fail(MB_ERR_INVALID, "mb_griffinlim_create: n_fft = %d is not a power of two in [256, 2048]", N);
  if (c.win_length <= 0 || c.win_length > N)
    return fail(MB_ERR_INVALID, "mb_griffinlim_create: win_length = %d must be in [1, n_fft = %d]", c.win_length, N);
  if (c.hop_length <= 0 || c.hop_length > c.win_length)
    return fail(MB_ERR_INVALID, "mb_griffinlim_create: hop_length = %d must be in [1, win_length = %d]", c.hop_length,
                c.win_length);
  if (c.n_mels <= 0 || c.n_mels > 1024)
    return fail(MB_ERR_INVALID, "mb_griffinlim_create: n_mels = %d must be in [1, 1024]", c.n_mels);
  if (c.pad_mode != 0 && c.pad_mode != 1)
    return fail(MB_ERR_INVALID, "mb_griffinlim_create: pad_mode = %d (0 reflect, 1 constant)", c.pad_mode);
  if (!(c.power > 0.f) || !std::isfinite(c.power))
    return fail(MB_ERR_INVALID, "mb_griffinlim_create: power = %g must be positive", (double)c.power);
  if (c.signal_normalization && !(c.max_abs_value > 0.f))
    return fail(MB_ERR_INVALID, "mb_griffinlim_create: max_abs_value = %g must be positive", (double)c.max_abs_value);
  if (!(c.preemphasis >= 0.0 && c.preemphasis < 1.0))
    return fail(MB_ERR_INVALID, "mb_griffinlim_create: preemphasis = %g must be in [0, 1)", c.preemphasis);
  int warm = 0;
  if (c.preemphasis > 0.0) {  // k^W < 2^-30
    const double w = std::ceil(30.0 * std::log(2.0) / -std::log(c.preemphasis));
    if (w > kMaxWarm)
      return fail(MB_ERR_INVALID, "mb_griffinlim_create: preemphasis = %g needs a warm-up of %.0f samples, more than %d",
                  c.preemphasis, w, kMaxWarm);
    warm = (int)w;
  }
  mb_griffinlim* h = new mb_griffinlim();
  h->cfg = c;
  h->n_bins = N / 2 + 1;
  h->warm = warm;
  h->w.add("inv_mel_basis", {h->n_bins, c.n_mels});
  h->w.add_derived("window", N);
  h->w.add_derived("twiddles", 2 * (size_t)N);
  h->tables.assign(3 * (size_t)N, 0.f);
  const double PI = 3.14159265358979323846;
  const int lpad = (N - c.win_length) / 2;  // periodic Hann of win_length, centred in n_fft (librosa.util.pad_center)
  for (int i = 0; i < c.win_length; ++i) h->tables[lpad + i] = (float)(0.5 - 0.5 * std::cos(2.0 * PI * i / c.win_length));
  fft_twiddles(N, h->tables.data() + N);
  *out = h;
  return MB_OK;
}

void mb_griffinlim_destroy(mb_griffinlim* h) { delete h; }

size_t mb_griffinlim_arena_bytes(const mb_griffinlim* h) { return h ? h->w.floats() * sizeof(float) : 0; }

int mb_griffinlim_set_arena(mb_griffinlim* h, void* arena, size_t bytes) {
  if (int rc = check_arena("mb_griffinlim_set_arena", h, arena, bytes, mb_griffinlim_arena_bytes(h), 256)) return rc;
  h->w.attach((float*)arena);
  h->arena = (float*)arena;
  h->finalized = false;
  return MB_OK;
}

int mb_griffinlim_set_weight(mb_griffinlim* h, const char* name, const float* w, const int64_t* dims, int32_t ndim,
                             void* stream) {
  if (!h) return fail(MB_ERR_INVALID, "mb_griffinlim_set_weight: null argument");
  if (int rc = h->w.set("mb_griffinlim_set_weight", name, w, dims, ndim, stream)) return rc;
  h->finalized = false;
  return MB_OK;
}

int mb_griffinlim_finalize(mb_griffinlim* h, void* stream) {
  if (!h || !h->arena) return fail(MB_ERR_STATE, "mb_griffinlim_finalize: no arena");
  if (int rc = h->w.check_all_set("mb_griffinlim_finalize")) return rc;
  const int N = h->cfg.n_fft;
  cudaStream_t st = (cudaStream_t)stream;
  MB_CUDA_CHECK(cudaMemcpyAsync(h->w.ptr("window"), h->tables.data(), sizeof(float) * N, cudaMemcpyHostToDevice, st));
  MB_CUDA_CHECK(cudaMemcpyAsync(h->w.ptr("twiddles"), h->tables.data() + N, sizeof(float) * 2 * N, cudaMemcpyHostToDevice, st));
  MB_CUDA_CHECK(cudaStreamSynchronize(st));  // the source is pageable host memory owned by the handle
  h->finalized = true;
  return MB_OK;
}

size_t mb_griffinlim_workspace_bytes(const mb_griffinlim* h, int32_t batch, const int32_t* frames_host) {
  if (!h || batch <= 0 || !frames_host) return 0;
  for (int b = 0; b < batch; ++b)
    if (frames_host[b] < 1) return 0;
  return layout(h->cfg.n_fft, h->n_bins, h->cfg.hop_length, batch, frames_host).total;
}

int mb_griffinlim_forward(mb_griffinlim* h, const float* mels, const int32_t* frames_host, int32_t batch,
                          const double* uniforms, const uint64_t* seeds_host, int32_t n_iters, float* out, void* workspace,
                          size_t workspace_bytes, void* stream) {
  if (!h || !mels || !frames_host || !out) return fail(MB_ERR_INVALID, "mb_griffinlim_forward: null argument");
  if (!h->finalized) return fail(MB_ERR_STATE, "mb_griffinlim_forward: weights not finalized");
  if (batch <= 0) return fail(MB_ERR_INVALID, "mb_griffinlim_forward: batch = %d", batch);
  if (n_iters < 0) return fail(MB_ERR_INVALID, "mb_griffinlim_forward: n_iters = %d is negative", n_iters);
  if ((uniforms == nullptr) == (seeds_host == nullptr))
    return fail(MB_ERR_INVALID, "mb_griffinlim_forward: pass exactly one of uniforms and seeds_host");
  const mb_griffinlim_config& c = h->cfg;
  const int N = c.n_fft, H = c.hop_length;
  int64_t F = 0;
  for (int b = 0; b < batch; ++b) {
    const int64_t T = frames_host[b];
    if (c.pad_mode == 0 && !(T >= 2 && (int64_t)H * (T - 1) > N / 2))
      return fail(MB_ERR_INVALID,
                  "mb_griffinlim_forward: utterance %d has %d frames; reflect padding needs hop * (T - 1) > n_fft / 2 = %d", b,
                  (int)T, N / 2);
    if (c.pad_mode == 1 && T < 2)
      return fail(MB_ERR_INVALID, "mb_griffinlim_forward: utterance %d has %d frames; at least 2 are needed", b, (int)T);
    F += T;
  }
  if (F > ((int64_t)1 << 28))
    return fail(MB_ERR_INVALID, "mb_griffinlim_forward: %lld frames are too many for one call", (long long)F);
  const Layout l = layout(N, h->n_bins, H, batch, frames_host);
  char* ws;
  if (int rc = bind("mb_griffinlim_forward", workspace, workspace_bytes, l.total, &ws)) return rc;
  // host row tables: pair -> (utterance, first local frame); utterance -> offsets and seed
  std::vector<char> host(l.S - l.pairs);
  int2* pairs = (int2*)host.data();
  GlUtt* utt = (GlUtt*)(host.data() + (l.utt - l.pairs));
  int64_t f0 = 0, o = 0, np = 0;
  for (int b = 0; b < batch; ++b) {
    const int T = frames_host[b];
    utt[b] = GlUtt{(int32_t)f0, T, o, seeds_host ? seeds_host[b] : 0};
    for (int t = 0; t < T; t += 2) pairs[np++] = make_int2(b, t);
    f0 += T;
    o += (int64_t)H * (T - 1);
  }
  cudaStream_t st = (cudaStream_t)stream;
  MB_CUDA_CHECK(cudaMemcpyAsync(ws + l.pairs, host.data(), host.size(), cudaMemcpyHostToDevice, st));

  GlParams p;
  memset(&p, 0, sizeof(p));
  p.n_fft = N;
  p.hop = H;
  p.n_bins = h->n_bins;
  p.n_mels = c.n_mels;
  p.pad_mode = c.pad_mode;
  p.warm = h->warm;
  p.signal_normalization = c.signal_normalization;
  p.allow_clipping = c.allow_clipping;
  p.symmetric = c.symmetric;
  p.power = c.power;
  p.preemphasis = c.preemphasis;
  p.max_abs_value = c.max_abs_value;
  p.min_level_db = c.min_level_db;
  p.ref_level_db = c.ref_level_db;
  p.basis = h->w.ptr("inv_mel_basis");
  p.window = h->w.ptr("window");
  p.tw = (const float2*)h->w.ptr("twiddles");
  p.pairs = (const int2*)(ws + l.pairs);
  p.utt = (const GlUtt*)(ws + l.utt);
  p.mels = mels;
  p.uniforms = uniforms;
  p.S = (float*)(ws + l.S);
  p.frames = (float*)(ws + l.frames);
  p.y = (float*)(ws + l.y);
  p.out = out;
  const unsigned P = (unsigned)l.n_pairs;
  const size_t fsmem = 2 * sizeof(float2) * N;
  gl_mag_kernel<<<P, kThreads, 2 * sizeof(double) * c.n_mels, st>>>(p);
  MB_LAUNCH_CHECK("gl_mag_kernel");
  if (uniforms) gl_frame_kernel<0><<<P, kThreads, fsmem, st>>>(p);
  else gl_frame_kernel<1><<<P, kThreads, fsmem, st>>>(p);
  MB_LAUNCH_CHECK("gl_frame_kernel");
  gl_ola_kernel<<<P, kThreads, 0, st>>>(p);
  MB_LAUNCH_CHECK("gl_ola_kernel");
  for (int it = 0; it < n_iters; ++it) {
    gl_frame_kernel<2><<<P, kThreads, fsmem, st>>>(p);
    MB_LAUNCH_CHECK("gl_frame_kernel");
    gl_ola_kernel<<<P, kThreads, 0, st>>>(p);
    MB_LAUNCH_CHECK("gl_ola_kernel");
  }
  gl_deemph_kernel<<<(P + 127) / 128, 128, 0, st>>>(p, (int)P);
  MB_LAUNCH_CHECK("gl_deemph_kernel");
  return MB_OK;
}

}  // extern "C"
