// Device post-processing of WaveRNN.generate (mb_wavernn_postprocess): class indices -> float64 waveform.
// mb_wavernn_postprocess_f32 runs the same kernels on the float samples of the MOL sampler (cast to float64, no mu-law).
//
//   sample            2 * idx.float() / (n_classes - 1.) - 1.   in float32, then float64   fatchord_version.py:226, 236-238
//                     (MOL: the float32 sample itself, then float64                          fatchord_version.py:211-216)
//   xfade_and_unfold  equal-power fades sqrt(0.5 (1 +- t)), t = linspace(-1, 1, overlap - overlap//2), silence overlap//2;
//                     overlap-add of the folds                                              fatchord_version.py:340-402
//   decode_mu_law     sign(y) / mu * ((1 + mu) ** |y| - 1), mu = n_classes - 1              wavernn/audio.py:102-107
//   de_emphasis       lfilter([1], [1, -0.97], x): y[n] = x[n] + 0.97 y[n-1]                wavernn/audio.py:92-93
//   trim / fade-out   out[:wave_len]; out[-fade_len:] *= linspace(1, 0, fade_len)           fatchord_version.py:251-253
//
// All float64 with separate multiplies and adds in the reference's order (the library is built with -fmad=false), numpy's
// linspace formula (start + i*step, last point = stop) and IEEE sqrt, so the fades are bit-identical; `pow` may differ from
// glibc's by an ulp (<= 1e-15 relative).  The serial IIR is evaluated in parallel WITHOUT changing its arithmetic: every
// thread runs the same two-rounding recurrence over its own 64 outputs after a 2048-sample run-in from zero; 0.97^2048 =
// 8e-28, so the run-in state has converged to the serial filter's state (to the last bit, the map being contractive).
#include <cstring>

#include "mb_common.h"

namespace {

// In: int16_t class indices (RAW) or float samples (MOL)
template <typename In>
struct PostParams {
  const In* idx;       // [folds][steps]
  int folds, steps, batched, target, overlap;
  int n_classes, mu_law;
  double preemph;      // 0: no de-emphasis
  long long total_len; // unfolded length
  long long n_out;     // after the trim
  int fade_len;
  double* tmp;         // [total_len] mu-law decoded, before the filter
  double* out;         // [n_out]
};

__device__ __forceinline__ double linspace_at(double start, double stop, int num, int i) {
  if (num == 1) return start;
  if (i == num - 1) return stop;
  const double step = (stop - start) / (double)(num - 1);
  return start + (double)i * step;
}

__device__ __forceinline__ double sample_of(const PostParams<int16_t>& p, int fold, int j) {
  const float v = 2.f * (float)p.idx[(size_t)fold * p.steps + j] / (float)(p.n_classes - 1) - 1.f;
  return (double)v;
}

__device__ __forceinline__ double sample_of(const PostParams<float>& p, int fold, int j) {
  return (double)p.idx[(size_t)fold * p.steps + j];
}

// fold value at in-fold position j with the cross-fade applied (y[:, :overlap] *= fade_in; y[:, -overlap:] *= fade_out)
template <typename In>
__device__ __forceinline__ double faded(const PostParams<In>& p, int fold, int j) {
  double v = sample_of(p, fold, j);
  const int silence = p.overlap / 2, fl = p.overlap - silence;
  if (j < p.overlap) {
    const double f = j < silence ? 0.0 : sqrt(0.5 * (1.0 + linspace_at(-1.0, 1.0, fl, j - silence)));
    v = v * f;
  }
  const int jj = j - (p.steps - p.overlap);
  if (jj >= 0) {
    const double f = jj < fl ? sqrt(0.5 * (1.0 - linspace_at(-1.0, 1.0, fl, jj))) : 0.0;
    v = v * f;
  }
  return v;
}

template <typename In>
__global__ void k_unfold_decode(PostParams<In> p) {
  const long long n = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= p.total_len) return;
  double y;
  if (!p.batched) {
    y = sample_of(p, 0, (int)n);
  } else {
    const int S = p.target + p.overlap;
    const int i = (int)(n / S);
    const int j = (int)(n - (long long)i * S);
    y = 0.0;
    if (i >= 1 && j < p.overlap) y = y + faded(p, i - 1, j + S);  // the tail of the previous fold comes first (loop order)
    if (i < p.folds) y = y + faded(p, i, j);
  }
  if (p.mu_law) {
    const double mu = (double)(p.n_classes - 1);
    const double s = y > 0.0 ? 1.0 : (y < 0.0 ? -1.0 : 0.0);
    y = s / mu * (pow(1.0 + mu, fabs(y)) - 1.0);
  }
  p.tmp[n] = y;
}

constexpr int kSeg = 64, kRunIn = 2048;

template <typename In>
__global__ void k_deemph_fade(PostParams<In> p) {
  const long long seg = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long n0 = seg * kSeg;
  if (n0 >= p.n_out) return;
  double y = 0.0;
  if (p.preemph != 0.0) {
    long long s = n0 - kRunIn;
    if (s < 0) s = 0;
    for (long long n = s; n < n0; ++n) y = p.tmp[n] + p.preemph * y;
  }
  const long long n1 = n0 + kSeg < p.n_out ? n0 + kSeg : p.n_out;
  for (long long n = n0; n < n1; ++n) {
    y = p.preemph != 0.0 ? p.tmp[n] + p.preemph * y : p.tmp[n];
    double o = y;
    const long long k = n - (p.n_out - p.fade_len);
    if (k >= 0) o = o * linspace_at(1.0, 0.0, p.fade_len, (int)k);
    p.out[n] = o;
  }
}

size_t workspace_bytes_of(int32_t folds, int32_t steps, int32_t batched, int32_t target, int32_t overlap) {
  const long long total = batched ? (long long)folds * (target + overlap) + overlap : (long long)steps;
  return (size_t)(total > 0 ? total : 0) * sizeof(double) + 256;
}

template <typename In>
int postprocess(const In* idx, int32_t folds, int32_t steps, int32_t batched, int32_t target, int32_t overlap,
                int32_t n_classes, int32_t mu_law, double preemphasis, int64_t wave_len, int32_t fade_len,
                double* out, int64_t* n_out, void* workspace, size_t workspace_bytes, void* stream) {
  if (!idx || !out || !n_out) return mb::fail(MB_ERR_INVALID, "mb_wavernn_postprocess: null argument");
  if (folds <= 0 || steps <= 0 || n_classes < 2) return mb::fail(MB_ERR_INVALID, "mb_wavernn_postprocess: empty input");
  if (batched && (steps != target + 2 * overlap || overlap < 0 || target <= 0))
    return mb::fail(MB_ERR_INVALID, "mb_wavernn_postprocess: folds must be target + 2*overlap = %d steps long, got %d", target + 2 * overlap, steps);
  if (!batched && folds != 1) return mb::fail(MB_ERR_INVALID, "mb_wavernn_postprocess: unbatched output has one row");
  PostParams<In> p;
  memset(&p, 0, sizeof(p));
  p.idx = idx;
  p.folds = folds;
  p.steps = steps;
  p.batched = batched;
  p.target = target;
  p.overlap = overlap;
  p.n_classes = n_classes;
  p.mu_law = mu_law;
  p.preemph = preemphasis;
  p.total_len = batched ? (long long)folds * (target + overlap) + overlap : (long long)steps;
  p.n_out = wave_len < p.total_len ? (wave_len < 0 ? 0 : wave_len) : p.total_len;  // out[:wave_len]
  p.fade_len = fade_len;
  if (p.n_out < fade_len) return mb::fail(MB_ERR_INVALID, "mb_wavernn_postprocess: output of %lld samples is shorter than the %d-sample fade "
                                          "(the reference raises here too)", p.n_out, fade_len);
  if (int rc = mb::bind("mb_wavernn_postprocess", workspace, workspace_bytes, workspace_bytes_of(folds, steps, batched, target, overlap),
                        &p.tmp))
    return rc;
  p.out = out;
  cudaStream_t st = (cudaStream_t)stream;
  k_unfold_decode<In><<<(unsigned)((p.total_len + 255) / 256), 256, 0, st>>>(p);
  MB_LAUNCH_CHECK("k_unfold_decode");
  if (p.n_out > 0) {
    const long long segs = (p.n_out + kSeg - 1) / kSeg;
    k_deemph_fade<In><<<(unsigned)((segs + 127) / 128), 128, 0, st>>>(p);
    MB_LAUNCH_CHECK("k_deemph_fade");
  }
  *n_out = p.n_out;
  return MB_OK;
}

}  // namespace

extern "C" {

size_t mb_wavernn_postprocess_workspace_bytes(int32_t folds, int32_t steps, int32_t batched, int32_t target, int32_t overlap) {
  return workspace_bytes_of(folds, steps, batched, target, overlap);
}

int mb_wavernn_postprocess(const int16_t* idx, int32_t folds, int32_t steps, int32_t batched, int32_t target, int32_t overlap,
                           int32_t n_classes, int32_t mu_law, double preemphasis, int64_t wave_len, int32_t fade_len,
                           double* out, int64_t* n_out, void* workspace, size_t workspace_bytes, void* stream) {
  return postprocess<int16_t>(idx, folds, steps, batched, target, overlap, n_classes, mu_law, preemphasis, wave_len, fade_len,
                              out, n_out, workspace, workspace_bytes, stream);
}

int mb_wavernn_postprocess_f32(const float* samples, int32_t folds, int32_t steps, int32_t batched, int32_t target,
                               int32_t overlap, double preemphasis, int64_t wave_len, int32_t fade_len, double* out,
                               int64_t* n_out, void* workspace, size_t workspace_bytes, void* stream) {
  // n_classes is not read for float input; 2 passes the argument check
  return postprocess<float>(samples, folds, steps, batched, target, overlap, 2, 0, preemphasis, wave_len, fade_len, out, n_out,
                            workspace, workspace_bytes, stream);
}

}  // extern "C"
