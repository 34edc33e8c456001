// Mel-spectrogram front-ends on H100 (mb_melspec_*): SURVEY.md section 8f rows N1 / N2.
//
//   N2  models/encoder/audio.py:53-65      wav_to_mel_spectrogram = librosa.feature.melspectrogram(y, sr=16000,
//       n_fft=400, hop_length=160, n_mels=40) (power spectrogram, no log), transposed to [frames][40]
//   N1  models/synthesizer/audio.py:59-65  melspectrogram = normalize(amp_to_db(mel_basis @ |stft(preemphasis(wav))|)
//       - ref_level_db) with librosa.stft(n_fft, hop, win) and librosa.filters.mel(sr, n_fft, n_mels, fmin, fmax)
//
// librosa is not vendored in the reference (requirements.txt: unpinned "librosa"); the algorithm restated here is
// librosa's published one: centered frames (reflect or zero padding of n_fft/2), periodic Hann window of win_length
// zero-padded to n_fft, rfft, Slaney mel scale with area normalisation.  The window, the DFT twiddles and the mel
// basis are computed on the host in float64 at create time.
//
// One CTA per frame: windowed frame -> shared memory, direct DFT (n_fft <= 2048: O(N^2) is ~0.5 MFLOP per frame),
// magnitude / power -> shared memory, mel projection (one warp per mel band, shuffle reduction), dB / normalise.
#include <cmath>
#include <cstring>
#include <vector>

#include "mb_common.h"

using namespace mb;

struct mb_melspec {
  mb_melspec_config cfg{};
  int n_bins = 0;
  std::vector<float> host;  // window [n_fft] | cos [n_fft] | sin [n_fft] | basis [n_mels][n_bins]
  float* arena = nullptr;
};

namespace {

double hz_to_mel(double f) {  // Slaney (librosa htk=False)
  const double f_sp = 200.0 / 3.0, min_log_hz = 1000.0, min_log_mel = min_log_hz / f_sp, logstep = std::log(6.4) / 27.0;
  return f >= min_log_hz ? min_log_mel + std::log(f / min_log_hz) / logstep : f / f_sp;
}
double mel_to_hz(double m) {
  const double f_sp = 200.0 / 3.0, min_log_hz = 1000.0, min_log_mel = min_log_hz / f_sp, logstep = std::log(6.4) / 27.0;
  return m >= min_log_mel ? min_log_hz * std::exp(logstep * (m - min_log_mel)) : f_sp * m;
}

struct MelParams {
  const float* wav;
  int n_samples, n_frames;
  int n_fft, hop, n_bins, n_mels, pad_mode, power, to_db, normalize, symmetric, transpose_out;
  float preemphasis, min_level, ref_level_db, min_level_db, max_abs_value;
  const float* window;
  const float* cs;
  const float* sn;
  const float* basis;
  float* out;
};

__device__ __forceinline__ float sample_at(const MelParams& p, int i) {
  // centered framing: index i of the padded signal refers to sample i - n_fft/2; reflect (or zero) outside
  int j = i;
  if (j < 0) {
    if (p.pad_mode != 0) return 0.f;
    j = -j;
  } else if (j >= p.n_samples) {
    if (p.pad_mode != 0) return 0.f;
    j = 2 * (p.n_samples - 1) - j;
  }
  if (j < 0 || j >= p.n_samples) return 0.f;
  float v = p.wav[j];
  if (p.preemphasis != 0.f && j > 0) v -= p.preemphasis * p.wav[j - 1];  // lfilter([1, -k], [1], wav)
  return v;
}

__global__ void __launch_bounds__(256) melspec_kernel(const MelParams p) {
  extern __shared__ float sm[];
  float* fr = sm;                  // [n_fft]
  float* tc = fr + p.n_fft;        // [n_fft] cos
  float* ts = tc + p.n_fft;        // [n_fft] sin
  float* mag = ts + p.n_fft;       // [n_bins]
  const int f = blockIdx.x, tid = threadIdx.x;
  const int start = f * p.hop - p.n_fft / 2;
  for (int j = tid; j < p.n_fft; j += blockDim.x) {
    fr[j] = sample_at(p, start + j) * p.window[j];
    tc[j] = p.cs[j];
    ts[j] = p.sn[j];
  }
  __syncthreads();
  for (int k = tid; k < p.n_bins; k += blockDim.x) {
    float re = 0.f, im = 0.f;
    int idx = 0;
    for (int j = 0; j < p.n_fft; ++j) {
      re = fmaf(fr[j], tc[idx], re);
      im = fmaf(fr[j], ts[idx], im);
      idx += k;
      if (idx >= p.n_fft) idx -= p.n_fft;
    }
    const float pw = re * re + im * im;
    mag[k] = p.power == 2 ? pw : sqrtf(pw);
  }
  __syncthreads();
  const int warp = tid >> 5, lane = tid & 31, nw = blockDim.x >> 5;
  for (int m = warp; m < p.n_mels; m += nw) {
    const float* b = p.basis + (size_t)m * p.n_bins;
    float a = 0.f;
    for (int k = lane; k < p.n_bins; k += 32) a = fmaf(b[k], mag[k], a);
    for (int o = 16; o; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
    if (lane == 0) {
      float v = a;
      if (p.to_db) v = 20.f * log10f(fmaxf(p.min_level, v)) - p.ref_level_db;
      if (p.normalize) {
        const float u = (v - p.min_level_db) / (-p.min_level_db);
        v = p.symmetric ? fminf(fmaxf(2.f * p.max_abs_value * u - p.max_abs_value, -p.max_abs_value), p.max_abs_value)
                        : fminf(fmaxf(p.max_abs_value * u, 0.f), p.max_abs_value);
      }
      if (p.transpose_out) p.out[(size_t)f * p.n_mels + m] = v;
      else p.out[(size_t)m * p.n_frames + f] = v;
    }
  }
}

}  // namespace

extern "C" {

int mb_melspec_create(const mb_melspec_config* cfg, mb_melspec** out) {
  if (!cfg || !out) return fail(MB_ERR_INVALID, "mb_melspec_create: null argument");
  const mb_melspec_config& c = *cfg;
  if (c.n_fft < 16 || c.n_fft > 2048 || c.hop_length <= 0 || c.win_length <= 0 || c.win_length > c.n_fft || c.n_mels <= 0 ||
      c.sample_rate <= 0 || (c.power != 1 && c.power != 2) || c.fmax <= c.fmin || c.fmax > c.sample_rate * 0.5f + 1e-3f)
    return fail(MB_ERR_INVALID, "mb_melspec_create: unsupported parameters");
  mb_melspec* h = new mb_melspec();
  h->cfg = c;
  const int N = c.n_fft, nb = N / 2 + 1;
  h->n_bins = nb;
  h->host.assign((size_t)3 * N + (size_t)c.n_mels * nb, 0.f);
  float* win = h->host.data();
  float* cs = win + N;
  float* sn = cs + N;
  float* basis = sn + N;
  const double PI = 3.14159265358979323846;
  // periodic Hann window of win_length, centered zero padding to n_fft (librosa.util.pad_center)
  const int lpad = (N - c.win_length) / 2;
  for (int i = 0; i < c.win_length; ++i) win[lpad + i] = (float)(0.5 - 0.5 * std::cos(2.0 * PI * i / c.win_length));
  for (int i = 0; i < N; ++i) {
    cs[i] = (float)std::cos(2.0 * PI * i / N);
    sn[i] = (float)(-std::sin(2.0 * PI * i / N));
  }
  // librosa.filters.mel: triangles between n_mels + 2 Slaney-mel-spaced edges, area ("slaney") normalisation
  std::vector<double> edges(c.n_mels + 2);
  const double m0 = hz_to_mel(c.fmin), m1 = hz_to_mel(c.fmax);
  for (int i = 0; i < c.n_mels + 2; ++i) edges[i] = mel_to_hz(m0 + (m1 - m0) * i / (c.n_mels + 1));
  for (int m = 0; m < c.n_mels; ++m) {
    const double lo = edges[m], ce = edges[m + 1], hi = edges[m + 2];
    const double enorm = 2.0 / (hi - lo);
    for (int k = 0; k < nb; ++k) {
      const double fk = (double)k * c.sample_rate / N;
      const double lower = (fk - lo) / (ce - lo), upper = (hi - fk) / (hi - ce);
      const double w = std::fmax(0.0, std::fmin(lower, upper));
      basis[(size_t)m * nb + k] = (float)(w * enorm);
    }
  }
  *out = h;
  return MB_OK;
}

void mb_melspec_destroy(mb_melspec* h) { delete h; }

size_t mb_melspec_arena_bytes(const mb_melspec* h) { return h ? h->host.size() * sizeof(float) : 0; }

int mb_melspec_set_arena(mb_melspec* h, void* arena, size_t bytes, void* stream) {
  if (!h || !arena) return fail(MB_ERR_INVALID, "mb_melspec_set_arena: null argument");
  if (bytes < mb_melspec_arena_bytes(h)) return fail(MB_ERR_WORKSPACE, "mb_melspec_set_arena: arena too small");
  MB_CUDA_CHECK(cudaMemcpyAsync(arena, h->host.data(), h->host.size() * sizeof(float), cudaMemcpyHostToDevice,
                                (cudaStream_t)stream));
  MB_CUDA_CHECK(cudaStreamSynchronize((cudaStream_t)stream));  // the source is pageable host memory owned by the handle
  h->arena = (float*)arena;
  return MB_OK;
}

int32_t mb_melspec_num_frames(const mb_melspec* h, int32_t n_samples) {
  if (!h || n_samples <= 0) return 0;
  return 1 + n_samples / h->cfg.hop_length;  // librosa center=True
}

int mb_melspec_forward(mb_melspec* h, const float* wav, int32_t n_samples, float* out, void* stream) {
  if (!h || !wav || !out) return fail(MB_ERR_INVALID, "mb_melspec_forward: null argument");
  if (!h->arena) return fail(MB_ERR_STATE, "mb_melspec_forward: call mb_melspec_set_arena first");
  const mb_melspec_config& c = h->cfg;
  if (n_samples <= 0) return fail(MB_ERR_INVALID, "mb_melspec_forward: empty signal");
  if (c.pad_mode == 0 && n_samples <= c.n_fft / 2)
    return fail(MB_ERR_INVALID, "mb_melspec_forward: reflect padding needs more than n_fft/2 = %d samples", c.n_fft / 2);
  MelParams p;
  memset(&p, 0, sizeof(p));
  p.wav = wav;
  p.n_samples = n_samples;
  p.n_frames = mb_melspec_num_frames(h, n_samples);
  p.n_fft = c.n_fft;
  p.hop = c.hop_length;
  p.n_bins = h->n_bins;
  p.n_mels = c.n_mels;
  p.pad_mode = c.pad_mode;
  p.power = c.power;
  p.to_db = c.to_db;
  p.normalize = c.normalize;
  p.symmetric = c.symmetric;
  p.transpose_out = c.transpose_out;
  p.preemphasis = c.preemphasis;
  p.min_level = expf(c.min_level_db / 20.f * logf(10.f));
  p.ref_level_db = c.ref_level_db;
  p.min_level_db = c.min_level_db;
  p.max_abs_value = c.max_abs_value;
  p.window = h->arena;
  p.cs = h->arena + c.n_fft;
  p.sn = h->arena + 2 * c.n_fft;
  p.basis = h->arena + 3 * c.n_fft;
  p.out = out;
  const size_t smem = sizeof(float) * ((size_t)3 * c.n_fft + h->n_bins);
  melspec_kernel<<<p.n_frames, 256, smem, (cudaStream_t)stream>>>(p);
  MB_LAUNCH_CHECK("melspec_kernel");
  return MB_OK;
}

}  // extern "C"
