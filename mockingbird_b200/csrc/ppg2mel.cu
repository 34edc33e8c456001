// Voice-conversion mel decoder (ppg2mel MelDecoderMOLv2.inference) on sm_90a.
//
//   encoder  models/ppg2mel/__init__.py:172-180   bnf_prenet / pitch_convs (Conv1d k1 -> LeakyReLU -> InstanceNorm ->
//                                                 2 x [Conv1d k4 s2 p1 -> LeakyReLU -> InstanceNorm]), sum, reduce_proj
//   decoder  models/ppg2mel/rnn_decoder_mol.py:267-315 + utils/mol_attention.py:69-122
//   postnet  models/ppg2mel/utils/cnn_postnet.py  (eval BatchNorm, dropout off)
//
// Every row of a padded batch is computed as its own B = 1 call: per-row lengths drive the instance-norm statistics,
// the zero padding every convolution reads past a row's end, the MoL position range and the step limits, and a
// finished row is frozen (all decoder kernels skip it) while the others run on.  No arithmetic of a row depends on the
// batch: every dot product has a fixed summation order that does not depend on B or on the row's position.
//
// All arithmetic is FP32 (FFMA-free: the library is compiled with -fmad=false), with accurate expf / log1pf and IEEE
// division.  See DESIGN.md section 4g for the kernel map and the precision study of the MoL attention.
#include <cuda_runtime.h>

#include <atomic>
#include <climits>
#include <cstring>
#include <string>
#include <vector>

#include "../../include/mb_wavernn_math.h"
#include "mb_common.h"

using mb::check_arena;
using mb::fail;
using mb::WeightTable;

namespace {

constexpr int kMaxRows = 128;    // rows per call (the Python layer splits larger batches)
constexpr int kE = 256;          // encoder_dim
constexpr int kH = 512;          // attention_rnn_dim = decoder_rnn_dim
constexpr int kP1 = 256, kP2 = 128;
constexpr int kNM = 80;          // num_mels
constexpr int kR = 2;            // frames_per_step
constexpr int kM = 5;            // num_mixtures
constexpr int kQ = 256;          // MoL query hidden width
constexpr int kGroup = 16;       // decoder steps per captured graph (even: the h ping-pong parity repeats)
constexpr int kRowsPerWarp = 8;  // rows sharing one weight fetch in the skinny dot kernels

// ---------------------------------------------------------------------------------------------- small helpers
__device__ __forceinline__ float sigmoidf_(float x) { return 1.0f / (1.0f + expf(-x)); }
__device__ __forceinline__ float softplusf_(float x) { return x > 20.0f ? x : log1pf(expf(x)); }  // threshold 20

__device__ __forceinline__ bool row_active(const int* done_at, int b, int step) { return step < done_at[b]; }

__device__ __forceinline__ bool keep_flag(const uint8_t* masks, int width, int B, int b, int step, int unit, int layer,
                                          uint64_t seed) {
  if (masks) return masks[((size_t)step * B + b) * width + unit] != 0;
  uint32_t o[4];
  mb_philox4x32((uint32_t)unit >> 2, (uint32_t)b, (uint32_t)step, 0x70326d00u + (uint32_t)layer, (uint32_t)seed,
                (uint32_t)(seed >> 32), o);
  return ((o[unit & 3] >> 16) & 1u) != 0;
}

struct Lens {
  int v[kMaxRows];
};

// per-call device state: lengths of each stage, the step counter and the freeze / stop bookkeeping
struct State {
  int* len0;     // PPG frames
  int* len1;     // after the first stride-2 conv
  int* tenc;     // T_enc
  int* done_at;  // step count at which the row stopped (INT_MAX while running)
  int* steps;    // = done_at once stopped
  int* mel_len;  // 2 * steps
  int* g_step;   // decoder step being computed
  int* flag;     // 1 once every row has stopped
};

__global__ void init_state_kernel(Lens L, int B, State s) {
  const int b = threadIdx.x;
  if (b < B) {
    const int t = L.v[b];
    s.len0[b] = t;
    s.len1[b] = t / 2;        // Conv1d(k4, s2, p1): floor((t + 2 - 4) / 2) + 1
    s.tenc[b] = (t / 2) / 2;
    s.done_at[b] = INT_MAX;
    s.steps[b] = 0;
    s.mel_len[b] = 0;
  }
  if (b == 0) {
    *s.g_step = 0;
    *s.flag = 0;
  }
}

// ---------------------------------------------------------------------------------------------- encoder / postnet
// y[b, t, n] = epilogue(sum_{c, tap} w[n, c, tap] * x[b, t * stride - pad + tap, c]) for t < len_out[b] (0 past it);
// x reads past len_in[b] (or before 0) are zero: exactly the zero padding a B = 1 Conv1d sees.
struct ConvP {
  const float* x;
  int xT, ldx, Cin;
  const int* len_in;
  int stride, pad, ks;
  const float* w;
  int ldw;
  const float* bias;
  int bias_ld;  // 0: one bias vector; N: a per-row bias [B][N]
  const float *bn_mean, *bn_var, *bn_w, *bn_b;  // eval BatchNorm after the bias (optional)
  int act;      // 0 none, 1 LeakyReLU(0.1), 2 tanh
  const float* res;  // added last, same layout as y (optional)
  float* y;
  int yT, ldy, N, T_out;
  const int* len_out;
  int B;
};

constexpr int kBM = 64, kBN = 64, kBK = 16;

__global__ void __launch_bounds__(256) conv_gemm_kernel(ConvP p) {
  __shared__ float As[kBK][kBM + 4];
  __shared__ float Bs[kBK][kBN + 4];
  const int tid = threadIdx.x;
  const int M = p.B * p.T_out;
  const int K = p.Cin * p.ks;
  const int m0 = blockIdx.x * kBM, n0 = blockIdx.y * kBN;
  const int tx = tid & 15, ty = tid >> 4;
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.0f;
  for (int k0 = 0; k0 < K; k0 += kBK) {
    const int kk = tid & 15;
    const int k = k0 + kk;
    const int c = k / p.ks, tap = k - c * p.ks;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int mr = (tid >> 4) + 16 * i;
      const int m = m0 + mr;
      float v = 0.0f;
      if (k < K && m < M) {
        const int b = m / p.T_out, t = m - b * p.T_out;
        const int ti = t * p.stride - p.pad + tap;
        const int li = p.len_in ? p.len_in[b] : p.xT;
        if (ti >= 0 && ti < li) v = p.x[((size_t)b * p.xT + ti) * p.ldx + c];
      }
      As[kk][mr] = v;
      const int n = n0 + mr;
      Bs[kk][mr] = (k < K && n < p.N) ? p.w[(size_t)n * p.ldw + k] : 0.0f;
    }
    __syncthreads();
#pragma unroll
    for (int q = 0; q < kBK; ++q) {
      float a[4], bb[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) a[i] = As[q][ty * 4 + i];
#pragma unroll
      for (int j = 0; j < 4; ++j) bb[j] = Bs[q][tx * 4 + j];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] += a[i] * bb[j];
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int m = m0 + ty * 4 + i;
    if (m >= M) continue;
    const int b = m / p.T_out, t = m - b * p.T_out;
    const int L = p.len_out ? p.len_out[b] : p.T_out;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int n = n0 + tx * 4 + j;
      if (n >= p.N) continue;
      float v = 0.0f;
      const size_t yi = ((size_t)b * p.yT + t) * p.ldy + n;
      if (t < L) {
        v = acc[i][j];
        if (p.bias) v += p.bias[(size_t)b * p.bias_ld + n];
        if (p.bn_mean) {
          const float alpha = p.bn_w[n] / sqrtf(p.bn_var[n] + 1e-5f);
          v = v * alpha + (p.bn_b[n] - p.bn_mean[n] * alpha);
        }
        if (p.act == 1) v = v > 0.0f ? v : 0.1f * v;
        else if (p.act == 2) v = tanhf(v);
        if (p.res) v += p.res[yi];
      }
      p.y[yi] = v;
    }
  }
}

// InstanceNorm1d(affine=False), eps 1e-5, biased variance over the row's own frames t < len[b]; frames past the
// row's end are set to 0.  x [B][T][C] in place; `add` (same layout, optional) is added after normalising.
// grid (C / 32, B), block (32, 8): thread (c, g) sums the frames t = g (mod 8) in double, combined in a fixed order.
__global__ void __launch_bounds__(256) instance_norm_kernel(float* x, int T, int C, const int* len, const float* add) {
  __shared__ double part[8][33];
  __shared__ float stat[2][32];
  const int c = blockIdx.x * 32 + threadIdx.x, g = threadIdx.y, b = blockIdx.y;
  const int L = len[b];
  float* xb = x + (size_t)b * T * C;
  double s = 0.0;
  for (int t = g; t < L; t += 8) s += (double)xb[(size_t)t * C + c];
  part[g][threadIdx.x] = s;
  __syncthreads();
  if (g == 0) {
    double tot = 0.0;
    for (int i = 0; i < 8; ++i) tot += part[i][threadIdx.x];
    stat[0][threadIdx.x] = (float)(tot / L);
  }
  __syncthreads();
  const double mean = (double)stat[0][threadIdx.x];
  s = 0.0;
  for (int t = g; t < L; t += 8) {
    const double d = (double)xb[(size_t)t * C + c] - mean;
    s += d * d;
  }
  __syncthreads();
  part[g][threadIdx.x] = s;
  __syncthreads();
  if (g == 0) {
    double tot = 0.0;
    for (int i = 0; i < 8; ++i) tot += part[i][threadIdx.x];
    stat[1][threadIdx.x] = 1.0f / sqrtf((float)(tot / L) + 1e-5f);
  }
  __syncthreads();
  const float mu = stat[0][threadIdx.x], inv = stat[1][threadIdx.x];
  for (int t = g; t < T; t += 8) {
    const size_t i = ((size_t)b * T + t) * C + c;
    float v = 0.0f;
    if (t < L) {
      v = (x[i] - mu) * inv;
      if (add) v = add[i] + v;
    }
    x[i] = v;
  }
}

// per-row bias of reduce_proj: bias + W[:, E:] . F.normalize(spk) (eps 1e-12); the speaker half of the input is the
// same for every frame of a row.  grid B, block 256 (= E)
__global__ void __launch_bounds__(256) spk_bias_kernel(const float* spk, int D, const float* W, int ldw,
                                                       const float* bias, float* out) {
  __shared__ float sn[1024];
  __shared__ float red[256];
  const int b = blockIdx.x, tid = threadIdx.x;
  float s = 0.0f;
  for (int k = tid; k < D; k += 256) {
    const float v = spk[(size_t)b * D + k];
    s += v * v;
  }
  red[tid] = s;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if (tid < o) red[tid] += red[tid + o];
    __syncthreads();
  }
  const float den = fmaxf(sqrtf(red[0]), 1e-12f);
  for (int k = tid; k < D; k += 256) sn[k] = spk[(size_t)b * D + k] / den;
  __syncthreads();
  float acc = 0.0f;
  const float* wr = W + (size_t)tid * ldw + kE;
  for (int k = 0; k < D; ++k) acc += wr[k] * sn[k];
  out[(size_t)b * kE + tid] = bias[tid] + acc;
}

// ---------------------------------------------------------------------------------------------- decoder step
// x rows of up to three concatenated input segments times weight rows; warp-per-output, lanes split K in float4
// slices, butterfly reduction (every lane ends with the same bits; the order depends on neither B nor the row).
struct Seg {
  const float* x;
  int ldx, k;
  const float* w;
  int ldw;
};
struct Segs {
  Seg s[3];
  int n;
};

template <int G>
__device__ __forceinline__ void dot_rows(const Segs& sg, const int (&wrow)[G], int b0, const bool (&act)[kRowsPerWarp],
                                         float (&acc)[G][kRowsPerWarp]) {
  const int lane = threadIdx.x & 31;
#pragma unroll
  for (int g = 0; g < G; ++g)
#pragma unroll
    for (int r = 0; r < kRowsPerWarp; ++r) acc[g][r] = 0.0f;
  for (int si = 0; si < sg.n; ++si) {
    const Seg s = sg.s[si];
    for (int k = lane * 4; k < s.k; k += 128) {
      float4 w[G];
#pragma unroll
      for (int g = 0; g < G; ++g) w[g] = __ldg(reinterpret_cast<const float4*>(s.w + (size_t)wrow[g] * s.ldw + k));
#pragma unroll
      for (int r = 0; r < kRowsPerWarp; ++r) {
        if (!act[r]) continue;
        const float4 x = *reinterpret_cast<const float4*>(s.x + (size_t)(b0 + r) * s.ldx + k);
#pragma unroll
        for (int g = 0; g < G; ++g) {
          float a = acc[g][r];
          a += w[g].x * x.x;
          a += w[g].y * x.y;
          a += w[g].z * x.z;
          a += w[g].w * x.w;
          acc[g][r] = a;
        }
      }
    }
  }
#pragma unroll
  for (int g = 0; g < G; ++g)
#pragma unroll
    for (int r = 0; r < kRowsPerWarp; ++r) {
      float v = acc[g][r];
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
      acc[g][r] = v;
    }
}

__device__ __forceinline__ void rows_active(int B, const int* done_at, int step, int b0, bool (&act)[kRowsPerWarp]) {
#pragma unroll
  for (int r = 0; r < kRowsPerWarp; ++r) act[r] = (b0 + r < B) && row_active(done_at, b0 + r, step);
}

// PreNet: Linear 80->256 (no bias) -> ReLU -> dropout(0.5, always on) -> Linear 256->128 -> ReLU -> dropout.
// Weights transposed ([in][out]) so that the per-unit loops read coalesced.  grid B, block 256
__global__ void __launch_bounds__(256) prenet_kernel(const float* frame, const float* W1t, const float* W2t,
                                                     const uint8_t* m1, const uint8_t* m2, uint64_t seed, int B,
                                                     const int* done_at, const int* g_step, float* out) {
  __shared__ float x[kNM], h1[kP1];
  const int b = blockIdx.x, tid = threadIdx.x, step = *g_step;
  if (!row_active(done_at, b, step)) return;
  if (tid < kNM) x[tid] = frame[(size_t)b * kNM + tid];
  __syncthreads();
  float a = 0.0f;
  for (int k = 0; k < kNM; ++k) a += W1t[k * kP1 + tid] * x[k];
  a = a > 0.0f ? a : 0.0f;
  h1[tid] = keep_flag(m1, kP1, B, b, step, tid, 1, seed) ? a * 2.0f : 0.0f;
  __syncthreads();
  if (tid < kP2) {
    float c = 0.0f;
    for (int k = 0; k < kP1; ++k) c += W2t[k * kP2 + tid] * h1[k];
    c = c > 0.0f ? c : 0.0f;
    out[(size_t)b * kP2 + tid] = keep_flag(m2, kP2, B, b, step, tid, 2, seed) ? c * 2.0f : 0.0f;
  }
}

// LSTMCell: gates = W_ih x + W_hh h + (b_ih + b_hh) (gate order i, f, g, o); warp = hidden unit j, 8 rows per warp.
// h is read from h_in and written to h_out (ping-pong: other warps still read h_in); c is updated in place.
// grid (H / 8, ceil(B / 8)), block 256
__global__ void __launch_bounds__(256) lstm_kernel(Segs sg, const float* bias, const float* h_in, float* h_out, float* c,
                                                   int B, const int* done_at, const int* g_step) {
  const int j = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  const int b0 = blockIdx.y * kRowsPerWarp, step = *g_step;
  bool act[kRowsPerWarp];
  rows_active(B, done_at, step, b0, act);
  bool any = false;
#pragma unroll
  for (int r = 0; r < kRowsPerWarp; ++r) any |= act[r];
  if (!any) return;
  sg.s[sg.n].x = h_in;
  sg.s[sg.n].ldx = kH;
  sg.n += 1;
  const int wrow[4] = {j, kH + j, 2 * kH + j, 3 * kH + j};
  float acc[4][kRowsPerWarp];
  dot_rows<4>(sg, wrow, b0, act, acc);
#pragma unroll
  for (int r = 0; r < kRowsPerWarp; ++r) {
    if (lane != r || !act[r]) continue;
    const size_t o = (size_t)(b0 + r) * kH + j;
    const float gi = sigmoidf_(acc[0][r] + bias[j]);
    const float gf = sigmoidf_(acc[1][r] + bias[kH + j]);
    const float gg = tanhf(acc[2][r] + bias[2 * kH + j]);
    const float go = sigmoidf_(acc[3][r] + bias[3 * kH + j]);
    const float cn = gf * c[o] + gi * gg;
    c[o] = cn;
    h_out[o] = go * tanhf(cn);
  }
}

// first layer of the MoL query: relu(W x + b), N = 256.  grid (N / 8, ceil(B / 8)), block 256
__global__ void __launch_bounds__(256) query_kernel(Segs sg, const float* bias, float* out, int N, int B,
                                                    const int* done_at, const int* g_step) {
  const int n = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  const int b0 = blockIdx.y * kRowsPerWarp, step = *g_step;
  if (n >= N) return;
  bool act[kRowsPerWarp];
  rows_active(B, done_at, step, b0, act);
  const int wrow[1] = {n};
  float acc[1][kRowsPerWarp];
  dot_rows<1>(sg, wrow, b0, act, acc);
#pragma unroll
  for (int r = 0; r < kRowsPerWarp; ++r)
    if (lane == r && act[r]) out[(size_t)(b0 + r) * N + n] = fmaxf(acc[0][r] + bias[n], 0.0f);
}

// MoL attention (mol_attention.py:76-118, eval): mixture parameters from the query hidden q, phi at j = k + 0.5 for
// k = 0..T_enc (fp32, the reference's order: sum over m = 0..4, then the adjacent difference), alpha == 0 -> 1e-5,
// context = alpha . memory.  grid B, block 256, dynamic smem (2 * Te_buf + 1) floats
__global__ void __launch_bounds__(256) mol_attention_kernel(const float* q, const float* W2, const float* b2,
                                                            float* mu_state, const float* memory, int Te_buf,
                                                            const int* tenc, const int* done_at, const int* g_step,
                                                            float* ctx, float* align, int S) {
  extern __shared__ float sm[];
  float* phi = sm;
  float* alpha = sm + Te_buf + 1;
  __shared__ float prm[3 * kM], mw[kM], msig[kM], mmu[kM];
  const int b = blockIdx.x, tid = threadIdx.x, step = *g_step;
  if (!row_active(done_at, b, step)) return;
  const int warp = tid >> 5, lane = tid & 31;
  for (int o = warp; o < 3 * kM; o += 8) {
    float s = 0.0f;
#pragma unroll
    for (int i = 0; i < kQ / 32; ++i) s += W2[o * kQ + lane + 32 * i] * q[(size_t)b * kQ + lane + 32 * i];
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) s += __shfl_xor_sync(0xffffffffu, s, d);
    if (lane == 0) prm[o] = s + b2[o];
  }
  __syncthreads();
  if (tid == 0) {
    float mx = prm[0];
    for (int m = 1; m < kM; ++m) mx = fmaxf(mx, prm[m]);
    float e[kM], sum = 0.0f;
    for (int m = 0; m < kM; ++m) {
      e[m] = expf(prm[m] - mx);
      sum += e[m];
    }
    for (int m = 0; m < kM; ++m) {
      mw[m] = e[m] / sum + 1e-5f;
      msig[m] = softplusf_(prm[kM + m]) + 1e-5f;
      const float mu = mu_state[b * 8 + m] + softplusf_(prm[2 * kM + m]);
      mmu[m] = mu;
      mu_state[b * 8 + m] = mu;
    }
  }
  __syncthreads();
  const int Te = tenc[b];
  for (int j = tid; j <= Te; j += 256) {
    const float jv = (float)j + 0.5f;
    float a = 0.0f;
#pragma unroll
    for (int m = 0; m < kM; ++m) {
      const float sgm = 1.0f / (1.0f + expf(-((mmu[m] - jv) / msig[m])));
      a += mw[m] * (1.0f / (1.0f + sgm));
    }
    phi[j] = a;
  }
  __syncthreads();
  float* arow = align + ((size_t)b * S + step) * Te_buf;
  for (int j = tid; j < Te; j += 256) {
    float a = phi[j + 1] - phi[j];
    if (a == 0.0f) a = 1e-5f;
    alpha[j] = a;
    arow[j] = a;
  }
  __syncthreads();
  const float* mb = memory + (size_t)b * Te_buf * kE + tid;
  float c = 0.0f;
  for (int j = 0; j < Te; ++j) c += alpha[j] * mb[(size_t)j * kE];
  ctx[(size_t)b * kE + tid] = c;
}

// mel = W [h | ctx] + b (160 = 2 frames), stop = w [h | ctx] + b, and the stop / freeze rule of
// rnn_decoder_mol.py:303-307 for each row.  grid (ceil(161 / 8), ceil(B / 8)), block 256
__global__ void __launch_bounds__(256) proj_kernel(Segs sg, const float* Wstop, const float* bias, const float* bstop,
                                                   int B, int S, int* done_at, const int* tenc, int* steps, int* mel_len,
                                                   const int* g_step, float* mel, float* frame, float* stop_out) {
  const int n = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  const int b0 = blockIdx.y * kRowsPerWarp, step = *g_step;
  constexpr int N = kNM * kR;
  if (n > N) return;
  bool act[kRowsPerWarp];
  rows_active(B, done_at, step, b0, act);
  float acc[1][kRowsPerWarp];
  if (n < N) {
    const int wrow[1] = {n};
    dot_rows<1>(sg, wrow, b0, act, acc);
  } else {
    const float* base = sg.s[0].w;
    for (int i = 0; i < sg.n; ++i) {
      sg.s[i].w = Wstop + (sg.s[i].w - base);  // same column offsets in the [1][768] stop weight
      sg.s[i].ldw = 0;
    }
    const int wrow[1] = {0};
    dot_rows<1>(sg, wrow, b0, act, acc);
  }
#pragma unroll
  for (int r = 0; r < kRowsPerWarp; ++r) {
    if (lane != r || !act[r]) continue;
    const int b = b0 + r;
    if (n < N) {
      const float v = acc[0][r] + bias[n];
      mel[((size_t)b * (2 * S) + kR * step + n / kNM) * kNM + n % kNM] = v;
      if (n >= N - kNM) frame[(size_t)b * kNM + n - (N - kNM)] = v;
    } else {
      const float v = acc[0][r] + bstop[0];
      if (stop_out) stop_out[(size_t)b * S + step] = v;
      const int ns = step + 1, mx = 2 * tenc[b], mn = mx - 5;
      if ((sigmoidf_(v) > 0.5f && ns >= mn) || ns >= mx) {
        done_at[b] = ns;
        steps[b] = ns;
        mel_len[b] = kR * ns;
      }
    }
  }
}

__global__ void step_end_kernel(State s, int B) {
  const int step = *s.g_step;
  bool done = true;
  for (int b = threadIdx.x; b < B; b += blockDim.x) done &= s.done_at[b] <= step + 1;
  done = __syncthreads_and(done);
  if (threadIdx.x == 0) {
    *s.flag = done ? 1 : 0;
    *s.g_step = step + 1;
  }
}

__global__ void transpose_kernel(const float* src, float* dst, int rows, int cols) {  // dst[c][r] = src[r][c]
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= rows * cols) return;
  const int r = i / cols, c = i - r * cols;
  dst[(size_t)c * rows + r] = src[i];
}

__global__ void add_kernel(const float* a, const float* b, float* dst, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) dst[i] = a[i] + b[i];
}

}  // namespace

struct mb_ppg2mel {
  mb_ppg2mel_config cfg{};
  WeightTable w;
  size_t total_floats = 0;
  size_t d_w1t = 0, d_w2t = 0, d_att_b = 0, d_dec_b = 0;
  float* arena = nullptr;
  bool finalized = false;
  cudaStream_t st = nullptr;
  cudaEvent_t ev_in = nullptr, ev_out = nullptr;

  const float* p(const std::string& name) const { return w.ptr(name); }
};

namespace {

void build_specs(mb_ppg2mel* h) {
  const int D = h->cfg.bottle_neck_feature_dim, Ds = h->cfg.spk_embed_dim;
  for (const char* br : {"bnf_prenet", "pitch_convs"}) {
    const std::string b = br;
    h->w.add(b + ".0.weight", {kE, b == "bnf_prenet" ? D : 2, 1});
    for (const char* i : {".3", ".6"}) {
      h->w.add(b + i + ".weight", {kE, kE, 4});
      h->w.add(b + i + ".bias", {kE});
    }
  }
  h->w.add("reduce_proj.weight", {kE, kE + Ds});
  h->w.add("reduce_proj.bias", {kE});
  h->w.add("decoder.prenet.layers.0.linear_layer.weight", {kP1, kNM});
  h->w.add("decoder.prenet.layers.1.linear_layer.weight", {kP2, kP1});
  for (const auto& pr : {std::make_pair("decoder.attention_rnn", kP2 + kE),
                         std::make_pair("decoder.decoder_rnn_layers.0", kH + kE)}) {
    const std::string b = pr.first;
    h->w.add(b + ".weight_ih", {4 * kH, pr.second});
    h->w.add(b + ".weight_hh", {4 * kH, kH});
    h->w.add(b + ".bias_ih", {4 * kH});
    h->w.add(b + ".bias_hh", {4 * kH});
  }
  h->w.add("decoder.attention_layer.query_layer.0.weight", {kQ, kH});
  h->w.add("decoder.attention_layer.query_layer.0.bias", {kQ});
  h->w.add("decoder.attention_layer.query_layer.2.weight", {3 * kM, kQ});
  h->w.add("decoder.attention_layer.query_layer.2.bias", {3 * kM});
  h->w.add("decoder.linear_projection.linear_layer.weight", {kNM * kR, kH + kE});
  h->w.add("decoder.linear_projection.linear_layer.bias", {kNM * kR});
  h->w.add("decoder.stop_layer.linear_layer.weight", {1, kH + kE});
  h->w.add("decoder.stop_layer.linear_layer.bias", {1});
  const int ch[6] = {kNM, 512, 512, 512, 512, kNM};
  for (int i = 0; i < 5; ++i) {
    const std::string b = "postnet.convolutions." + std::to_string(i);
    h->w.add(b + ".0.conv.weight", {ch[i + 1], ch[i], 5});
    h->w.add(b + ".0.conv.bias", {ch[i + 1]});
    for (const char* leaf : {".1.weight", ".1.bias", ".1.running_mean", ".1.running_var"}) h->w.add(b + leaf, {ch[i + 1]});
  }
  // the model's own derived region follows the table
  size_t off = h->w.floats();
  h->d_w1t = off;
  off += mb::align_up((size_t)kNM * kP1, 64);
  h->d_w2t = off;
  off += mb::align_up((size_t)kP1 * kP2, 64);
  h->d_att_b = off;
  off += 4 * kH;
  h->d_dec_b = off;
  off += 4 * kH;
  h->total_floats = off;
}

// per-call workspace layout (bytes, 256-aligned regions)
struct WsLayout {
  size_t ints, rowbias, x0, x1, e1, e2, mem, ah, ac, dh, dc, ctx, mu, frame, pre, q, p0, p1, total;
};

WsLayout ws_layout(int B, int T) {
  WsLayout L{};
  const size_t T1 = T / 2, T2 = T1 / 2, S = 2 * T2;
  size_t o = 0;
  auto take = [&](size_t floats) {
    const size_t r = o;
    o += mb::align_up(floats * 4, 256);
    return r;
  };
  L.ints = take(8 * kMaxRows + 8);
  L.rowbias = take((size_t)B * kE);
  L.x0 = take((size_t)B * T * kE);
  L.x1 = take((size_t)B * T1 * kE);
  L.e1 = take((size_t)B * T2 * kE);
  L.e2 = take((size_t)B * T2 * kE);
  L.mem = take((size_t)B * T2 * kE);
  L.ah = take((size_t)2 * B * kH);
  L.ac = take((size_t)B * kH);
  L.dh = take((size_t)2 * B * kH);
  L.dc = take((size_t)B * kH);
  L.ctx = take((size_t)B * kE);
  L.mu = take((size_t)B * 8);
  L.frame = take((size_t)B * kNM);
  L.pre = take((size_t)B * kP2);
  L.q = take((size_t)B * kQ);
  L.p0 = take((size_t)B * 2 * S * 512);
  L.p1 = take((size_t)B * 2 * S * 512);
  L.total = o;
  return L;
}

int launch_conv(const ConvP& p, cudaStream_t st) {
  const int M = p.B * p.T_out;
  if (M <= 0) return MB_OK;
  dim3 grid((M + kBM - 1) / kBM, (p.N + kBN - 1) / kBN);
  conv_gemm_kernel<<<grid, 256, 0, st>>>(p);
  MB_LAUNCH_CHECK("conv_gemm_kernel");
  return MB_OK;
}

ConvP conv_base(int B) {
  ConvP p{};
  p.B = B;
  p.stride = 1;
  p.ks = 1;
  return p;
}

int launch_in(float* x, int T, const int* len, const float* add, int B, cudaStream_t st) {
  instance_norm_kernel<<<dim3(kE / 32, B), dim3(32, 8), 0, st>>>(x, T, kE, len, add);
  MB_LAUNCH_CHECK("instance_norm_kernel");
  return MB_OK;
}

// dynamic shared memory of mol_attention_kernel: phi [Te_buf + 1] and alpha [Te_buf]
size_t att_smem_bytes(int Te_buf) { return sizeof(float) * (2 * (size_t)Te_buf + 1); }

// largest Te_buf whose attention shared memory fits one block: the device's opt-in limit less the kernel's static
// arrays, queried once per device; 0 (with a message) when the device cannot be queried
int max_att_tenc() {
  constexpr int kMaxDevices = 64;
  static std::atomic<int> cached[kMaxDevices];
  int dev = 0, optin = 0;
  cudaFuncAttributes fa{};
  if (cudaGetDevice(&dev) != cudaSuccess) {
    const cudaError_t e = cudaGetLastError();
    fail(MB_ERR_CUDA, "ppg2mel: no current device for the attention's shared-memory limit: %s", cudaGetErrorString(e));
    return 0;
  }
  if (dev < kMaxDevices) {
    const int te = cached[dev].load(std::memory_order_relaxed);
    if (te > 0) return te;
  }
  if (cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev) != cudaSuccess ||
      cudaFuncGetAttributes(&fa, mol_attention_kernel) != cudaSuccess) {
    const cudaError_t e = cudaGetLastError();
    fail(MB_ERR_CUDA, "ppg2mel: cannot query the attention kernel's shared-memory limit: %s", cudaGetErrorString(e));
    return 0;
  }
  const size_t room = (size_t)optin - fa.sharedSizeBytes;
  int te = (int)((room / sizeof(float) - 1) / 2);
  while (te > 0 && att_smem_bytes(te) > room) --te;
  while (att_smem_bytes(te + 1) <= room) ++te;
  if (dev < kMaxDevices) cached[dev].store(te, std::memory_order_relaxed);
  return te;
}

#define MB_TRY(x)               \
  do {                          \
    const int _rc = (x);        \
    if (_rc != MB_OK) return _rc; \
  } while (0)

}  // namespace

extern "C" {

int mb_ppg2mel_create(const mb_ppg2mel_config* cfg, mb_ppg2mel** out) {
  if (!cfg || !out) return fail(MB_ERR_INVALID, "mb_ppg2mel_create: null argument");
  const mb_ppg2mel_config& c = *cfg;
  if (c.bottle_neck_feature_dim < 1 || c.bottle_neck_feature_dim > 1024)
    return fail(MB_ERR_INVALID, "mb_ppg2mel_create: bottle_neck_feature_dim %d outside 1..1024", c.bottle_neck_feature_dim);
  if (c.spk_embed_dim < 1 || c.spk_embed_dim > 1024)
    return fail(MB_ERR_INVALID, "mb_ppg2mel_create: spk_embed_dim %d outside 1..1024", c.spk_embed_dim);
  struct {
    const char* name;
    int got, want;
  } fixed[] = {{"encoder_dim", c.encoder_dim, kE},
               {"encoder_downsample_rates[0]", c.encoder_downsample_rates[0], 2},
               {"encoder_downsample_rates[1]", c.encoder_downsample_rates[1], 2},
               {"attention_rnn_dim", c.attention_rnn_dim, kH},
               {"decoder_rnn_dim", c.decoder_rnn_dim, kH},
               {"num_decoder_rnn_layer", c.num_decoder_rnn_layer, 1},
               {"concat_context_to_last", c.concat_context_to_last, 1},
               {"prenet_dims[0]", c.prenet_dims[0], kP1},
               {"prenet_dims[1]", c.prenet_dims[1], kP2},
               {"num_mixtures", c.num_mixtures, kM},
               {"frames_per_step", c.frames_per_step, kR},
               {"num_mels", c.num_mels, kNM}};
  for (const auto& f : fixed)
    if (f.got != f.want)
      return fail(MB_ERR_INVALID, "mb_ppg2mel_create: %s = %d is not supported (the kernels are built for %d)", f.name,
                  f.got, f.want);
  auto* h = new mb_ppg2mel();
  h->cfg = c;
  build_specs(h);
  h->w.ignored = [](const std::string& n) {  // in the checkpoint, never read by inference
    return n.rfind("decoder.prenet_pitch.", 0) == 0 || n.find("num_batches_tracked") != std::string::npos;
  };
  *out = h;
  return MB_OK;
}

void mb_ppg2mel_destroy(mb_ppg2mel* h) {
  if (!h) return;
  if (h->ev_in) cudaEventDestroy(h->ev_in);
  if (h->ev_out) cudaEventDestroy(h->ev_out);
  if (h->st) cudaStreamDestroy(h->st);
  delete h;
}

size_t mb_ppg2mel_arena_bytes(const mb_ppg2mel* h) { return h ? h->total_floats * sizeof(float) : 0; }

int mb_ppg2mel_set_arena(mb_ppg2mel* h, void* arena, size_t bytes) {
  if (int rc = check_arena("mb_ppg2mel_set_arena", h, arena, bytes, mb_ppg2mel_arena_bytes(h), 256)) return rc;
  h->w.attach(static_cast<float*>(arena));
  h->arena = static_cast<float*>(arena);
  h->finalized = false;
  return MB_OK;
}

int mb_ppg2mel_set_weight(mb_ppg2mel* h, const char* name, const float* w, const int64_t* dims, int32_t ndim,
                          void* stream) {
  if (!h) return fail(MB_ERR_INVALID, "mb_ppg2mel_set_weight: null argument");
  if (int rc = h->w.set("mb_ppg2mel_set_weight", name, w, dims, ndim, stream)) return rc;
  h->finalized = false;
  return MB_OK;
}

int mb_ppg2mel_finalize(mb_ppg2mel* h, void* stream) {
  if (!h) return fail(MB_ERR_INVALID, "mb_ppg2mel_finalize: null handle");
  if (int rc = h->w.check_all_set("mb_ppg2mel_finalize")) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  float* A = h->arena;
  transpose_kernel<<<(kP1 * kNM + 255) / 256, 256, 0, st>>>(h->p("decoder.prenet.layers.0.linear_layer.weight"),
                                                            A + h->d_w1t, kP1, kNM);
  MB_LAUNCH_CHECK("transpose_kernel");
  transpose_kernel<<<(kP2 * kP1 + 255) / 256, 256, 0, st>>>(h->p("decoder.prenet.layers.1.linear_layer.weight"),
                                                            A + h->d_w2t, kP2, kP1);
  MB_LAUNCH_CHECK("transpose_kernel");
  add_kernel<<<(4 * kH + 255) / 256, 256, 0, st>>>(h->p("decoder.attention_rnn.bias_ih"),
                                                   h->p("decoder.attention_rnn.bias_hh"), A + h->d_att_b, 4 * kH);
  MB_LAUNCH_CHECK("add_kernel");
  add_kernel<<<(4 * kH + 255) / 256, 256, 0, st>>>(h->p("decoder.decoder_rnn_layers.0.bias_ih"),
                                                   h->p("decoder.decoder_rnn_layers.0.bias_hh"), A + h->d_dec_b, 4 * kH);
  MB_LAUNCH_CHECK("add_kernel");
  h->finalized = true;
  return MB_OK;
}

size_t mb_ppg2mel_workspace_bytes(const mb_ppg2mel* h, int32_t batch, int32_t frames) {
  if (!h || batch < 1 || frames < 4) return 0;
  int dev = 0;
  if (cudaGetDevice(&dev) == cudaSuccess) {  // without a device nothing can run: the size alone is still answered
    const int te_max = max_att_tenc();
    if (te_max == 0) return 0;  // the query failed: mb_last_error says why
    if (frames / 4 > te_max) {
      fail(MB_ERR_INVALID, "mb_ppg2mel_workspace_bytes: frames %d gives T_enc %d > %d, the most the MoL attention's shared "
           "memory holds (frames <= %d)", frames, frames / 4, te_max, 4 * te_max + 3);
      return 0;
    }
  } else {
    cudaGetLastError();
  }
  return ws_layout(batch, frames).total;
}

int mb_ppg2mel_inference(mb_ppg2mel* h, const float* ppg, const float* lf0_uv, const float* spk, const int32_t* lengths,
                         int32_t batch, int32_t frames, const uint8_t* mask1, const uint8_t* mask2, uint64_t seed,
                         float* mel, float* mel_post, float* align, float* stop, int32_t* steps_host, void* workspace,
                         size_t workspace_bytes, void* stream) {
  if (!h) return fail(MB_ERR_INVALID, "mb_ppg2mel_inference: null handle");
  if (!h->finalized) return fail(MB_ERR_STATE, "mb_ppg2mel_inference: weights not finalized");
  if (batch < 1 || batch > kMaxRows) return fail(MB_ERR_INVALID, "mb_ppg2mel_inference: batch %d outside 1..%d", batch, kMaxRows);
  if (frames < 4) return fail(MB_ERR_INVALID, "mb_ppg2mel_inference: frames %d < 4", frames);
  const int te_max = max_att_tenc();
  if (te_max == 0) return MB_ERR_CUDA;
  if (frames / 4 > te_max)
    return fail(MB_ERR_INVALID, "mb_ppg2mel_inference: frames %d gives T_enc %d > %d, the most the MoL attention's shared "
                "memory holds (frames <= %d)", frames, frames / 4, te_max, 4 * te_max + 3);
  if (!ppg || !lf0_uv || !spk || !lengths || !mel || !mel_post || !align || !steps_host || !workspace)
    return fail(MB_ERR_INVALID, "mb_ppg2mel_inference: null argument");
  if ((mask1 == nullptr) != (mask2 == nullptr))
    return fail(MB_ERR_INVALID, "mb_ppg2mel_inference: pass both dropout masks or neither");
  Lens lens{};
  for (int b = 0; b < batch; ++b) {
    if (lengths[b] < 4 || lengths[b] > frames)
      return fail(MB_ERR_INVALID, "mb_ppg2mel_inference: lengths[%d] = %d outside 4..%d", b, lengths[b], frames);
    lens.v[b] = lengths[b];
  }
  const WsLayout L = ws_layout(batch, frames);
  if (workspace_bytes < L.total) return fail(MB_ERR_WORKSPACE, "mb_ppg2mel_inference: workspace too small");
  const int B = batch, T = frames, T1 = T / 2, T2 = T1 / 2, S = 2 * T2;
  const int Dp = h->cfg.bottle_neck_feature_dim, Ds = h->cfg.spk_embed_dim;
  char* ws = static_cast<char*>(workspace);
  auto F = [&](size_t off) { return reinterpret_cast<float*>(ws + off); };
  int* ints = reinterpret_cast<int*>(ws + L.ints);
  State s{ints, ints + kMaxRows, ints + 2 * kMaxRows, ints + 3 * kMaxRows, ints + 4 * kMaxRows, ints + 5 * kMaxRows,
          ints + 6 * kMaxRows, ints + 6 * kMaxRows + 1};

  if (!h->st) {
    MB_CUDA_CHECK(cudaStreamCreateWithFlags(&h->st, cudaStreamNonBlocking));
    MB_CUDA_CHECK(cudaEventCreateWithFlags(&h->ev_in, cudaEventDisableTiming));
    MB_CUDA_CHECK(cudaEventCreateWithFlags(&h->ev_out, cudaEventDisableTiming));
  }
  cudaStream_t caller = static_cast<cudaStream_t>(stream);
  cudaStream_t st = h->st;
  MB_CUDA_CHECK(cudaEventRecord(h->ev_in, caller));
  MB_CUDA_CHECK(cudaStreamWaitEvent(st, h->ev_in, 0));

  // ------------------------------------------------------------------ outputs and recurrent state start at zero
  MB_CUDA_CHECK(cudaMemsetAsync(mel, 0, sizeof(float) * B * 2 * S * kNM, st));
  MB_CUDA_CHECK(cudaMemsetAsync(mel_post, 0, sizeof(float) * B * 2 * S * kNM, st));
  MB_CUDA_CHECK(cudaMemsetAsync(align, 0, sizeof(float) * B * S * T2, st));
  if (stop) MB_CUDA_CHECK(cudaMemsetAsync(stop, 0, sizeof(float) * B * S, st));
  MB_CUDA_CHECK(cudaMemsetAsync(ws + L.ah, 0, L.p0 - L.ah, st));
  init_state_kernel<<<1, kMaxRows, 0, st>>>(lens, B, s);
  MB_LAUNCH_CHECK("init_state_kernel");

  // ------------------------------------------------------------------ encoder (__init__.py:172-180)
  spk_bias_kernel<<<B, 256, 0, st>>>(spk, Ds, h->p("reduce_proj.weight"), kE + Ds, h->p("reduce_proj.bias"),
                                     F(L.rowbias));
  MB_LAUNCH_CHECK("spk_bias_kernel");
  for (int br = 0; br < 2; ++br) {
    const std::string pre = br == 0 ? "bnf_prenet" : "pitch_convs";
    const int Cin = br == 0 ? Dp : 2;
    float* out = br == 0 ? F(L.e1) : F(L.e2);
    ConvP p = conv_base(B);
    p.x = br == 0 ? ppg : lf0_uv;
    p.xT = T, p.ldx = Cin, p.Cin = Cin, p.len_in = s.len0;
    p.w = h->p((pre + ".0.weight").c_str()), p.ldw = Cin;
    p.act = 1;
    p.y = F(L.x0), p.yT = T, p.ldy = kE, p.N = kE, p.T_out = T, p.len_out = s.len0;
    MB_TRY(launch_conv(p, st));
    MB_TRY(launch_in(F(L.x0), T, s.len0, nullptr, B, st));
    for (int layer = 0; layer < 2; ++layer) {
      const std::string wn = pre + (layer == 0 ? ".3" : ".6");
      ConvP c = conv_base(B);
      c.x = layer == 0 ? F(L.x0) : F(L.x1);
      c.xT = layer == 0 ? T : T1, c.ldx = kE, c.Cin = kE, c.len_in = layer == 0 ? s.len0 : s.len1;
      c.stride = 2, c.pad = 1, c.ks = 4;
      c.w = h->p((wn + ".weight").c_str()), c.ldw = kE * 4;
      c.bias = h->p((wn + ".bias").c_str());
      c.act = 1;
      c.y = layer == 0 ? F(L.x1) : out, c.yT = layer == 0 ? T1 : T2, c.ldy = kE, c.N = kE;
      c.T_out = layer == 0 ? T1 : T2, c.len_out = layer == 0 ? s.len1 : s.tenc;
      MB_TRY(launch_conv(c, st));
      const bool last = layer == 1;
      MB_TRY(launch_in(c.y, c.yT, c.len_out, (last && br == 1) ? F(L.e1) : nullptr, B, st));
    }
  }
  {
    ConvP p = conv_base(B);
    p.x = F(L.e2), p.xT = T2, p.ldx = kE, p.Cin = kE, p.len_in = s.tenc;
    p.w = h->p("reduce_proj.weight"), p.ldw = kE + Ds;
    p.bias = F(L.rowbias), p.bias_ld = kE;
    p.y = F(L.mem), p.yT = T2, p.ldy = kE, p.N = kE, p.T_out = T2, p.len_out = s.tenc;
    MB_TRY(launch_conv(p, st));
  }

  // ------------------------------------------------------------------ decoder loop (rnn_decoder_mol.py:286-309)
  float* ah[2] = {F(L.ah), F(L.ah) + (size_t)B * kH};
  float* dh[2] = {F(L.dh), F(L.dh) + (size_t)B * kH};
  const dim3 rows_grid_h(kH / 8, (B + kRowsPerWarp - 1) / kRowsPerWarp);
  const size_t att_smem = att_smem_bytes(T2);
  if (att_smem > 48 * 1024)
    MB_CUDA_CHECK(cudaFuncSetAttribute(mol_attention_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)att_smem));
  const float* A = h->arena;
  auto emit_step = [&](int parity) -> int {
    const float* ah_in = ah[parity];
    float* ah_out = ah[parity ^ 1];
    const float* dh_in = dh[parity];
    float* dh_out = dh[parity ^ 1];
    prenet_kernel<<<B, 256, 0, st>>>(F(L.frame), A + h->d_w1t, A + h->d_w2t, mask1, mask2, seed, B, s.done_at, s.g_step,
                                     F(L.pre));
    MB_LAUNCH_CHECK("prenet_kernel");
    Segs a{};
    a.s[0] = {F(L.pre), kP2, kP2, h->p("decoder.attention_rnn.weight_ih"), kP2 + kE};
    a.s[1] = {F(L.ctx), kE, kE, h->p("decoder.attention_rnn.weight_ih") + kP2, kP2 + kE};
    a.s[2] = {nullptr, kH, kH, h->p("decoder.attention_rnn.weight_hh"), kH};
    a.n = 2;
    lstm_kernel<<<rows_grid_h, 256, 0, st>>>(a, A + h->d_att_b, ah_in, ah_out, F(L.ac), B, s.done_at, s.g_step);
    MB_LAUNCH_CHECK("lstm_kernel");
    Segs q{};
    q.s[0] = {ah_out, kH, kH, h->p("decoder.attention_layer.query_layer.0.weight"), kH};
    q.n = 1;
    query_kernel<<<dim3(kQ / 8, rows_grid_h.y), 256, 0, st>>>(q, h->p("decoder.attention_layer.query_layer.0.bias"),
                                                              F(L.q), kQ, B, s.done_at, s.g_step);
    MB_LAUNCH_CHECK("query_kernel");
    mol_attention_kernel<<<B, 256, att_smem, st>>>(F(L.q), h->p("decoder.attention_layer.query_layer.2.weight"),
                                                   h->p("decoder.attention_layer.query_layer.2.bias"), F(L.mu), F(L.mem),
                                                   T2, s.tenc, s.done_at, s.g_step, F(L.ctx), align, S);
    MB_LAUNCH_CHECK("mol_attention_kernel");
    Segs d{};
    d.s[0] = {ah_out, kH, kH, h->p("decoder.decoder_rnn_layers.0.weight_ih"), kH + kE};
    d.s[1] = {F(L.ctx), kE, kE, h->p("decoder.decoder_rnn_layers.0.weight_ih") + kH, kH + kE};
    d.s[2] = {nullptr, kH, kH, h->p("decoder.decoder_rnn_layers.0.weight_hh"), kH};
    d.n = 2;
    lstm_kernel<<<rows_grid_h, 256, 0, st>>>(d, A + h->d_dec_b, dh_in, dh_out, F(L.dc), B, s.done_at, s.g_step);
    MB_LAUNCH_CHECK("lstm_kernel");
    Segs pj{};
    pj.s[0] = {dh_out, kH, kH, h->p("decoder.linear_projection.linear_layer.weight"), kH + kE};
    pj.s[1] = {F(L.ctx), kE, kE, h->p("decoder.linear_projection.linear_layer.weight") + kH, kH + kE};
    pj.n = 2;
    proj_kernel<<<dim3((kNM * kR + 1 + 7) / 8, rows_grid_h.y), 256, 0, st>>>(
        pj, h->p("decoder.stop_layer.linear_layer.weight"), h->p("decoder.linear_projection.linear_layer.bias"),
        h->p("decoder.stop_layer.linear_layer.bias"), B, S, s.done_at, s.tenc, s.steps, s.mel_len, s.g_step, mel,
        F(L.frame), stop);
    MB_LAUNCH_CHECK("proj_kernel");
    step_end_kernel<<<1, kMaxRows, 0, st>>>(s, B);
    MB_LAUNCH_CHECK("step_end_kernel");
    return MB_OK;
  };

  cudaGraph_t graph = nullptr;
  cudaGraphExec_t exec = nullptr;
  const uint64_t before = mb_launch_count();
  MB_CUDA_CHECK(cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal));
  int rc = MB_OK;
  for (int j = 0; j < kGroup && rc == MB_OK; ++j) rc = emit_step(j & 1);
  const cudaError_t ec = cudaStreamEndCapture(st, &graph);
  const int per_graph = (int)(mb_launch_count() - before);
  mb::count_launch(-per_graph);  // captured, not launched; every replay below counts them
  if (rc != MB_OK) {
    if (graph) cudaGraphDestroy(graph);
    return rc;
  }
  if (ec != cudaSuccess || !graph) return fail(MB_ERR_CUDA, "mb_ppg2mel_inference: graph capture failed: %s", cudaGetErrorString(ec));
  if (cudaGraphInstantiate(&exec, graph, 0) != cudaSuccess) {
    cudaGraphDestroy(graph);
    return fail(MB_ERR_CUDA, "mb_ppg2mel_inference: cudaGraphInstantiate failed");
  }
  int flag = 0;
  const int groups = (S + kGroup - 1) / kGroup;
  for (int g = 0; g < groups && !flag && rc == MB_OK; ++g) {
    if (cudaGraphLaunch(exec, st) != cudaSuccess) rc = fail(MB_ERR_CUDA, "mb_ppg2mel_inference: cudaGraphLaunch failed");
    mb::count_launch(per_graph);
    if (rc == MB_OK && cudaMemcpyAsync(&flag, s.flag, sizeof(int), cudaMemcpyDeviceToHost, st) != cudaSuccess)
      rc = fail(MB_ERR_CUDA, "mb_ppg2mel_inference: flag copy failed");
    if (rc == MB_OK && cudaStreamSynchronize(st) != cudaSuccess)
      rc = fail(MB_ERR_CUDA, "mb_ppg2mel_inference: decoder step failed: %s", cudaGetErrorString(cudaGetLastError()));
  }
  cudaGraphExecDestroy(exec);
  cudaGraphDestroy(graph);
  if (rc != MB_OK) return rc;
  if (!flag) return fail(MB_ERR_STATE, "mb_ppg2mel_inference: rows still running after the step limit");
  MB_CUDA_CHECK(cudaMemcpy(steps_host, s.steps, sizeof(int) * B, cudaMemcpyDeviceToHost));
  int nmax = 0;
  for (int b = 0; b < B; ++b) nmax = steps_host[b] > nmax ? steps_host[b] : nmax;

  // ------------------------------------------------------------------ postnet (cnn_postnet.py:47-52) + residual
  const int Tp = kR * nmax;
  const float* xin = mel;
  float* bufs[2] = {F(L.p0), F(L.p1)};
  for (int i = 0; i < 5; ++i) {
    const std::string b = "postnet.convolutions." + std::to_string(i);
    const int Cin = i == 0 ? kNM : 512, Cout = i == 4 ? kNM : 512;
    ConvP p = conv_base(B);
    p.x = xin, p.xT = 2 * S, p.ldx = Cin, p.Cin = Cin, p.len_in = s.mel_len;
    p.pad = 2, p.ks = 5;
    p.w = h->p((b + ".0.conv.weight").c_str()), p.ldw = Cin * 5;
    p.bias = h->p((b + ".0.conv.bias").c_str());
    p.bn_mean = h->p((b + ".1.running_mean").c_str()), p.bn_var = h->p((b + ".1.running_var").c_str());
    p.bn_w = h->p((b + ".1.weight").c_str()), p.bn_b = h->p((b + ".1.bias").c_str());
    p.act = i < 4 ? 2 : 0;
    p.res = i == 4 ? mel : nullptr;
    p.y = i == 4 ? mel_post : bufs[i & 1], p.yT = 2 * S, p.ldy = Cout, p.N = Cout, p.T_out = Tp, p.len_out = s.mel_len;
    MB_TRY(launch_conv(p, st));
    xin = p.y;
  }
  MB_CUDA_CHECK(cudaEventRecord(h->ev_out, st));
  MB_CUDA_CHECK(cudaStreamWaitEvent(caller, h->ev_out, 0));
  return MB_OK;
}

}  // extern "C"
