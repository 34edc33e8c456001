// fatchord WaveRNN on H100: conditioning network + the persistent, weight-stationary sample loop.
//
// reference: models/vocoder/wavernn/models/fatchord_version.py
//   UpsampleNetwork / MelResNet :27-85, sample loop of WaveRNN.generate :176-234
//
// Sample loop design (SURVEY.md section 7, hard part 2): 8.14 MFLOP and 16.3 MB of FP32 weights per
// sample-row, ~9k strictly sequential steps, only a few dozen rows (folds).  The weights are made
// STATIONARY: 128 persistent CTAs (one per SM, cooperative launch) each own 4 of the 512 units of
// every layer and keep their 120 KB weight slice in shared memory for the whole call.  Per step the
// CTAs exchange the [512 x rows] activation matrices through L2-resident global buffers laid out
// [unit][row] (so every consumer reads them with coalesced 16-byte loads) and meet at 6 grid barriers
// (after rnn1, rnn2, fc1, fc2, fc3, sampling).  All arithmetic is FP32 FFMA in a fixed, documented
// order (k-slices -> pair sum -> binary tree; include/mb_wavernn_math.h for exp/sigmoid/tanh) so that
// the CPU twin (oracle/wavernn_twin.c) reproduces every logit and therefore every sample bit for
// bit.  Tensor cores are deliberately not used here: fp16/tf32 operand rounding (1e-3) would flip
// ~0.1-1% of the argmax(p/q) draws (SURVEY.md section 7), FP32 keeps the integer samples exact.
#include <cooperative_groups.h>
#include <cuda_runtime.h>

#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include "../../include/mb_wavernn_math.h"
#include "mb_common.h"

namespace cg = cooperative_groups;

namespace mb {
namespace {

constexpr int RNN = 512;
constexpr int NCLS = 512;
constexpr int AUXD = 32;
constexpr int FEAT = 80;
constexpr int CDIM = 128;
constexpr int HOP = 200;
constexpr int NCTA = 128;       // 4 units per CTA
constexpr int UPC = 4;          // units per CTA
constexpr int RB = 64;          // rows per row block
constexpr int kThreads = 512;

// ------------------------------------------------------------------------------------------------
// conditioning kernels: one thread per output, sequential fmaf chains in the twin's order
// ------------------------------------------------------------------------------------------------
__global__ void k_conv_in(const float* __restrict__ w, const float* __restrict__ mel, int T, float* __restrict__ y) {
  // y[o][t] = sum_{ci,k} w[o][ci][k] * P[ci][t+k],  P = mel padded by 2 zero frames on both sides
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= CDIM * T) return;
  const int o = i / T, t = i - o * T;
  float acc = 0.0f;
  for (int ci = 0; ci < FEAT; ++ci)
    for (int k = 0; k < 5; ++k) {
      const int s = t + k - 2;
      const float v = (s >= 0 && s < T) ? mel[ci * T + s] : 0.0f;
      acc = fmaf(w[(o * FEAT + ci) * 5 + k], v, acc);
    }
  y[i] = acc;
}

__global__ void k_bn(const float* __restrict__ g, const float* __restrict__ b, const float* __restrict__ mean,
                     const float* __restrict__ var, float* __restrict__ x, int T, int relu, const float* res) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= CDIM * T) return;
  const int c = i / T;
  const float invstd = 1.0f / sqrtf(var[c] + 1e-5f);
  const float alpha = g[c] * invstd;
  const float beta = b[c] - mean[c] * alpha;
  float v = fmaf(x[i], alpha, beta);
  if (relu && v < 0.0f) v = 0.0f;
  if (res) v = v + res[i];
  x[i] = v;
}

__global__ void k_conv1x1(const float* __restrict__ w, const float* __restrict__ x, int T, float* __restrict__ y,
                          const float* __restrict__ bias, int transpose_out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= CDIM * T) return;
  const int o = i / T, t = i - o * T;
  float acc = 0.0f;
  for (int c = 0; c < CDIM; ++c) acc = fmaf(w[o * CDIM + c], x[c * T + t], acc);
  if (bias) acc = acc + bias[o];
  if (transpose_out) y[t * CDIM + o] = acc;
  else y[i] = acc;
}

// one ladder stage: y[c][i] = sum_j w[j] * rep(x)[i + j - s]
__global__ void k_ladder(const float* __restrict__ w, const float* __restrict__ x, int len, int s,
                         float* __restrict__ y) {
  const int nl = len * s;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= FEAT * nl) return;
  const int c = i / nl, p = i - c * nl;
  float acc = 0.0f;
  for (int j = 0; j <= 2 * s; ++j) {
    const int src = p + j - s;
    const float v = (src >= 0 && src < nl) ? x[c * len + src / s] : 0.0f;
    acc = fmaf(w[j], v, acc);
  }
  y[i] = acc;
}

__global__ void k_pad_mel(const float* __restrict__ mel, int T, float* __restrict__ P) {
  const int Tp = T + 4;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= FEAT * Tp) return;
  const int c = i / Tp, t = i - c * Tp;
  P[i] = (t >= 2 && t < T + 2) ? mel[c * T + t - 2] : 0.0f;
}

__global__ void k_crop_melup(const float* __restrict__ y3, int len, int T, float* __restrict__ melup) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= HOP * T * FEAT) return;
  const int t = i / FEAT, c = i - t * FEAT;
  melup[i] = y3[c * len + t + 2 * HOP];
}

// frame-rate tables: out[f][g] = dot_seq(W[g][K0 : K0+32], aux[f][a0 : a0+32]) + bias[g]; row f == T is
// the "past the end" row (zero conditioning)
__global__ void k_aux_table(const float* __restrict__ W, int ld, int K0, const float* __restrict__ bias,
                            const float* __restrict__ aux, int a0, int T, int G, float* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (T + 1) * G) return;
  const int f = i / G, g = i - f * G;
  float acc = 0.0f;
  for (int j = 0; j < AUXD; ++j) {
    const float a = (f < T) ? aux[f * CDIM + a0 + j] : 0.0f;
    acc = fmaf(W[(size_t)g * ld + K0 + j], a, acc);
  }
  out[i] = acc + bias[g];
}

// per-chunk conditioning of the I layer in the exchange layout:
//   condI[i][u][r] = dot_seq(I_w[u][1:113], [melup[t]; aux[t/200][0:32]]) + I_b[u],  t = start[r] + step0 + i
__global__ void __launch_bounds__(256) k_condI(const float* __restrict__ I_w, const float* __restrict__ I_b,
                                               const float* __restrict__ melup, const float* __restrict__ aux,
                                               int T, const int* __restrict__ starts, int B, int Bpad, int step0,
                                               int nsteps, float* __restrict__ out) {
  __shared__ float c[FEAT + AUXD];
  const int r = blockIdx.x % Bpad;
  const int i = blockIdx.x / Bpad;
  if (i >= nsteps) return;
  const int t = (r < B) ? starts[r] + step0 + i : -1;
  const bool live = (t >= 0 && t < HOP * T);
  for (int j = threadIdx.x; j < FEAT + AUXD; j += blockDim.x) {
    float v = 0.0f;
    if (live) v = (j < FEAT) ? melup[(size_t)t * FEAT + j] : aux[(size_t)(t / HOP) * CDIM + (j - FEAT)];
    c[j] = v;
  }
  __syncthreads();
  for (int u = threadIdx.x; u < RNN; u += blockDim.x) {
    float acc = 0.0f;
    const float* wr = I_w + (size_t)u * 113 + 1;
    for (int j = 0; j < FEAT + AUXD; ++j) acc = fmaf(wr[j], c[j], acc);
    out[((size_t)i * RNN + u) * Bpad + r] = (r < B) ? acc + I_b[u] : 0.0f;
  }
}

// ------------------------------------------------------------------------------------------------
// the sample loop
// ------------------------------------------------------------------------------------------------
struct LoopParams {
  // packed per-CTA weights (global): see pack kernel
  const float* wpack;       // [NCTA][WPACK_FLOATS]
  const float* I0;          // [512]  I_w[:, 0]
  // frame-rate tables
  const float* aux2P;       // [T+1][1536]
  const float* aux3P;       // [T+1][512]
  const float* aux4P;       // [T+1][512]
  const float* condI;       // [nsteps][512][Bpad]
  const int* starts;        // [B]
  int T, B, Bpad, step0, nsteps, steps_total;
  // state / exchange buffers (global, [unit][Bpad])
  float* h1;                // [2][512][Bpad]
  float* h2;                // [2][512][Bpad]
  float* f1;                // [512][Bpad]
  float* f2;                // [512][Bpad]
  float* logits;            // [512][Bpad]
  float* xprev;             // [Bpad]
  const float* noise;       // [nsteps][noise_B][512] or nullptr (this call's rows are noise rows row0 .. row0+B)
  int noise_B, row0;        // row0: global fold index of local row 0 (fold sharding across GPUs)
  uint64_t seed;
  int16_t* out_idx;         // [B][steps_total]
  unsigned int* barrier;    // grid barrier counter / per-CTA epoch flags [NCTA] (zeroed by the host before launch)
  int flagbar;              // 1: flag barrier, 0: single atomic counter
};

// per-CTA weight pack (floats):
//   W1ih [512][12] | W1hh [512][12] | W2ih [512][12] | W2hh [512][12] | fc1 [512][4] | fc2 [512][4] | fc3 [512][4]
//   | b1ih[12] b1hh[12] b2hh[12] fc3b[4] (aux tables carry b2ih / fc1b / fc2b)
constexpr int OFF_W1IH = 0;
constexpr int OFF_W1HH = OFF_W1IH + RNN * 12;
constexpr int OFF_W2IH = OFF_W1HH + RNN * 12;
constexpr int OFF_W2HH = OFF_W2IH + RNN * 12;
constexpr int OFF_FC1 = OFF_W2HH + RNN * 12;
constexpr int OFF_FC2 = OFF_FC1 + RNN * 4;
constexpr int OFF_FC3 = OFF_FC2 + RNN * 4;
constexpr int OFF_B1IH = OFF_FC3 + RNN * 4;
constexpr int OFF_B1HH = OFF_B1IH + 12;
constexpr int OFF_B2HH = OFF_B1HH + 12;
constexpr int OFF_FC3B = OFF_B2HH + 12;
constexpr int WPACK_FLOATS = ((OFF_FC3B + 4 + 31) / 32) * 32;   // 30784 floats = 123 KB
constexpr int SCRATCH_FLOATS = 2 * 8 * RB * 12;                  // [matrix][slice][row][col] = 12288 floats = 48 KB
constexpr int SMEM_FLOATS = WPACK_FLOATS + SCRATCH_FLOATS + RNN + NCLS; // + I0 + this step's noise row (prefetched)

struct PackSrc {
  const float *r1_wih, *r1_whh, *r1_bih, *r1_bhh, *r2_wih, *r2_whh, *r2_bhh, *fc1_w, *fc2_w, *fc3_w, *fc3_b;
};

__global__ void k_pack(PackSrc s, float* __restrict__ wpack) {
  const int c = blockIdx.x;
  float* dst = wpack + (size_t)c * WPACK_FLOATS;
  for (int i = threadIdx.x; i < WPACK_FLOATS; i += blockDim.x) {
    float v = 0.0f;
    if (i < OFF_FC1) {
      const int m = i / (RNN * 12);
      const int rem = i - m * RNN * 12;
      const int k = rem / 12, col = rem - k * 12;
      const int g = col / 4, j = col - g * 4;
      const int row = g * RNN + c * UPC + j;
      const float* W = (m == 0) ? s.r1_wih : (m == 1) ? s.r1_whh : (m == 2) ? s.r2_wih : s.r2_whh;
      const int ld = (m == 2) ? (RNN + AUXD) : RNN;
      v = W[(size_t)row * ld + k];
    } else if (i < OFF_B1IH) {
      const int m = (i - OFF_FC1) / (RNN * 4);
      const int rem = (i - OFF_FC1) - m * RNN * 4;
      const int k = rem / 4, j = rem - k * 4;
      const int row = c * UPC + j;
      const float* W = (m == 0) ? s.fc1_w : (m == 1) ? s.fc2_w : s.fc3_w;
      const int ld = (m == 2) ? RNN : (RNN + AUXD);
      v = W[(size_t)row * ld + k];
    } else if (i < OFF_FC3B) {
      const int m = (i - OFF_B1IH) / 12;
      const int col = (i - OFF_B1IH) - m * 12;
      const int g = col / 4, j = col - g * 4;
      const float* b = (m == 0) ? s.r1_bih : (m == 1) ? s.r1_bhh : s.r2_bhh;
      v = b[g * RNN + c * UPC + j];
    } else if (i < OFF_FC3B + 4) {
      v = s.fc3_b[c * UPC + (i - OFF_FC3B)];
    }
    dst[i] = v;
  }
}

// Flag barrier (p.flagbar): every CTA publishes its epoch in its own word, threads 0..gridDim-1 of every CTA each poll one
// word - no 128-way serialised atomic on a single L2 line, the polls run in parallel.  The counter variant is kept for A/B.
__device__ __forceinline__ void grid_barrier_flags(unsigned int* flags, unsigned int& epoch) {
  __syncthreads();
  epoch += 1;
  if (threadIdx.x == 0) {
    __threadfence();
    asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(flags + blockIdx.x), "r"(epoch) : "memory");
  }
  if (threadIdx.x < gridDim.x) {
    unsigned int v;
    do {
      asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(flags + threadIdx.x) : "memory");
    } while (v < epoch);
    __threadfence();
  }
  __syncthreads();
}

__device__ __forceinline__ void grid_barrier_counter(unsigned int* counter, unsigned int& target) {
  __syncthreads();
  if (threadIdx.x == 0) {
    target += gridDim.x;
    __threadfence();
    atomicAdd(counter, 1u);
    unsigned int v;
    do {
      asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(counter) : "memory");
    } while (v < target);
    __threadfence();  // also invalidates this SM's L1 so the plain loads below see the new data
  }
  __syncthreads();
}

__device__ __forceinline__ void grid_barrier(const LoopParams& p, unsigned int& target) {
  if (p.flagbar) grid_barrier_flags(p.barrier, target);
  else grid_barrier_counter(p.barrier, target);
}

// 4 rows x NC columns register tile over the k-range [k0, k0+klen) of one matrix:
//   acc[rr][col] += W[k][col] * act(k, row 4*rt + rr)
template <int NC, class ActFn>
__device__ __forceinline__ void tile_gemv(const float* __restrict__ wsm /*[512][NC]*/, int k0, int klen, ActFn act,
                                          float (&acc)[4][NC]) {
#pragma unroll
  for (int rr = 0; rr < 4; ++rr)
#pragma unroll
    for (int cidx = 0; cidx < NC; ++cidx) acc[rr][cidx] = 0.0f;
#pragma unroll 4
  for (int kk = 0; kk < klen; ++kk) {
    const int k = k0 + kk;
    const float4 a = act(k);
    const float av[4] = {a.x, a.y, a.z, a.w};
    float wv[NC];
#pragma unroll
    for (int q = 0; q < NC / 4; ++q) {
      const float4 w4 = *reinterpret_cast<const float4*>(wsm + k * NC + q * 4);
      wv[q * 4 + 0] = w4.x; wv[q * 4 + 1] = w4.y; wv[q * 4 + 2] = w4.z; wv[q * 4 + 3] = w4.w;
    }
#pragma unroll
    for (int rr = 0; rr < 4; ++rr)
#pragma unroll
      for (int cidx = 0; cidx < NC; ++cidx) acc[rr][cidx] = fmaf(wv[cidx], av[rr], acc[rr][cidx]);
  }
}

__device__ __forceinline__ float4 ld4(const float* p) { return *reinterpret_cast<const float4*>(p); }

__global__ void __launch_bounds__(kThreads, 1) k_sample_loop(const LoopParams p) {
  extern __shared__ __align__(16) float sm[];
  float* wsm = sm;
  float* scratch = sm + WPACK_FLOATS;
  float* I0 = scratch + SCRATCH_FLOATS;
  float* qsm = I0 + RNN;  // Exp(1) noise of this CTA's row for the current step (cp.async at the top of the step)

  const int tid = threadIdx.x;
  const int warp = tid >> 5, lane = tid & 31;
  const int rt = lane & 15;   // row tile: rows 4*rt .. 4*rt+3 of the row block
  const int kh = lane >> 4;   // k half within the warp's slice
  const int cta = blockIdx.x;
  const int Bpad = p.Bpad;
  const int nrb = Bpad / RB;

  {  // one-time: weights -> shared memory
    const float4* src = reinterpret_cast<const float4*>(p.wpack + (size_t)cta * WPACK_FLOATS);
    float4* dst = reinterpret_cast<float4*>(wsm);
    for (int i = tid; i < WPACK_FLOATS / 4; i += kThreads) dst[i] = src[i];
    for (int i = tid; i < RNN; i += kThreads) I0[i] = p.I0[i];
  }
  __syncthreads();

  unsigned int bar_target = 0;
  const size_t HS = (size_t)RNN * Bpad;  // one [512][Bpad] matrix

  for (int i = 0; i < p.nsteps; ++i) {
    const int gstep = p.step0 + i;
    const int par = gstep & 1;
    const float* h1_old = p.h1 + (size_t)par * HS;
    float* h1_new = p.h1 + (size_t)(par ^ 1) * HS;
    const float* h2_old = p.h2 + (size_t)par * HS;
    float* h2_new = p.h2 + (size_t)(par ^ 1) * HS;
    const float* condI = p.condI + (size_t)i * HS;
    // The 512 noise values of this CTA's row are needed only by the sampling phase at the END of the step: start their copy
    // into shared memory now (cp.async: no registers), so that their HBM/L2 latency hides behind phases A-E instead of sitting
    // on the dependent chain (measured: +2 us per step with noise in global memory).
    if (p.noise && cta < p.B && tid < NCLS / 4) {
      const float* src = p.noise + ((size_t)i * p.noise_B + (size_t)(p.row0 + cta)) * NCLS + tid * 4;
      const uint32_t dst = (uint32_t)__cvta_generic_to_shared(qsm + tid * 4);
      asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory");
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
    // built-in generator: the same 512 values, one per thread, computed here instead of inside the sampling phase
    if (!p.noise && cta < p.B && tid < NCLS) qsm[tid] = mb_exp1_noise(p.seed, (uint32_t)gstep, (uint32_t)(p.row0 + cta), (uint32_t)tid);

    // ================= phase A: rnn1 =================
    for (int rb = 0; rb < nrb; ++rb) {
      const int r0 = rb * RB + 4 * rt;
      const float4 xp = ld4(p.xprev + r0);
      {
        const int m = warp >> 3;       // 0: W_ih x,  1: W_hh h
        const int slice = warp & 7;    // 64 k per warp
        const int k0 = slice * 64 + kh * 32;
        float acc[4][12];
        if (m == 0) {
          tile_gemv<12>(wsm + OFF_W1IH, k0, 32,
                        [&](int k) {
                          const float4 c = ld4(condI + (size_t)k * Bpad + r0);
                          const float w0 = I0[k];
                          return make_float4(fmaf(w0, xp.x, c.x), fmaf(w0, xp.y, c.y), fmaf(w0, xp.z, c.z),
                                             fmaf(w0, xp.w, c.w));
                        },
                        acc);
        } else {
          tile_gemv<12>(wsm + OFF_W1HH, k0, 32, [&](int k) { return ld4(h1_old + (size_t)k * Bpad + r0); }, acc);
        }
#pragma unroll
        for (int rr = 0; rr < 4; ++rr)
#pragma unroll
          for (int cidx = 0; cidx < 12; ++cidx) acc[rr][cidx] = acc[rr][cidx] + __shfl_xor_sync(0xffffffffu, acc[rr][cidx], 16);
        if (kh == 0) {
          float* dst = scratch + ((size_t)(m * 8 + slice) * RB + 4 * rt) * 12;
#pragma unroll
          for (int rr = 0; rr < 4; ++rr)
#pragma unroll
            for (int cidx = 0; cidx < 12; ++cidx) dst[rr * 12 + cidx] = acc[rr][cidx];
        }
      }
      __syncthreads();
      if (tid < RB * UPC) {
        const int r = tid & (RB - 1), j = tid >> 6;
        const int row = rb * RB + r;
        const int unit = cta * UPC + j;
        float g[2][3];
#pragma unroll
        for (int m = 0; m < 2; ++m)
#pragma unroll
          for (int gt = 0; gt < 3; ++gt) {
            float s[8];
#pragma unroll
            for (int w = 0; w < 8; ++w) s[w] = scratch[((size_t)(m * 8 + w) * RB + r) * 12 + gt * 4 + j];
            const float t = ((s[0] + s[1]) + (s[2] + s[3])) + ((s[4] + s[5]) + (s[6] + s[7]));
            g[m][gt] = t + wsm[(m == 0 ? OFF_B1IH : OFF_B1HH) + gt * 4 + j];
          }
        const float hold = h1_old[(size_t)unit * Bpad + row];
        const float rg = mb_sigmoidf(g[1][0] + g[0][0]);
        const float zg = mb_sigmoidf(g[1][1] + g[0][1]);
        const float ng = mb_tanhf(g[0][2] + g[1][2] * rg);
        h1_new[(size_t)unit * Bpad + row] = (hold - ng) * zg + ng;
      }
      __syncthreads();
    }
    grid_barrier(p, bar_target);

    // ================= phase B: rnn2 =================
    for (int rb = 0; rb < nrb; ++rb) {
      const int r0 = rb * RB + 4 * rt;
      const float4 xp = ld4(p.xprev + r0);
      {
        const int m = warp >> 3;
        const int slice = warp & 7;
        const int k0 = slice * 64 + kh * 32;
        float acc[4][12];
        if (m == 0) {
          tile_gemv<12>(wsm + OFF_W2IH, k0, 32,
                        [&](int k) {
                          const float4 c = ld4(condI + (size_t)k * Bpad + r0);
                          const float4 h = ld4(h1_new + (size_t)k * Bpad + r0);
                          const float w0 = I0[k];
                          return make_float4(fmaf(w0, xp.x, c.x) + h.x, fmaf(w0, xp.y, c.y) + h.y,
                                             fmaf(w0, xp.z, c.z) + h.z, fmaf(w0, xp.w, c.w) + h.w);
                        },
                        acc);
        } else {
          tile_gemv<12>(wsm + OFF_W2HH, k0, 32, [&](int k) { return ld4(h2_old + (size_t)k * Bpad + r0); }, acc);
        }
#pragma unroll
        for (int rr = 0; rr < 4; ++rr)
#pragma unroll
          for (int cidx = 0; cidx < 12; ++cidx) acc[rr][cidx] = acc[rr][cidx] + __shfl_xor_sync(0xffffffffu, acc[rr][cidx], 16);
        if (kh == 0) {
          float* dst = scratch + ((size_t)(m * 8 + slice) * RB + 4 * rt) * 12;
#pragma unroll
          for (int rr = 0; rr < 4; ++rr)
#pragma unroll
            for (int cidx = 0; cidx < 12; ++cidx) dst[rr * 12 + cidx] = acc[rr][cidx];
        }
      }
      __syncthreads();
      if (tid < RB * UPC) {
        const int r = tid & (RB - 1), j = tid >> 6;
        const int row = rb * RB + r;
        const int unit = cta * UPC + j;
        int frame = p.T;  // "past the end" row of the tables
        if (row < p.B) {
          const int t = p.starts[row] + gstep;
          if (t < HOP * p.T) frame = t / HOP;
        }
        float g[2][3];
#pragma unroll
        for (int m = 0; m < 2; ++m)
#pragma unroll
          for (int gt = 0; gt < 3; ++gt) {
            float s[8];
#pragma unroll
            for (int w = 0; w < 8; ++w) s[w] = scratch[((size_t)(m * 8 + w) * RB + r) * 12 + gt * 4 + j];
            const float t = ((s[0] + s[1]) + (s[2] + s[3])) + ((s[4] + s[5]) + (s[6] + s[7]));
            g[m][gt] = t + (m == 0 ? p.aux2P[(size_t)frame * (3 * RNN) + gt * RNN + unit] : wsm[OFF_B2HH + gt * 4 + j]);
          }
        const float hold = h2_old[(size_t)unit * Bpad + row];
        const float rg = mb_sigmoidf(g[1][0] + g[0][0]);
        const float zg = mb_sigmoidf(g[1][1] + g[0][1]);
        const float ng = mb_tanhf(g[0][2] + g[1][2] * rg);
        h2_new[(size_t)unit * Bpad + row] = (hold - ng) * zg + ng;
      }
      __syncthreads();
    }
    grid_barrier(p, bar_target);

    // ================= phases C, D, E: fc1, fc2, fc3 =================
#pragma unroll 1
    for (int layer = 0; layer < 3; ++layer) {
      const float* wl = wsm + (layer == 0 ? OFF_FC1 : layer == 1 ? OFF_FC2 : OFF_FC3);
      for (int rb = 0; rb < nrb; ++rb) {
        const int r0 = rb * RB + 4 * rt;
        const float4 xp = ld4(p.xprev + r0);
        const int k0 = warp * 32 + kh * 16;  // 32 sub-slices of 16
        float acc[4][4];
        if (layer == 0) {
          tile_gemv<4>(wl, k0, 16,
                       [&](int k) {
                         const float4 c = ld4(condI + (size_t)k * Bpad + r0);
                         const float4 ha = ld4(h1_new + (size_t)k * Bpad + r0);
                         const float4 hb = ld4(h2_new + (size_t)k * Bpad + r0);
                         const float w0 = I0[k];
                         return make_float4((fmaf(w0, xp.x, c.x) + ha.x) + hb.x, (fmaf(w0, xp.y, c.y) + ha.y) + hb.y,
                                            (fmaf(w0, xp.z, c.z) + ha.z) + hb.z, (fmaf(w0, xp.w, c.w) + ha.w) + hb.w);
                       },
                       acc);
        } else {
          const float* a = (layer == 1) ? p.f1 : p.f2;
          tile_gemv<4>(wl, k0, 16, [&](int k) { return ld4(a + (size_t)k * Bpad + r0); }, acc);
        }
#pragma unroll
        for (int rr = 0; rr < 4; ++rr)
#pragma unroll
          for (int cidx = 0; cidx < 4; ++cidx) acc[rr][cidx] = acc[rr][cidx] + __shfl_xor_sync(0xffffffffu, acc[rr][cidx], 16);
        if (kh == 0) {
          float* dst = scratch + ((size_t)warp * RB + 4 * rt) * 4;
#pragma unroll
          for (int rr = 0; rr < 4; ++rr)
#pragma unroll
            for (int cidx = 0; cidx < 4; ++cidx) dst[rr * 4 + cidx] = acc[rr][cidx];
        }
        __syncthreads();
        if (tid < RB * UPC) {
          const int r = tid & (RB - 1), j = tid >> 6;
          const int row = rb * RB + r;
          const int unit = cta * UPC + j;
          float s[16];
#pragma unroll
          for (int w = 0; w < 16; ++w) s[w] = scratch[((size_t)w * RB + r) * 4 + j];
#pragma unroll
          for (int n = 8; n >= 1; n >>= 1)
#pragma unroll
            for (int q = 0; q < n; ++q) s[q] = s[2 * q] + s[2 * q + 1];
          float v = s[0];
          if (layer < 2) {
            int frame = p.T;
            if (row < p.B) {
              const int t = p.starts[row] + gstep;
              if (t < HOP * p.T) frame = t / HOP;
            }
            v = v + (layer == 0 ? p.aux3P : p.aux4P)[(size_t)frame * RNN + unit];
            v = v > 0.0f ? v : 0.0f;
            (layer == 0 ? p.f1 : p.f2)[(size_t)unit * Bpad + row] = v;
          } else {
            p.logits[(size_t)unit * Bpad + row] = v + wsm[OFF_FC3B + j];
          }
        }
        __syncthreads();
      }
      asm volatile("cp.async.wait_group 0;" ::: "memory");  // this step's noise row has landed (issued at the top of the step)
      grid_barrier(p, bar_target);
    }

    // ================= phase F: softmax + Categorical sample (one warp per row) =================
    // (the copies issued at the top of the step were waited for before the grid barrier above: qsm is complete and visible)
    if (warp == 0) {
      for (int row = cta; row < p.B; row += gridDim.x) {
        float lg[16], e[16];
        float m = -3.0e38f;
#pragma unroll
        for (int jj = 0; jj < 16; ++jj) {
          lg[jj] = p.logits[(size_t)(lane + 32 * jj) * Bpad + row];
          m = lg[jj] > m ? lg[jj] : m;
        }
#pragma unroll
        for (int off = 16; off >= 1; off >>= 1) {
          const float o = __shfl_xor_sync(0xffffffffu, m, off);
          m = o > m ? o : m;
        }
        float s = 0.0f;
#pragma unroll
        for (int jj = 0; jj < 16; ++jj) {
          e[jj] = mb_expf(lg[jj] - m);
          s = s + e[jj];
        }
#pragma unroll
        for (int off = 16; off >= 1; off >>= 1) s = s + __shfl_xor_sync(0xffffffffu, s, off);
        const float S = s;
        float s2 = 0.0f;
#pragma unroll
        for (int jj = 0; jj < 16; ++jj) {
          e[jj] = e[jj] / S;
          s2 = s2 + e[jj];
        }
#pragma unroll
        for (int off = 16; off >= 1; off >>= 1) s2 = s2 + __shfl_xor_sync(0xffffffffu, s2, off);
        const float S2 = s2;
        float bestv = -1.0f;
        int best = 0;
#pragma unroll
        for (int jj = 0; jj < 16; ++jj) {
          const int cls = lane + 32 * jj;
          const float q = (row == cta) ? qsm[cls]
                          : (p.noise ? p.noise[((size_t)i * p.noise_B + (size_t)(p.row0 + row)) * NCLS + cls]
                                     : mb_exp1_noise(p.seed, (uint32_t)gstep, (uint32_t)(p.row0 + row), (uint32_t)cls));
          const float v = (e[jj] / S2) / q;
          if (v > bestv) {  // ascending class order within the lane: first maximum wins
            bestv = v;
            best = cls;
          }
        }
#pragma unroll
        for (int off = 16; off >= 1; off >>= 1) {
          const float ov = __shfl_xor_sync(0xffffffffu, bestv, off);
          const int ob = __shfl_xor_sync(0xffffffffu, best, off);
          if (ov > bestv || (ov == bestv && ob < best)) {
            bestv = ov;
            best = ob;
          }
        }
        if (lane == 0) {
          p.out_idx[(size_t)row * p.steps_total + gstep] = (int16_t)best;
          p.xprev[row] = (2.0f * (float)best) / 511.0f - 1.0f;
        }
      }
    }
    grid_barrier(p, bar_target);
  }
}

}  // namespace
}  // namespace mb

// =================================================================================================
// C ABI
// =================================================================================================
using namespace mb;

namespace {
struct WSlot {
  std::string name;
  std::vector<int64_t> dims;
  size_t off = 0;  // float offset in the arena
  bool set = false;
};
}  // namespace

struct mb_wavernn {
  mb_wavernn_config cfg{};
  std::vector<WSlot> slots;
  size_t raw_floats = 0;   // raw weights as given
  size_t pack_off = 0;     // per-CTA packs
  size_t total_floats = 0;
  float* arena = nullptr;
  bool finalized = false;
  // conditioning of the current utterance (workspace-resident)
  int cond_T = 0;
  void* cond_ws = nullptr;
};

namespace {

const float* W(const mb_wavernn* h, const std::string& name) {
  for (const WSlot& s : h->slots)
    if (s.name == name) return h->arena + s.off;
  return nullptr;
}

void add_slot(mb_wavernn* h, const std::string& name, std::vector<int64_t> dims) {
  WSlot s;
  s.name = name;
  s.dims = dims;
  size_t n = 1;
  for (int64_t d : dims) n *= (size_t)d;
  s.off = h->raw_floats;
  h->raw_floats += align_up(n, 64);
  h->slots.push_back(s);
}

struct WsLayout {
  size_t aux, melup, aux2P, aux3P, aux4P, tmpA, tmpB, tmpR, padP, lad5, lad25, lad200, starts, condI, h1, h2, f1, f2, logits, xprev,
      barrier, total;
};

WsLayout ws_layout(int T, int Bpad, int chunk_steps) {
  WsLayout L{};
  size_t o = 0;
  auto take = [&](size_t floats) {
    size_t r = o;
    o += align_up(floats, 64);
    return r;
  };
  L.aux = take((size_t)T * CDIM);
  L.melup = take((size_t)HOP * T * FEAT);
  L.aux2P = take((size_t)(T + 1) * 3 * RNN);
  L.aux3P = take((size_t)(T + 1) * RNN);
  L.aux4P = take((size_t)(T + 1) * RNN);
  L.tmpA = take((size_t)CDIM * T);
  L.tmpB = take((size_t)CDIM * T);
  L.tmpR = take((size_t)CDIM * T);
  L.padP = take((size_t)FEAT * (T + 4));
  L.lad5 = take((size_t)FEAT * (T + 4) * 5);
  L.lad25 = take((size_t)FEAT * (T + 4) * 25);
  L.lad200 = take((size_t)FEAT * (T + 4) * HOP);
  L.starts = take((size_t)Bpad);
  L.condI = take((size_t)chunk_steps * RNN * Bpad);
  L.h1 = take((size_t)2 * RNN * Bpad);
  L.h2 = take((size_t)2 * RNN * Bpad);
  L.f1 = take((size_t)RNN * Bpad);
  L.f2 = take((size_t)RNN * Bpad);
  L.logits = take((size_t)RNN * Bpad);
  L.xprev = take((size_t)Bpad);
  L.barrier = take(256);  // 1 KB: counter, or one epoch word per CTA
  L.total = o;
  return L;
}

constexpr int kChunkMax = 128;  // steps per mb_wavernn_generate call

int bpad_of(int B) { return ((B + RB - 1) / RB) * RB; }

}  // namespace

extern "C" {

int mb_wavernn_create(const mb_wavernn_config* cfg, mb_wavernn** out) {
  if (!cfg || !out) return fail(MB_ERR_INVALID, "mb_wavernn_create: null argument");
  if (cfg->rnn_dims != RNN || cfg->fc_dims != RNN || cfg->bits != 9 || cfg->pad != 2 || cfg->num_upsample != 3 ||
      cfg->upsample_factors[0] * cfg->upsample_factors[1] * cfg->upsample_factors[2] != HOP ||
      cfg->upsample_factors[0] != 5 || cfg->upsample_factors[1] != 5 || cfg->feat_dims != FEAT ||
      cfg->compute_dims != CDIM || cfg->res_out_dims != CDIM || cfg->res_blocks < 1 || cfg->res_blocks > 16)
    return fail(MB_ERR_INVALID,
                "mb_wavernn_create: only the reference hparams are built (rnn/fc 512, 9 bits, pad 2, "
                "upsample (5,5,8), 80 mels, compute/res_out 128)");
  mb_wavernn* h = new mb_wavernn();
  h->cfg = *cfg;
  add_slot(h, "upsample.resnet.conv_in.weight", {CDIM, FEAT, 5});
  auto bn = [&](const std::string& p) {
    for (const char* leaf : {".weight", ".bias", ".running_mean", ".running_var"}) add_slot(h, p + leaf, {CDIM});
  };
  bn("upsample.resnet.batch_norm");
  for (int i = 0; i < cfg->res_blocks; ++i) {
    const std::string b = "upsample.resnet.layers." + std::to_string(i);
    add_slot(h, b + ".conv1.weight", {CDIM, CDIM, 1});
    add_slot(h, b + ".conv2.weight", {CDIM, CDIM, 1});
    bn(b + ".batch_norm1");
    bn(b + ".batch_norm2");
  }
  add_slot(h, "upsample.resnet.conv_out.weight", {CDIM, CDIM, 1});
  add_slot(h, "upsample.resnet.conv_out.bias", {CDIM});
  for (int j = 0; j < 3; ++j)
    add_slot(h, "upsample.up_layers." + std::to_string(2 * j + 1) + ".weight", {1, 1, 1, 2 * cfg->upsample_factors[j] + 1});
  add_slot(h, "I.weight", {RNN, FEAT + AUXD + 1});
  add_slot(h, "I.bias", {RNN});
  add_slot(h, "rnn1.weight_ih_l0", {3 * RNN, RNN});
  add_slot(h, "rnn1.weight_hh_l0", {3 * RNN, RNN});
  add_slot(h, "rnn1.bias_ih_l0", {3 * RNN});
  add_slot(h, "rnn1.bias_hh_l0", {3 * RNN});
  add_slot(h, "rnn2.weight_ih_l0", {3 * RNN, RNN + AUXD});
  add_slot(h, "rnn2.weight_hh_l0", {3 * RNN, RNN});
  add_slot(h, "rnn2.bias_ih_l0", {3 * RNN});
  add_slot(h, "rnn2.bias_hh_l0", {3 * RNN});
  add_slot(h, "fc1.weight", {RNN, RNN + AUXD});
  add_slot(h, "fc1.bias", {RNN});
  add_slot(h, "fc2.weight", {RNN, RNN + AUXD});
  add_slot(h, "fc2.bias", {RNN});
  add_slot(h, "fc3.weight", {NCLS, RNN});
  add_slot(h, "fc3.bias", {NCLS});
  h->pack_off = h->raw_floats;
  h->total_floats = h->pack_off + (size_t)NCTA * WPACK_FLOATS + RNN;
  *out = h;
  return MB_OK;
}

void mb_wavernn_destroy(mb_wavernn* h) { delete h; }

size_t mb_wavernn_arena_bytes(const mb_wavernn* h) { return h ? h->total_floats * sizeof(float) : 0; }

int mb_wavernn_set_arena(mb_wavernn* h, void* arena, size_t bytes) {
  if (!h || !arena) return fail(MB_ERR_INVALID, "mb_wavernn_set_arena: null argument");
  if (bytes < mb_wavernn_arena_bytes(h)) return fail(MB_ERR_WORKSPACE, "mb_wavernn_set_arena: arena too small");
  if (((uintptr_t)arena & 255) != 0) return fail(MB_ERR_INVALID, "mb_wavernn_set_arena: arena must be 256-byte aligned");
  h->arena = (float*)arena;
  return MB_OK;
}

int mb_wavernn_set_weight(mb_wavernn* h, const char* name, const float* w, const int64_t* dims, int32_t ndim,
                          void* stream) {
  if (!h || !name || !w || !dims) return fail(MB_ERR_INVALID, "mb_wavernn_set_weight: null argument");
  if (!h->arena) return fail(MB_ERR_STATE, "mb_wavernn_set_weight: call mb_wavernn_set_arena first");
  for (WSlot& s : h->slots) {
    if (s.name != name) continue;
    size_t n = 1, given = 1;
    for (int64_t d : s.dims) n *= (size_t)d;
    for (int i = 0; i < ndim; ++i) given *= (size_t)dims[i];
    if (given != n) return fail(MB_ERR_INVALID, "mb_wavernn_set_weight: %s has %zu elements, expected %zu", name, given, n);
    MB_CUDA_CHECK(cudaMemcpyAsync(h->arena + s.off, w, n * sizeof(float), cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
    s.set = true;
    h->finalized = false;
    return MB_OK;
  }
  return fail(MB_ERR_INVALID, "mb_wavernn_set_weight: unknown tensor '%s'", name);
}

int mb_wavernn_finalize(mb_wavernn* h, void* stream) {
  if (!h) return fail(MB_ERR_INVALID, "mb_wavernn_finalize: null handle");
  for (const WSlot& s : h->slots)
    if (!s.set) return fail(MB_ERR_STATE, "mb_wavernn_finalize: tensor %s was never set", s.name.c_str());
  PackSrc ps;
  ps.r1_wih = W(h, "rnn1.weight_ih_l0");
  ps.r1_whh = W(h, "rnn1.weight_hh_l0");
  ps.r1_bih = W(h, "rnn1.bias_ih_l0");
  ps.r1_bhh = W(h, "rnn1.bias_hh_l0");
  ps.r2_wih = W(h, "rnn2.weight_ih_l0");
  ps.r2_whh = W(h, "rnn2.weight_hh_l0");
  ps.r2_bhh = W(h, "rnn2.bias_hh_l0");
  ps.fc1_w = W(h, "fc1.weight");
  ps.fc2_w = W(h, "fc2.weight");
  ps.fc3_w = W(h, "fc3.weight");
  ps.fc3_b = W(h, "fc3.bias");
  cudaStream_t st = (cudaStream_t)stream;
  k_pack<<<NCTA, 256, 0, st>>>(ps, h->arena + h->pack_off);
  MB_LAUNCH_CHECK("k_pack");
  // I0 = I.weight[:, 0]
  MB_CUDA_CHECK(cudaMemcpy2DAsync(h->arena + h->pack_off + (size_t)NCTA * WPACK_FLOATS, sizeof(float), W(h, "I.weight"),
                                  sizeof(float) * (FEAT + AUXD + 1), sizeof(float), RNN, cudaMemcpyDeviceToDevice, st));
  h->finalized = true;
  return MB_OK;
}

size_t mb_wavernn_workspace_bytes(const mb_wavernn* h, int32_t frames, int32_t folds, int32_t steps) {
  if (!h || frames <= 0 || folds <= 0) return 0;
  (void)steps;
  return ws_layout(frames, bpad_of(folds), kChunkMax).total * sizeof(float) + 256;
}

int mb_wavernn_condition(mb_wavernn* h, const float* mel, int32_t T, void* workspace, size_t workspace_bytes,
                         void* stream) {
  if (!h || !mel || !workspace || T <= 0) return fail(MB_ERR_INVALID, "mb_wavernn_condition: bad argument");
  if (!h->finalized) return fail(MB_ERR_STATE, "mb_wavernn_condition: weights not finalized");
  // the conditioning part of the layout does not depend on the fold count
  const WsLayout L = ws_layout(T, RB, kChunkMax);
  if (workspace_bytes < (L.starts) * sizeof(float) + 256)
    return fail(MB_ERR_WORKSPACE, "mb_wavernn_condition: workspace too small");
  float* ws = (float*)(((uintptr_t)workspace + 255) & ~(uintptr_t)255);
  cudaStream_t st = (cudaStream_t)stream;
  const int n = CDIM * T, nb = (n + 255) / 256;
  float *x = ws + L.tmpA, *y = ws + L.tmpB, *r = ws + L.tmpR;
  k_conv_in<<<nb, 256, 0, st>>>(W(h, "upsample.resnet.conv_in.weight"), mel, T, x);
  MB_LAUNCH_CHECK("k_conv_in");
  auto bnrun = [&](const std::string& p, float* buf, int relu, const float* res) -> int {
    k_bn<<<nb, 256, 0, st>>>(W(h, p + ".weight"), W(h, p + ".bias"), W(h, p + ".running_mean"), W(h, p + ".running_var"),
                             buf, T, relu, res);
    MB_LAUNCH_CHECK("k_bn");
    return MB_OK;
  };
  int rc = bnrun("upsample.resnet.batch_norm", x, 1, nullptr);
  if (rc) return rc;
  for (int i = 0; i < h->cfg.res_blocks; ++i) {
    const std::string b = "upsample.resnet.layers." + std::to_string(i);
    MB_CUDA_CHECK(cudaMemcpyAsync(r, x, sizeof(float) * n, cudaMemcpyDeviceToDevice, st));
    k_conv1x1<<<nb, 256, 0, st>>>(W(h, b + ".conv1.weight"), x, T, y, nullptr, 0);
    MB_LAUNCH_CHECK("k_conv1x1");
    if ((rc = bnrun(b + ".batch_norm1", y, 1, nullptr))) return rc;
    k_conv1x1<<<nb, 256, 0, st>>>(W(h, b + ".conv2.weight"), y, T, x, nullptr, 0);
    MB_LAUNCH_CHECK("k_conv1x1");
    if ((rc = bnrun(b + ".batch_norm2", x, 0, r))) return rc;
  }
  k_conv1x1<<<nb, 256, 0, st>>>(W(h, "upsample.resnet.conv_out.weight"), x, T, ws + L.aux,
                                W(h, "upsample.resnet.conv_out.bias"), 1);
  MB_LAUNCH_CHECK("k_conv1x1");
  // mel ladder: P (Tp) -> x5 -> x25 -> x200, then crop
  const int Tp = T + 4;
  float* P = ws + L.padP;
  float* l5 = ws + L.lad5;
  float* l25 = ws + L.lad25;
  float* l1 = ws + L.lad200;
  k_pad_mel<<<(FEAT * Tp + 255) / 256, 256, 0, st>>>(mel, T, P);
  MB_LAUNCH_CHECK("k_pad_mel");
  const int s0 = h->cfg.upsample_factors[0], s1 = h->cfg.upsample_factors[1], s2 = h->cfg.upsample_factors[2];
  k_ladder<<<(FEAT * Tp * s0 + 255) / 256, 256, 0, st>>>(W(h, "upsample.up_layers.1.weight"), P, Tp, s0, l5);
  MB_LAUNCH_CHECK("k_ladder");
  k_ladder<<<(FEAT * Tp * s0 * s1 + 255) / 256, 256, 0, st>>>(W(h, "upsample.up_layers.3.weight"), l5, Tp * s0, s1, l25);
  MB_LAUNCH_CHECK("k_ladder");
  k_ladder<<<(int)(((size_t)FEAT * Tp * HOP + 255) / 256), 256, 0, st>>>(W(h, "upsample.up_layers.5.weight"), l25,
                                                                          Tp * s0 * s1, s2, l1);
  MB_LAUNCH_CHECK("k_ladder");
  k_crop_melup<<<(int)(((size_t)HOP * T * FEAT + 255) / 256), 256, 0, st>>>(l1, Tp * HOP, T, ws + L.melup);
  MB_LAUNCH_CHECK("k_crop_melup");
  // frame-rate tables of the aux contributions
  k_aux_table<<<((T + 1) * 3 * RNN + 255) / 256, 256, 0, st>>>(W(h, "rnn2.weight_ih_l0"), RNN + AUXD, RNN,
                                                               W(h, "rnn2.bias_ih_l0"), ws + L.aux, AUXD, T, 3 * RNN,
                                                               ws + L.aux2P);
  MB_LAUNCH_CHECK("k_aux_table");
  k_aux_table<<<((T + 1) * RNN + 255) / 256, 256, 0, st>>>(W(h, "fc1.weight"), RNN + AUXD, RNN, W(h, "fc1.bias"),
                                                           ws + L.aux, 2 * AUXD, T, RNN, ws + L.aux3P);
  MB_LAUNCH_CHECK("k_aux_table");
  k_aux_table<<<((T + 1) * RNN + 255) / 256, 256, 0, st>>>(W(h, "fc2.weight"), RNN + AUXD, RNN, W(h, "fc2.bias"),
                                                           ws + L.aux, 3 * AUXD, T, RNN, ws + L.aux4P);
  MB_LAUNCH_CHECK("k_aux_table");
  h->cond_T = T;
  h->cond_ws = workspace;
  return MB_OK;
}

int mb_wavernn_generate(mb_wavernn* h, const int32_t* fold_starts_host, int32_t B, int32_t steps, int32_t step0,
                        int32_t nsteps, const float* noise, uint64_t seed, int16_t* out_idx, void* workspace,
                        size_t workspace_bytes, void* stream) {
  return mb_wavernn_generate_rows(h, fold_starts_host, B, steps, step0, nsteps, noise, B, 0, seed, out_idx, workspace,
                                  workspace_bytes, stream);
}

int mb_wavernn_generate_rows(mb_wavernn* h, const int32_t* fold_starts_host, int32_t B, int32_t steps, int32_t step0,
                             int32_t nsteps, const float* noise, int32_t noise_folds, int32_t row0, uint64_t seed,
                             int16_t* out_idx, void* workspace, size_t workspace_bytes, void* stream) {
  if (!h || !fold_starts_host || !out_idx || !workspace) return fail(MB_ERR_INVALID, "mb_wavernn_generate: null argument");
  if (row0 < 0 || (noise && row0 + B > noise_folds))
    return fail(MB_ERR_INVALID, "mb_wavernn_generate_rows: rows [%d, %d) outside the %d noise rows", row0, row0 + B, noise_folds);
  if (!h->finalized) return fail(MB_ERR_STATE, "mb_wavernn_generate: weights not finalized");
  if (h->cond_T <= 0 || h->cond_ws != workspace)
    return fail(MB_ERR_STATE, "mb_wavernn_generate: call mb_wavernn_condition on this workspace first");
  if (B <= 0 || nsteps <= 0 || nsteps > kChunkMax || step0 < 0 || step0 + nsteps > steps)
    return fail(MB_ERR_INVALID, "mb_wavernn_generate: bad step range (at most %d steps per call)", kChunkMax);
  const int T = h->cond_T;
  const int Bpad = bpad_of(B);
  const WsLayout L = ws_layout(T, Bpad, kChunkMax);
  if (workspace_bytes < L.total * sizeof(float) + 256) return fail(MB_ERR_WORKSPACE, "mb_wavernn_generate: workspace too small");
  float* ws = (float*)(((uintptr_t)workspace + 255) & ~(uintptr_t)255);
  cudaStream_t st = (cudaStream_t)stream;
  if (step0 == 0) {
    // zero initial state (fatchord_version.py:178-185) and upload the fold starts
    MB_CUDA_CHECK(cudaMemsetAsync(ws + L.h1, 0, sizeof(float) * (L.xprev + align_up((size_t)Bpad, 64) - L.h1), st));
    std::vector<int32_t> tmp(Bpad, 0);
    memcpy(tmp.data(), fold_starts_host, sizeof(int32_t) * B);
    MB_CUDA_CHECK(cudaMemcpyAsync(ws + L.starts, tmp.data(), sizeof(int32_t) * Bpad, cudaMemcpyHostToDevice, st));
    MB_CUDA_CHECK(cudaStreamSynchronize(st));  // tmp goes out of scope
  }
  const int* starts = reinterpret_cast<const int*>(ws + L.starts);
  k_condI<<<nsteps * Bpad, 256, 0, st>>>(W(h, "I.weight"), W(h, "I.bias"), ws + L.melup, ws + L.aux, T, starts, B, Bpad,
                                         step0, nsteps, ws + L.condI);
  MB_LAUNCH_CHECK("k_condI");
  MB_CUDA_CHECK(cudaMemsetAsync(ws + L.barrier, 0, 1024, st));
  LoopParams p;
  memset(&p, 0, sizeof(p));
  p.wpack = h->arena + h->pack_off;
  p.I0 = h->arena + h->pack_off + (size_t)NCTA * WPACK_FLOATS;
  p.aux2P = ws + L.aux2P;
  p.aux3P = ws + L.aux3P;
  p.aux4P = ws + L.aux4P;
  p.condI = ws + L.condI;
  p.starts = starts;
  p.T = T;
  p.B = B;
  p.Bpad = Bpad;
  p.step0 = step0;
  p.nsteps = nsteps;
  p.steps_total = steps;
  p.h1 = ws + L.h1;
  p.h2 = ws + L.h2;
  p.f1 = ws + L.f1;
  p.f2 = ws + L.f2;
  p.logits = ws + L.logits;
  p.xprev = ws + L.xprev;
  p.noise = noise;
  p.noise_B = noise_folds;
  p.row0 = row0;
  p.seed = seed;
  p.out_idx = out_idx;
  p.barrier = reinterpret_cast<unsigned int*>(ws + L.barrier);
  static const int flagbar = [] {
    // A/B switch.  Measured: the flag barrier is much SLOWER (604 vs 428 ms per cfg-3 call: 128 x 128 polling threads swamp the
    // four flag lines); the single-counter barrier stays the default.
    const char* e = getenv("MB_WAVERNN_FLAGBAR");
    return e ? atoi(e) : 0;
  }();
  p.flagbar = flagbar;
  const size_t smem = sizeof(float) * SMEM_FLOATS;
  static bool attr = false;
  if (!attr) {
    MB_CUDA_CHECK(cudaFuncSetAttribute(k_sample_loop, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    attr = true;
  }
  void* args[] = {(void*)&p};
  MB_CUDA_CHECK(cudaLaunchCooperativeKernel((void*)k_sample_loop, dim3(NCTA), dim3(kThreads), args, smem, st));
  count_launch();
  return MB_OK;
}

int mb_wavernn_last_logits(mb_wavernn* h, float* logits, int32_t B, void* workspace, void* stream) {
  if (!h || !logits || !workspace || h->cond_T <= 0) return fail(MB_ERR_INVALID, "mb_wavernn_last_logits: bad argument");
  const int Bpad = bpad_of(B);
  const WsLayout L = ws_layout(h->cond_T, Bpad, kChunkMax);
  float* ws = (float*)(((uintptr_t)workspace + 255) & ~(uintptr_t)255);
  // logits are stored [class][Bpad]; return [B][512]
  MB_CUDA_CHECK(cudaMemcpy2DAsync(logits, sizeof(float) * NCLS, ws + L.logits, sizeof(float), sizeof(float), 1,
                                  cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
  // generic strided transpose through a tiny loop of 2D copies (debug hook, B is small)
  for (int r = 0; r < B; ++r)
    MB_CUDA_CHECK(cudaMemcpy2DAsync(logits + (size_t)r * NCLS, sizeof(float), ws + L.logits + r, sizeof(float) * Bpad,
                                    sizeof(float), NCLS, cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
  return MB_OK;
}

}  // extern "C"
