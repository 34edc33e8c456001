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
// conditioning kernels: one thread per output, sequential fmaf chains in the twin's order.  The frames of the call's
// utterances are concatenated (one utterance is the case n_utts = 1): utterance u owns frames [segF[u], segF[u] + segT[u]) of
// the [C][Ttot] activations, of aux [Ttot][128] and (x200) of melup, padded frames [segF[u] + 4u, + segT[u] + 4) of the ladder
// buffers and rows [segF[u] + u, + segT[u] + 1) of the aux tables (the last one is its "past the end" row).  k_bn / k_conv1x1
// are frame-wise and run over Ttot frames; the kernels after them must not look across an utterance boundary.
// fseg / pseg: utterance of a frame / padded frame.
// ------------------------------------------------------------------------------------------------
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

// y[o][t] = sum_{ci,k} w[o][ci][k] * P[ci][t+k],  P = the utterance's mel padded by 2 zero frames on both sides
__global__ void k_conv_in(const float* __restrict__ w, const float* __restrict__ mel, int Ttot, const int* __restrict__ fseg,
                          const int* __restrict__ segF, const int* __restrict__ segT, float* __restrict__ y) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= CDIM * Ttot) return;
  const int o = i / Ttot, tg = i - o * Ttot;
  const int u = fseg[tg], F = segF[u], T = segT[u], t = tg - F;
  const float* m = mel + (size_t)FEAT * F;  // mels [80, T_u] back to back
  float acc = 0.0f;
  for (int ci = 0; ci < FEAT; ++ci)
    for (int k = 0; k < 5; ++k) {
      const int s = t + k - 2;
      const float v = (s >= 0 && s < T) ? m[ci * T + s] : 0.0f;
      acc = fmaf(w[(o * FEAT + ci) * 5 + k], v, acc);
    }
  y[i] = acc;
}

__global__ void k_pad_mel(const float* __restrict__ mel, int Tptot, const int* __restrict__ pseg, const int* __restrict__ segF,
                          const int* __restrict__ segT, float* __restrict__ P) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= FEAT * Tptot) return;
  const int c = i / Tptot, pg = i - c * Tptot;
  const int u = pseg[pg], F = segF[u], T = segT[u], t = pg - (F + 4 * u);
  P[i] = (t >= 2 && t < T + 2) ? mel[(size_t)FEAT * F + c * T + t - 2] : 0.0f;
}

// one ladder stage, y[c][i] = sum_j w[j] * rep(x)[i + j - s] within each utterance; `per` = input positions per padded frame
// (1, 5, 25)
__global__ void k_ladder(const float* __restrict__ w, const float* __restrict__ x, int len, int s, int per,
                         const int* __restrict__ pseg, const int* __restrict__ segF, const int* __restrict__ segT,
                         float* __restrict__ y) {
  const size_t nl = (size_t)len * s;
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= FEAT * nl) return;
  const int c = (int)(i / nl), pg = (int)(i - c * nl);
  const int u = pseg[pg / (per * s)];
  const int seg0 = (segF[u] + 4 * u) * per * s, seglen = (segT[u] + 4) * per * s;
  const int p = pg - seg0;
  float acc = 0.0f;
  for (int j = 0; j <= 2 * s; ++j) {
    const int src = p + j - s;
    const float v = (src >= 0 && src < seglen) ? x[(size_t)c * len + (seg0 + src) / s] : 0.0f;
    acc = fmaf(w[j], v, acc);
  }
  y[i] = acc;
}

__global__ void k_crop_melup(const float* __restrict__ y3, int len, int Ttot, const int* __restrict__ fseg,
                             float* __restrict__ melup) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)HOP * Ttot * FEAT) return;
  const int tg = (int)(i / FEAT), c = (int)(i - (size_t)tg * FEAT);
  const int u = fseg[tg / HOP];
  melup[i] = y3[(size_t)c * len + tg + HOP * (4 * u) + 2 * HOP];
}

// frame-rate tables: out[f][g] = dot_seq(W[g][K0 : K0+32], aux[tsrc[f]][a0 : a0+32]) + bias[g]; tsrc[f] = -1 marks an
// utterance's "past the end" row (zero conditioning)
__global__ void k_aux_table(const float* __restrict__ W, int ld, int K0, const float* __restrict__ bias,
                            const float* __restrict__ aux, int a0, const int* __restrict__ tsrc, int R, int G,
                            float* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= R * G) return;
  const int f = i / G, g = i - f * G;
  const int src = tsrc[f];
  float acc = 0.0f;
  for (int j = 0; j < AUXD; ++j) {
    const float a = (src >= 0) ? aux[(size_t)src * CDIM + a0 + j] : 0.0f;
    acc = fmaf(W[(size_t)g * ld + K0 + j], a, acc);
  }
  out[i] = acc + bias[g];
}

// per-chunk conditioning of the I layer in the exchange layout:
//   condI[i][u][r] = dot_seq(I_w[u][1:113], [melup[t]; aux[t/200][0:32]]) + I_b[u],  t = start[r] + step0 + i
// row r is described by rowc[r] = {start, T_u, table base, frame base}; only the W = 64 * (live row blocks) leading rows are
// written, and the dot product is skipped for the padding rows past the table (T_u == 0: most of a row block when there are
// only a few rows)
__global__ void __launch_bounds__(256) k_condI(const float* __restrict__ I_w, const float* __restrict__ I_b,
                                               const float* __restrict__ melup, const float* __restrict__ aux,
                                               const int4* __restrict__ rowc, int W, int Bpad, int step0, int nsteps,
                                               float* __restrict__ out) {
  __shared__ float c[FEAT + AUXD];
  const int r = blockIdx.x % W;
  const int i = blockIdx.x / W;
  if (i >= nsteps) return;
  const int4 d = rowc[r];
  const int t = d.x + step0 + i;
  const bool live = t < HOP * d.y;
  for (int j = threadIdx.x; j < FEAT + AUXD; j += blockDim.x) {
    float v = 0.0f;
    if (live) v = (j < FEAT) ? melup[((size_t)HOP * d.w + t) * FEAT + j] : aux[(size_t)(d.w + t / HOP) * CDIM + (j - FEAT)];
    c[j] = v;
  }
  __syncthreads();
  for (int u = threadIdx.x; u < RNN; u += blockDim.x) {
    float acc = 0.0f;
    const float* wr = I_w + (size_t)u * 113 + 1;
    if (d.y > 0)
      for (int j = 0; j < FEAT + AUXD; ++j) acc = fmaf(wr[j], c[j], acc);
    out[((size_t)i * RNN + u) * Bpad + r] = acc + I_b[u];
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
  int B, Bpad, step0, nsteps, steps_total;  // B: live rows, a prefix (rows are ordered longest first); steps_total: row 0's
  // state / exchange buffers (global, [unit][Bpad])
  float* h1;                // [2][512][Bpad]
  float* h2;                // [2][512][Bpad]
  float* f1;                // [512][Bpad]
  float* f2;                // [512][Bpad]
  float* logits;            // [512][Bpad]
  float* xprev;             // [Bpad]
  const float* noise;       // RAW: [nsteps][noise_B][512] Exp(1), row r at noise row rown.z + rown.y; MOL: per step, every
                            // block of n noise rows from rown.z holds its [n*10 mixture | n logistic] uniforms; or nullptr
  int noise_B;              // noise rows per step
  int16_t* out_idx;         // RAW: class indices [B][steps_total]
  float* out_x;             // MOL: float samples [B][steps_total]
  unsigned int* barrier;    // grid barrier counter (zeroed by the host before launch)
  // per-row descriptors [Bpad]
  const int4* rowc;         // {start, T_u, first table row of its utterance, first frame of its utterance}
  const int4* rown;         // {steps, noise / generator key, first noise row of its block, rows in that block}
  const uint64_t* rowseed;  // built-in generator: keyed by (seed, step, key, slot)
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
  int fc3_rows;  // 512 (RAW) or 30 (MOL): the slices of units past it are zero
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
      v = (m < 2 || row < s.fc3_rows) ? W[(size_t)row * ld + k] : 0.0f;
    } else if (i < OFF_FC3B) {
      const int m = (i - OFF_B1IH) / 12;
      const int col = (i - OFF_B1IH) - m * 12;
      const int g = col / 4, j = col - g * 4;
      const float* b = (m == 0) ? s.r1_bih : (m == 1) ? s.r1_bhh : s.r2_bhh;
      v = b[g * RNN + c * UPC + j];
    } else if (i < OFF_FC3B + 4) {
      const int row = c * UPC + (i - OFF_FC3B);
      v = row < s.fc3_rows ? s.fc3_b[row] : 0.0f;
    }
    dst[i] = v;
  }
}

__device__ __forceinline__ void grid_barrier(unsigned int* counter, unsigned int& target) {
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

// the aux-table row that `row` reads at step gstep: its frame, or its utterance's "past the end" row
__device__ __forceinline__ int table_row(const LoopParams& p, int row, int gstep) {
  const int4 d = p.rowc[row];
  const int t = d.x + gstep;
  return d.z + (t < HOP * d.y ? t / HOP : d.y);
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

// Rows of one or several utterances with their own lengths (LoopParams::rowc / rown / rowseed); only the row blocks that hold
// a live row run, and a row stores nothing past its own last step.
// MOL: fc3 has 30 outputs (units of CTAs 0..7; the other CTAs skip phase E) and phase F is the mixture-of-logistics draw
template <bool MOL>
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
  const int nrb = (p.B + RB - 1) / RB;
  // descriptors of this CTA's own row (the first row of phase F): the same at every step, so read once and kept in shared
  // memory (in registers they would add spills to the GEMV phases)
  __shared__ int4 own;
  __shared__ uint64_t own_seed;

  {  // one-time: weights -> shared memory
    const float4* src = reinterpret_cast<const float4*>(p.wpack + (size_t)cta * WPACK_FLOATS);
    float4* dst = reinterpret_cast<float4*>(wsm);
    for (int i = tid; i < WPACK_FLOATS / 4; i += kThreads) dst[i] = src[i];
    for (int i = tid; i < RNN; i += kThreads) I0[i] = p.I0[i];
    if (tid == 0) {
      own = cta < p.B ? p.rown[cta] : make_int4(0, 0, 0, 0);
      own_seed = cta < p.B ? p.rowseed[cta] : 0;
    }
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
    if (!MOL && p.noise && cta < p.B && tid < NCLS / 4) {
      const float* src = p.noise + ((size_t)i * p.noise_B + (size_t)(own.z + own.y)) * NCLS + tid * 4;
      const uint32_t dst = (uint32_t)__cvta_generic_to_shared(qsm + tid * 4);
      asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory");
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
    // MOL: the 11 uniforms of this CTA's first row, one per lane of warp 0, loaded now and used after phase E
    float mol_pre = 0.0f;
    if (MOL && p.noise && cta < p.B && warp == 0 && lane < MB_MOL_UNIFORMS) {
      const size_t base = (size_t)i * MB_MOL_UNIFORMS * p.noise_B;
      mol_pre = p.noise[base + (size_t)MB_MOL_UNIFORMS * own.z +
                        (lane < MB_MOL_NMIX ? own.y * MB_MOL_NMIX + lane : MB_MOL_NMIX * own.w + own.y)];
    }
    // built-in generator: the same 512 values, one per thread, computed here instead of inside the sampling phase
    if (!MOL && !p.noise && cta < p.B && tid < NCLS) qsm[tid] = mb_exp1_noise(own_seed, (uint32_t)gstep, (uint32_t)own.y, (uint32_t)tid);

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
    grid_barrier(p.barrier, bar_target);

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
        const int frame = table_row(p, row, gstep);
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
    grid_barrier(p.barrier, bar_target);

    // ================= phases C, D, E: fc1, fc2, fc3 =================
#pragma unroll 1
    for (int layer = 0; layer < 3; ++layer) {
      const float* wl = wsm + (layer == 0 ? OFF_FC1 : layer == 1 ? OFF_FC2 : OFF_FC3);
      const int nrb_l = (MOL && layer == 2 && cta * UPC >= MB_MOL_NOUT) ? 0 : nrb;  // MOL: no fc3 unit on this CTA
      for (int rb = 0; rb < nrb_l; ++rb) {
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
            const int frame = table_row(p, row, gstep);
            v = v + (layer == 0 ? p.aux3P : p.aux4P)[(size_t)frame * RNN + unit];
            v = v > 0.0f ? v : 0.0f;
            (layer == 0 ? p.f1 : p.f2)[(size_t)unit * Bpad + row] = v;
          } else if (!MOL || unit < MB_MOL_NOUT) {
            p.logits[(size_t)unit * Bpad + row] = v + wsm[OFF_FC3B + j];
          }
        }
        __syncthreads();
      }
      asm volatile("cp.async.wait_group 0;" ::: "memory");  // this step's noise row has landed (issued at the top of the step)
      grid_barrier(p.barrier, bar_target);
    }

    if constexpr (MOL) {
      // ================= phase F (MOL): mixture pick + logistic draw (one warp per row) =================
      // lanes 0..9 score one component each; first maximum wins (the butterfly breaks ties towards the lower index)
      if (warp == 0) {
        const size_t base = (size_t)i * MB_MOL_UNIFORMS * p.noise_B;
        for (int row = cta; row < p.B; row += gridDim.x) {
          const int4 dn = row == cta ? own : p.rown[row];
          const uint64_t seed = row == cta ? own_seed : p.rowseed[row];
          // element offsets of the row's mixture uniforms and of its logistic uniform within the step
          const size_t mix0 = (size_t)MB_MOL_UNIFORMS * dn.z + (size_t)dn.y * MB_MOL_NMIX;
          const size_t log0 = (size_t)MB_MOL_UNIFORMS * dn.z + (size_t)MB_MOL_NMIX * dn.w + dn.y;
          float sc = -3.0e38f;
          if (lane < MB_MOL_NMIX) {
            const float t = (row == cta && p.noise) ? mol_pre
                            : (p.noise ? p.noise[base + mix0 + lane]
                                       : mb_mol_uniform(seed, (uint32_t)gstep, (uint32_t)dn.y, (uint32_t)lane));
            sc = mb_mol_score(p.logits[(size_t)lane * Bpad + row], t);
          }
          int best = lane;
#pragma unroll
          for (int off = 16; off >= 1; off >>= 1) {
            const float ov = __shfl_xor_sync(0xffffffffu, sc, off);
            const int ob = __shfl_xor_sync(0xffffffffu, best, off);
            if (ov > sc || (ov == sc && ob < best)) {
              sc = ov;
              best = ob;
            }
          }
          const float u_pre = __shfl_sync(0xffffffffu, mol_pre, MB_MOL_NMIX);
          if (lane == 0) {
            const float u = (row == cta && p.noise) ? u_pre
                            : (p.noise ? p.noise[base + log0]
                                       : mb_mol_uniform(seed, (uint32_t)gstep, (uint32_t)dn.y, MB_MOL_NMIX));
            const float x = mb_mol_sample(p.logits[(size_t)(MB_MOL_NMIX + best) * Bpad + row],
                                          p.logits[(size_t)(2 * MB_MOL_NMIX + best) * Bpad + row], u);
            if (gstep < dn.x) p.out_x[(size_t)row * p.steps_total + gstep] = x;
            p.xprev[row] = x;
          }
        }
      }
    } else if (warp == 0) {
    // ================= phase F: softmax + Categorical sample (one warp per row) =================
    // (the copies issued at the top of the step were waited for before the grid barrier above: qsm is complete and visible)
      for (int row = cta; row < p.B; row += gridDim.x) {
        const int4 dn = row == cta ? own : p.rown[row];
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
                          : (p.noise ? p.noise[((size_t)i * p.noise_B + (size_t)(dn.z + dn.y)) * NCLS + cls]
                                     : mb_exp1_noise(p.rowseed[row], (uint32_t)gstep, (uint32_t)dn.y, (uint32_t)cls));
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
          if (gstep < dn.x) p.out_idx[(size_t)row * p.steps_total + gstep] = (int16_t)best;
          p.xprev[row] = (2.0f * (float)best) / 511.0f - 1.0f;
        }
      }
    }
    grid_barrier(p.barrier, bar_target);
  }
}

}  // namespace
}  // namespace mb

// =================================================================================================
// C ABI
// =================================================================================================
using namespace mb;

struct mb_wavernn {
  mb_wavernn_config cfg{};
  int mode = MB_WAVERNN_RAW;  // fixed at create: MB_WAVERNN_RAW (512-way Categorical) or MB_WAVERNN_MOL (mixture of logistics)
  int ncls = NCLS;          // fc3 outputs: 512 or 30
  WeightTable w;           // raw weights as given
  size_t pack_off = 0;     // per-CTA packs
  size_t total_floats = 0;
  float* arena = nullptr;
  bool finalized = false;
  // conditioning held in the workspace cond_ws: frames per utterance of the last mb_wavernn_condition[_multi]; empty before
  std::vector<int32_t> cond_frames;
  void* cond_ws = nullptr;
};

namespace {

const float* W(const mb_wavernn* h, const std::string& name) { return h->w.ptr(name); }

struct Ws {
  size_t aux, melup, aux2P, aux3P, aux4P, tmpA, tmpB, tmpR, padP, lad5, lad25, lad200, segs, condI, h1, h2, f1, f2, logits,
      xprev, barrier, rowdesc;  // floats
  size_t total;                 // bytes
};

// T frames of U utterances in all (each utterance has its own "past the end" table row and its own 4 frames of ladder padding);
// the segment tables of the conditioning kernels and the row descriptors of the sample loop are always laid out
Ws ws_layout(int T, int Bpad, int chunk_steps, int U) {
  Ws L{};
  WsLayout W;
  L.aux = W.take<float>((size_t)T * CDIM);
  L.melup = W.take<float>((size_t)HOP * T * FEAT);
  L.aux2P = W.take<float>((size_t)(T + U) * 3 * RNN);
  L.aux3P = W.take<float>((size_t)(T + U) * RNN);
  L.aux4P = W.take<float>((size_t)(T + U) * RNN);
  L.tmpA = W.take<float>((size_t)CDIM * T);
  L.tmpB = W.take<float>((size_t)CDIM * T);
  L.tmpR = W.take<float>((size_t)CDIM * T);
  L.padP = W.take<float>((size_t)FEAT * (T + 4 * U));
  L.lad5 = W.take<float>((size_t)FEAT * (T + 4 * U) * 5);
  L.lad25 = W.take<float>((size_t)FEAT * (T + 4 * U) * 25);
  L.lad200 = W.take<float>((size_t)FEAT * (T + 4 * U) * HOP);
  L.segs = W.take<float>((size_t)3 * T + 7 * U);  // int32: fseg[T] pseg[T+4U] tsrc[T+U] segF[U] segT[U]
  L.condI = W.take<float>((size_t)chunk_steps * RNN * Bpad);
  L.h1 = W.take<float>((size_t)2 * RNN * Bpad);
  L.h2 = W.take<float>((size_t)2 * RNN * Bpad);
  L.f1 = W.take<float>((size_t)RNN * Bpad);
  L.f2 = W.take<float>((size_t)RNN * Bpad);
  L.logits = W.take<float>((size_t)RNN * Bpad);
  L.xprev = W.take<float>((size_t)Bpad);
  L.barrier = W.take<float>(1);  // the grid barrier's counter
  L.rowdesc = W.take<float>((size_t)10 * Bpad);  // int4 rowc[Bpad] | int4 rown[Bpad] | uint64 rowseed[Bpad]
  L.total = W.total();
  return L;
}

constexpr int kChunkMax = 128;  // steps per mb_wavernn_generate call

int bpad_of(int B) { return ((B + RB - 1) / RB) * RB; }

// total frames of a set of utterances, or -1 when the list is not usable
int64_t total_frames(const int32_t* frames, int32_t n_utts) {
  if (!frames || n_utts <= 0) return -1;
  int64_t tot = 0;
  for (int u = 0; u < n_utts; ++u) {
    if (frames[u] <= 0) return -1;
    tot += frames[u];
  }
  // the kernels index the x200 upsampled, 80-channel ladder with 32-bit ints
  return ((tot + 4 * (int64_t)n_utts) * HOP * FEAT < (int64_t)1 << 31) ? tot : -1;
}

// conditioning of n_utts utterances (mb_wavernn_condition is the case n_utts = 1): MelResNet, the x200 mel ladder and the three
// frame-rate aux tables of every utterance, written into the workspace for the sample loop
int condition_impl(const char* fn, mb_wavernn* h, const float* mel_concat, const int32_t* frames, int32_t n_utts,
                   void* workspace, size_t workspace_bytes, void* stream) {
  if (!h || !mel_concat || !frames) return fail(MB_ERR_INVALID, "%s: null argument", fn);
  const int64_t tot = total_frames(frames, n_utts);
  if (tot < 0) return fail(MB_ERR_INVALID, "%s: bad utterance lengths (each > 0, %d frames in all at most)", fn,
                           (int)(((int64_t)1 << 31) / (HOP * FEAT)));
  const int U = n_utts, Ttot = (int)tot, Tptot = Ttot + 4 * U, R = Ttot + U;
  // the conditioning part of the layout does not depend on the row count; the check asks for the smallest full workspace
  const Ws L = ws_layout(Ttot, RB, kChunkMax, U);
  float* ws;
  if (int rc = bind(fn, workspace, workspace_bytes, L.total, &ws)) return rc;
  if (!h->finalized) return fail(MB_ERR_STATE, "%s: weights not finalized", fn);
  cudaStream_t st = (cudaStream_t)stream;
  // segment tables
  std::vector<int32_t> seg((size_t)3 * Ttot + 7 * U);
  int32_t* fseg_h = seg.data();
  int32_t* pseg_h = fseg_h + Ttot;
  int32_t* tsrc_h = pseg_h + Tptot;
  int32_t* segF_h = tsrc_h + R;
  int32_t* segT_h = segF_h + U;
  for (int u = 0, F = 0; u < U; F += frames[u], ++u) {
    const int T = frames[u];
    segF_h[u] = F;
    segT_h[u] = T;
    for (int t = 0; t < T; ++t) fseg_h[F + t] = u;
    for (int t = 0; t < T + 4; ++t) pseg_h[F + 4 * u + t] = u;
    for (int t = 0; t <= T; ++t) tsrc_h[F + u + t] = t < T ? F + t : -1;
  }
  int* fseg = reinterpret_cast<int*>(ws + L.segs);
  const int *pseg = fseg + Ttot, *tsrc = pseg + Tptot, *segF = tsrc + R, *segT = segF + U;
  MB_CUDA_CHECK(cudaMemcpyAsync(fseg, seg.data(), sizeof(int32_t) * seg.size(), cudaMemcpyHostToDevice, st));
  MB_CUDA_CHECK(cudaStreamSynchronize(st));  // seg goes out of scope
  const int n = CDIM * Ttot, nb = (n + 255) / 256;
  float *x = ws + L.tmpA, *y = ws + L.tmpB, *r = ws + L.tmpR;
  k_conv_in<<<nb, 256, 0, st>>>(W(h, "upsample.resnet.conv_in.weight"), mel_concat, Ttot, fseg, segF, segT, x);
  MB_LAUNCH_CHECK("k_conv_in");
  auto bnrun = [&](const std::string& p, float* buf, int relu, const float* res) -> int {
    k_bn<<<nb, 256, 0, st>>>(W(h, p + ".weight"), W(h, p + ".bias"), W(h, p + ".running_mean"), W(h, p + ".running_var"),
                             buf, Ttot, relu, res);
    MB_LAUNCH_CHECK("k_bn");
    return MB_OK;
  };
  int rc = bnrun("upsample.resnet.batch_norm", x, 1, nullptr);
  if (rc) return rc;
  for (int i = 0; i < h->cfg.res_blocks; ++i) {
    const std::string b = "upsample.resnet.layers." + std::to_string(i);
    MB_CUDA_CHECK(cudaMemcpyAsync(r, x, sizeof(float) * n, cudaMemcpyDeviceToDevice, st));
    k_conv1x1<<<nb, 256, 0, st>>>(W(h, b + ".conv1.weight"), x, Ttot, y, nullptr, 0);
    MB_LAUNCH_CHECK("k_conv1x1");
    if ((rc = bnrun(b + ".batch_norm1", y, 1, nullptr))) return rc;
    k_conv1x1<<<nb, 256, 0, st>>>(W(h, b + ".conv2.weight"), y, Ttot, x, nullptr, 0);
    MB_LAUNCH_CHECK("k_conv1x1");
    if ((rc = bnrun(b + ".batch_norm2", x, 0, r))) return rc;
  }
  k_conv1x1<<<nb, 256, 0, st>>>(W(h, "upsample.resnet.conv_out.weight"), x, Ttot, ws + L.aux,
                                W(h, "upsample.resnet.conv_out.bias"), 1);
  MB_LAUNCH_CHECK("k_conv1x1");
  // mel ladder: P (each utterance padded by 2 frames on both sides) -> x5 -> x25 -> x200, then crop
  float* P = ws + L.padP;
  float* l5 = ws + L.lad5;
  float* l25 = ws + L.lad25;
  float* l1 = ws + L.lad200;
  k_pad_mel<<<(FEAT * Tptot + 255) / 256, 256, 0, st>>>(mel_concat, Tptot, pseg, segF, segT, P);
  MB_LAUNCH_CHECK("k_pad_mel");
  const int s0 = h->cfg.upsample_factors[0], s1 = h->cfg.upsample_factors[1], s2 = h->cfg.upsample_factors[2];
  auto blocks = [](size_t n_out) { return (unsigned)((n_out + 255) / 256); };
  k_ladder<<<blocks((size_t)FEAT * Tptot * s0), 256, 0, st>>>(W(h, "upsample.up_layers.1.weight"), P, Tptot, s0, 1, pseg, segF,
                                                             segT, l5);
  MB_LAUNCH_CHECK("k_ladder");
  k_ladder<<<blocks((size_t)FEAT * Tptot * s0 * s1), 256, 0, st>>>(W(h, "upsample.up_layers.3.weight"), l5, Tptot * s0, s1, s0,
                                                                  pseg, segF, segT, l25);
  MB_LAUNCH_CHECK("k_ladder");
  k_ladder<<<blocks((size_t)FEAT * Tptot * HOP), 256, 0, st>>>(W(h, "upsample.up_layers.5.weight"), l25, Tptot * s0 * s1, s2,
                                                              s0 * s1, pseg, segF, segT, l1);
  MB_LAUNCH_CHECK("k_ladder");
  k_crop_melup<<<blocks((size_t)HOP * Ttot * FEAT), 256, 0, st>>>(l1, Tptot * HOP, Ttot, fseg, ws + L.melup);
  MB_LAUNCH_CHECK("k_crop_melup");
  // frame-rate tables of the aux contributions
  k_aux_table<<<(R * 3 * RNN + 255) / 256, 256, 0, st>>>(W(h, "rnn2.weight_ih_l0"), RNN + AUXD, RNN, W(h, "rnn2.bias_ih_l0"),
                                                         ws + L.aux, AUXD, tsrc, R, 3 * RNN, ws + L.aux2P);
  MB_LAUNCH_CHECK("k_aux_table");
  k_aux_table<<<(R * RNN + 255) / 256, 256, 0, st>>>(W(h, "fc1.weight"), RNN + AUXD, RNN, W(h, "fc1.bias"), ws + L.aux,
                                                     2 * AUXD, tsrc, R, RNN, ws + L.aux3P);
  MB_LAUNCH_CHECK("k_aux_table");
  k_aux_table<<<(R * RNN + 255) / 256, 256, 0, st>>>(W(h, "fc2.weight"), RNN + AUXD, RNN, W(h, "fc2.bias"), ws + L.aux,
                                                     3 * AUXD, tsrc, R, RNN, ws + L.aux4P);
  MB_LAUNCH_CHECK("k_aux_table");
  h->cond_ws = workspace;
  h->cond_frames.assign(frames, frames + U);
  return MB_OK;
}

}  // namespace

extern "C" {

int mb_wavernn_create(const mb_wavernn_config* cfg, mb_wavernn** out) {
  return mb_wavernn_create_mode(cfg, MB_WAVERNN_RAW, out);
}

int mb_wavernn_create_mode(const mb_wavernn_config* cfg, int32_t mode, mb_wavernn** out) {
  if (!cfg || !out) return fail(MB_ERR_INVALID, "mb_wavernn_create: null argument");
  if (mode != MB_WAVERNN_RAW && mode != MB_WAVERNN_MOL) return fail(MB_ERR_INVALID, "mb_wavernn_create_mode: unknown mode %d", mode);
  if (cfg->rnn_dims != RNN || cfg->fc_dims != RNN || cfg->bits != 9 || cfg->pad != 2 || cfg->num_upsample != 3 ||
      cfg->upsample_factors[0] * cfg->upsample_factors[1] * cfg->upsample_factors[2] != HOP ||
      cfg->upsample_factors[0] != 5 || cfg->upsample_factors[1] != 5 || cfg->feat_dims != FEAT ||
      cfg->compute_dims != CDIM || cfg->res_out_dims != CDIM || cfg->res_blocks < 1 || cfg->res_blocks > 16)
    return fail(MB_ERR_INVALID,
                "mb_wavernn_create: only the reference hparams are built (rnn/fc 512, 9 bits, pad 2, "
                "upsample (5,5,8), 80 mels, compute/res_out 128)");
  mb_wavernn* h = new mb_wavernn();
  h->cfg = *cfg;
  h->mode = mode;
  h->ncls = mode == MB_WAVERNN_MOL ? MB_MOL_NOUT : NCLS;
  h->w.add("upsample.resnet.conv_in.weight", {CDIM, FEAT, 5});
  auto bn = [&](const std::string& p) {
    for (const char* leaf : {".weight", ".bias", ".running_mean", ".running_var"}) h->w.add(p + leaf, {CDIM});
  };
  bn("upsample.resnet.batch_norm");
  for (int i = 0; i < cfg->res_blocks; ++i) {
    const std::string b = "upsample.resnet.layers." + std::to_string(i);
    h->w.add(b + ".conv1.weight", {CDIM, CDIM, 1});
    h->w.add(b + ".conv2.weight", {CDIM, CDIM, 1});
    bn(b + ".batch_norm1");
    bn(b + ".batch_norm2");
  }
  h->w.add("upsample.resnet.conv_out.weight", {CDIM, CDIM, 1});
  h->w.add("upsample.resnet.conv_out.bias", {CDIM});
  for (int j = 0; j < 3; ++j)
    h->w.add("upsample.up_layers." + std::to_string(2 * j + 1) + ".weight", {1, 1, 1, 2 * cfg->upsample_factors[j] + 1});
  h->w.add("I.weight", {RNN, FEAT + AUXD + 1});
  h->w.add("I.bias", {RNN});
  h->w.add("rnn1.weight_ih_l0", {3 * RNN, RNN});
  h->w.add("rnn1.weight_hh_l0", {3 * RNN, RNN});
  h->w.add("rnn1.bias_ih_l0", {3 * RNN});
  h->w.add("rnn1.bias_hh_l0", {3 * RNN});
  h->w.add("rnn2.weight_ih_l0", {3 * RNN, RNN + AUXD});
  h->w.add("rnn2.weight_hh_l0", {3 * RNN, RNN});
  h->w.add("rnn2.bias_ih_l0", {3 * RNN});
  h->w.add("rnn2.bias_hh_l0", {3 * RNN});
  h->w.add("fc1.weight", {RNN, RNN + AUXD});
  h->w.add("fc1.bias", {RNN});
  h->w.add("fc2.weight", {RNN, RNN + AUXD});
  h->w.add("fc2.bias", {RNN});
  h->w.add("fc3.weight", {h->ncls, RNN});
  h->w.add("fc3.bias", {h->ncls});
  h->pack_off = h->w.floats();
  h->total_floats = h->pack_off + (size_t)NCTA * WPACK_FLOATS + RNN;
  *out = h;
  return MB_OK;
}

void mb_wavernn_destroy(mb_wavernn* h) { delete h; }

size_t mb_wavernn_arena_bytes(const mb_wavernn* h) { return h ? h->total_floats * sizeof(float) : 0; }

int mb_wavernn_set_arena(mb_wavernn* h, void* arena, size_t bytes) {
  if (int rc = check_arena("mb_wavernn_set_arena", h, arena, bytes, mb_wavernn_arena_bytes(h), 256)) return rc;
  h->w.attach((float*)arena);
  h->arena = (float*)arena;
  h->finalized = false;
  return MB_OK;
}

int mb_wavernn_set_weight(mb_wavernn* h, const char* name, const float* w, const int64_t* dims, int32_t ndim,
                          void* stream) {
  if (!h) return fail(MB_ERR_INVALID, "mb_wavernn_set_weight: null argument");
  if (int rc = h->w.set("mb_wavernn_set_weight", name, w, dims, ndim, stream)) return rc;
  h->finalized = false;
  return MB_OK;
}

int mb_wavernn_finalize(mb_wavernn* h, void* stream) {
  if (!h) return fail(MB_ERR_INVALID, "mb_wavernn_finalize: null handle");
  if (int rc = h->w.check_all_set("mb_wavernn_finalize")) return rc;
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
  ps.fc3_rows = h->ncls;
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
  return mb_wavernn_workspace_bytes_multi(h, 1, &frames, folds, steps);
}

size_t mb_wavernn_workspace_bytes_multi(const mb_wavernn* h, int32_t n_utts, const int32_t* frames, int32_t rows,
                                        int32_t max_steps) {
  const int64_t Ttot = total_frames(frames, n_utts);
  if (!h || Ttot < 0 || rows <= 0) return 0;
  (void)max_steps;
  return ws_layout((int)Ttot, bpad_of(rows), kChunkMax, n_utts).total;
}

int mb_wavernn_condition(mb_wavernn* h, const float* mel, int32_t T, void* workspace, size_t workspace_bytes,
                         void* stream) {
  return condition_impl("mb_wavernn_condition", h, mel, &T, 1, workspace, workspace_bytes, stream);
}

int mb_wavernn_condition_multi(mb_wavernn* h, const float* mel_concat, const int32_t* frames, int32_t n_utts, void* workspace,
                               size_t workspace_bytes, void* stream) {
  return condition_impl("mb_wavernn_condition_multi", h, mel_concat, frames, n_utts, workspace, workspace_bytes, stream);
}

}  // extern "C"

namespace {

// One chunk of the sample loop over a row table the caller has checked: `rows` rows, of which the first n_live are alive, and
// `noise_rows` rows of injected noise per step.  At step0 == 0 the state is reset and the row descriptors are uploaded, as
// describe(rowc, rown, rowseed) writes them for the `rows` rows (int32 [4] per row for rowc and rown; LoopParams).  Exactly one
// of out_idx (RAW handle) / out_x (MOL handle) is given.
template <class Describe>
int sample_chunk(const char* fn, mb_wavernn* h, int rows, int n_live, int noise_rows, int max_steps, int step0, int nsteps,
                 const float* noise, int16_t* out_idx, float* out_x, void* workspace, size_t workspace_bytes, void* stream,
                 Describe describe) {
  int Ttot = 0;
  for (int t : h->cond_frames) Ttot += t;
  const int Bpad = bpad_of(rows);
  const Ws L = ws_layout(Ttot, Bpad, kChunkMax, (int)h->cond_frames.size());
  float* ws;
  if (int rc = bind(fn, workspace, workspace_bytes, L.total, &ws)) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  int4* rowc = reinterpret_cast<int4*>(ws + L.rowdesc);
  int4* rown = rowc + Bpad;
  uint64_t* rowseed = reinterpret_cast<uint64_t*>(rown + Bpad);
  if (step0 == 0) {
    // zero initial state (fatchord_version.py:178-185) and upload the row descriptors (rows past the table: T_u == 0, never
    // live)
    MB_CUDA_CHECK(cudaMemsetAsync(ws + L.h1, 0, sizeof(float) * (L.xprev + align_up((size_t)Bpad, 64) - L.h1), st));
    std::vector<int32_t> tmp((size_t)10 * Bpad, 0);
    describe(tmp.data(), tmp.data() + 4 * Bpad, reinterpret_cast<uint64_t*>(tmp.data() + 8 * Bpad));
    MB_CUDA_CHECK(cudaMemcpyAsync(rowc, tmp.data(), sizeof(int32_t) * tmp.size(), cudaMemcpyHostToDevice, st));
    MB_CUDA_CHECK(cudaStreamSynchronize(st));  // tmp goes out of scope
  }
  const int Wl = bpad_of(n_live);  // rows of the live row blocks
  k_condI<<<nsteps * Wl, 256, 0, st>>>(W(h, "I.weight"), W(h, "I.bias"), ws + L.melup, ws + L.aux, rowc, Wl, Bpad, step0, nsteps,
                                       ws + L.condI);
  MB_LAUNCH_CHECK("k_condI");
  MB_CUDA_CHECK(cudaMemsetAsync(ws + L.barrier, 0, sizeof(unsigned int), st));
  LoopParams p;
  memset(&p, 0, sizeof(p));
  p.wpack = h->arena + h->pack_off;
  p.I0 = h->arena + h->pack_off + (size_t)NCTA * WPACK_FLOATS;
  p.aux2P = ws + L.aux2P;
  p.aux3P = ws + L.aux3P;
  p.aux4P = ws + L.aux4P;
  p.condI = ws + L.condI;
  p.B = n_live;
  p.Bpad = Bpad;
  p.step0 = step0;
  p.nsteps = nsteps;
  p.steps_total = max_steps;
  p.h1 = ws + L.h1;
  p.h2 = ws + L.h2;
  p.f1 = ws + L.f1;
  p.f2 = ws + L.f2;
  p.logits = ws + L.logits;
  p.xprev = ws + L.xprev;
  p.noise = noise;
  p.noise_B = noise_rows;
  p.out_idx = out_idx;
  p.out_x = out_x;
  p.barrier = reinterpret_cast<unsigned int*>(ws + L.barrier);
  p.rowc = rowc;
  p.rown = rown;
  p.rowseed = rowseed;
  const bool mol = h->mode == MB_WAVERNN_MOL;
  const void* kern = mol ? (const void*)k_sample_loop<true> : (const void*)k_sample_loop<false>;
  const size_t smem = sizeof(float) * SMEM_FLOATS;
  static bool attr[2] = {false, false};
  if (!attr[mol]) {
    MB_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    attr[mol] = true;
  }
  void* args[] = {(void*)&p};
  MB_CUDA_CHECK(cudaLaunchCooperativeKernel(kern, dim3(NCTA), dim3(kThreads), args, smem, st));
  count_launch();
  return MB_OK;
}

// mb_wavernn_generate_rows[_mol]: the folds of the one conditioned utterance as a one-utterance row table.  Row r is fold
// row0 + r of a block of noise_folds noise rows, which is also its generator key, so a fold draws the same noise however the
// folds are dealt to calls.
int generate_folds(mb_wavernn* h, const int32_t* fold_starts_host, int32_t B, int32_t steps, int32_t step0, int32_t nsteps,
                   const float* noise, int32_t noise_folds, int32_t row0, uint64_t seed, int16_t* out_idx, float* out_x,
                   void* workspace, size_t workspace_bytes, void* stream) {
  if (row0 < 0 || (noise && row0 + B > noise_folds))
    return fail(MB_ERR_INVALID, "mb_wavernn_generate_rows: rows [%d, %d) outside the %d noise rows", row0, row0 + B, noise_folds);
  if (B <= 0 || nsteps <= 0 || nsteps > kChunkMax || step0 < 0 || step0 + nsteps > steps)
    return fail(MB_ERR_INVALID, "mb_wavernn_generate: bad step range (at most %d steps per call)", kChunkMax);
  for (int r = 0; r < B; ++r)
    if (fold_starts_host[r] < 0 || fold_starts_host[r] > INT32_MAX - steps)
      return fail(MB_ERR_INVALID, "mb_wavernn_generate: fold start %d of row %d outside [0, %d]", fold_starts_host[r], r,
                  INT32_MAX - steps);
  if (!h->finalized) return fail(MB_ERR_STATE, "mb_wavernn_generate: weights not finalized");
  if (h->cond_frames.size() != 1 || h->cond_ws != workspace)
    return fail(MB_ERR_STATE, "mb_wavernn_generate: call mb_wavernn_condition on this workspace first");
  const int T = h->cond_frames[0];
  return sample_chunk("mb_wavernn_generate", h, B, B, noise_folds, steps, step0, nsteps, noise, out_idx, out_x, workspace,
                      workspace_bytes, stream, [&](int32_t* c, int32_t* n, uint64_t* sd) {
                        for (int r = 0; r < B; ++r) {
                          c[4 * r + 0] = fold_starts_host[r];
                          c[4 * r + 1] = T;
                          n[4 * r + 0] = steps;
                          n[4 * r + 1] = row0 + r;
                          n[4 * r + 3] = noise_folds;
                          sd[r] = seed;
                        }
                      });
}

// mb_wavernn_generate_multi[_mol]: whole utterances side by side (folds 0 .. n-1 of one utterance, all of one length), longest
// rows first.  Row r is fold row_fold[r] of its utterance's block of noise rows.
int generate_multi_impl(const char* fn, mb_wavernn* h, const int32_t* row_utt, const int32_t* row_start,
                        const int32_t* row_steps, const int32_t* row_fold, int32_t rows, const uint64_t* utt_seeds,
                        int32_t max_steps, int32_t step0, int32_t nsteps, int32_t n_live, const float* noise, int16_t* out_idx,
                        float* out_x, void* workspace, size_t workspace_bytes, void* stream) {
  if (rows <= 0 || max_steps <= 0 || nsteps <= 0 || nsteps > kChunkMax || step0 < 0 || step0 + nsteps > max_steps)
    return fail(MB_ERR_INVALID, "%s: bad row count or step range (at most %d steps per call)", fn, kChunkMax);
  int alive = 0;
  for (int r = 0; r < rows; ++r) {
    if (row_utt[r] < 0 || row_start[r] < 0 || row_start[r] > INT32_MAX - max_steps || row_steps[r] <= 0 ||
        row_steps[r] > max_steps || row_fold[r] < 0)
      return fail(MB_ERR_INVALID, "%s: row %d (utterance %d, start %d, steps %d, fold %d) outside the table", fn, r, row_utt[r],
                  row_start[r], row_steps[r], row_fold[r]);
    if (r > 0 && row_steps[r] > row_steps[r - 1]) return fail(MB_ERR_INVALID, "%s: rows must be ordered longest first (row %d)", fn, r);
    const bool cont = r > 0 && row_utt[r] == row_utt[r - 1];
    if (cont ? (row_fold[r] != row_fold[r - 1] + 1 || row_steps[r] != row_steps[r - 1]) : row_fold[r] != 0)
      return fail(MB_ERR_INVALID, "%s: the folds of an utterance must be adjacent rows 0, 1, .. of one length (row %d)", fn, r);
    alive += row_steps[r] > step0;
  }
  if (n_live != alive)
    return fail(MB_ERR_INVALID, "%s: %d rows are alive at step %d, the call says %d", fn, alive, step0, n_live);
  if (n_live < rows && row_utt[n_live] == row_utt[n_live - 1])
    return fail(MB_ERR_INVALID, "%s: the live rows end inside utterance %d", fn, row_utt[n_live]);
  if (!h->finalized) return fail(MB_ERR_STATE, "%s: weights not finalized", fn);
  if (h->cond_frames.empty() || h->cond_ws != workspace)
    return fail(MB_ERR_STATE, "%s: call mb_wavernn_condition_multi on this workspace first", fn);
  const int U = (int)h->cond_frames.size();
  for (int r = 0; r < rows; ++r)
    if (row_utt[r] >= U) return fail(MB_ERR_INVALID, "%s: row %d names utterance %d of %d", fn, r, row_utt[r], U);
  return sample_chunk(fn, h, rows, n_live, n_live, max_steps, step0, nsteps, noise, out_idx, out_x, workspace, workspace_bytes,
                      stream, [&](int32_t* c, int32_t* n, uint64_t* sd) {
                        std::vector<int32_t> fbase(U);
                        for (int u = 0, f = 0; u < U; f += h->cond_frames[u], ++u) fbase[u] = f;
                        for (int r = 0, first = 0; r < rows; ++r) {
                          const int u = row_utt[r];
                          if (row_fold[r] == 0) first = r;
                          c[4 * r + 0] = row_start[r];
                          c[4 * r + 1] = h->cond_frames[u];
                          c[4 * r + 2] = fbase[u] + u;
                          c[4 * r + 3] = fbase[u];
                          n[4 * r + 0] = row_steps[r];
                          n[4 * r + 1] = row_fold[r];
                          n[4 * r + 2] = first;
                          sd[r] = utt_seeds ? utt_seeds[u] : 0;
                        }
                        for (int r = rows - 1, nf = 0; r >= 0; --r) {  // folds of the row's utterance
                          if (r == rows - 1 || row_fold[r + 1] == 0) nf = row_fold[r] + 1;
                          n[4 * r + 3] = nf;
                        }
                      });
}

}  // namespace

extern "C" {

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
  if (h->mode != MB_WAVERNN_RAW) return fail(MB_ERR_INVALID, "mb_wavernn_generate_rows: a MOL handle samples floats (mb_wavernn_generate_rows_mol)");
  return generate_folds(h, fold_starts_host, B, steps, step0, nsteps, noise, noise_folds, row0, seed, out_idx, nullptr, workspace,
                        workspace_bytes, stream);
}

int mb_wavernn_generate_rows_mol(mb_wavernn* h, const int32_t* fold_starts_host, int32_t B, int32_t steps, int32_t step0,
                                 int32_t nsteps, const float* uniforms, int32_t noise_folds, int32_t row0, uint64_t seed,
                                 float* out_x, void* workspace, size_t workspace_bytes, void* stream) {
  if (!h || !fold_starts_host || !out_x || !workspace) return fail(MB_ERR_INVALID, "mb_wavernn_generate_rows_mol: null argument");
  if (h->mode != MB_WAVERNN_MOL) return fail(MB_ERR_INVALID, "mb_wavernn_generate_rows_mol: the handle was not created in MOL mode");
  return generate_folds(h, fold_starts_host, B, steps, step0, nsteps, uniforms, noise_folds, row0, seed, nullptr, out_x, workspace,
                        workspace_bytes, stream);
}

int mb_wavernn_last_logits(mb_wavernn* h, float* logits, int32_t B, void* workspace, void* stream) {
  if (!h || !logits || !workspace || h->cond_frames.size() != 1)
    return fail(MB_ERR_INVALID, "mb_wavernn_last_logits: bad argument");
  const int Bpad = bpad_of(B);
  const Ws L = ws_layout(h->cond_frames[0], Bpad, kChunkMax, 1);
  float* ws = aligned<float>(workspace);
  // logits are stored [class][Bpad]; return [B][ncls] (512 RAW, 30 MOL)
  const int ncls = h->ncls;
  MB_CUDA_CHECK(cudaMemcpy2DAsync(logits, sizeof(float) * ncls, ws + L.logits, sizeof(float), sizeof(float), 1,
                                  cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
  // generic strided transpose through a tiny loop of 2D copies (debug hook, B is small)
  for (int r = 0; r < B; ++r)
    MB_CUDA_CHECK(cudaMemcpy2DAsync(logits + (size_t)r * ncls, sizeof(float), ws + L.logits + r, sizeof(float) * Bpad,
                                    sizeof(float), ncls, cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
  return MB_OK;
}

int mb_wavernn_generate_multi(mb_wavernn* h, const int32_t* row_utt, const int32_t* row_start, const int32_t* row_steps,
                              const int32_t* row_fold, int32_t rows, const uint64_t* utt_seeds, int32_t max_steps,
                              int32_t step0, int32_t nsteps, int32_t n_live, const float* noise, int16_t* out_idx,
                              void* workspace, size_t workspace_bytes, void* stream) {
  if (!h || !row_utt || !row_start || !row_steps || !row_fold || !out_idx || !workspace || (!noise && !utt_seeds))
    return fail(MB_ERR_INVALID, "mb_wavernn_generate_multi: null argument");
  if (h->mode != MB_WAVERNN_RAW)
    return fail(MB_ERR_INVALID, "mb_wavernn_generate_multi: a MOL handle samples floats (mb_wavernn_generate_multi_mol)");
  return generate_multi_impl("mb_wavernn_generate_multi", h, row_utt, row_start, row_steps, row_fold, rows, utt_seeds, max_steps,
                             step0, nsteps, n_live, noise, out_idx, nullptr, workspace, workspace_bytes, stream);
}

int mb_wavernn_generate_multi_mol(mb_wavernn* h, const int32_t* row_utt, const int32_t* row_start, const int32_t* row_steps,
                                  const int32_t* row_fold, int32_t rows, const uint64_t* utt_seeds, int32_t max_steps,
                                  int32_t step0, int32_t nsteps, int32_t n_live, const float* uniforms, float* out_x,
                                  void* workspace, size_t workspace_bytes, void* stream) {
  if (!h || !row_utt || !row_start || !row_steps || !row_fold || !out_x || !workspace || (!uniforms && !utt_seeds))
    return fail(MB_ERR_INVALID, "mb_wavernn_generate_multi_mol: null argument");
  if (h->mode != MB_WAVERNN_MOL)
    return fail(MB_ERR_INVALID, "mb_wavernn_generate_multi_mol: the handle was not created in MOL mode");
  return generate_multi_impl("mb_wavernn_generate_multi_mol", h, row_utt, row_start, row_steps, row_fold, rows, utt_seeds,
                             max_steps, step0, nsteps, n_live, uniforms, nullptr, out_x, workspace, workspace_bytes, stream);
}

}  // extern "C"
