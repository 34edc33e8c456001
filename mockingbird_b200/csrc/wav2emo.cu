// wav2vec2 emotion model (models/synthesizer/models/wav2emo.py: EmotionExtractorModel, the encoder of extract_emo) on the H100:
// the feature extractor's normalisation, the LayerNorm conv feature encoder, the feature projection, the grouped positional
// conv and the pre-LN (stable layer norm) transformer, then the per-clip mean and the regression head.  Every clip of a
// ragged batch is computed as its own B = 1 call: no sum's order depends on the batch or on the clip's slot, the positional
// conv reads zeros outside the clip, attention sees only the clip's frames and the mean runs over the clip's frames.
//
//   norm_kernel        one CTA per clip: (x - mean) / sqrt(var + 1e-7) with numpy's float32 pairwise sums (mb_pairwise.cuh)
//   conv0_kernel       conv_layers.0 (1 -> C, FFMA) -> fp32 rows
//   ln_act_rows_kernel LayerNorm (eps 1e-5) + GELU of each conv layer, in place; rows past the clip's frames zeroed
//   im2col + tc_big    conv_layers.1.. as 3-term-split tensor-core GEMMs: the input viewed as rows of `stride` frames
//                      (ld = stride C) turns tap j into segment (j % stride, row shift j / stride)
//   ln_tiles / tc_big  feature projection, QKV (one N = 3D GEMM), out_proj (+ residual), FF1 / FF2 (+ residual)
//   posconv_tc_kernel  grouped Conv1d (weight norm folded by the host) as an implicit GEMM on the tensor cores (3-term split):
//                      each tap's operand is the clip's hi / lo window shifted by one row; SamePad, GELU, + residual
//   attn_tc_kernel     flash-style attention on the tensor cores (3-term split Q K^T and P V, online FP32 softmax) over the
//                      clip's own keys
//   ln_rows / mean / head  final LayerNorm, per-clip mean in frame order, dense + tanh + out_proj
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <mma.h>

#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <string>
#include <vector>

#include "encoder_layers.cuh"
#include "mb_common.h"
#include "mb_pairwise.cuh"
#include "tacotron_kernels.cuh"

using namespace mb;
using namespace mb::enc;

namespace {

constexpr int kMaxRows = 128;
constexpr int kMaxConv = 8;
constexpr int kNormThreads = 256;
constexpr int kPcT = 64;  // frames per positional-conv CTA
constexpr int kPcC = 64;  // output channels per positional-conv CTA
constexpr size_t kPcMaxSmem = 220 * 1024;  // create refuses a group width x taps whose window needs more

int kb_of(int K) { return (K + 63) / 64; }
size_t ceil128(size_t m) { return (m + 127) / 128 * 128; }

#define MB_TRY(x)                 \
  do {                            \
    const int _rc = (x);          \
    if (_rc != MB_OK) return _rc; \
  } while (0)

struct NormClip {
  int64_t off;
  int32_t n, depth;
};

// Wav2Vec2FeatureExtractor.zero_mean_unit_var_norm on float32: mean = sum / n, var = sum((x - mean)^2) / n (numpy's pairwise
// sums), y = (x - mean) / sqrt(var + 1e-7), every step one rounded float32 operation
__global__ void __launch_bounds__(kNormThreads) norm_kernel(const float* __restrict__ x, const NormClip* clips,
                                                            float* __restrict__ y) {
  __shared__ float part[kNormThreads];
  const NormClip c = clips[blockIdx.x];
  const float* a = x + c.off;
  const float fn = (float)c.n;
  const float mean = __fdiv_rn(pairwise_sum_block([a](int64_t i) { return a[i]; }, c.n, c.depth, part), fn);
  const float ss = pairwise_sum_block(
      [a, mean](int64_t i) {
        const float d = __fsub_rn(a[i], mean);
        return __fmul_rn(d, d);
      },
      c.n, c.depth, part);
  const float sd = __fsqrt_rn(__fadd_rn(__fdiv_rn(ss, fn), 1e-7f));
  for (int64_t i = threadIdx.x; i < c.n; i += blockDim.x) y[c.off + i] = __fdiv_rn(__fsub_rn(a[i], mean), sd);
}

// conv_layers.0 (one input channel): y[b S + t][c] = bias[c] + sum_j w[c][j] x_b[t s + j] for t < len[b], zero for t in [len[b], S)
__global__ void conv0_kernel(const float* __restrict__ x, const int64_t* __restrict__ off, const int* __restrict__ len, int S,
                             const float* __restrict__ w, const float* __restrict__ bias, int C, int k, int s,
                             float* __restrict__ y) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int b = blockIdx.y;
  if (i >= (size_t)S * C) return;
  const int c = (int)(i % C), t = (int)(i / C);
  float acc = 0.f;
  if (t < len[b]) {
    const float* xb = x + off[b] + (int64_t)t * s;
    for (int j = 0; j < k; ++j) acc += w[c * k + j] * xb[j];
    if (bias) acc += bias[c];
  }
  y[((size_t)b * S + t) * C + c] = acc;
}

// LayerNorm (eps) + activation of rows [B][S] in place, one warp per row; rows t >= len[b] are written as zeros
__global__ void ln_act_rows_kernel(float* x, int M, int D, float eps, const float* __restrict__ g, const float* __restrict__ be,
                                   int act, const int* __restrict__ len, int S) {
  const int m = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (m >= M) return;
  float* xr = x + (size_t)m * D;
  if (m % S >= len[m / S]) {
    for (int n = lane; n < D; n += 32) xr[n] = 0.f;
    return;
  }
  float mean, rstd;
  row_stats(xr, D, lane, eps, mean, rstd);
  __syncwarp();
  for (int n = lane; n < D; n += 32) xr[n] = act_f((xr[n] - mean) * rstd * g[n] + be[n], act);
}

// Positional conv of one (clip b, 64 frames, 64 output channels of group g) as an implicit GEMM on the tensor cores:
// out = x + gelu(bias + sum_{j, ci} w[co][ci][j] x[t + j - k/2][ci]), zeros outside the clip's frames (the even-k SamePad drops
// output T, which this never computes).  The clip's window of frames [t0 - k/2, t0 + 63 - k/2 + k) is split once into fp16
// hi / lo rows in shared memory; tap j's A operand is that window shifted by j rows, so no im2col is built.  B is the packed
// weight image [g][j][ci][co] (hi | lo, scaled by a power of two) read straight from global memory.  3-term split
// (hi hi + lo hi + hi lo) with FP32 accumulation in (tap, 16-channel step) order; 4 warps of 16 frames x 64 channels.
__global__ void __launch_bounds__(128) posconv_tc_kernel(const float* __restrict__ x, const __half* __restrict__ w_hi,
                                                         const __half* __restrict__ w_lo, float inv_scale,
                                                         const float* __restrict__ bias, const int* __restrict__ len, int S,
                                                         int D, int cg, int k, float* __restrict__ out) {
  using namespace nvcuda;
  extern __shared__ __align__(128) unsigned char pc_sm[];
  const int rows = kPcT + k - 1;
  __half* xh = reinterpret_cast<__half*>(pc_sm);           // [rows][cg]
  __half* xl = xh + (size_t)rows * cg;                     // [rows][cg]
  float* of = reinterpret_cast<float*>(xl + (size_t)rows * cg);  // [4 warps][16][64]
  const int b = blockIdx.z, t0 = blockIdx.x * kPcT;
  const int chunks = cg / kPcC;
  const int g = blockIdx.y / chunks, cc = blockIdx.y % chunks;
  const int T = len[b];
  const int pad = k / 2;
  const float* xb = x + (size_t)b * S * D + g * cg;
  for (int e = threadIdx.x; e < rows * cg; e += blockDim.x) {
    const int r = e / cg, ci = e - r * cg;
    const int tt = t0 - pad + r;
    const float v = (tt >= 0 && tt < T) ? xb[(size_t)tt * D + ci] : 0.f;
    const __half hi = __float2half_rn(v);
    xh[e] = hi;
    xl[e] = __float2half_rn(v - __half2float(hi));
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  wmma::fragment<wmma::accumulator, 16, 16, 16, float> acc[4];
#pragma unroll
  for (int n = 0; n < 4; ++n) wmma::fill_fragment(acc[n], 0.f);
  wmma::fragment<wmma::matrix_a, 16, 16, 16, __half, wmma::row_major> ah, al;
  wmma::fragment<wmma::matrix_b, 16, 16, 16, __half, wmma::row_major> bh, bl;
  for (int j = 0; j < k; ++j) {
    for (int kk = 0; kk < cg / 16; ++kk) {
      const size_t ao = (size_t)(warp * 16 + j) * cg + kk * 16;
      wmma::load_matrix_sync(ah, xh + ao, cg);
      wmma::load_matrix_sync(al, xl + ao, cg);
      const size_t wo = (((size_t)g * k + j) * cg + kk * 16) * cg + cc * kPcC;
#pragma unroll
      for (int n = 0; n < 4; ++n) {
        wmma::load_matrix_sync(bh, w_hi + wo + n * 16, cg);
        wmma::load_matrix_sync(bl, w_lo + wo + n * 16, cg);
        wmma::mma_sync(acc[n], ah, bh, acc[n]);
        wmma::mma_sync(acc[n], al, bh, acc[n]);
        wmma::mma_sync(acc[n], ah, bl, acc[n]);
      }
    }
  }
  float* o = of + warp * 16 * 64;
#pragma unroll
  for (int n = 0; n < 4; ++n) wmma::store_matrix_sync(o + n * 16, acc[n], 64, wmma::mem_row_major);
  __syncwarp();
  for (int e = lane; e < 16 * 64; e += 32) {
    const int r = e >> 6, c = e & 63;
    const int tt = t0 + warp * 16 + r;
    if (tt >= S) continue;
    const int n = g * cg + cc * kPcC + c;
    const size_t oo = ((size_t)b * S + tt) * D + n;
    out[oo] = tt < T ? x[oo] + gelu_erf(o[e] * inv_scale + bias[n]) : 0.f;
  }
}

// packed image [g][j][ci][co] = w[g cg + co][ci][j] * scale as fp16 hi and lo
__global__ void posconv_pack_kernel(const float* __restrict__ w, int D, int cg, int k, float scale, __half* __restrict__ w_hi,
                                    __half* __restrict__ w_lo) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)D * cg * k) return;
  const int co = (int)(i % cg), ci = (int)((i / cg) % cg), j = (int)((i / ((size_t)cg * cg)) % k);
  const int g = (int)(i / ((size_t)cg * cg * k));
  const float v = w[((size_t)(g * cg + co) * cg + ci) * k + j] * scale;
  const __half hi = __float2half_rn(v);
  w_hi[i] = hi;
  w_lo[i] = __float2half_rn(v - __half2float(hi));
}

// Multi-head attention of one (clip b, head h, 64 queries) per CTA on the tensor cores, flash style: for each tile of 64 of the
// clip's keys, S = Q K^T (3-term fp16 split, FP32 accumulation) scaled by 1/8, an online softmax in FP32 (running max and sum
// per query row), then O = O corr + P V with P and V split the same way.  Keys at and past the clip's length are excluded;
// query rows in [len, S) are written as zeros.  dk = 64; 4 warps of 16 query rows; two lanes per row in the softmax.
__global__ void __launch_bounds__(128) attn_tc_kernel(const float* __restrict__ qkv, const int* __restrict__ len, int S, int D,
                                                      float* __restrict__ ctx) {
  using namespace nvcuda;
  constexpr int Q = 64, KT = 64, DK = 64;
  extern __shared__ __align__(128) unsigned char at_sm[];
  __half* qh = reinterpret_cast<__half*>(at_sm);  // [Q][DK]
  __half* ql = qh + Q * DK;
  __half* kh = ql + Q * DK;                       // [KT][DK]
  __half* kl = kh + KT * DK;
  __half* vh = kl + KT * DK;
  __half* vl = vh + KT * DK;
  float* sf = reinterpret_cast<float*>(vl + KT * DK);  // per warp [16][KT] scores
  float* of = sf + 4 * 16 * KT;                         // per warp [16][DK] running output
  __half* ph = reinterpret_cast<__half*>(of + 4 * 16 * DK);  // per warp [16][KT]
  __half* pl = ph + 4 * 16 * KT;
  const int b = blockIdx.z, h = blockIdx.y, i0 = blockIdx.x * Q;
  const int T = len[b];
  const size_t ld = 3 * (size_t)D, rb = (size_t)b * S;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (i0 >= T) {  // every query row of this CTA lies past the clip
    for (int e = threadIdx.x; e < Q * DK; e += blockDim.x) {
      const int i = i0 + e / DK;
      if (i < S) ctx[(rb + i) * D + h * DK + (e % DK)] = 0.f;
    }
    return;
  }
  auto split = [](float v, __half* hi, __half* lo, int e) {
    const __half a = __float2half_rn(v);
    hi[e] = a;
    lo[e] = __float2half_rn(v - __half2float(a));
  };
  for (int e = threadIdx.x; e < Q * DK; e += blockDim.x) {
    const int i = i0 + e / DK;
    split(i < T ? qkv[(rb + i) * ld + h * DK + e % DK] : 0.f, qh, ql, e);
  }
  float* s_w = sf + warp * 16 * KT;
  float* o_w = of + warp * 16 * DK;
  __half* ph_w = ph + warp * 16 * KT;
  __half* pl_w = pl + warp * 16 * KT;
  for (int e = lane; e < 16 * DK; e += 32) o_w[e] = 0.f;
  const int r = lane & 15, half = lane >> 4;  // softmax: row r, columns [32 half, 32 half + 32)
  float m = -INFINITY, l = 0.f;
  wmma::fragment<wmma::matrix_a, 16, 16, 16, __half, wmma::row_major> fa_h, fa_l;
  wmma::fragment<wmma::matrix_b, 16, 16, 16, __half, wmma::col_major> fk_h, fk_l;
  wmma::fragment<wmma::matrix_b, 16, 16, 16, __half, wmma::row_major> fv_h, fv_l;
  wmma::fragment<wmma::accumulator, 16, 16, 16, float> acc;
  for (int j0 = 0; j0 < T; j0 += KT) {
    __syncthreads();  // the previous tile's K / V are no longer read
    for (int e = threadIdx.x; e < KT * DK; e += blockDim.x) {
      const int j = j0 + e / DK, d = e % DK;
      const bool ok = j < T;
      split(ok ? qkv[(rb + j) * ld + D + h * DK + d] : 0.f, kh, kl, e);
      split(ok ? qkv[(rb + j) * ld + 2 * D + h * DK + d] : 0.f, vh, vl, e);
    }
    __syncthreads();
    // S = Q K^T for this warp's 16 rows
#pragma unroll
    for (int n = 0; n < KT / 16; ++n) {
      wmma::fill_fragment(acc, 0.f);
#pragma unroll
      for (int kk = 0; kk < DK / 16; ++kk) {
        wmma::load_matrix_sync(fa_h, qh + warp * 16 * DK + kk * 16, DK);
        wmma::load_matrix_sync(fa_l, ql + warp * 16 * DK + kk * 16, DK);
        wmma::load_matrix_sync(fk_h, kh + n * 16 * DK + kk * 16, DK);
        wmma::load_matrix_sync(fk_l, kl + n * 16 * DK + kk * 16, DK);
        wmma::mma_sync(acc, fa_h, fk_h, acc);
        wmma::mma_sync(acc, fa_l, fk_h, acc);
        wmma::mma_sync(acc, fa_h, fk_l, acc);
      }
      wmma::store_matrix_sync(s_w + n * 16, acc, KT, wmma::mem_row_major);
    }
    __syncwarp();
    // online softmax: two lanes per row, 32 columns each, combined in a fixed order
    float* srow = s_w + r * KT + half * 32;
    float mt = -INFINITY;
    for (int c = 0; c < 32; ++c) {
      const bool ok = j0 + half * 32 + c < T;
      const float s = ok ? srow[c] * 0.125f : -INFINITY;
      srow[c] = s;
      mt = fmaxf(mt, s);
    }
    mt = fmaxf(mt, __shfl_xor_sync(0xffffffffu, mt, 16));
    const float mn = fmaxf(m, mt);
    const float corr = m == -INFINITY ? 0.f : expf(m - mn);
    float ps = 0.f;
    for (int c = 0; c < 32; ++c) {
      const float p = srow[c] == -INFINITY ? 0.f : expf(srow[c] - mn);
      ps += p;
      split(p, ph_w, pl_w, r * KT + half * 32 + c);
    }
    ps += __shfl_xor_sync(0xffffffffu, ps, 16);
    l = l * corr + ps;
    m = mn;
    for (int c = 0; c < 32; ++c) o_w[r * DK + half * 32 + c] *= corr;
    __syncwarp();
    // O += P V
#pragma unroll
    for (int n = 0; n < DK / 16; ++n) {
      wmma::load_matrix_sync(acc, o_w + n * 16, DK, wmma::mem_row_major);
#pragma unroll
      for (int kk = 0; kk < KT / 16; ++kk) {
        wmma::load_matrix_sync(fa_h, ph_w + kk * 16, KT);
        wmma::load_matrix_sync(fa_l, pl_w + kk * 16, KT);
        wmma::load_matrix_sync(fv_h, vh + kk * 16 * DK + n * 16, DK);
        wmma::load_matrix_sync(fv_l, vl + kk * 16 * DK + n * 16, DK);
        wmma::mma_sync(acc, fa_h, fv_h, acc);
        wmma::mma_sync(acc, fa_l, fv_h, acc);
        wmma::mma_sync(acc, fa_h, fv_l, acc);
      }
      wmma::store_matrix_sync(o_w + n * 16, acc, DK, wmma::mem_row_major);
    }
    __syncwarp();
  }
  const int i = i0 + warp * 16 + r;
  if (i < S) {
    float* dst = ctx + (rb + i) * D + h * DK + half * 32;
    for (int c = 0; c < 32; ++c) dst[c] = i < T ? o_w[r * DK + half * 32 + c] / l : 0.f;
  }
}

// emb[b][n] = mean over t < len[b] of h[b S + t][n], summed in frame order
__global__ void mean_kernel(const float* __restrict__ h, const int* __restrict__ len, int S, int D, float* __restrict__ emb) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x, b = blockIdx.y;
  if (n >= D) return;
  const int T = len[b];
  const float* hb = h + (size_t)b * S * D + n;
  float s = 0.f;
  for (int t = 0; t < T; ++t) s += hb[(size_t)t * D];
  emb[(size_t)b * D + n] = s / T;
}

// y[b][n] = act(bias[n] + x[b] . W[n]), one warp per output, lanes over k then a fixed butterfly; act 1 = tanh
__global__ void head_linear_kernel(const float* __restrict__ x, const float* __restrict__ W, const float* __restrict__ bias, int N,
                                   int K, int act, float* __restrict__ y) {
  const int n = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31, b = blockIdx.y;
  if (n >= N) return;
  const float* xb = x + (size_t)b * K;
  const float* w = W + (size_t)n * K;
  float s = 0.f;
  for (int i = lane; i < K; i += 32) s += xb[i] * w[i];
#pragma unroll
  for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if (lane == 0) {
    s += bias[n];
    y[(size_t)b * N + n] = act == 1 ? tanhf(s) : s;
  }
}

// out[b][t][n] = h[b S + t][n] for t < T_out (rows past len[b] are already zero)
__global__ void copy_rows_kernel(const float* __restrict__ h, int S, int D, int T_out, float* __restrict__ out) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int b = blockIdx.y;
  if (i >= (size_t)T_out * D) return;
  out[(size_t)b * T_out * D + i] = h[(size_t)b * S * D + i];
}

struct Gemm {
  std::vector<std::string> w, b;  // row blocks concatenated along N (QKV)
  int N = 0, K = 0, nseg = 1, taps = 1;  // conv layers: nseg = taps, K = input channels, weight [N][K][taps]
  bool cat = false;               // weights and biases concatenated into the derived qkv.* regions
  size_t img = 0;
  float inv_scale = 1.f;
  const float* bias = nullptr;
};

struct LayerW {
  const float *ln[2], *fln[2];
};

}  // namespace

struct mb_emo {
  mb_emo_config cfg{};
  int D = 0, H = 0, U = 0, L = 0, C = 0, nconv = 0, G = 0, cg = 0, kp = 0, nlab = 0;
  int P = 1;  // product of the strides of conv layers 1..
  WeightTable w;
  std::vector<Gemm> g;  // conv 1.., projection, then per layer: qkv, out, ff1, ff2
  int g_proj = 0;
  size_t total_bytes = 0;
  char* arena = nullptr;
  bool finalized = false;
  std::vector<LayerW> lw;
  const float *conv_ln[kMaxConv][2] = {}, *conv0_w = nullptr, *conv0_b = nullptr, *fp_ln[2] = {}, *pc_b = nullptr,
              *enc_ln[2] = {}, *dense_w = nullptr, *dense_b = nullptr, *out_w = nullptr, *out_b = nullptr;
  const __half *pc_hi = nullptr, *pc_lo = nullptr;  // packed positional-conv image
  float pc_inv_scale = 1.f;
  std::vector<int> host_ints;
  std::vector<int64_t> host_off;
  std::vector<NormClip> host_clips;

  const float* p(const std::string& n) const { return w.ptr(n); }
  float* fl(size_t off) const { return reinterpret_cast<float*>(arena) + off; }
  // frames after conv layer l of an n-sample clip: floor((n - k) / s) + 1 per layer (0 when too short)
  int frames_at(int n, int l) const {
    int t = n;
    for (int i = 0; i <= l; ++i) {
      if (t < cfg.conv_kernel[i]) return 0;
      t = (t - cfg.conv_kernel[i]) / cfg.conv_stride[i] + 1;
    }
    return t;
  }
  int frames(int n) const { return frames_at(n, nconv - 1); }
};

namespace {

struct Ws {
  size_t ints, offs, clips, normed, a, b, t_hi, t_lo, x, x2, y, ctx, emb, hid, total;
  int S[kMaxConv], M, RT;
};

Ws ws_layout(const mb_emo* h, int B, int n_max) {
  Ws L{};
  const int T0 = h->frames_at(n_max, 0);
  L.S[0] = (T0 + h->P - 1) / h->P * h->P;
  for (int l = 1; l < h->nconv; ++l) L.S[l] = L.S[l - 1] / h->cfg.conv_stride[l];
  const int S = L.S[h->nconv - 1];
  L.M = B * S;
  L.RT = (int)ceil128(L.M);
  size_t tiles = (size_t)std::max(kb_of(h->D), kb_of(h->U)) * L.RT * 64;
  tiles = std::max(tiles, (size_t)kb_of(h->C) * L.RT * 64);
  for (int l = 1; l < h->nconv; ++l)
    tiles = std::max(tiles, (size_t)h->cfg.conv_kernel[l] * kb_of(h->C) * ceil128((size_t)B * L.S[l]) * 64);
  WsLayout W;
  L.ints = W.take(sizeof(int) * 2 * kMaxConv * kMaxRows);
  L.offs = W.take(sizeof(int64_t) * kMaxRows);
  L.clips = W.take(sizeof(NormClip) * kMaxRows);
  L.normed = W.take(sizeof(float) * (size_t)B * n_max);
  L.a = W.take(sizeof(float) * (size_t)B * L.S[0] * h->C);
  L.b = W.take(sizeof(float) * (size_t)B * (h->nconv > 1 ? L.S[1] : 1) * h->C);
  L.t_hi = W.take(sizeof(__half) * tiles);
  L.t_lo = W.take(sizeof(__half) * tiles);
  L.x = W.take(sizeof(float) * (size_t)L.M * h->D);
  L.x2 = W.take(sizeof(float) * (size_t)L.M * h->D);
  L.y = W.take(sizeof(float) * (size_t)L.M * std::max(3 * h->D, h->U));
  L.ctx = W.take(sizeof(float) * (size_t)L.M * h->D);
  L.emb = W.take(sizeof(float) * (size_t)B * h->D);
  L.hid = W.take(sizeof(float) * (size_t)B * h->D);
  L.total = W.total();
  return L;
}

int run_gemm(const mb_emo* h, const Gemm& gm, const __half* a_hi, const __half* a_lo, int M, int rows_total, const float* res,
             float* y, int ldy, cudaStream_t st) {
  taco::TcBigArgs a{};
  a.a_hi = a_hi;
  a.a_lo = a_lo;
  a.w = reinterpret_cast<const __half*>(h->arena + gm.img);
  a.bias = gm.bias;
  a.KB = gm.nseg * kb_of(gm.K);
  a.M = M;
  a.N = gm.N;
  a.rows_total = rows_total;
  a.act = taco::ACT_NONE;
  a.inv_scale = gm.inv_scale;
  a.res = res;
  a.ldres = res ? ldy : 0;
  a.y = y;
  a.ldy = ldy;
  const cudaError_t e = taco::launch_tc_big(a, st, 0);
  if (e != cudaSuccess) return fail(MB_ERR_CUDA, "tc_big launch failed: %s", cudaGetErrorString(e));
  count_launch();
  return MB_OK;
}

int ln_tiles(const float* x, int M, int D, int RT, float eps, const float* g, const float* be, __half* hi, __half* lo,
             cudaStream_t st) {
  ln_tiles_kernel<<<RT / 8, 256, 0, st>>>(x, M, D, kb_of(D), RT, eps, g, be, hi, lo);
  MB_LAUNCH_CHECK("ln_tiles_kernel");
  return MB_OK;
}

int act_tiles(const float* src, int M, int K, int RT, int act, __half* hi, __half* lo, cudaStream_t st) {
  const size_t n = (size_t)kb_of(K) * RT * 8;
  act_tiles_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(src, K, M, K, kb_of(K), RT, act, hi, lo);
  MB_LAUNCH_CHECK("act_tiles_kernel");
  return MB_OK;
}

int ln_act_rows(float* x, int M, int D, float eps, const float* g, const float* be, int act, const int* len, int S,
                cudaStream_t st) {
  ln_act_rows_kernel<<<(M + 7) / 8, 256, 0, st>>>(x, M, D, eps, g, be, act, len, S);
  MB_LAUNCH_CHECK("ln_act_rows_kernel");
  return MB_OK;
}

size_t posconv_smem(int cg, int k) { return 2 * sizeof(__half) * (size_t)(kPcT + k - 1) * cg + sizeof(float) * 4 * 16 * 64; }
// Q hi / lo, K and V hi / lo (64 x 64 halves each), per warp: scores, running output (16 x 64 floats), P hi / lo
constexpr size_t kAttnSmem = 6 * 64 * 64 * sizeof(__half) + 4 * (2 * 16 * 64 * sizeof(float) + 2 * 16 * 64 * sizeof(__half));

int pack_posconv(const float* w, int D, int cg, int k, float scale, __half* img, cudaStream_t st) {
  const size_t n = (size_t)D * cg * k;
  posconv_pack_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(w, D, cg, k, scale, img, img + n);
  MB_LAUNCH_CHECK("posconv_pack_kernel");
  return MB_OK;
}

// x, out [B][S][D] (out = x + gelu(posconv(x)) on the clip's frames, zeros past them); image from pack_posconv
int launch_posconv(const float* x, const __half* w_hi, const __half* w_lo, float inv_scale, const float* bias, const int* len,
                   int B, int S, int D, int G, int k, float* out, cudaStream_t st) {
  static bool attr = false;  // per kernel, not per handle: once, to the most any handle may launch with
  if (!attr) {
    MB_CUDA_CHECK(cudaFuncSetAttribute(posconv_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kPcMaxSmem));
    attr = true;
  }
  const int cg = D / G;
  const dim3 grid((S + kPcT - 1) / kPcT, G * (cg / kPcC), B);
  posconv_tc_kernel<<<grid, 128, posconv_smem(cg, k), st>>>(x, w_hi, w_lo, inv_scale, bias, len, S, D, cg, k, out);
  MB_LAUNCH_CHECK("posconv_tc_kernel");
  return MB_OK;
}

// qkv [B][S][3 D] (q | k | v, heads of 64) -> ctx [B][S][D], zeros past each clip's frames
int launch_attn(const float* qkv, const int* len, int B, int S, int H, float* ctx, cudaStream_t st) {
  static bool attr = false;
  if (!attr) {
    MB_CUDA_CHECK(cudaFuncSetAttribute(attn_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kAttnSmem));
    attr = true;
  }
  attn_tc_kernel<<<dim3((S + 63) / 64, H, B), 128, kAttnSmem, st>>>(qkv, len, S, 64 * H, ctx);
  MB_LAUNCH_CHECK("attn_tc_kernel");
  return MB_OK;
}

}  // namespace

extern "C" {

int mb_emo_create(const mb_emo_config* cfg, mb_emo** out) {
  if (!cfg || !out) return fail(MB_ERR_INVALID, "mb_emo_create: null argument");
  const mb_emo_config& c = *cfg;
  const char* me = "mb_emo_create";
  if (c.feat_extract_norm != MB_EMO_NORM_LAYER)
    return fail(MB_ERR_INVALID, "%s: feat_extract_norm %d is not supported (only \"layer\")", me, c.feat_extract_norm);
  if (!c.do_stable_layer_norm) return fail(MB_ERR_INVALID, "%s: do_stable_layer_norm=False is not supported", me);
  if (c.feat_extract_activation != MB_EMO_ACT_GELU || c.hidden_act != MB_EMO_ACT_GELU)
    return fail(MB_ERR_INVALID, "%s: activations other than gelu are not supported", me);
  if (c.add_adapter) return fail(MB_ERR_INVALID, "%s: add_adapter is not supported", me);
  if (c.num_attention_heads < 1 || c.hidden_size != 64 * c.num_attention_heads)
    return fail(MB_ERR_INVALID, "%s: head size hidden_size / num_attention_heads = %d / %d is not 64", me, c.hidden_size,
                c.num_attention_heads);
  if (c.intermediate_size < 64 || c.intermediate_size % 64)
    return fail(MB_ERR_INVALID, "%s: intermediate_size %d is not a multiple of 64", me, c.intermediate_size);
  if (c.num_hidden_layers < 1 || c.num_hidden_layers > 64)
    return fail(MB_ERR_INVALID, "%s: num_hidden_layers %d outside 1..64", me, c.num_hidden_layers);
  if (c.num_conv_layers < 1 || c.num_conv_layers > kMaxConv)
    return fail(MB_ERR_INVALID, "%s: num_conv_layers %d outside 1..%d", me, c.num_conv_layers, kMaxConv);
  long long P = 1;
  for (int l = 0; l < c.num_conv_layers; ++l) {
    if (c.conv_dim[l] != c.conv_dim[0] || c.conv_dim[0] < 64 || c.conv_dim[0] % 64)
      return fail(MB_ERR_INVALID, "%s: conv_dim must be one width, a multiple of 64 (layer %d: %d)", me, l, c.conv_dim[l]);
    if (c.conv_stride[l] < 1 || c.conv_kernel[l] < 1 || c.conv_kernel[l] > (l == 0 ? 64 : taco::kMaxSeg))
      return fail(MB_ERR_INVALID, "%s: conv layer %d kernel %d / stride %d unsupported (kernel <= %d)", me, l, c.conv_kernel[l],
                  c.conv_stride[l], l == 0 ? 64 : taco::kMaxSeg);
    if (l > 0) P *= c.conv_stride[l];
  }
  if (P > 4096) return fail(MB_ERR_INVALID, "%s: conv strides multiply to %lld > 4096", me, P);
  if (c.num_conv_pos_embedding_groups < 1 || c.hidden_size % c.num_conv_pos_embedding_groups ||
      (c.hidden_size / c.num_conv_pos_embedding_groups) % 64)
    return fail(MB_ERR_INVALID, "%s: hidden_size / num_conv_pos_embedding_groups = %d / %d is not a multiple of 64", me,
                c.hidden_size, c.num_conv_pos_embedding_groups);
  if (c.num_conv_pos_embeddings < 1 || c.num_conv_pos_embeddings > 256)
    return fail(MB_ERR_INVALID, "%s: num_conv_pos_embeddings %d outside 1..256", me, c.num_conv_pos_embeddings);
  if (posconv_smem(c.hidden_size / c.num_conv_pos_embedding_groups, c.num_conv_pos_embeddings) > kPcMaxSmem)
    return fail(MB_ERR_INVALID, "%s: positional conv group width %d x %d taps exceeds shared memory", me,
                c.hidden_size / c.num_conv_pos_embedding_groups, c.num_conv_pos_embeddings);
  if (c.num_labels < 1) return fail(MB_ERR_INVALID, "%s: num_labels %d < 1", me, c.num_labels);
  if (!(c.layer_norm_eps > 0.f)) return fail(MB_ERR_INVALID, "%s: layer_norm_eps must be positive", me);

  auto* h = new mb_emo();
  h->cfg = c;
  h->D = c.hidden_size;
  h->H = c.num_attention_heads;
  h->U = c.intermediate_size;
  h->L = c.num_hidden_layers;
  h->C = c.conv_dim[0];
  h->nconv = c.num_conv_layers;
  h->G = c.num_conv_pos_embedding_groups;
  h->cg = h->D / h->G;
  h->kp = c.num_conv_pos_embeddings;
  h->nlab = c.num_labels;
  h->P = (int)P;
  const int D = h->D, C = h->C, U = h->U;
  WeightTable& w = h->w;
  const std::string fe = "wav2vec2.feature_extractor.conv_layers.";
  for (int l = 0; l < h->nconv; ++l) {
    const std::string b = fe + std::to_string(l) + ".";
    w.add(b + "conv.weight", {C, l == 0 ? 1 : C, c.conv_kernel[l]});
    if (c.conv_bias) w.add(b + "conv.bias", {C});
    w.add(b + "layer_norm.weight", {C});
    w.add(b + "layer_norm.bias", {C});
    if (l > 0) {
      Gemm gm;
      gm.w = {b + "conv.weight"};
      if (c.conv_bias) gm.b = {b + "conv.bias"};
      gm.N = C, gm.K = C, gm.nseg = gm.taps = c.conv_kernel[l];
      h->g.push_back(gm);
    }
  }
  w.add("wav2vec2.feature_projection.layer_norm.weight", {C});
  w.add("wav2vec2.feature_projection.layer_norm.bias", {C});
  w.add("wav2vec2.feature_projection.projection.weight", {D, C});
  w.add("wav2vec2.feature_projection.projection.bias", {D});
  h->g_proj = (int)h->g.size();
  {
    Gemm gm;
    gm.w = {"wav2vec2.feature_projection.projection.weight"};
    gm.b = {"wav2vec2.feature_projection.projection.bias"};
    gm.N = D, gm.K = C;
    h->g.push_back(gm);
  }
  w.add("wav2vec2.encoder.pos_conv_embed.conv.weight", {D, h->cg, h->kp});
  w.add("wav2vec2.encoder.pos_conv_embed.conv.bias", {D});
  for (int i = 0; i < h->L; ++i) {
    const std::string b = "wav2vec2.encoder.layers." + std::to_string(i) + ".";
    for (const char* n : {"q_proj", "k_proj", "v_proj", "out_proj"}) {
      w.add(b + "attention." + n + ".weight", {D, D});
      w.add(b + "attention." + n + ".bias", {D});
    }
    for (const char* n : {"layer_norm", "final_layer_norm"}) {
      w.add(b + n + ".weight", {D});
      w.add(b + n + ".bias", {D});
    }
    w.add(b + "feed_forward.intermediate_dense.weight", {U, D});
    w.add(b + "feed_forward.intermediate_dense.bias", {U});
    w.add(b + "feed_forward.output_dense.weight", {D, U});
    w.add(b + "feed_forward.output_dense.bias", {D});
    Gemm q, o, f1, f2;
    q.w = {b + "attention.q_proj.weight", b + "attention.k_proj.weight", b + "attention.v_proj.weight"};
    q.b = {b + "attention.q_proj.bias", b + "attention.k_proj.bias", b + "attention.v_proj.bias"};
    q.N = 3 * D, q.K = D;
    o.w = {b + "attention.out_proj.weight"};
    o.b = {b + "attention.out_proj.bias"};
    o.N = D, o.K = D;
    f1.w = {b + "feed_forward.intermediate_dense.weight"};
    f1.b = {b + "feed_forward.intermediate_dense.bias"};
    f1.N = U, f1.K = D;
    f2.w = {b + "feed_forward.output_dense.weight"};
    f2.b = {b + "feed_forward.output_dense.bias"};
    f2.N = D, f2.K = U;
    for (Gemm* gm : {&q, &o, &f1, &f2}) h->g.push_back(*gm);
  }
  w.add("wav2vec2.encoder.layer_norm.weight", {D});
  w.add("wav2vec2.encoder.layer_norm.bias", {D});
  w.add("classifier.dense.weight", {D, D});
  w.add("classifier.dense.bias", {D});
  w.add("classifier.out_proj.weight", {h->nlab, D});
  w.add("classifier.out_proj.bias", {h->nlab});
  for (size_t i = 0; i < h->g.size(); ++i) {
    Gemm& gm = h->g[i];
    if (gm.w.size() > 1) {
      w.add_derived("qkv.weight." + std::to_string(i), (size_t)gm.N * gm.K);
      w.add_derived("qkv.bias." + std::to_string(i), (size_t)gm.N);
    }
  }
  w.add_derived("pos_conv.packed", (size_t)D * h->cg * h->kp);  // fp16 hi then lo: 2 halves per float
  w.add_derived("absmax", h->g.size() + 1);
  w.ignored = [](const std::string& n) { return n == "wav2vec2.masked_spec_embed"; };
  size_t bytes = mb::align_up(w.floats() * sizeof(float), 1024);
  for (auto& gm : h->g) {
    gm.img = bytes;
    bytes += mb::align_up(taco::tc_big_weight_bytes(gm.N, gm.nseg, gm.K), 1024);
  }
  h->total_bytes = bytes;
  *out = h;
  return MB_OK;
}

void mb_emo_destroy(mb_emo* h) { delete h; }

size_t mb_emo_arena_bytes(const mb_emo* h) { return h ? h->total_bytes : 0; }

int mb_emo_set_arena(mb_emo* h, void* arena, size_t bytes) {
  if (int rc = check_arena("mb_emo_set_arena", h, arena, bytes, mb_emo_arena_bytes(h), 1024)) return rc;
  h->w.attach(static_cast<float*>(arena));
  h->arena = static_cast<char*>(arena);
  h->finalized = false;
  return MB_OK;
}

int mb_emo_set_weight(mb_emo* h, const char* name, const float* w, const int64_t* dims, int32_t ndim, void* stream) {
  if (!h) return fail(MB_ERR_INVALID, "mb_emo_set_weight: null argument");
  if (int rc = h->w.set("mb_emo_set_weight", name, w, dims, ndim, stream)) return rc;
  h->finalized = false;
  return MB_OK;
}

int mb_emo_finalize(mb_emo* h, void* stream) {
  if (!h) return fail(MB_ERR_INVALID, "mb_emo_finalize: null handle");
  if (int rc = h->w.check_all_set("mb_emo_finalize")) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int D = h->D;
  for (size_t i = 0; i < h->g.size(); ++i) {
    Gemm& gm = h->g[i];
    if (gm.w.size() > 1) {  // QKV: weights and biases concatenated along N
      float* wc = h->w.ptr("qkv.weight." + std::to_string(i));
      float* bc = h->w.ptr("qkv.bias." + std::to_string(i));
      for (size_t s = 0; s < gm.w.size(); ++s) {
        MB_CUDA_CHECK(cudaMemcpyAsync(wc + s * (size_t)D * gm.K, h->p(gm.w[s]), sizeof(float) * D * gm.K, cudaMemcpyDeviceToDevice, st));
        MB_CUDA_CHECK(cudaMemcpyAsync(bc + s * (size_t)D, h->p(gm.b[s]), sizeof(float) * D, cudaMemcpyDeviceToDevice, st));
      }
      gm.cat = true;
    }
  }
  auto src = [&](size_t i) {
    return h->g[i].cat ? h->w.ptr("qkv.weight." + std::to_string(i)) : h->p(h->g[i].w[0]);
  };
  unsigned int* d_abs = reinterpret_cast<unsigned int*>(h->w.ptr("absmax"));
  const size_t ng = h->g.size();
  const float* pc_w = h->p("wav2vec2.encoder.pos_conv_embed.conv.weight");
  const size_t pc_n = (size_t)D * h->cg * h->kp;
  MB_CUDA_CHECK(cudaMemsetAsync(d_abs, 0, (ng + 1) * sizeof(unsigned int), st));
  for (size_t i = 0; i <= ng; ++i) {  // slot ng: the positional conv
    const cudaError_t e = i < ng ? taco::tc_skinny_absmax(src(i), (size_t)h->g[i].N * h->g[i].K * h->g[i].taps, d_abs + i, st)
                                 : taco::tc_skinny_absmax(pc_w, pc_n, d_abs + i, st);
    if (e != cudaSuccess) return fail(MB_ERR_CUDA, "absmax: %s", cudaGetErrorString(e));
  }
  std::vector<unsigned int> bits(ng + 1);
  MB_CUDA_CHECK(cudaMemcpyAsync(bits.data(), d_abs, (ng + 1) * sizeof(unsigned int), cudaMemcpyDeviceToHost, st));
  MB_CUDA_CHECK(cudaStreamSynchronize(st));
  for (size_t i = 0; i < ng; ++i) {
    Gemm& gm = h->g[i];
    const float scale = taco::tc_weight_scale(bits[i]);
    gm.inv_scale = 1.f / scale;
    taco::TcBigPack q{};
    q.W = src(i);
    q.ldw = gm.K * gm.taps;
    q.N = gm.N;
    q.nseg = gm.nseg;
    q.K = gm.K;
    q.KBs = kb_of(gm.K);
    for (int s = 0; s < gm.nseg; ++s) {  // Conv1d weight [N][K][taps]: tap s at column s, stride taps
      q.w_off[s] = s;
      q.w_stride[s] = gm.taps;
    }
    q.scale = scale;
    const cudaError_t e = taco::launch_pack_big_w(q, reinterpret_cast<__half*>(h->arena + gm.img), st);
    if (e != cudaSuccess) return fail(MB_ERR_CUDA, "pack: %s", cudaGetErrorString(e));
    count_launch();
    gm.bias = gm.b.empty() ? nullptr : gm.cat ? h->w.ptr("qkv.bias." + std::to_string(i)) : h->p(gm.b[0]);
  }
  {
    const float scale = taco::tc_weight_scale(bits[ng]);
    h->pc_inv_scale = 1.f / scale;
    __half* img = reinterpret_cast<__half*>(h->w.ptr("pos_conv.packed"));
    MB_TRY(pack_posconv(pc_w, D, h->cg, h->kp, scale, img, st));
    h->pc_hi = img;
    h->pc_lo = img + pc_n;
  }
  const std::string fe = "wav2vec2.feature_extractor.conv_layers.";
  for (int l = 0; l < h->nconv; ++l) {
    h->conv_ln[l][0] = h->p(fe + std::to_string(l) + ".layer_norm.weight");
    h->conv_ln[l][1] = h->p(fe + std::to_string(l) + ".layer_norm.bias");
  }
  h->conv0_w = h->p(fe + "0.conv.weight");
  h->conv0_b = h->cfg.conv_bias ? h->p(fe + "0.conv.bias") : nullptr;
  h->fp_ln[0] = h->p("wav2vec2.feature_projection.layer_norm.weight");
  h->fp_ln[1] = h->p("wav2vec2.feature_projection.layer_norm.bias");
  h->pc_b = h->p("wav2vec2.encoder.pos_conv_embed.conv.bias");
  h->enc_ln[0] = h->p("wav2vec2.encoder.layer_norm.weight");
  h->enc_ln[1] = h->p("wav2vec2.encoder.layer_norm.bias");
  h->dense_w = h->p("classifier.dense.weight");
  h->dense_b = h->p("classifier.dense.bias");
  h->out_w = h->p("classifier.out_proj.weight");
  h->out_b = h->p("classifier.out_proj.bias");
  h->lw.assign(h->L, LayerW{});
  for (int i = 0; i < h->L; ++i) {
    const std::string b = "wav2vec2.encoder.layers." + std::to_string(i) + ".";
    h->lw[i].ln[0] = h->p(b + "layer_norm.weight");
    h->lw[i].ln[1] = h->p(b + "layer_norm.bias");
    h->lw[i].fln[0] = h->p(b + "final_layer_norm.weight");
    h->lw[i].fln[1] = h->p(b + "final_layer_norm.bias");
  }
  h->finalized = true;
  return MB_OK;
}

int32_t mb_emo_num_frames(const mb_emo* h, int32_t n_samples) {
  if (!h || n_samples < 0) return 0;
  return h->frames(n_samples);
}

size_t mb_emo_workspace_bytes(const mb_emo* h, int32_t batch, int32_t n_samples_max) {
  if (!h || batch < 1 || batch > kMaxRows || h->frames(n_samples_max) < 1) return 0;
  return ws_layout(h, batch, n_samples_max).total;
}

int mb_emo_forward(mb_emo* h, const float* wav, const int32_t* n_samples, int32_t batch, int32_t normalize, float* emb,
                   float* logits, float* normed, float* hidden, void* workspace, size_t workspace_bytes, void* stream) {
  const char* me = "mb_emo_forward";
  if (!h) return fail(MB_ERR_INVALID, "%s: null handle", me);
  if (!h->finalized) return fail(MB_ERR_STATE, "%s: weights not finalized", me);
  if (batch < 1 || batch > kMaxRows) return fail(MB_ERR_INVALID, "%s: batch %d outside 1..%d", me, batch, kMaxRows);
  if (!wav || !n_samples || !emb || !logits) return fail(MB_ERR_INVALID, "%s: null argument", me);
  int n_max = 0;
  for (int b = 0; b < batch; ++b) {
    if (h->frames(n_samples[b]) < 1)
      return fail(MB_ERR_INVALID, "%s: clip %d has %d samples, too short for one frame", me, b, n_samples[b]);
    n_max = std::max(n_max, (int)n_samples[b]);
  }
  const Ws L = ws_layout(h, batch, n_max);
  char* ws;
  if (int rc = bind(me, workspace, workspace_bytes, L.total, &ws)) return rc;
  const int B = batch, nc = h->nconv, C = h->C, D = h->D, U = h->U, M = L.M, RT = L.RT, S = L.S[nc - 1];
  h->host_ints.assign((size_t)2 * kMaxConv * kMaxRows, 0);
  h->host_off.assign(kMaxRows, 0);
  h->host_clips.assign(kMaxRows, NormClip{});
  int64_t off = 0;
  for (int b = 0; b < B; ++b) {
    for (int l = 0; l < nc; ++l) {
      h->host_ints[(size_t)l * kMaxRows + b] = h->frames_at(n_samples[b], l);
      if (l > 0)  // rows of conv_stride[l] input frames holding at least one of the clip's frames
        h->host_ints[(size_t)(kMaxConv + l) * kMaxRows + b] =
            (h->host_ints[(size_t)(l - 1) * kMaxRows + b] + h->cfg.conv_stride[l] - 1) / h->cfg.conv_stride[l];
    }
    h->host_off[b] = off;
    h->host_clips[b] = NormClip{off, n_samples[b], pairwise_depth(n_samples[b])};
    off += n_samples[b];
  }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  // [layer][clip]: frames after each conv layer, then [kMaxConv + layer][clip]: the input rows of conv layer l >= 1
  int* d_len = reinterpret_cast<int*>(ws + L.ints);
  int64_t* d_off = reinterpret_cast<int64_t*>(ws + L.offs);
  NormClip* d_clips = reinterpret_cast<NormClip*>(ws + L.clips);
  MB_CUDA_CHECK(cudaMemcpyAsync(d_len, h->host_ints.data(), sizeof(int) * h->host_ints.size(), cudaMemcpyHostToDevice, st));
  MB_CUDA_CHECK(cudaMemcpyAsync(d_off, h->host_off.data(), sizeof(int64_t) * kMaxRows, cudaMemcpyHostToDevice, st));
  MB_CUDA_CHECK(cudaMemcpyAsync(d_clips, h->host_clips.data(), sizeof(NormClip) * kMaxRows, cudaMemcpyHostToDevice, st));
  const int* d_T = d_len + (size_t)(nc - 1) * kMaxRows;
  auto fp = [&](size_t o) { return reinterpret_cast<float*>(ws + o); };
  __half *th = reinterpret_cast<__half*>(ws + L.t_hi), *tl = reinterpret_cast<__half*>(ws + L.t_lo);
  const float* xn = wav;
  if (normalize) {
    float* y = normed ? normed : fp(L.normed);
    norm_kernel<<<B, kNormThreads, 0, st>>>(wav, d_clips, y);
    MB_LAUNCH_CHECK("norm_kernel");
    xn = y;
  }
  // feature encoder
  {
    const size_t n = (size_t)L.S[0] * C;
    conv0_kernel<<<dim3((unsigned)((n + 255) / 256), B), 256, 0, st>>>(xn, d_off, d_len, L.S[0], h->conv0_w, h->conv0_b, C,
                                                                        h->cfg.conv_kernel[0], h->cfg.conv_stride[0], fp(L.a));
    MB_LAUNCH_CHECK("conv0_kernel");
  }
  MB_TRY(ln_act_rows(fp(L.a), B * L.S[0], C, 1e-5f, h->conv_ln[0][0], h->conv_ln[0][1], ENC_ACT_GELU, d_len, L.S[0], st));
  float* cur = fp(L.a);
  for (int l = 1; l < nc; ++l) {
    const int s = h->cfg.conv_stride[l], k = h->cfg.conv_kernel[l], Sl = L.S[l], Ml = B * Sl, RTl = (int)ceil128(Ml);
    float* nxt = (l % 2) ? fp(L.b) : fp(L.a);
    // the input as rows of s frames: tap j is segment (j % s) of row t + j / s; a row at or past ceil(T_in / s) reads zeros
    taco::TcIm2col q{};
    for (int j = 0; j < k; ++j) {
      q.x[j] = cur + (size_t)(j % s) * C;
      q.ld[j] = s * C;
      q.shift[j] = j / s;
    }
    q.nseg = k, q.K = C, q.KBs = kb_of(C);
    q.M = Ml, q.T = Sl, q.rows_total = RTl;
    q.len = d_len + (size_t)(kMaxConv + l) * kMaxRows;
    cudaError_t e = taco::launch_im2col_split(q, th, tl, st);
    if (e != cudaSuccess) return fail(MB_ERR_CUDA, "im2col launch failed: %s", cudaGetErrorString(e));
    count_launch();
    MB_TRY(run_gemm(h, h->g[l - 1], th, tl, Ml, RTl, nullptr, nxt, C, st));
    MB_TRY(ln_act_rows(nxt, Ml, C, 1e-5f, h->conv_ln[l][0], h->conv_ln[l][1], ENC_ACT_GELU, d_len + (size_t)l * kMaxRows, Sl, st));
    cur = nxt;
  }
  // feature projection
  float* x = fp(L.x);
  float* y = fp(L.y);
  float* ctx = fp(L.ctx);
  const float eps = h->cfg.layer_norm_eps;
  MB_TRY(ln_tiles(cur, M, C, RT, eps, h->fp_ln[0], h->fp_ln[1], th, tl, st));
  MB_TRY(run_gemm(h, h->g[h->g_proj], th, tl, M, RT, nullptr, x, D, st));
  // positional conv: x2 = x + gelu(conv(x)), the residual stream from here on
  {
    float* x2 = fp(L.x2);
    MB_TRY(launch_posconv(x, h->pc_hi, h->pc_lo, h->pc_inv_scale, h->pc_b, d_T, B, S, D, h->G, h->kp, x2, st));
    x = x2;
  }
  for (int i = 0; i < h->L; ++i) {
    const Gemm* gq = &h->g[h->g_proj + 1 + 4 * i];
    MB_TRY(ln_tiles(x, M, D, RT, eps, h->lw[i].ln[0], h->lw[i].ln[1], th, tl, st));
    MB_TRY(run_gemm(h, gq[0], th, tl, M, RT, nullptr, y, 3 * D, st));
    MB_TRY(launch_attn(y, d_T, B, S, h->H, ctx, st));
    MB_TRY(act_tiles(ctx, M, D, RT, ENC_ACT_NONE, th, tl, st));
    MB_TRY(run_gemm(h, gq[1], th, tl, M, RT, x, x, D, st));
    MB_TRY(ln_tiles(x, M, D, RT, eps, h->lw[i].fln[0], h->lw[i].fln[1], th, tl, st));
    MB_TRY(run_gemm(h, gq[2], th, tl, M, RT, nullptr, y, U, st));
    MB_TRY(act_tiles(y, M, U, RT, ENC_ACT_GELU, th, tl, st));
    MB_TRY(run_gemm(h, gq[3], th, tl, M, RT, x, x, D, st));
  }
  MB_TRY(ln_act_rows(x, M, D, eps, h->enc_ln[0], h->enc_ln[1], ENC_ACT_NONE, d_T, S, st));
  mean_kernel<<<dim3((D + 127) / 128, B), 128, 0, st>>>(x, d_T, S, D, emb);
  MB_LAUNCH_CHECK("mean_kernel");
  float* hid = fp(L.hid);
  head_linear_kernel<<<dim3((D + 7) / 8, B), 256, 0, st>>>(emb, h->dense_w, h->dense_b, D, D, 1, hid);
  MB_LAUNCH_CHECK("head_linear_kernel");
  head_linear_kernel<<<dim3((h->nlab + 7) / 8, B), 256, 0, st>>>(hid, h->out_w, h->out_b, h->nlab, D, 0, logits);
  MB_LAUNCH_CHECK("head_linear_kernel");
  if (hidden) {
    const int T_out = h->frames(n_max);
    const size_t n = (size_t)T_out * D;
    copy_rows_kernel<<<dim3((unsigned)((n + 255) / 256), B), 256, 0, st>>>(x, S, D, T_out, hidden);
    MB_LAUNCH_CHECK("copy_rows_kernel");
  }
  return MB_OK;
}

// ---------------------------------------------------------------------------------------------- one-launch test hook
namespace {
struct DbgWs {
  size_t ints, offs, clips, img, abs, total;
};
DbgWs dbg_layout(const mb_emo_debug_spec* s) {
  DbgWs L{};
  WsLayout W;
  L.ints = W.take(sizeof(int) * kMaxRows);
  L.offs = W.take(sizeof(int64_t) * kMaxRows);
  L.clips = W.take(sizeof(NormClip) * kMaxRows);
  const bool pc = s->kind == MB_EMO_DBG_POSCONV && s->groups > 0 && s->kernel > 0;
  L.img = W.take(pc ? 2 * sizeof(__half) * (size_t)s->dim * (s->dim / s->groups) * s->kernel : 0);
  L.abs = W.take(sizeof(unsigned int));
  L.total = W.total();
  return L;
}
}  // namespace

size_t mb_emo_debug_workspace_bytes(const mb_emo_debug_spec* s) { return s ? dbg_layout(s).total : 0; }

int mb_emo_debug(const mb_emo_debug_spec* spec, void* workspace, size_t workspace_bytes, void* stream) {
  const char* me = "mb_emo_debug";
  if (!spec) return fail(MB_ERR_INVALID, "%s: null argument", me);
  const mb_emo_debug_spec& s = *spec;
  const DbgWs L = dbg_layout(spec);
  char* ws;
  if (int rc = bind(me, workspace, workspace_bytes, L.total, &ws)) return rc;
  const int B = s.batch;
  if (B < 1 || B > kMaxRows || !s.lengths || !s.x || !s.y) return fail(MB_ERR_INVALID, "%s: batch %d / null argument", me, B);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  int* d_len = reinterpret_cast<int*>(ws + L.ints);
  int64_t* d_off = reinterpret_cast<int64_t*>(ws + L.offs);
  NormClip* d_clips = reinterpret_cast<NormClip*>(ws + L.clips);
  std::vector<int> lens(kMaxRows, 0);
  std::vector<int64_t> offs(kMaxRows, 0);
  std::vector<NormClip> clips(kMaxRows, NormClip{});
  int64_t off = 0;
  for (int b = 0; b < B; ++b) {
    lens[b] = s.lengths[b];
    if (lens[b] < 1 || (s.kind != MB_EMO_DBG_NORM && s.kind != MB_EMO_DBG_CONV0 && lens[b] > s.frames))
      return fail(MB_ERR_INVALID, "%s: lengths[%d] = %d outside 1..%d", me, b, lens[b], s.frames);
    offs[b] = off;
    clips[b] = NormClip{off, lens[b], pairwise_depth(lens[b])};
    off += lens[b];
  }
  MB_CUDA_CHECK(cudaMemcpyAsync(d_off, offs.data(), sizeof(int64_t) * kMaxRows, cudaMemcpyHostToDevice, st));
  MB_CUDA_CHECK(cudaMemcpyAsync(d_clips, clips.data(), sizeof(NormClip) * kMaxRows, cudaMemcpyHostToDevice, st));
  const int S = s.frames, D = s.dim;
  switch (s.kind) {
    case MB_EMO_DBG_NORM:
      norm_kernel<<<B, kNormThreads, 0, st>>>(s.x, d_clips, s.y);
      MB_LAUNCH_CHECK("norm_kernel");
      break;
    case MB_EMO_DBG_CONV0: {
      // lengths are samples; frames of clip b: floor((n - k) / s) + 1, rows [frames, S) written as zeros
      if (s.kernel < 1 || s.stride < 1 || D < 1 || S < 1 || !s.w) return fail(MB_ERR_INVALID, "%s: conv0 shape", me);
      for (int b = 0; b < B; ++b) {
        const int n = lens[b] < s.kernel ? 0 : (lens[b] - s.kernel) / s.stride + 1;
        if (n < 1 || n > S) return fail(MB_ERR_INVALID, "%s: clip %d gives %d frames outside 1..%d", me, b, n, S);
        lens[b] = n;
      }
      MB_CUDA_CHECK(cudaMemcpyAsync(d_len, lens.data(), sizeof(int) * kMaxRows, cudaMemcpyHostToDevice, st));
      const size_t n = (size_t)S * D;
      conv0_kernel<<<dim3((unsigned)((n + 255) / 256), B), 256, 0, st>>>(s.x, d_off, d_len, S, s.w, s.bias, D, s.kernel, s.stride,
                                                                          s.y);
      MB_LAUNCH_CHECK("conv0_kernel");
      break;
    }
    case MB_EMO_DBG_LN_ACT:
      if (!s.gamma || !s.beta || D < 1) return fail(MB_ERR_INVALID, "%s: ln_act arguments", me);
      MB_CUDA_CHECK(cudaMemcpyAsync(d_len, lens.data(), sizeof(int) * kMaxRows, cudaMemcpyHostToDevice, st));
      if (s.y != s.x) MB_CUDA_CHECK(cudaMemcpyAsync(s.y, s.x, sizeof(float) * (size_t)B * S * D, cudaMemcpyDeviceToDevice, st));
      MB_TRY(ln_act_rows(s.y, B * S, D, s.eps, s.gamma, s.beta, s.act, d_len, S, st));
      break;
    case MB_EMO_DBG_POSCONV: {
      if (s.groups < 1 || D % s.groups || (D / s.groups) % 64 || s.kernel < 1 || !s.w || !s.bias ||
          posconv_smem(D / s.groups, s.kernel) > kPcMaxSmem)
        return fail(MB_ERR_INVALID, "%s: posconv dim %d / groups %d / kernel %d", me, D, s.groups, s.kernel);
      MB_CUDA_CHECK(cudaMemcpyAsync(d_len, lens.data(), sizeof(int) * kMaxRows, cudaMemcpyHostToDevice, st));
      // as finalize: max |w| -> power-of-two scale (one host read-back) -> packed image
      const size_t n = (size_t)D * (D / s.groups) * s.kernel;
      unsigned int* d_abs = reinterpret_cast<unsigned int*>(ws + L.abs);
      MB_CUDA_CHECK(cudaMemsetAsync(d_abs, 0, sizeof(unsigned int), st));
      const cudaError_t e = taco::tc_skinny_absmax(s.w, n, d_abs, st);
      if (e != cudaSuccess) return fail(MB_ERR_CUDA, "absmax: %s", cudaGetErrorString(e));
      unsigned int bits = 0;
      MB_CUDA_CHECK(cudaMemcpyAsync(&bits, d_abs, sizeof(bits), cudaMemcpyDeviceToHost, st));
      MB_CUDA_CHECK(cudaStreamSynchronize(st));
      const float scale = taco::tc_weight_scale(bits);
      __half* img = reinterpret_cast<__half*>(ws + L.img);
      MB_TRY(pack_posconv(s.w, D, D / s.groups, s.kernel, scale, img, st));
      MB_TRY(launch_posconv(s.x, img, img + n, 1.f / scale, s.bias, d_len, B, S, D, s.groups, s.kernel, s.y, st));
      break;
    }
    case MB_EMO_DBG_ATTN:
      if (s.heads < 1 || D != 64 * s.heads) return fail(MB_ERR_INVALID, "%s: dim %d is not 64 heads x %d", me, D, s.heads);
      MB_CUDA_CHECK(cudaMemcpyAsync(d_len, lens.data(), sizeof(int) * kMaxRows, cudaMemcpyHostToDevice, st));
      MB_TRY(launch_attn(s.x, d_len, B, S, s.heads, s.y, st));
      break;
    case MB_EMO_DBG_MEAN:
      MB_CUDA_CHECK(cudaMemcpyAsync(d_len, lens.data(), sizeof(int) * kMaxRows, cudaMemcpyHostToDevice, st));
      mean_kernel<<<dim3((D + 127) / 128, B), 128, 0, st>>>(s.x, d_len, S, D, s.y);
      MB_LAUNCH_CHECK("mean_kernel");
      break;
    case MB_EMO_DBG_HEAD:
      if (!s.w || !s.bias || s.n_out < 1) return fail(MB_ERR_INVALID, "%s: head arguments", me);
      head_linear_kernel<<<dim3((s.n_out + 7) / 8, B), 256, 0, st>>>(s.x, s.w, s.bias, s.n_out, D, s.act, s.y);
      MB_LAUNCH_CHECK("head_linear_kernel");
      break;
    default:
      return fail(MB_ERR_INVALID, "%s: bad kind %d", me, s.kind);
  }
  MB_CUDA_CHECK(cudaStreamSynchronize(st));
  return MB_OK;
}

}  // extern "C"
