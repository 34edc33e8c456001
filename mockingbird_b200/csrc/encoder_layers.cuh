// Transformer-encoder building blocks shared by the PPG extractor (csrc/ppg_extractor.cu) and the wav2vec2 emotion model
// (csrc/wav2emo.cu): LayerNorm and activations straight into the hi / lo operand tiles of the tensor-core GEMMs
// (taco::tc_big), and the FP32 multi-head attention over each row's own keys.  Each includer gets its own copies of the
// kernels (static, or templates).
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include <cmath>
#include <cstdint>

#include "tacotron_kernels.cuh"

namespace mb {
namespace enc {

constexpr int kLanes = 4;  // threads per query in the attention kernel, each taking every kLanes-th key
constexpr int kQ = 128 / kLanes;  // queries per attention CTA
constexpr int kKT = 32; // keys per shared-memory tile
static_assert(kQ - 1 + kKT <= 2 * kKT, "the p-row windows of a tile pair hold 2 kKT rows");

__device__ __forceinline__ float sigmoidf_(float x) { return 1.f / (1.f + expf(-x)); }
// exact (erf) GELU, torch.nn.functional.gelu's default
__device__ __forceinline__ float gelu_erf(float x) { return 0.5f * x * (1.f + erff(x * 0.70710678118654752f)); }
enum EncAct : int { ENC_ACT_NONE = 0, ENC_ACT_RELU = 1, ENC_ACT_SWISH = 2, ENC_ACT_GELU = 3 };
__device__ __forceinline__ float act_f(float x, int act) {
  return act == ENC_ACT_RELU ? fmaxf(x, 0.f) : act == ENC_ACT_SWISH ? x * sigmoidf_(x) : act == ENC_ACT_GELU ? gelu_erf(x) : x;
}

// fp32 [M][ld] (columns [0, K)) with an activation -> operand tiles [KB][rows_total][64]; zeros elsewhere
static __global__ void act_tiles_kernel(const float* __restrict__ src, int ld, int M, int K, int KB, int rows_total, int act,
                                        __half* __restrict__ t_hi, __half* __restrict__ t_lo) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;  // one 16-byte chunk
  const size_t total = (size_t)KB * rows_total * 8;
  if (i >= total) return;
  const int c8 = (int)(i & 7);
  const int m = (int)((i >> 3) % rows_total);
  const int kb = (int)(i / ((size_t)8 * rows_total));
  __align__(16) __half hi[8], lo[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    const int k = kb * 64 + c8 * 8 + e;
    const float v = (m < M && k < K) ? act_f(src[(size_t)m * ld + k], act) : 0.f;
    hi[e] = __float2half_rn(v);
    lo[e] = __float2half_rn(v - __half2float(hi[e]));
  }
  const size_t o = ((size_t)kb * rows_total + m) * 8 + (size_t)(c8 ^ (m & 7));
  reinterpret_cast<uint4*>(t_hi)[o] = *reinterpret_cast<const uint4*>(hi);
  reinterpret_cast<uint4*>(t_lo)[o] = *reinterpret_cast<const uint4*>(lo);
}

// one warp per row: the row's mean / biased variance in a fixed order, rstd = 1 / sqrt(var + eps)
__device__ __forceinline__ void row_stats(const float* x, int D, int lane, float eps, float& mean, float& rstd) {
  float s = 0.f;
  for (int n = lane; n < D; n += 32) s += x[n];
#pragma unroll
  for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  mean = s / D;
  float v = 0.f;
  for (int n = lane; n < D; n += 32) {
    const float d = x[n] - mean;
    v += d * d;
  }
#pragma unroll
  for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  rstd = 1.f / sqrtf(v / D + eps);
}

// LayerNorm (eps) rows [0, M) of x -> operand tiles (rows [M, rows_total) and columns [D, 64 KB) zero)
static __global__ void ln_tiles_kernel(const float* __restrict__ x, int M, int D, int KB, int rows_total, float eps,
                                       const float* __restrict__ g, const float* __restrict__ be, __half* __restrict__ t_hi,
                                       __half* __restrict__ t_lo) {
  const int m = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (m >= rows_total) return;
  float mean = 0.f, rstd = 0.f;
  const float* xr = x + (size_t)m * D;
  if (m < M) row_stats(xr, D, lane, eps, mean, rstd);
  for (int k = lane; k < KB * 64; k += 32) {
    const float v = (m < M && k < D) ? (xr[k] - mean) * rstd * g[k] + be[k] : 0.f;
    taco::store_split_scalar(v, m, rows_total, k, t_hi, t_lo);
  }
}

// Multi-head attention of one (row b, head h, kQ queries) per CTA, kLanes threads per query splitting the keys, merged at
// the end in a fixed order.  qkv [M][3D] (q | k | v), P [T_max][ldp] = linear_pos(pos_emb) of this block (rel only).
// rel: score(i, j) = ((q_i + u) . k_j + bd(i, j)) / sqrt(dk) with the legacy rel_shift in closed form:
//   bd(i, j) = (q_i + v) . p[T - 1 - i + j] for j <= i,  0 for j = i + 1,  (q_{i+1} + v) . p[j - i - 2] for j > i + 1.
template <int DK>
__global__ void __launch_bounds__(128) attn_kernel(const float* __restrict__ qkv, const float* __restrict__ P, int ldp,
                                                   const float* __restrict__ pu, const float* __restrict__ pv,
                                                   const int* __restrict__ len, int T_max, int D, int dk, int rel,
                                                   float* __restrict__ ctx) {
  extern __shared__ float asm_[];
  float* Ks = asm_;                 // [kKT][dk]
  float* Vs = Ks + kKT * dk;        // [kKT][dk]
  float* Pl = Vs + kKT * dk;        // [2 kKT][dk]: p rows [lo0, lo0 + 2 kKT)
  float* Pu = Pl + 2 * kKT * dk;    // [2 kKT][dk]: p rows [up0, up0 + 2 kKT)
  const int b = blockIdx.z, h = blockIdx.y;
  const int T = len[b];
  const int i0 = blockIdx.x * kQ;
  if (i0 >= T_max) return;
  const int qi = threadIdx.x / kLanes, sub = threadIdx.x % kLanes;
  const int i = i0 + qi;
  const bool active = i < T;
  const size_t ld = 3 * (size_t)D;
  const size_t rb = (size_t)b * T_max;
  float qu[DK], qv[DK], qn[DK], acc[DK];
#pragma unroll
  for (int d = 0; d < DK; ++d) {
    qu[d] = qv[d] = qn[d] = acc[d] = 0.f;
    if (d < dk && active) {
      const float q = qkv[(rb + i) * ld + h * dk + d];
      qu[d] = rel ? q + pu[h * dk + d] : q;
      qv[d] = rel ? q + pv[h * dk + d] : 0.f;
      if (rel && i + 1 < T) qn[d] = qkv[(rb + i + 1) * ld + h * dk + d] + pv[h * dk + d];
    }
  }
  const float sq = sqrtf((float)dk);
  float mx = -INFINITY, l = 0.f;
  const int nkt = i0 < T ? (T + kKT - 1) / kKT : 0;
  for (int kt = 0; kt < nkt; ++kt) {
    const int j0 = kt * kKT;
    const int lo0 = T - 1 - (i0 + kQ - 1) + j0;  // smallest T - 1 - i + j of this tile pair
    const int up0 = j0 - (i0 + kQ - 1) - 2;      // smallest j - i - 2
    __syncthreads();
    for (int e = threadIdx.x; e < kKT * dk; e += blockDim.x) {
      const int r = e / dk, d = e - r * dk;
      const int j = j0 + r;
      Ks[e] = j < T ? qkv[(rb + j) * ld + D + h * dk + d] : 0.f;
      Vs[e] = j < T ? qkv[(rb + j) * ld + 2 * D + h * dk + d] : 0.f;
    }
    if (rel) {
      for (int e = threadIdx.x; e < 2 * kKT * dk; e += blockDim.x) {
        const int r = e / dk, d = e - r * dk;
        const int a = lo0 + r, c = up0 + r;
        Pl[e] = (a >= 0 && a < T) ? P[(size_t)a * ldp + h * dk + d] : 0.f;
        Pu[e] = (c >= 0 && c < T) ? P[(size_t)c * ldp + h * dk + d] : 0.f;
      }
    }
    __syncthreads();
    if (!active) continue;
    for (int r = sub; r < kKT; r += kLanes) {
      const int j = j0 + r;
      if (j >= T) break;
      float ac = 0.f;
#pragma unroll
      for (int d = 0; d < DK; ++d)
        if (d < dk) ac += qu[d] * Ks[r * dk + d];
      float bd = 0.f;
      if (rel) {
        if (j <= i) {
          const float* pr = Pl + (T - 1 - i + j - lo0) * dk;
#pragma unroll
          for (int d = 0; d < DK; ++d)
            if (d < dk) bd += qv[d] * pr[d];
        } else if (j > i + 1) {
          const float* pr = Pu + (j - i - 2 - up0) * dk;
#pragma unroll
          for (int d = 0; d < DK; ++d)
            if (d < dk) bd += qn[d] * pr[d];
        }
      }
      const float s = (ac + bd) / sq;
      if (s > mx) {
        const float corr = expf(mx - s);
        l *= corr;
#pragma unroll
        for (int d = 0; d < DK; ++d) acc[d] *= corr;
        mx = s;
      }
      const float pexp = expf(s - mx);
      l += pexp;
#pragma unroll
      for (int d = 0; d < DK; ++d)
        if (d < dk) acc[d] += pexp * Vs[r * dk + d];
    }
  }
  // merge the kLanes key subsets (lanes kLanes qi + 0 .. kLanes - 1) in a fixed butterfly order
#pragma unroll
  for (int o = 1; o < kLanes; o <<= 1) {
    const float mo = __shfl_xor_sync(0xffffffffu, mx, o);
    const float lo_ = __shfl_xor_sync(0xffffffffu, l, o);
    const float mn = fmaxf(mx, mo);
    const float a = mx == -INFINITY ? 0.f : expf(mx - mn), c = mo == -INFINITY ? 0.f : expf(mo - mn);
#pragma unroll
    for (int d = 0; d < DK; ++d) {
      const float ao = __shfl_xor_sync(0xffffffffu, acc[d], o);
      acc[d] = acc[d] * a + ao * c;
    }
    l = l * a + lo_ * c;
    mx = mn;
  }
  if (sub == 0 && i < T_max) {
    float* out = ctx + (rb + i) * D + h * dk;
    for (int d = 0; d < dk; ++d) out[d] = active ? acc[d] / l : 0.f;
  }
}

}  // namespace enc
}  // namespace mb
