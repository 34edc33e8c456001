// Voice-conversion PPG extractor (models/ppg_extractor: PPGModel.forward) on the H100.  Every padded-batch row is computed
// as its own B = 1 call: the STFT, MVN statistics, both Conv2d layers and the depthwise conv read only the row's own frames
// (zeros past its end), attention runs over the row's own keys, and no summation order depends on B or on the row's slot.
//
//   frontend_kernel    reflect-padded frame, rectangular window (torch.stft without window=), direct DFT in double,
//                      power, melmat, log(. + 1e-20)                                         (stft.py, log_mel.py)
//   mvn_kernel         per-row mean / var over the row's frames in double; norm_vars divides by var^(1/4)
//                                                                                            (utterance_mvn.py:39-74)
//   conv0_kernel       embed.conv.0 (1 -> D), FFMA, bias + ReLU -> channels-last fp16 hi / lo planes
//   conv2d_tc          embed.conv.2 implicit GEMM on wgmma (conv2d_tc.cu) -> embed.out.0's operand tiles
//   taco::tc_big       every Linear / pointwise conv (3-term split, FP32-equivalent); ff_scale 1/2 folded into w_2's
//                      inverse scale and bias (both powers of two: res + (y / 2) exactly as the reference rounds it)
//   ln_tiles_kernel    LayerNorm (eps 1e-12) straight into the next GEMM's hi / lo operand tiles
//   act_tiles_kernel   fp32 activations (+ swish / ReLU) -> operand tiles
//   attn_kernel        (row, head, 32 queries): ac and the legacy rel_shift'ed bd in closed form, online softmax, . V
//   dw_kernel          GLU + depthwise conv (zeros past the row's end) + eval BatchNorm + activation -> operand tiles
//   ln_rows_kernel     norm_final / after_norm
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include <climits>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

#include "mb_common.h"
#include "ppgx_kernels.cuh"
#include "tacotron_kernels.cuh"

using namespace mb;

namespace {

constexpr int kMaxRows = 128;
constexpr int kMaxFft = 1024;
constexpr int kLanes = 4;  // threads per query in the attention kernel, each taking every kLanes-th key
constexpr int kQ = 128 / kLanes;  // queries per attention CTA
constexpr int kKT = 32; // keys per shared-memory tile
static_assert(kQ - 1 + kKT <= 2 * kKT, "the p-row windows of a tile pair hold 2 kKT rows");

__device__ __forceinline__ float sigmoidf_(float x) { return 1.f / (1.f + expf(-x)); }
__device__ __forceinline__ float act_f(float x, int act) {  // 0 none, 1 relu, 2 swish
  return act == 1 ? fmaxf(x, 0.f) : act == 2 ? x * sigmoidf_(x) : x;
}

// ---------------------------------------------------------------------------------------------- frontend
// grid (T_stft_max, B); one frame per CTA
__global__ void frontend_kernel(const float* __restrict__ wav, int n_max, const int* __restrict__ nsamp,
                                const int* __restrict__ tf_len, int Tf_max, int n_fft, int win, int hop,
                                const float* __restrict__ melmat, int n_mels, float* __restrict__ out) {
  extern __shared__ double fsm[];
  double* cs = fsm;             // cos(2 pi n / n_fft)
  double* sn = cs + n_fft;      // sin
  double* frame = sn + n_fft;   // windowed frame
  double* power = frame + n_fft;
  const int b = blockIdx.y, t = blockIdx.x;
  float* o = out + ((size_t)b * Tf_max + t) * n_mels;
  if (t >= tf_len[b]) {
    for (int m = threadIdx.x; m < n_mels; m += blockDim.x) o[m] = 0.f;
    return;
  }
  const int L = nsamp[b];
  const float* x = wav + (size_t)b * n_max;
  const int left = (n_fft - win) / 2;
  for (int n = threadIdx.x; n < n_fft; n += blockDim.x) {
    double s, c;
    sincospi(2.0 * n / n_fft, &s, &c);
    cs[n] = c;
    sn[n] = s;
    int i = t * hop - n_fft / 2 + n;  // center=True: reflect padding by n_fft / 2
    if (i < 0) i = -i;
    if (i >= L) i = 2 * (L - 1) - i;
    frame[n] = (n >= left && n < left + win) ? (double)x[i] : 0.0;
  }
  __syncthreads();
  const int n_freq = n_fft / 2 + 1;
  for (int k = threadIdx.x; k < n_freq; k += blockDim.x) {
    double re = 0.0, im = 0.0;
    int idx = (int)(((long long)k * left) % n_fft);
    for (int n = left; n < left + win; ++n) {
      re += frame[n] * cs[idx];
      im -= frame[n] * sn[idx];
      idx += k;
      if (idx >= n_fft) idx -= n_fft;
    }
    const float fr = (float)re, fi = (float)im;
    power[k] = (double)(fr * fr + fi * fi);
  }
  __syncthreads();
  for (int m = threadIdx.x; m < n_mels; m += blockDim.x) {
    double acc = 0.0;
    for (int k = 0; k < n_freq; ++k) acc += power[k] * (double)melmat[(size_t)k * n_mels + m];
    o[m] = logf((float)acc + 1e-20f);
  }
}

// grid B; one thread per mel bin, the row's frames in order (double accumulation)
__global__ void mvn_kernel(float* __restrict__ x, const int* __restrict__ tf_len, int Tf_max, int F, int norm_means,
                           int norm_vars) {
  const int b = blockIdx.x;
  const int n = tf_len[b];
  for (int f = threadIdx.x; f < F; f += blockDim.x) {
    float* c = x + (size_t)b * Tf_max * F + f;
    double s = 0.0;
    for (int t = 0; t < n; ++t) s += c[(size_t)t * F];
    const float mean = (float)(s / n);
    if (!norm_means && !norm_vars) continue;
    double v = 0.0;
    for (int t = 0; t < n; ++t) {
      const float d = c[(size_t)t * F] - mean;
      v += (double)d * d;
    }
    const float sd = fmaxf(sqrtf((float)(v / n)), 1e-20f);
    const float div = norm_means ? sqrtf(sd) : sd;  // utterance_mvn.py:62-73: var^(1/4) with norm_means, the std without
    for (int t = 0; t < n; ++t) {
      float y = c[(size_t)t * F];
      if (norm_means) y -= mean;
      if (norm_vars) y /= div;
      c[(size_t)t * F] = y;
    }
  }
}

// embed.conv.0: [B][Tf][F] (1 channel) -> relu(conv) as channels-last hi / lo planes [B][T1][F1][D]
__global__ void conv0_kernel(const float* __restrict__ x, const int* __restrict__ tf_len, int Tf_max, int F,
                             const float* __restrict__ w, const float* __restrict__ bias, int D, int k, int s, int p,
                             int T1_max, int F1, __half* __restrict__ y_hi, __half* __restrict__ y_lo) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int b = blockIdx.y;
  const size_t per = (size_t)T1_max * F1 * D;
  if (i >= per) return;
  const int c = (int)(i % D);
  const int f = (int)((i / D) % F1);
  const int t = (int)(i / ((size_t)D * F1));
  const int n = tf_len[b];
  const float* xb = x + (size_t)b * Tf_max * F;
  float acc = bias[c];
  for (int dt = 0; dt < k; ++dt) {
    const int ti = t * s + dt - p;
    if (ti < 0 || ti >= n) continue;
    for (int df = 0; df < k; ++df) {
      const int fi = f * s + df - p;
      if (fi < 0 || fi >= F) continue;
      acc += w[((size_t)c * k + dt) * k + df] * xb[(size_t)ti * F + fi];
    }
  }
  const float v = fmaxf(acc, 0.f);
  const __half h = __float2half_rn(v);
  const size_t o = (size_t)b * per + i;
  y_hi[o] = h;
  y_lo[o] = __float2half_rn(v - __half2float(h));
}

// x[m][n] = y[m][n] * xscale (+ pe[t][n] for abs_pos)
__global__ void embed_finish_kernel(const float* __restrict__ y, float* __restrict__ x, int M, int D, int T_max, float xscale,
                                    const float* __restrict__ pe) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)M * D) return;
  float v = y[i] * xscale;
  if (pe) v += pe[(size_t)((i / D) % T_max) * D + i % D];
  x[i] = v;
}

// fp32 [M][ld] (columns [0, K)) with an activation -> operand tiles [KB][rows_total][64]; zeros elsewhere
__global__ void act_tiles_kernel(const float* __restrict__ src, int ld, int M, int K, int KB, int rows_total, int act,
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

// one warp per row: the row's mean / biased variance in a fixed order
__device__ __forceinline__ void row_stats(const float* x, int D, int lane, float& mean, float& rstd) {
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
  rstd = 1.f / sqrtf(v / D + 1e-12f);
}

// LayerNorm rows [0, M) of x -> operand tiles (rows [M, rows_total) and columns [D, 64 KB) zero)
__global__ void ln_tiles_kernel(const float* __restrict__ x, int M, int D, int KB, int rows_total, const float* __restrict__ g,
                                const float* __restrict__ be, __half* __restrict__ t_hi, __half* __restrict__ t_lo) {
  const int m = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (m >= rows_total) return;
  float mean = 0.f, rstd = 0.f;
  const float* xr = x + (size_t)m * D;
  if (m < M) row_stats(xr, D, lane, mean, rstd);
  for (int k = lane; k < KB * 64; k += 32) {
    const float v = (m < M && k < D) ? (xr[k] - mean) * rstd * g[k] + be[k] : 0.f;
    taco::store_split_scalar(v, m, rows_total, k, t_hi, t_lo);
  }
}

// LayerNorm of rows [0, M) of x -> dst (may alias x); zero_pad: rows t >= len[b] of [B][T_max] are written as zeros
__global__ void ln_rows_kernel(const float* x, float* dst, int M, int D, const float* __restrict__ g, const float* __restrict__ be,
                               const int* __restrict__ len, int T_max, int zero_pad) {
  const int m = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (m >= M) return;
  const float* xr = x + (size_t)m * D;
  float* yr = dst + (size_t)m * D;
  if (zero_pad && m % T_max >= len[m / T_max]) {
    for (int n = lane; n < D; n += 32) yr[n] = 0.f;
    return;
  }
  float mean, rstd;
  row_stats(xr, D, lane, mean, rstd);
  __syncwarp();
  for (int n = lane; n < D; n += 32) yr[n] = (xr[n] - mean) * rstd * g[n] + be[n];
}

// taps[m][n] = x[m][n], zero for rows past the row's frames
__global__ void tap_kernel(const float* __restrict__ x, float* __restrict__ tap, int M, int D, const int* __restrict__ len,
                           int T_max) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)M * D) return;
  const int m = (int)(i / D);
  tap[i] = (m % T_max < len[m / T_max]) ? x[i] : 0.f;
}

// conv module: GLU(pw1) -> depthwise conv (zeros outside [0, len)) -> eval BatchNorm -> activation -> operand tiles.
// One thread per (row, 8 channels).
__global__ void dw_kernel(const float* __restrict__ pw, int D, int M, int T_max, const int* __restrict__ len,
                          const float* __restrict__ w, const float* __restrict__ bias, int K, const float* __restrict__ bn_w,
                          const float* __restrict__ bn_b, const float* __restrict__ bn_m, const float* __restrict__ bn_v,
                          int act, int KB, int rows_total, __half* __restrict__ t_hi, __half* __restrict__ t_lo) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t total = (size_t)KB * rows_total * 8;
  if (i >= total) return;
  const int c8 = (int)(i & 7);
  const int m = (int)((i >> 3) % rows_total);
  const int kb = (int)(i / ((size_t)8 * rows_total));
  const int b = m / T_max, t = m - b * T_max;
  const bool row_ok = m < M && t < len[b];
  const int pad = (K - 1) / 2;
  __align__(16) __half hi[8], lo[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    const int c = kb * 64 + c8 * 8 + e;
    float v = 0.f;
    if (row_ok && c < D) {
      float s = bias[c];
      for (int kk = 0; kk < K; ++kk) {
        const int tt = t + kk - pad;
        if (tt < 0 || tt >= len[b]) continue;
        const float* r = pw + (size_t)(b * T_max + tt) * 2 * D;
        s += w[(size_t)c * K + kk] * (r[c] * sigmoidf_(r[D + c]));
      }
      v = act_f((s - bn_m[c]) / sqrtf(bn_v[c] + 1e-5f) * bn_w[c] + bn_b[c], act);
    }
    hi[e] = __float2half_rn(v);
    lo[e] = __float2half_rn(v - __half2float(hi[e]));
  }
  const size_t o = ((size_t)kb * rows_total + m) * 8 + (size_t)(c8 ^ (m & 7));
  reinterpret_cast<uint4*>(t_hi)[o] = *reinterpret_cast<const uint4*>(hi);
  reinterpret_cast<uint4*>(t_lo)[o] = *reinterpret_cast<const uint4*>(lo);
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

// ---------------------------------------------------------------------------------------------- weights
// one tensor-core GEMM: packed weight image + the fp32 sources it is packed from
struct Gemm {
  std::vector<std::string> w;  // row blocks concatenated along N (QKV, linear_pos of all blocks)
  std::vector<std::string> b;  // biases (empty: none)
  int N = 0, K = 0;
  bool half = false;           // ff_scale 1/2 folded into the inverse scale and the bias
  size_t w_cat = 0, b_cat = 0; // fp32 concatenation / scaled bias in the arena (floats), when needed
  size_t img = 0;              // byte offset of the packed image
  float inv_scale = 1.f;
  const float* bias = nullptr; // resolved by finalize
};

// parameters the forward reads per block, resolved by name once in finalize (none are looked up per call)
struct BlockW {
  const float *ln_mac[2] = {}, *ln_mha[2] = {}, *ln_conv[2] = {}, *ln_ff[2] = {}, *ln_final[2] = {};  // weight, bias
  const float *pu = nullptr, *pv = nullptr;
  const float *dw_w = nullptr, *dw_b = nullptr, *bn_w = nullptr, *bn_b = nullptr, *bn_m = nullptr, *bn_v = nullptr;
};

}  // namespace

struct mb_ppgx {
  mb_ppgx_config cfg{};
  int D = 0, H = 0, dk = 0, U = 0, nb = 0, F = 0, n_freq = 0;
  int k0 = 5, s0 = 1, p0 = 2, k2 = 5, s2 = 1, p2 = 2, F1 = 0, F2 = 0;
  bool rel = false;
  WeightTable w;
  std::vector<Gemm> g;     // [0] embed.out, [1] linear_pos (rel), then per block: qkv, out, (mac w1, mac w2), w1, w2, (pw1, pw2)
  int g_pos = -1;
  std::vector<int> g_block;  // first GEMM of each block
  size_t floats = 0, abs_off = 0, conv_img = 0, total_bytes = 0;
  float conv_inv_scale = 1.f;
  char* arena = nullptr;
  bool finalized = false;
  std::vector<int> host_ints;
  std::vector<BlockW> bw;
  const float *melmat = nullptr, *conv0_w = nullptr, *conv0_b = nullptr, *conv2_b = nullptr, *after_w = nullptr,
              *after_b = nullptr;

  const float* p(const std::string& name) const { return w.ptr(name); }
  float* fl(size_t off) const { return reinterpret_cast<float*>(arena) + off; }
  int frames_stft(int n) const { return 1 + n / cfg.hop_length; }
  // torch's conv output length floor((L + 2p - k) / s) + 1, with a floor (not truncating) division
  static int conv_len(int L, int k, int s, int p) {
    const int a = L + 2 * p - k;
    return (a >= 0 ? a / s : -((-a + s - 1) / s)) + 1;
  }
  int frames1(int n) const { return conv_len(frames_stft(n), k0, s0, p0); }
  int frames(int n) const { return conv_len(frames1(n), k2, s2, p2); }
};

namespace {

int kb_of(int K) { return (K + 63) / 64; }
size_t ceil128(size_t m) { return (m + 127) / 128 * 128; }

void build_specs(mb_ppgx* h) {
  const int D = h->D, U = h->U;
  h->w.add("frontend.logmel.melmat", {h->n_freq, h->F});
  h->w.add("encoder.embed.conv.0.weight", {D, 1, h->k0, h->k0});
  h->w.add("encoder.embed.conv.0.bias", {D});
  h->w.add("encoder.embed.conv.2.weight", {D, D, h->k2, h->k2});
  h->w.add("encoder.embed.conv.2.bias", {D});
  h->w.add("encoder.embed.out.0.weight", {D, (int64_t)D * h->F2});
  h->w.add("encoder.embed.out.0.bias", {D});
  Gemm ge;
  ge.w = {"encoder.embed.out.0.weight"};
  ge.b = {"encoder.embed.out.0.bias"};
  ge.N = D, ge.K = D * h->F2;
  h->g.push_back(ge);
  if (h->rel) {
    Gemm gp;
    for (int i = 0; i < h->nb; ++i) gp.w.push_back("encoder.encoders." + std::to_string(i) + ".self_attn.linear_pos.weight");
    gp.N = D * h->nb, gp.K = D;
    h->g_pos = (int)h->g.size();
    h->g.push_back(gp);
  }
  const bool mac = h->cfg.macaron_style, cnn = h->cfg.use_cnn_module;
  for (int i = 0; i < h->nb; ++i) {
    const std::string b = "encoder.encoders." + std::to_string(i) + ".";
    for (const char* n : {"linear_q", "linear_k", "linear_v", "linear_out"}) {
      h->w.add(b + "self_attn." + n + ".weight", {D, D});
      h->w.add(b + "self_attn." + n + ".bias", {D});
    }
    if (h->rel) {
      h->w.add(b + "self_attn.linear_pos.weight", {D, D});
      h->w.add(b + "self_attn.pos_bias_u", {h->H, h->dk});
      h->w.add(b + "self_attn.pos_bias_v", {h->H, h->dk});
    }
    std::vector<std::string> ffs = {"feed_forward"};
    if (mac) ffs.push_back("feed_forward_macaron");
    for (const auto& f : ffs) {
      h->w.add(b + f + ".w_1.weight", {U, D});
      h->w.add(b + f + ".w_1.bias", {U});
      h->w.add(b + f + ".w_2.weight", {D, U});
      h->w.add(b + f + ".w_2.bias", {D});
    }
    if (cnn) {
      const std::string c = b + "conv_module.";
      h->w.add(c + "pointwise_conv1.weight", {2 * D, D, 1});
      h->w.add(c + "pointwise_conv1.bias", {2 * D});
      h->w.add(c + "depthwise_conv.weight", {D, 1, h->cfg.cnn_module_kernel});
      h->w.add(c + "depthwise_conv.bias", {D});
      for (const char* n : {"weight", "bias", "running_mean", "running_var"}) h->w.add(c + "norm." + n, {D});
      h->w.add(c + "pointwise_conv2.weight", {D, D, 1});
      h->w.add(c + "pointwise_conv2.bias", {D});
    }
    std::vector<std::string> norms = {"norm_ff", "norm_mha"};
    if (mac) norms.push_back("norm_ff_macaron");
    if (cnn) {
      norms.push_back("norm_conv");
      norms.push_back("norm_final");
    }
    for (const auto& n : norms) {
      h->w.add(b + n + ".weight", {D});
      h->w.add(b + n + ".bias", {D});
    }
    h->g_block.push_back((int)h->g.size());
    Gemm q;
    q.w = {b + "self_attn.linear_q.weight", b + "self_attn.linear_k.weight", b + "self_attn.linear_v.weight"};
    q.b = {b + "self_attn.linear_q.bias", b + "self_attn.linear_k.bias", b + "self_attn.linear_v.bias"};
    q.N = 3 * D, q.K = D;
    h->g.push_back(q);
    Gemm o;
    o.w = {b + "self_attn.linear_out.weight"};
    o.b = {b + "self_attn.linear_out.bias"};
    o.N = D, o.K = D;
    h->g.push_back(o);
    for (int r = (int)ffs.size() - 1; r >= 0; --r) {  // macaron first: the order the block runs them
      Gemm w1, w2;
      w1.w = {b + ffs[r] + ".w_1.weight"};
      w1.b = {b + ffs[r] + ".w_1.bias"};
      w1.N = U, w1.K = D;
      w2.w = {b + ffs[r] + ".w_2.weight"};
      w2.b = {b + ffs[r] + ".w_2.bias"};
      w2.N = D, w2.K = U;
      w2.half = mac;
      h->g.push_back(w1);
      h->g.push_back(w2);
    }
    if (cnn) {
      Gemm a, c2;
      a.w = {b + "conv_module.pointwise_conv1.weight"};
      a.b = {b + "conv_module.pointwise_conv1.bias"};
      a.N = 2 * D, a.K = D;
      c2.w = {b + "conv_module.pointwise_conv2.weight"};
      c2.b = {b + "conv_module.pointwise_conv2.bias"};
      c2.N = D, c2.K = D;
      h->g.push_back(a);
      h->g.push_back(c2);
    }
  }
  h->w.add("encoder.after_norm.weight", {D});
  h->w.add("encoder.after_norm.bias", {D});
  size_t off = h->w.floats();  // the model's own derived regions follow the table
  for (auto& gm : h->g) {
    if (gm.w.size() > 1) {
      gm.w_cat = off;
      off += mb::align_up((size_t)gm.N * gm.K, 64);
    }
    if (!gm.b.empty() && (gm.b.size() > 1 || gm.half)) {
      gm.b_cat = off;
      off += mb::align_up((size_t)gm.N, 64);
    }
  }
  h->abs_off = off;  // max |w| slots of finalize (one per GEMM + the conv)
  off += mb::align_up(h->g.size() + 1, 64);
  h->floats = off;
  size_t bytes = mb::align_up(off * sizeof(float), 1024);
  h->conv_img = bytes;
  bytes += mb::align_up(ppgx::conv2d_tc_weight_bytes(D, D, h->k2, h->k2), 1024);
  for (auto& gm : h->g) {
    gm.img = bytes;
    bytes += mb::align_up(taco::tc_big_weight_bytes(gm.N, 1, gm.K), 1024);
  }
  h->total_bytes = bytes;
}

struct WsLayout {
  size_t ints, feat, pl_hi, pl_lo, e_hi, e_lo, x, y, ctx, t_hi, t_lo, pt_hi, pt_lo, P, total;
  int Tf, T1, T, M, RT, RTp, KBe, KBt, KBd;
};

WsLayout ws_layout(const mb_ppgx* h, int B, int n_max) {
  WsLayout L{};
  L.Tf = h->frames_stft(n_max);
  L.T1 = h->frames1(n_max);
  L.T = h->frames(n_max);
  L.M = B * L.T;
  L.RT = (int)ceil128(L.M);
  L.RTp = (int)ceil128(L.T);
  L.KBe = kb_of(h->D * h->F2);
  L.KBd = kb_of(h->D);
  L.KBt = std::max(kb_of(h->D), kb_of(h->U));
  const int wide = std::max(std::max(3 * h->D, h->U), 2 * h->D);
  size_t o = 0;
  auto take = [&](size_t bytes) {
    const size_t r = o;
    o += mb::align_up(bytes, 256);
    return r;
  };
  L.ints = take(sizeof(int) * 4 * kMaxRows);
  L.feat = take(sizeof(float) * (size_t)B * L.Tf * h->F);
  L.pl_hi = take(sizeof(__half) * (size_t)B * L.T1 * h->F1 * h->D);
  L.pl_lo = take(sizeof(__half) * (size_t)B * L.T1 * h->F1 * h->D);
  L.e_hi = take(sizeof(__half) * (size_t)L.KBe * L.RT * 64);
  L.e_lo = take(sizeof(__half) * (size_t)L.KBe * L.RT * 64);
  L.x = take(sizeof(float) * (size_t)L.M * h->D);
  L.y = take(sizeof(float) * (size_t)L.M * wide);
  L.ctx = take(sizeof(float) * (size_t)L.M * h->D);
  L.t_hi = take(sizeof(__half) * (size_t)L.KBt * L.RT * 64);
  L.t_lo = take(sizeof(__half) * (size_t)L.KBt * L.RT * 64);
  if (h->rel) {
    L.pt_hi = take(sizeof(__half) * (size_t)L.KBd * L.RTp * 64);
    L.pt_lo = take(sizeof(__half) * (size_t)L.KBd * L.RTp * 64);
    L.P = take(sizeof(float) * (size_t)L.T * h->nb * h->D);
  }
  L.total = o;
  return L;
}

#define MB_TRY(x)                 \
  do {                            \
    const int _rc = (x);          \
    if (_rc != MB_OK) return _rc; \
  } while (0)

int run_gemm(const mb_ppgx* h, const Gemm& gm, const __half* a_hi, const __half* a_lo, int M, int rows_total, const float* res,
             float* y, int ldy, cudaStream_t st) {
  taco::TcBigArgs a{};
  a.a_hi = a_hi;
  a.a_lo = a_lo;
  a.w = reinterpret_cast<const __half*>(h->arena + gm.img);
  a.bias = gm.bias;
  a.KB = kb_of(gm.K);
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

int to_tiles(const float* src, int ld, int M, int K, int KB, int rows_total, int act, __half* hi, __half* lo, cudaStream_t st) {
  const size_t n = (size_t)KB * rows_total * 8;
  act_tiles_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(src, ld, M, K, KB, rows_total, act, hi, lo);
  MB_LAUNCH_CHECK("act_tiles_kernel");
  return MB_OK;
}

int ln_tiles(int D, const float* x, int M, int RT, const float* g, const float* be, __half* hi, __half* lo, cudaStream_t st) {
  ln_tiles_kernel<<<RT / 8, 256, 0, st>>>(x, M, D, kb_of(D), RT, g, be, hi, lo);
  MB_LAUNCH_CHECK("ln_tiles_kernel");
  return MB_OK;
}

int ln_rows(const float* x, float* dst, int M, int D, const float* g, const float* be, const int* len, int T, int zero_pad,
            cudaStream_t st) {
  ln_rows_kernel<<<(M + 7) / 8, 256, 0, st>>>(x, dst, M, D, g, be, len, T, zero_pad);
  MB_LAUNCH_CHECK("ln_rows_kernel");
  return MB_OK;
}

int launch_frontend(const float* wav, int n_max, const int* nsamp, const int* tf_len, int B, int Tf, int n_fft, int win, int hop,
                    const float* melmat, int n_mels, float* feat, cudaStream_t st) {
  const size_t smem = sizeof(double) * (3 * n_fft + n_fft / 2 + 1);
  frontend_kernel<<<dim3(Tf, B), 256, smem, st>>>(wav, n_max, nsamp, tf_len, Tf, n_fft, win, hop, melmat, n_mels, feat);
  MB_LAUNCH_CHECK("frontend_kernel");
  return MB_OK;
}

int launch_mvn(float* feat, const int* tf_len, int B, int Tf, int F, int norm_means, int norm_vars, cudaStream_t st) {
  mvn_kernel<<<B, 128, 0, st>>>(feat, tf_len, Tf, F, norm_means, norm_vars);
  MB_LAUNCH_CHECK("mvn_kernel");
  return MB_OK;
}

int launch_conv0(const float* feat, const int* tf_len, int B, int Tf, int F, const float* w, const float* bias, int D, int k, int s,
                 int p, int T1, int F1, __half* y_hi, __half* y_lo, cudaStream_t st) {
  const size_t per = (size_t)T1 * F1 * D;
  conv0_kernel<<<dim3((unsigned)((per + 255) / 256), B), 256, 0, st>>>(feat, tf_len, Tf, F, w, bias, D, k, s, p, T1, F1, y_hi,
                                                                         y_lo);
  MB_LAUNCH_CHECK("conv0_kernel");
  return MB_OK;
}

// embed.conv.2 into embed.out.0's operand tiles [kb_of(N F_out)][rows_total][64], zeroed first: the rows past M and the
// columns past N F_out are read by the GEMM
int run_conv2d(const ppgx::Conv2dTcArgs& c, cudaStream_t st) {
  const size_t bytes = sizeof(__half) * (size_t)kb_of(c.N * c.F_out) * c.rows_total * 64;
  MB_CUDA_CHECK(cudaMemsetAsync(c.y_hi, 0, bytes, st));
  MB_CUDA_CHECK(cudaMemsetAsync(c.y_lo, 0, bytes, st));
  const cudaError_t e = ppgx::launch_conv2d_tc(c, st);
  if (e != cudaSuccess) return fail(MB_ERR_CUDA, "conv2d_tc launch failed: %s", cudaGetErrorString(e));
  count_launch();
  return MB_OK;
}

int launch_dw(const float* pw, int D, int M, int T, const int* len, const float* w, const float* bias, int K, const float* bn_w,
              const float* bn_b, const float* bn_m, const float* bn_v, int act, int RT, __half* hi, __half* lo, cudaStream_t st) {
  const size_t n = (size_t)kb_of(D) * RT * 8;
  dw_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(pw, D, M, T, len, w, bias, K, bn_w, bn_b, bn_m, bn_v, act, kb_of(D), RT,
                                                         hi, lo);
  MB_LAUNCH_CHECK("dw_kernel");
  return MB_OK;
}

int attention_dk(int dk) { return dk <= 16 ? 16 : dk <= 32 ? 32 : dk <= 40 ? 40 : dk <= 64 ? 64 : 0; }

// attention of B rows of T padded frames: qkv [B T][3 D], heads of dk at column h dk, P rows at stride ldp (rel only)
int launch_attn(const float* qkv, const float* P, int ldp, const float* pu, const float* pv, const int* len, int B, int T, int H,
                int dk, int D, int rel, float* ctx, cudaStream_t st) {
  dim3 grid((T + kQ - 1) / kQ, H, B);
  const size_t smem = sizeof(float) * 6 * kKT * dk;
  switch (attention_dk(dk)) {
#define MB_ATTN(DK)                                                                                                       \
  case DK:                                                                                                                \
    attn_kernel<DK><<<grid, 128, smem, st>>>(qkv, P, ldp, pu, pv, len, T, D, dk, rel, ctx);                              \
    break;
    MB_ATTN(16)
    MB_ATTN(32)
    MB_ATTN(40)
    MB_ATTN(64)
#undef MB_ATTN
    default:
      return fail(MB_ERR_INVALID, "attention head dim %d > 64", dk);
  }
  MB_LAUNCH_CHECK("attn_kernel");
  return MB_OK;
}

__global__ void scale_kernel(const float* a, float s, float* dst, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) dst[i] = a[i] * s;
}

}  // namespace

extern "C" {

int mb_ppgx_create(const mb_ppgx_config* cfg, mb_ppgx** out) {
  if (!cfg || !out) return fail(MB_ERR_INVALID, "mb_ppgx_create: null argument");
  const mb_ppgx_config& c = *cfg;
  if (c.input_layer != MB_PPGX_INPUT_CONV2D)
    return fail(MB_ERR_INVALID, "mb_ppgx_create: input_layer %d is not supported (only conv2d)", c.input_layer);
  if (c.pos_enc_layer_type == MB_PPGX_POS_SCALED_ABS)
    return fail(MB_ERR_INVALID, "mb_ppgx_create: pos_enc_layer_type scaled_abs_pos is not supported");
  if (c.pos_enc_layer_type != MB_PPGX_POS_ABS && c.pos_enc_layer_type != MB_PPGX_POS_REL)
    return fail(MB_ERR_INVALID, "mb_ppgx_create: pos_enc_layer_type %d unknown", c.pos_enc_layer_type);
  if ((c.pos_enc_layer_type == MB_PPGX_POS_REL) != (c.selfattention_layer_type == MB_PPGX_ATTN_REL))
    return fail(MB_ERR_INVALID, "mb_ppgx_create: selfattention_layer_type rel_selfattn goes with pos_enc_layer_type rel_pos "
                                "(the reference asserts it)");
  if (c.concat_after) return fail(MB_ERR_INVALID, "mb_ppgx_create: concat_after is not supported");
  if (!c.normalize_before) return fail(MB_ERR_INVALID, "mb_ppgx_create: normalize_before=False is not supported");
  if (c.positionwise_layer_type != MB_PPGX_FF_LINEAR)
    return fail(MB_ERR_INVALID, "mb_ppgx_create: positionwise_layer_type %d is not supported (only linear)",
                c.positionwise_layer_type);
  if (c.kaldi_padding_mode) return fail(MB_ERR_INVALID, "mb_ppgx_create: kaldi_padding_mode is not supported");
  if (c.downsample_rate > 1) return fail(MB_ERR_INVALID, "mb_ppgx_create: downsample_rate %d > 1 is not supported", c.downsample_rate);
  if (c.activation_type != MB_PPGX_ACT_SWISH && c.activation_type != MB_PPGX_ACT_RELU)
    return fail(MB_ERR_INVALID, "mb_ppgx_create: activation_type %d is not supported (swish or relu)", c.activation_type);
  if (c.attention_heads < 1 || c.attention_dim < 1 || c.attention_dim % c.attention_heads)
    return fail(MB_ERR_INVALID, "mb_ppgx_create: attention_dim %d not divisible by attention_heads %d", c.attention_dim,
                c.attention_heads);
  if (attention_dk(c.attention_dim / c.attention_heads) == 0)
    return fail(MB_ERR_INVALID, "mb_ppgx_create: attention_dim / attention_heads = %d > 64", c.attention_dim / c.attention_heads);
  if (ppgx::conv2d_tc_ntile(c.attention_dim) == 0)
    return fail(MB_ERR_INVALID, "mb_ppgx_create: attention_dim %d must be a multiple of 32 or of 144", c.attention_dim);
  if (c.linear_units < 4 || c.linear_units % 4) return fail(MB_ERR_INVALID, "mb_ppgx_create: linear_units %d not a multiple of 4", c.linear_units);
  if (c.num_blocks < 1 || c.num_blocks > 64) return fail(MB_ERR_INVALID, "mb_ppgx_create: num_blocks %d outside 1..64", c.num_blocks);
  if (c.use_cnn_module && (c.cnn_module_kernel < 1 || c.cnn_module_kernel % 2 == 0))
    return fail(MB_ERR_INVALID, "mb_ppgx_create: cnn_module_kernel %d must be odd", c.cnn_module_kernel);
  if (c.n_fft < 2 || c.n_fft > kMaxFft || c.win_length < 1 || c.win_length > c.n_fft || c.hop_length < 1)
    return fail(MB_ERR_INVALID, "mb_ppgx_create: n_fft %d / win_length %d / hop_length %d unsupported (n_fft <= %d)", c.n_fft,
                c.win_length, c.hop_length, kMaxFft);
  if (c.n_mels < 4 || c.n_mels > 1024) return fail(MB_ERR_INVALID, "mb_ppgx_create: n_mels %d outside 4..1024", c.n_mels);
  auto* h = new mb_ppgx();
  h->cfg = c;
  h->D = c.attention_dim;
  h->H = c.attention_heads;
  h->dk = h->D / h->H;
  h->U = c.linear_units;
  h->nb = c.num_blocks;
  h->F = c.n_mels;
  h->n_freq = c.n_fft / 2 + 1;
  h->rel = c.pos_enc_layer_type == MB_PPGX_POS_REL;
  if (!c.no_subsample) {
    h->k2 = 4, h->s2 = 2, h->p2 = 1;
    if (!c.subsample_by_2) h->k0 = 4, h->s0 = 2, h->p0 = 1;
  }
  h->F1 = (h->F + 2 * h->p0 - h->k0) / h->s0 + 1;
  h->F2 = (h->F1 + 2 * h->p2 - h->k2) / h->s2 + 1;
  build_specs(h);
  h->w.ignored = [](const std::string& n) {  // in the checkpoint, never read by inference
    return n == "frontend.logmel.inv_melmat" || n.find("num_batches_tracked") != std::string::npos;
  };
  *out = h;
  return MB_OK;
}

void mb_ppgx_destroy(mb_ppgx* h) { delete h; }

size_t mb_ppgx_arena_bytes(const mb_ppgx* h) { return h ? h->total_bytes : 0; }

int mb_ppgx_set_arena(mb_ppgx* h, void* arena, size_t bytes) {
  if (int rc = check_arena("mb_ppgx_set_arena", h, arena, bytes, mb_ppgx_arena_bytes(h), 1024)) return rc;
  h->w.attach(static_cast<float*>(arena));
  h->arena = static_cast<char*>(arena);
  h->finalized = false;
  return MB_OK;
}

int mb_ppgx_set_weight(mb_ppgx* h, const char* name, const float* w, const int64_t* dims, int32_t ndim, void* stream) {
  if (!h) return fail(MB_ERR_INVALID, "mb_ppgx_set_weight: null argument");
  if (int rc = h->w.set("mb_ppgx_set_weight", name, w, dims, ndim, stream)) return rc;
  h->finalized = false;
  return MB_OK;
}

int mb_ppgx_finalize(mb_ppgx* h, void* stream) {
  if (!h) return fail(MB_ERR_INVALID, "mb_ppgx_finalize: null handle");
  if (int rc = h->w.check_all_set("mb_ppgx_finalize")) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  // concatenations (QKV, linear_pos of all blocks) and their biases
  for (auto& gm : h->g) {
    if (gm.w_cat) {
      size_t o = 0;
      for (const auto& n : gm.w) {
        const size_t cnt = (size_t)gm.K * (gm.N / gm.w.size());
        MB_CUDA_CHECK(cudaMemcpyAsync(h->fl(gm.w_cat + o), h->p(n), cnt * sizeof(float), cudaMemcpyDeviceToDevice, st));
        o += cnt;
      }
    }
    if (gm.b_cat) {
      const int nb = gm.N / (int)gm.b.size();
      for (size_t i = 0; i < gm.b.size(); ++i) {
        scale_kernel<<<(nb + 255) / 256, 256, 0, st>>>(h->p(gm.b[i]), gm.half ? 0.5f : 1.f, h->fl(gm.b_cat) + i * nb, nb);
        MB_LAUNCH_CHECK("scale_kernel");
      }
    }
  }
  // power-of-two pack scales from each weight's max |w| (one host round trip)
  const size_t ng = h->g.size() + 1;
  unsigned int* d_abs = reinterpret_cast<unsigned int*>(h->fl(h->abs_off));
  MB_CUDA_CHECK(cudaMemsetAsync(d_abs, 0, ng * sizeof(unsigned int), st));
  auto src = [&](const Gemm& gm) { return gm.w_cat ? h->fl(gm.w_cat) : h->p(gm.w[0]); };
  for (size_t i = 0; i < h->g.size(); ++i) {
    const cudaError_t e = taco::tc_skinny_absmax(src(h->g[i]), (size_t)h->g[i].N * h->g[i].K, d_abs + i, st);
    if (e != cudaSuccess) return fail(MB_ERR_CUDA, "absmax: %s", cudaGetErrorString(e));
  }
  {
    const cudaError_t e = taco::tc_skinny_absmax(h->p("encoder.embed.conv.2.weight"), (size_t)h->D * h->D * h->k2 * h->k2,
                                                 d_abs + h->g.size(), st);
    if (e != cudaSuccess) return fail(MB_ERR_CUDA, "absmax: %s", cudaGetErrorString(e));
  }
  std::vector<unsigned int> bits(ng);
  MB_CUDA_CHECK(cudaMemcpyAsync(bits.data(), d_abs, ng * sizeof(unsigned int), cudaMemcpyDeviceToHost, st));
  MB_CUDA_CHECK(cudaStreamSynchronize(st));
  for (size_t i = 0; i < h->g.size(); ++i) {
    Gemm& gm = h->g[i];
    const float scale = taco::tc_weight_scale(bits[i]);
    gm.inv_scale = (gm.half ? 0.5f : 1.f) / scale;
    taco::TcBigPack q{};
    q.W = src(gm);
    q.ldw = gm.K;
    q.N = gm.N;
    q.nseg = 1;
    q.K = gm.K;
    q.KBs = kb_of(gm.K);
    q.w_off[0] = 0;
    q.w_stride[0] = 1;
    q.scale = scale;
    const cudaError_t e = taco::launch_pack_big_w(q, reinterpret_cast<__half*>(h->arena + gm.img), st);
    if (e != cudaSuccess) return fail(MB_ERR_CUDA, "pack: %s", cudaGetErrorString(e));
    count_launch();
  }
  for (auto& gm : h->g) gm.bias = gm.b.empty() ? nullptr : (gm.b_cat ? h->fl(gm.b_cat) : h->p(gm.b[0]));
  h->melmat = h->p("frontend.logmel.melmat");
  h->conv0_w = h->p("encoder.embed.conv.0.weight");
  h->conv0_b = h->p("encoder.embed.conv.0.bias");
  h->conv2_b = h->p("encoder.embed.conv.2.bias");
  h->after_w = h->p("encoder.after_norm.weight");
  h->after_b = h->p("encoder.after_norm.bias");
  h->bw.assign(h->nb, BlockW{});
  for (int i = 0; i < h->nb; ++i) {
    const std::string b = "encoder.encoders." + std::to_string(i) + ".";
    BlockW& w = h->bw[i];
    auto ln = [&](const char* n, const float* (&dst)[2]) {
      dst[0] = h->p(b + n + ".weight");
      dst[1] = h->p(b + n + ".bias");
    };
    ln("norm_ff_macaron", w.ln_mac);
    ln("norm_mha", w.ln_mha);
    ln("norm_conv", w.ln_conv);
    ln("norm_ff", w.ln_ff);
    ln("norm_final", w.ln_final);
    w.pu = h->p(b + "self_attn.pos_bias_u");
    w.pv = h->p(b + "self_attn.pos_bias_v");
    const std::string c = b + "conv_module.";
    w.dw_w = h->p(c + "depthwise_conv.weight");
    w.dw_b = h->p(c + "depthwise_conv.bias");
    w.bn_w = h->p(c + "norm.weight");
    w.bn_b = h->p(c + "norm.bias");
    w.bn_m = h->p(c + "norm.running_mean");
    w.bn_v = h->p(c + "norm.running_var");
  }
  const float cs = taco::tc_weight_scale(bits[h->g.size()]);
  h->conv_inv_scale = 1.f / cs;
  const cudaError_t e = ppgx::conv2d_tc_pack(h->p("encoder.embed.conv.2.weight"), h->D, h->D, h->k2, h->k2, cs,
                                             reinterpret_cast<__half*>(h->arena + h->conv_img), st);
  if (e != cudaSuccess) return fail(MB_ERR_CUDA, "conv2d pack: %s", cudaGetErrorString(e));
  count_launch();
  h->finalized = true;
  return MB_OK;
}

int32_t mb_ppgx_num_frames(const mb_ppgx* h, int32_t n_samples) {
  if (!h || n_samples < 0) return 0;
  return std::max(0, h->frames(n_samples));
}

size_t mb_ppgx_workspace_bytes(const mb_ppgx* h, int32_t batch, int32_t n_samples_max) {
  if (!h || batch < 1 || batch > kMaxRows || n_samples_max <= h->cfg.n_fft / 2 || h->frames(n_samples_max) < 1) return 0;
  return ws_layout(h, batch, n_samples_max).total;
}

int mb_ppgx_forward(mb_ppgx* h, const float* wav, const int32_t* n_samples, int32_t batch, int32_t n_max, int32_t pe_len,
                    const float* pos_table, float* out, float* taps, void* workspace, size_t workspace_bytes, void* stream) {
  if (!h) return fail(MB_ERR_INVALID, "mb_ppgx_forward: null handle");
  if (!h->finalized) return fail(MB_ERR_STATE, "mb_ppgx_forward: weights not finalized");
  if (batch < 1 || batch > kMaxRows) return fail(MB_ERR_INVALID, "mb_ppgx_forward: batch %d outside 1..%d", batch, kMaxRows);
  if (!wav || !n_samples || !pos_table || !out || !workspace) return fail(MB_ERR_INVALID, "mb_ppgx_forward: null argument");
  const size_t need = mb_ppgx_workspace_bytes(h, batch, n_max);
  if (need == 0) return fail(MB_ERR_INVALID, "mb_ppgx_forward: n_max %d gives no frames", n_max);
  if (workspace_bytes < need) return fail(MB_ERR_WORKSPACE, "mb_ppgx_forward: workspace %zu < %zu bytes", workspace_bytes, need);
  const WsLayout L = ws_layout(h, batch, n_max);
  if (h->rel && pe_len < L.T) return fail(MB_ERR_INVALID, "mb_ppgx_forward: pe_len %d < %d frames", pe_len, L.T);
  h->host_ints.assign(4 * kMaxRows, 0);
  for (int b = 0; b < batch; ++b) {
    const int n = n_samples[b];
    if (n <= h->cfg.n_fft / 2 || n > n_max || h->frames(n) < 1)
      return fail(MB_ERR_INVALID, "mb_ppgx_forward: n_samples[%d] = %d outside (%d, %d] or too short for one frame", b, n,
                  h->cfg.n_fft / 2, n_max);
    h->host_ints[b] = n;
    h->host_ints[kMaxRows + b] = h->frames_stft(n);
    h->host_ints[2 * kMaxRows + b] = h->frames1(n);
    h->host_ints[3 * kMaxRows + b] = h->frames(n);
  }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  char* ws = static_cast<char*>(workspace);
  int* d_ints = reinterpret_cast<int*>(ws + L.ints);
  const int *d_n = d_ints, *d_tf = d_ints + kMaxRows, *d_t1 = d_ints + 2 * kMaxRows, *d_t = d_ints + 3 * kMaxRows;
  MB_CUDA_CHECK(cudaMemcpyAsync(d_ints, h->host_ints.data(), sizeof(int) * 4 * kMaxRows, cudaMemcpyHostToDevice, st));
  const int D = h->D, B = batch, M = L.M, RT = L.RT, T = L.T;
  float* feat = reinterpret_cast<float*>(ws + L.feat);
  auto hp = [&](size_t o) { return reinterpret_cast<__half*>(ws + o); };
  float* x = reinterpret_cast<float*>(ws + L.x);
  float* y = reinterpret_cast<float*>(ws + L.y);
  float* ctx = reinterpret_cast<float*>(ws + L.ctx);

  // frontend + MVN
  MB_TRY(launch_frontend(wav, n_max, d_n, d_tf, B, L.Tf, h->cfg.n_fft, h->cfg.win_length, h->cfg.hop_length, h->melmat, h->F,
                         feat, st));
  MB_TRY(launch_mvn(feat, d_tf, B, L.Tf, h->F, h->cfg.norm_means, h->cfg.norm_vars, st));
  // input layer
  {
    MB_TRY(launch_conv0(feat, d_tf, B, L.Tf, h->F, h->conv0_w, h->conv0_b, D, h->k0, h->s0, h->p0, L.T1, h->F1, hp(L.pl_hi),
                        hp(L.pl_lo), st));
    ppgx::Conv2dTcArgs c{};
    c.x_hi = hp(L.pl_hi);
    c.x_lo = hp(L.pl_lo);
    c.len_in = d_t1;
    c.B = B, c.T_in = L.T1, c.F_in = h->F1, c.C = D;
    c.T_out = T, c.F_out = h->F2, c.kh = c.kw = h->k2, c.stride = h->s2, c.pad = h->p2;
    c.w = reinterpret_cast<const __half*>(h->arena + h->conv_img);
    c.bias = h->conv2_b;
    c.N = D, c.K = h->k2 * h->k2 * D, c.KB = kb_of(c.K);
    c.inv_scale = h->conv_inv_scale;
    c.y_hi = hp(L.e_hi);
    c.y_lo = hp(L.e_lo);
    c.rows_total = RT;
    MB_TRY(run_conv2d(c, st));
    MB_TRY(run_gemm(h, h->g[0], hp(L.e_hi), hp(L.e_lo), M, RT, nullptr, y, D, st));
    const size_t n = (size_t)M * D;
    embed_finish_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(y, x, M, D, T, sqrtf((float)D), h->rel ? nullptr : pos_table);
    MB_LAUNCH_CHECK("embed_finish_kernel");
  }
  const size_t MD = (size_t)M * D;
  auto tap = [&](int l) -> int {
    if (!taps) return MB_OK;
    tap_kernel<<<(unsigned)((MD + 255) / 256), 256, 0, st>>>(x, taps + (size_t)l * MD, M, D, d_t, T);
    MB_LAUNCH_CHECK("tap_kernel");
    return MB_OK;
  };
  MB_TRY(tap(0));
  float* P = h->rel ? reinterpret_cast<float*>(ws + L.P) : nullptr;
  if (h->rel) {  // linear_pos(pos_emb) of every block in one GEMM (N = num_blocks * D)
    MB_TRY(to_tiles(pos_table, D, T, D, L.KBd, L.RTp, 0, hp(L.pt_hi), hp(L.pt_lo), st));
    MB_TRY(run_gemm(h, h->g[h->g_pos], hp(L.pt_hi), hp(L.pt_lo), T, L.RTp, nullptr, P, h->nb * D, st));
  }
  const int act = h->cfg.activation_type == MB_PPGX_ACT_RELU ? 1 : 2;
  __half *th = hp(L.t_hi), *tl = hp(L.t_lo);
  for (int i = 0; i < h->nb; ++i) {
    const BlockW& w = h->bw[i];
    int gi = h->g_block[i];
    const Gemm &g_qkv = h->g[gi], &g_out = h->g[gi + 1];
    gi += 2;
    auto ffn = [&](const float* const (&norm)[2]) -> int {
      const Gemm &w1 = h->g[gi], &w2 = h->g[gi + 1];
      gi += 2;
      MB_TRY(ln_tiles(D, x, M, RT, norm[0], norm[1], th, tl, st));
      MB_TRY(run_gemm(h, w1, th, tl, M, RT, nullptr, y, h->U, st));
      MB_TRY(to_tiles(y, h->U, M, h->U, kb_of(h->U), RT, act, th, tl, st));
      return run_gemm(h, w2, th, tl, M, RT, x, x, D, st);  // x += ff_scale * w_2(.)
    };
    if (h->cfg.macaron_style) MB_TRY(ffn(w.ln_mac));
    MB_TRY(ln_tiles(D, x, M, RT, w.ln_mha[0], w.ln_mha[1], th, tl, st));
    MB_TRY(run_gemm(h, g_qkv, th, tl, M, RT, nullptr, y, 3 * D, st));
    MB_TRY(launch_attn(y, h->rel ? P + (size_t)i * D : nullptr, h->nb * D, w.pu, w.pv, d_t, B, T, h->H, h->dk, D, h->rel ? 1 : 0,
                       ctx, st));
    MB_TRY(to_tiles(ctx, D, M, D, kb_of(D), RT, 0, th, tl, st));
    MB_TRY(run_gemm(h, g_out, th, tl, M, RT, x, x, D, st));
    if (h->cfg.use_cnn_module) {
      // the block's GEMM order is qkv, out, (macaron), ffn, conv: the conv module's pair sits after the FFN pair(s)
      const int gc = gi + 2;
      MB_TRY(ln_tiles(D, x, M, RT, w.ln_conv[0], w.ln_conv[1], th, tl, st));
      MB_TRY(run_gemm(h, h->g[gc], th, tl, M, RT, nullptr, y, 2 * D, st));
      MB_TRY(launch_dw(y, D, M, T, d_t, w.dw_w, w.dw_b, h->cfg.cnn_module_kernel, w.bn_w, w.bn_b, w.bn_m, w.bn_v, act, RT, th, tl,
                       st));
      MB_TRY(run_gemm(h, h->g[gc + 1], th, tl, M, RT, x, x, D, st));
    }
    MB_TRY(ffn(w.ln_ff));
    if (h->cfg.use_cnn_module) MB_TRY(ln_rows(x, x, M, D, w.ln_final[0], w.ln_final[1], d_t, T, 0, st));
    MB_TRY(tap(i + 1));
  }
  return ln_rows(x, out, M, D, h->after_w, h->after_b, d_t, T, 1, st);
}

// ---------------------------------------------------------------------------------------------- one-launch test hook
size_t mb_ppgx_debug_workspace_bytes(const mb_ppgx_debug_spec* s) {
  if (!s) return 0;
  if (s->kind != MB_PPGX_DBG_CONV2D_TC) return 256;
  return 2048 + mb::align_up(ppgx::conv2d_tc_weight_bytes(s->N, s->C, s->k, s->k), 1024);  // absmax slot, then the image
}

int mb_ppgx_debug(const mb_ppgx_debug_spec* spec, void* workspace, size_t workspace_bytes, void* stream, char* report,
                  size_t report_len) {
  const char* me = "mb_ppgx_debug";
  if (!spec || !workspace) return fail(MB_ERR_INVALID, "%s: null argument", me);
  const mb_ppgx_debug_spec& s = *spec;
  const size_t need = mb_ppgx_debug_workspace_bytes(spec);
  if (workspace_bytes < need) return fail(MB_ERR_WORKSPACE, "%s: workspace %zu < %zu bytes", me, workspace_bytes, need);
  const bool rows = s.kind != MB_PPGX_DBG_LN_TILES && s.kind != MB_PPGX_DBG_ACT_TILES;  // kinds over a padded batch
  if (rows && (s.B < 1 || s.T < 1 || !s.len)) return fail(MB_ERR_INVALID, "%s: B %d / T %d / len", me, s.B, s.T);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  auto hp = [](void* p) { return static_cast<__half*>(p); };
  const char* kname = "";
  int inst = 0;
  dim3 grid(0, 0, 0);
  float inv_scale = 1.f;
  switch (s.kind) {
    case MB_PPGX_DBG_FRONTEND:
      if (s.n_fft < 2 || s.n_fft > kMaxFft || s.win_length < 1 || s.win_length > s.n_fft || s.hop_length < 1 || !s.len2)
        return fail(MB_ERR_INVALID, "%s: n_fft %d / win_length %d / hop_length %d", me, s.n_fft, s.win_length, s.hop_length);
      MB_TRY(launch_frontend(s.x, s.n_max, s.len, s.len2, s.B, s.T, s.n_fft, s.win_length, s.hop_length, s.w, s.F, s.y, st));
      kname = "frontend_kernel";
      grid = dim3(s.T, s.B);
      break;
    case MB_PPGX_DBG_MVN:
      MB_TRY(launch_mvn(s.y, s.len, s.B, s.T, s.F, s.flags & 1, (s.flags >> 1) & 1, st));
      kname = "mvn_kernel";
      grid = dim3(s.B);
      break;
    case MB_PPGX_DBG_CONV0: {
      const int T1 = mb_ppgx::conv_len(s.T, s.k, s.stride, s.pad), F1 = mb_ppgx::conv_len(s.F, s.k, s.stride, s.pad);
      if (T1 < 1 || F1 < 1) return fail(MB_ERR_INVALID, "%s: conv0 output %d x %d", me, T1, F1);
      MB_TRY(launch_conv0(s.x, s.len, s.B, s.T, s.F, s.w, s.bias, s.N, s.k, s.stride, s.pad, T1, F1, hp(s.y_hi), hp(s.y_lo), st));
      kname = "conv0_kernel";
      grid = dim3((unsigned)(((size_t)T1 * F1 * s.N + 255) / 256), s.B);
      break;
    }
    case MB_PPGX_DBG_CONV2D_TC: {
      const int NT = ppgx::conv2d_tc_ntile(s.N);
      ppgx::Conv2dTcArgs c{};
      c.x_hi = static_cast<const __half*>(s.x_hi);
      c.x_lo = static_cast<const __half*>(s.x_lo);
      c.len_in = s.len;
      c.B = s.B, c.T_in = s.T, c.F_in = s.F, c.C = s.C;
      c.T_out = mb_ppgx::conv_len(s.T, s.k, s.stride, s.pad), c.F_out = mb_ppgx::conv_len(s.F, s.k, s.stride, s.pad);
      c.kh = c.kw = s.k, c.stride = s.stride, c.pad = s.pad;
      c.N = s.N, c.K = s.k * s.k * s.C, c.KB = kb_of(c.K);
      c.bias = s.bias;
      c.y_hi = hp(s.y_hi);
      c.y_lo = hp(s.y_lo);
      c.rows_total = s.rows_total;
      if (NT == 0 || s.C % 8 || c.T_out < 1 || c.F_out < 1 || s.rows_total % 128 || s.rows_total < s.B * c.T_out)
        return fail(MB_ERR_INVALID, "%s: conv2d N %d / C %d / output %d x %d / rows_total %d", me, s.N, s.C, c.T_out, c.F_out,
                    s.rows_total);
      // as finalize: max |w| -> power-of-two scale (one host read-back) -> packed image
      char* ws = reinterpret_cast<char*>(((uintptr_t)workspace + 1023) & ~(uintptr_t)1023);
      unsigned int* d_abs = reinterpret_cast<unsigned int*>(ws);
      __half* img = reinterpret_cast<__half*>(ws + 1024);
      if (reinterpret_cast<char*>(img) + ppgx::conv2d_tc_weight_bytes(s.N, s.C, s.k, s.k) >
          static_cast<char*>(workspace) + workspace_bytes)
        return fail(MB_ERR_WORKSPACE, "%s: workspace too small for the weight image", me);
      MB_CUDA_CHECK(cudaMemsetAsync(d_abs, 0, sizeof(unsigned int), st));
      cudaError_t e = taco::tc_skinny_absmax(s.w, (size_t)s.N * s.C * s.k * s.k, d_abs, st);
      if (e != cudaSuccess) return fail(MB_ERR_CUDA, "absmax: %s", cudaGetErrorString(e));
      unsigned int bits = 0;
      MB_CUDA_CHECK(cudaMemcpyAsync(&bits, d_abs, sizeof(bits), cudaMemcpyDeviceToHost, st));
      MB_CUDA_CHECK(cudaStreamSynchronize(st));
      const float scale = taco::tc_weight_scale(bits);
      inv_scale = 1.f / scale;
      c.inv_scale = inv_scale;
      c.w = img;
      e = ppgx::conv2d_tc_pack(s.w, s.N, s.C, s.k, s.k, scale, img, st);
      if (e != cudaSuccess) return fail(MB_ERR_CUDA, "conv2d pack: %s", cudaGetErrorString(e));
      count_launch();
      MB_TRY(run_conv2d(c, st));
      kname = "conv2d_tc";
      inst = NT;
      grid = dim3((unsigned)((s.B * c.T_out * c.F_out + 127) / 128), (unsigned)(s.N / NT));
      break;
    }
    case MB_PPGX_DBG_LN_TILES:
      if (s.rows_total % 128 || s.M > s.rows_total) return fail(MB_ERR_INVALID, "%s: rows_total %d", me, s.rows_total);
      MB_TRY(ln_tiles(s.D, s.x, s.M, s.rows_total, s.w, s.bias, hp(s.y_hi), hp(s.y_lo), st));
      kname = "ln_tiles_kernel";
      grid = dim3(s.rows_total / 8);
      break;
    case MB_PPGX_DBG_ACT_TILES:
      if (s.rows_total % 128 || s.M > s.rows_total) return fail(MB_ERR_INVALID, "%s: rows_total %d", me, s.rows_total);
      MB_TRY(to_tiles(s.x, s.ld, s.M, s.D, kb_of(s.D), s.rows_total, s.act, hp(s.y_hi), hp(s.y_lo), st));
      kname = "act_tiles_kernel";
      grid = dim3((unsigned)(((size_t)kb_of(s.D) * s.rows_total * 8 + 255) / 256));
      break;
    case MB_PPGX_DBG_LN_ROWS:
      MB_TRY(ln_rows(s.x, s.y, s.B * s.T, s.D, s.w, s.bias, s.len, s.T, (s.flags >> 2) & 1, st));
      kname = "ln_rows_kernel";
      grid = dim3((s.B * s.T + 7) / 8);
      break;
    case MB_PPGX_DBG_DW:
      if (s.k < 1 || s.k % 2 == 0 || s.rows_total % 128 || s.B * s.T > s.rows_total)
        return fail(MB_ERR_INVALID, "%s: dw kernel %d / rows_total %d", me, s.k, s.rows_total);
      MB_TRY(launch_dw(s.x, s.D, s.B * s.T, s.T, s.len, s.w, s.bias, s.k, s.bn[0], s.bn[1], s.bn[2], s.bn[3], s.act, s.rows_total,
                       hp(s.y_hi), hp(s.y_lo), st));
      kname = "dw_kernel";
      grid = dim3((unsigned)(((size_t)kb_of(s.D) * s.rows_total * 8 + 255) / 256));
      break;
    case MB_PPGX_DBG_ATTN:
      if (s.H < 1 || s.dk < 1 || s.H * s.dk > s.D) return fail(MB_ERR_INVALID, "%s: H %d x dk %d > D %d", me, s.H, s.dk, s.D);
      MB_TRY(launch_attn(s.x, s.P, s.ldp, s.pu, s.pv, s.len, s.B, s.T, s.H, s.dk, s.D, s.rel, s.y, st));
      kname = "attn_kernel";
      inst = attention_dk(s.dk);
      grid = dim3((s.T + kQ - 1) / kQ, s.H, s.B);
      break;
    default:
      return fail(MB_ERR_INVALID, "%s: bad kind %d", me, s.kind);
  }
  MB_CUDA_CHECK(cudaStreamSynchronize(st));
  if (report && report_len)
    snprintf(report, report_len, "kernel=%s inst=%d grid=%u,%u,%u inv_scale=%.9e\n", kname, inst, grid.x, grid.y, grid.z,
             (double)inv_scale);
  return MB_OK;
}

}  // extern "C"
