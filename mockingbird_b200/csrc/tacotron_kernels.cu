// FP32 kernels of the Tacotron path (see tacotron_kernels.cuh).
#include "tacotron_kernels.cuh"

namespace mb {
namespace taco {

namespace {

constexpr int BM = 64;
constexpr int BK = 16;

__device__ __forceinline__ float act_fn(float v, int act) {
  if (act == ACT_RELU) return v > 0.f ? v : 0.f;
  if (act == ACT_SIGMOID) return 1.f / (1.f + expf(-v));
  if (act == ACT_TANH) return tanhf(v);
  return v;
}

// 64 x BN output tile, 256 threads, thread tile 4 x (BN/16); operands staged k-major in shared memory
__device__ __forceinline__ void step_seg0(const GemmArgs& a, Seg& sg) {
  if (!a.step_mode) return;
  const int si = step_index(a.step_ptr, a.step_j);
  if (si == 0 && a.x_first) {
    sg.x = a.x_first;
    sg.ld = 0;
  } else {
    sg.x += (long long)si * a.x_step;
  }
}
__device__ __forceinline__ const uint8_t* step_mask(const GemmArgs& a) {
  return a.step_mode ? a.mask + (size_t)step_index(a.step_ptr, a.step_j) * (size_t)a.mask_step : a.mask;
}

template <int BN>
__global__ void __launch_bounds__(256) gemm_kernel(const GemmArgs a) {
  constexpr int TN = BN / 16;
  __shared__ __align__(16) float As[BK][BM + 4];
  __shared__ __align__(16) float Bs[BK][BN + 4];
  const int tid = threadIdx.x;
  const int tx = tid & 15, ty = tid >> 4;
  const int m0 = blockIdx.y * BM, n0 = blockIdx.x * BN;
  float acc[4][TN];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;

  for (int s = 0; s < a.nseg; ++s) {
    Seg sg = a.seg[s];
    if (s == 0) step_seg0(a, sg);
    for (int k0 = 0; k0 < sg.K; k0 += BK) {
      // A tile: 64 rows x 16 k (k fastest -> coalesced along the feature axis)
      for (int i = tid; i < BM * BK; i += 256) {
        const int mm = i >> 4, kk = i & 15;
        const int m = m0 + mm;
        float v = 0.f;
        if (m < a.M && k0 + kk < sg.K) {
          int row = m;
          bool ok = true;
          if (sg.shift != 0) {
            const int t = m % a.T + sg.shift;
            ok = (t >= 0 && t < a.T);
            row = m + sg.shift;
          }
          if (ok) v = sg.x[(size_t)row * sg.ld + k0 + kk];
        }
        As[kk][mm] = v;
      }
      for (int i = tid; i < BN * BK; i += 256) {
        const int nn = i >> 4, kk = i & 15;
        const int n = n0 + nn;
        float v = 0.f;
        if (n < a.N && k0 + kk < sg.K) v = a.W[(size_t)n * a.ldw + sg.w_off + (size_t)(k0 + kk) * sg.w_stride];
        Bs[kk][nn] = v;
      }
      __syncthreads();
#pragma unroll
      for (int kk = 0; kk < BK; ++kk) {
        const float4 av = *reinterpret_cast<const float4*>(&As[kk][ty * 4]);
        const float ar[4] = {av.x, av.y, av.z, av.w};
        float br[TN];
#pragma unroll
        for (int j = 0; j < TN; j += 2) {
          const float2 bv = *reinterpret_cast<const float2*>(&Bs[kk][tx * TN + j]);
          br[j] = bv.x;
          br[j + 1] = bv.y;
        }
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int j = 0; j < TN; ++j) acc[i][j] = fmaf(ar[i], br[j], acc[i][j]);
      }
      __syncthreads();
    }
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int m = m0 + ty * 4 + i;
    if (m >= a.M) continue;
#pragma unroll
    for (int j = 0; j < TN; ++j) {
      const int n = n0 + tx * TN + j;
      if (n >= a.N) continue;
      float v = acc[i][j];
      if (a.bias) v += a.bias[n];
      v = act_fn(v, a.act);
      if (a.bn_scale) v = fmaf(v, a.bn_scale[n], a.bn_shift[n]);
      if (a.mask) v = step_mask(a)[(size_t)m * a.N + n] ? v * 2.f : 0.f;
      if (a.res) v += a.res[(size_t)m * a.ldres + n];
      a.Y[(size_t)m * a.ldy + n] = v;
    }
  }
}

// ---- large-M kernel: 128 x 128 tile, 8 x 8 per thread, k-major shared tiles ----------------------
constexpr int LBM = 128, LBN = 128, LBK = 8;

__global__ void __launch_bounds__(256) gemm_big_kernel(const GemmArgs a) {
  __shared__ __align__(16) float As[2][LBK][LBM + 4];
  __shared__ __align__(16) float Bs[2][LBK][LBN + 4];
  const int tid = threadIdx.x;
  const int tx = tid & 15, ty = tid >> 4;   // 16 x 16 threads, each 8 rows x 8 cols (two 4-wide halves)
  const int m0 = blockIdx.y * LBM, n0 = blockIdx.x * LBN;
  float acc[8][8];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;

  // loader mapping: 128 rows x 8 k = 1024 elements per operand -> 4 per thread
  const int lk = tid & 7;        // k within the chunk
  const int lr = tid >> 3;       // 0..31, rows lr + 32*i
  float ra[4], rb[4];

  // flat list of (segment, k0) chunks
  int nchunks = 0;
  for (int s = 0; s < a.nseg; ++s) nchunks += (a.seg[s].K + LBK - 1) / LBK;

  auto load = [&](int chunk) {
    int s = 0, c = chunk;
    while (c >= (a.seg[s].K + LBK - 1) / LBK) {
      c -= (a.seg[s].K + LBK - 1) / LBK;
      ++s;
    }
    Seg sg = a.seg[s];
    if (s == 0) step_seg0(a, sg);
    const int k = c * LBK + lk;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int m = m0 + lr + 32 * i;
      float v = 0.f;
      if (m < a.M && k < sg.K) {
        bool ok = true;
        int row = m;
        if (sg.shift != 0) {
          const int t = m % a.T + sg.shift;
          ok = (t >= 0 && t < a.T);
          row = m + sg.shift;
        }
        if (ok) v = sg.x[(size_t)row * sg.ld + k];
      }
      ra[i] = v;
      const int n = n0 + lr + 32 * i;
      float w = 0.f;
      if (n < a.N && k < sg.K) w = a.W[(size_t)n * a.ldw + sg.w_off + (size_t)k * sg.w_stride];
      rb[i] = w;
    }
  };
  auto stash = [&](int buf) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      As[buf][lk][lr + 32 * i] = ra[i];
      Bs[buf][lk][lr + 32 * i] = rb[i];
    }
  };

  load(0);
  stash(0);
  __syncthreads();
  for (int c = 0; c < nchunks; ++c) {
    const int buf = c & 1;
    if (c + 1 < nchunks) load(c + 1);
#pragma unroll
    for (int kk = 0; kk < LBK; ++kk) {
      const float4 a0 = *reinterpret_cast<const float4*>(&As[buf][kk][ty * 4]);
      const float4 a1 = *reinterpret_cast<const float4*>(&As[buf][kk][64 + ty * 4]);
      const float4 b0 = *reinterpret_cast<const float4*>(&Bs[buf][kk][tx * 4]);
      const float4 b1 = *reinterpret_cast<const float4*>(&Bs[buf][kk][64 + tx * 4]);
      const float ar[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
      const float br[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(ar[i], br[j], acc[i][j]);
    }
    if (c + 1 < nchunks) stash(buf ^ 1);
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int m = m0 + (i < 4 ? ty * 4 + i : 64 + ty * 4 + (i - 4));
    if (m >= a.M) continue;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int n = n0 + (j < 4 ? tx * 4 + j : 64 + tx * 4 + (j - 4));
      if (n >= a.N) continue;
      float v = acc[i][j];
      if (a.bias) v += a.bias[n];
      v = act_fn(v, a.act);
      if (a.bn_scale) v = fmaf(v, a.bn_scale[n], a.bn_shift[n]);
      if (a.mask) v = step_mask(a)[(size_t)m * a.N + n] ? v * 2.f : 0.f;
      if (a.res) v += a.res[(size_t)m * a.ldres + n];
      a.Y[(size_t)m * a.ldy + n] = v;
    }
  }
}

// ---- skinny kernel (M <= 64: decoder step, recurrent h projections): one CTA = all rows x 8 output
// columns, the 8 warps split K and reduce through shared memory -> N/8 CTAs keep every SM busy.
constexpr int SKK = 16;

// CG = column groups of 8 per CTA (1 -> 8 columns, 4 -> 32 columns: fewer re-reads of X for wide N)
template <int CG>
__global__ void __launch_bounds__(256) gemm_skinny_kernel(const GemmArgs a) {
  constexpr int SKN = 8 * CG;
  // Xs [8 warps][SKK][64+4] | Ws [8][SKK][SKN]; the cross-warp reduction buffer aliases Xs afterwards
  extern __shared__ __align__(16) float sm[];
  float (*Xs)[SKK][68] = reinterpret_cast<float (*)[SKK][68]>(sm);
  float (*Ws)[SKK][SKN] = reinterpret_cast<float (*)[SKK][SKN]>(sm + 8 * SKK * 68);
  float (*red)[64][9] = reinterpret_cast<float (*)[64][9]>(sm);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int rt = lane & 15, ct = lane >> 4;  // rows 4*rt.., cols 4*ct.. within a column group
  const int n0 = blockIdx.x * SKN;
  float acc[CG][4][4];
#pragma unroll
  for (int g = 0; g < CG; ++g)
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) acc[g][i][j] = 0.f;

  const int lq = lane & 3, lr = lane >> 2;  // staging: 4 lanes x float4 cover 16 k of a row, 8 rows per pass
  int chunk = 0;
  for (int s = 0; s < a.nseg; ++s) {
    Seg sg = a.seg[s];
    if (s == 0) step_seg0(a, sg);
    const bool vec = ((sg.ld & 3) == 0) && ((sg.K & 3) == 0) && ((reinterpret_cast<uintptr_t>(sg.x) & 15) == 0);
    const bool wvec = (sg.w_stride == 1) && ((a.ldw & 3) == 0) && ((sg.w_off & 3) == 0) && ((sg.K & 3) == 0) &&
                      ((reinterpret_cast<uintptr_t>(a.W) & 15) == 0);
    for (int k0 = 0; k0 < sg.K; k0 += SKK, ++chunk) {
      if ((chunk & 7) != warp) continue;
      const int k = k0 + 4 * lq;
#pragma unroll
      for (int pass = 0; pass < 8; ++pass) {
        const int m = pass * 8 + lr;
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (m < a.M) {
          const float* src = sg.x + (size_t)m * sg.ld + k;
          if (vec && k + 3 < sg.K) v = *reinterpret_cast<const float4*>(src);
          else {
            if (k < sg.K) v.x = src[0];
            if (k + 1 < sg.K) v.y = src[1];
            if (k + 2 < sg.K) v.z = src[2];
            if (k + 3 < sg.K) v.w = src[3];
          }
        }
        Xs[warp][4 * lq + 0][m] = v.x;
        Xs[warp][4 * lq + 1][m] = v.y;
        Xs[warp][4 * lq + 2][m] = v.z;
        Xs[warp][4 * lq + 3][m] = v.w;
      }
#pragma unroll
      for (int pass = 0; pass < CG; ++pass) {
        const int j = pass * 8 + lr;
        const int n = n0 + j;
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (n < a.N) {
          const float* src = a.W + (size_t)n * a.ldw + sg.w_off + (size_t)k * sg.w_stride;
          if (wvec && k + 3 < sg.K) v = *reinterpret_cast<const float4*>(src);
          else {
            if (k < sg.K) v.x = src[0];
            if (k + 1 < sg.K) v.y = src[(size_t)sg.w_stride];
            if (k + 2 < sg.K) v.z = src[(size_t)2 * sg.w_stride];
            if (k + 3 < sg.K) v.w = src[(size_t)3 * sg.w_stride];
          }
        }
        Ws[warp][4 * lq + 0][j] = v.x;
        Ws[warp][4 * lq + 1][j] = v.y;
        Ws[warp][4 * lq + 2][j] = v.z;
        Ws[warp][4 * lq + 3][j] = v.w;
      }
      __syncwarp();
#pragma unroll
      for (int kk = 0; kk < SKK; ++kk) {
        const float4 xv = *reinterpret_cast<const float4*>(&Xs[warp][kk][rt * 4]);
        const float xr[4] = {xv.x, xv.y, xv.z, xv.w};
#pragma unroll
        for (int g = 0; g < CG; ++g) {
          const float4 wv = *reinterpret_cast<const float4*>(&Ws[warp][kk][g * 8 + ct * 4]);
          const float wr[4] = {wv.x, wv.y, wv.z, wv.w};
#pragma unroll
          for (int i = 0; i < 4; ++i)
#pragma unroll
            for (int j = 0; j < 4; ++j) acc[g][i][j] = fmaf(xr[i], wr[j], acc[g][i][j]);
        }
      }
      __syncwarp();
    }
  }
#pragma unroll
  for (int g = 0; g < CG; ++g) {
    __syncthreads();  // Xs (first pass) / the previous group's partials are no longer needed
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) red[warp][rt * 4 + i][ct * 4 + j] = acc[g][i][j];
    __syncthreads();
    for (int o = tid; o < 64 * 8; o += 256) {
      const int m = o >> 3, j = o & 7;
      const int n = n0 + g * 8 + j;
      if (m >= a.M || n >= a.N) continue;
      float v = 0.f;
#pragma unroll
      for (int w = 0; w < 8; ++w) v += red[w][m][j];
      if (a.bias) v += a.bias[n];
      v = act_fn(v, a.act);
      if (a.bn_scale) v = fmaf(v, a.bn_scale[n], a.bn_shift[n]);
      if (a.mask) v = step_mask(a)[(size_t)m * a.N + n] ? v * 2.f : 0.f;
      if (a.res) v += a.res[(size_t)m * a.ldres + n];
      a.Y[(size_t)m * a.ldy + n] = v;
    }
  }
}

// y[m] = act(bias + sum_j x_j[m] . w[off_j : off_j + K_j])  for N == 1 (stop projection): one CTA per row
__global__ void __launch_bounds__(256) rowdot_kernel(const GemmArgs a) {
  __shared__ float red[8];
  const int m = blockIdx.x, tid = threadIdx.x;
  float s = 0.f;
  for (int sgi = 0; sgi < a.nseg; ++sgi) {
    Seg sg = a.seg[sgi];
    if (sgi == 0) step_seg0(a, sg);
    for (int k = tid; k < sg.K; k += 256) s = fmaf(sg.x[(size_t)m * sg.ld + k], a.W[sg.w_off + (size_t)k * sg.w_stride], s);
  }
  for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if ((tid & 31) == 0) red[tid >> 5] = s;
  __syncthreads();
  if (tid == 0) {
    float v = 0.f;
    for (int w = 0; w < 8; ++w) v += red[w];
    if (a.bias) v += a.bias[0];
    a.Y[(size_t)m * a.ldy] = act_fn(v, a.act);
  }
}

__global__ void gru_cell_kernel(const float* __restrict__ gi, int ldgi, const float* __restrict__ gh, float* h, int ldh,
                                float* out2, int ldout2, int M, int H) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= M * H) return;
  const int m = i / H, u = i - m * H;
  const float* a = gi + (size_t)m * ldgi;
  const float* b = gh + (size_t)m * 3 * H;
  const float r = 1.f / (1.f + expf(-(b[u] + a[u])));
  const float z = 1.f / (1.f + expf(-(b[H + u] + a[H + u])));
  const float n = tanhf(a[2 * H + u] + b[2 * H + u] * r);
  const float hv = h[(size_t)m * ldh + u];
  const float hn = (hv - n) * z + n;
  h[(size_t)m * ldh + u] = hn;
  if (out2) out2[(size_t)m * ldout2 + u] = hn;
}

__global__ void lstm_cell_kernel(const float* __restrict__ g, float* c, float* h, float* x, int M, int H) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= M * H) return;
  const int m = i / H, u = i - m * H;
  const float* gg = g + (size_t)m * 4 * H;
  const float ig = 1.f / (1.f + expf(-gg[u]));
  const float fg = 1.f / (1.f + expf(-gg[H + u]));
  const float cg = tanhf(gg[2 * H + u]);
  const float og = 1.f / (1.f + expf(-gg[3 * H + u]));
  const float cn = fg * c[i] + ig * cg;
  const float hn = og * tanhf(cn);
  c[i] = cn;
  h[i] = hn;
  if (x) x[i] = x[i] + hn;
}

__global__ void highway_kernel(const float* __restrict__ x12, float* y, int M, int C) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= M * C) return;
  const int m = i / C, c = i - m * C;
  const float x1 = x12[(size_t)m * 2 * C + c];
  const float x2 = x12[(size_t)m * 2 * C + C + c];
  const float g = 1.f / (1.f + expf(-x2));
  y[i] = g * (x1 > 0.f ? x1 : 0.f) + (1.f - g) * y[i];
}

__global__ void maxpool2_kernel(const float* __restrict__ x, float* __restrict__ y, int B, int T, int C) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)B * T * C) return;
  const int t = (int)((i / C) % T);
  const float v = x[i];
  y[i] = t > 0 ? fmaxf(v, x[i - C]) : v;
}

__global__ void embedding_kernel(const int32_t* __restrict__ ids, const float* __restrict__ table, float* __restrict__ y,
                                 int M, int D) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)M * D) return;
  const int m = (int)(i / D), d = (int)(i - (size_t)m * D);
  y[i] = table[(size_t)ids[m] * D + d];
}

__global__ void copy_cols_kernel(const float* __restrict__ src, int ldsrc, int rows_per_src, float* __restrict__ dst,
                                 int lddst, int off, int M, int n) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)M * n) return;
  const int m = (int)(i / n), j = (int)(i - (size_t)m * n);
  dst[(size_t)m * lddst + off + j] = src[(size_t)(m / rows_per_src) * ldsrc + j];
}

}  // namespace

constexpr int kPrenetRows = 4;     // batch rows per CTA
constexpr int kPrenetWarps = 16;   // 512 threads (128 registers: 8 x 4 accumulators + 16 weights in flight)
constexpr int kPrenetOut = 8;      // outputs per warp and pass: 16 warps x 8 = 128 outputs, two passes per layer

// one dense layer for kPrenetRows rows held in shared memory: out[r][n] = mask(relu(b[n] + W[n][:] . in[r][:])) * 2.
// The kernel is a chain of L2 round trips (16 CTAs read the same 344 KB of weights), so each lane keeps 16 independent weight loads
// in flight (8 outputs x 2 k: 12 dependent round trips per step instead of 22); the per-lane accumulation order (k = lane, lane + 32, ...) is that of the 4-output version.
template <int KMAX>
__device__ __forceinline__ void prenet_layer(const float* __restrict__ W, const float* __restrict__ bias, int K, int H,
                                             const float (*in)[KMAX], const uint8_t* __restrict__ mask, const long long* moff, int b0,
                                             int B, int warp, int lane,
                                             float (*out_s)[256], float* out_g, int ldy, __half* s_hi = nullptr,
                                             __half* s_lo = nullptr, int s_k0 = 0, int s_rows_pad = 0) {
  for (int n0 = warp * kPrenetOut; n0 < H; n0 += kPrenetWarps * kPrenetOut) {
    float acc[kPrenetOut][kPrenetRows];
#pragma unroll
    for (int o = 0; o < kPrenetOut; ++o)
#pragma unroll
      for (int r = 0; r < kPrenetRows; ++r) acc[o][r] = 0.f;
    for (int k = lane; k < K; k += 64) {
      const int k2 = k + 32;
      const bool two = k2 < K;
      float w0[kPrenetOut], w1[kPrenetOut];
#pragma unroll
      for (int o = 0; o < kPrenetOut; ++o) {
        const bool ok = n0 + o < H;
        w0[o] = ok ? W[(size_t)(n0 + o) * K + k] : 0.f;
        w1[o] = (ok && two) ? W[(size_t)(n0 + o) * K + k2] : 0.f;
      }
#pragma unroll
      for (int r = 0; r < kPrenetRows; ++r) {
        const float x0 = in[r][k];
#pragma unroll
        for (int o = 0; o < kPrenetOut; ++o) acc[o][r] = fmaf(w0[o], x0, acc[o][r]);
      }
      if (two) {
#pragma unroll
        for (int r = 0; r < kPrenetRows; ++r) {
          const float x1 = in[r][k2];
#pragma unroll
          for (int o = 0; o < kPrenetOut; ++o) acc[o][r] = fmaf(w1[o], x1, acc[o][r]);
        }
      }
    }
#pragma unroll
    for (int o = 0; o < kPrenetOut; ++o)
#pragma unroll
      for (int r = 0; r < kPrenetRows; ++r)
#pragma unroll
        for (int off = 16; off >= 1; off >>= 1) acc[o][r] += __shfl_xor_sync(0xffffffffu, acc[o][r], off);
    {
      const int o = lane >> 2, r = lane & 3;  // kPrenetOut * kPrenetRows == 32: one (output, row) per lane
      float v = 0.f;
#pragma unroll
      for (int oo = 0; oo < kPrenetOut; ++oo)
#pragma unroll
        for (int rr = 0; rr < kPrenetRows; ++rr) v = (oo == o && rr == r) ? acc[oo][rr] : v;
      const int n = n0 + o, b = b0 + r;
      if (n < H) {
        v += bias[n];
        v = v > 0.f ? v : 0.f;
        if (b < B) v = mask[(moff ? moff[r] : 0) + (long long)b * H + n] ? v * 2.f : 0.f;
        if (out_s) out_s[r][n] = v;
        if (out_g && b < B) out_g[(size_t)b * ldy + n] = v;
        if (s_hi && b < B) store_split_scalar(v, b, s_rows_pad, s_k0 + n, s_hi, s_lo);
      }
    }
  }
}

__global__ void __launch_bounds__(32 * kPrenetWarps) prenet_fused_kernel(const PrenetArgs a) {
  __shared__ float xs[kPrenetRows][128];
  __shared__ float hs[kPrenetRows][256];
  const int b0 = blockIdx.x * kPrenetRows;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int si = step_index(a.step_ptr, a.step_j);
  // with a per-row step origin each row reads at its own step (row_step): the go frame at its step 0, else the last frame of its
  // previous step, and the masks of its step; without one every row is at step si
  const bool per_row = a.row_start != nullptr;
  __shared__ long long moff[kPrenetRows];
  if (per_row && threadIdx.x < kPrenetRows) {
    const int b = b0 + threadIdx.x;
    moff[threadIdx.x] = b < a.B ? (long long)ring_slot(row_step(si, a.row_start, b), a.row_start, a.ring) * a.mask_step : 0;
  }
  const bool go = (si == 0 && a.x_first != nullptr);
  for (int i = threadIdx.x; i < kPrenetRows * a.K; i += blockDim.x) {
    const int r = i / a.K, k = i - r * a.K;
    const int b = b0 + r;
    float v = 0.f;
    if (b < a.B && !per_row) {
      v = go ? a.x_first[k] : a.x[(long long)b * a.x_ld + (long long)si * a.x_step + k];
    } else if (b < a.B) {
      const int s = row_step(si, a.row_start, b);
      // x + s * x_step is frame s * r - 1; in a ring, step s - 1's frames sit at slot (s - 1) % ring
      v = (s == 0 && a.x_first != nullptr) ? a.x_first[k] : a.x[(long long)b * a.x_ld + ((long long)((s - 1) % a.ring) + 1) * a.x_step + k];
    }
    xs[r][k] = v;
  }
  __syncthreads();
  const uint8_t* m1 = per_row ? a.m1 : a.m1 + (size_t)si * (size_t)a.mask_step;
  const uint8_t* m2 = per_row ? a.m2 : a.m2 + (size_t)si * (size_t)a.mask_step;
  prenet_layer<128>(a.W1, a.b1, a.K, a.H, xs, m1, per_row ? moff : nullptr, b0, a.B, warp, lane, hs, nullptr, 0);
  __syncthreads();
  prenet_layer<256>(a.W2, a.b2, a.H, a.H, hs, m2, per_row ? moff : nullptr, b0, a.B, warp, lane, nullptr, a.y, a.ldy, a.s_hi, a.s_lo, a.s_k0, a.s_rows_pad);
}

cudaError_t launch_prenet_fused(const PrenetArgs& a, cudaStream_t st) {
  if (a.K > 128 || a.H > 256 || a.B <= 0 || (a.row_start && a.ring <= 0)) return cudaErrorInvalidValue;
  prenet_fused_kernel<<<(a.B + kPrenetRows - 1) / kPrenetRows, 32 * kPrenetWarps, 0, st>>>(a);
  return cudaGetLastError();
}

cudaError_t launch_gemm(const GemmArgs& a, cudaStream_t st, GemmLaunchInfo* info) {
  if (a.M <= 0 || a.N <= 0) return cudaSuccess;
  bool shifted = false;
  for (int s = 0; s < a.nseg; ++s) shifted = shifted || a.seg[s].shift != 0;
  auto note = [&](const char* k, dim3 grid, size_t smem) {
    if (info) *info = GemmLaunchInfo{k, (int)grid.x, (int)grid.y, 256, smem};
  };
  if (a.N == 1 && !shifted && !a.mask && !a.res && !a.bn_scale && !a.fma_chain) {
    note("rowdot", dim3(a.M), 0);
    rowdot_kernel<<<a.M, 256, 0, st>>>(a);
    return cudaGetLastError();
  }
  if (a.M <= 64 && !shifted && !a.fma_chain) {
    if (a.N >= 2048) {
      constexpr size_t smem = sizeof(float) * (8 * SKK * 68 + 8 * SKK * 32);
      static bool attr = false;
      if (!attr) {
        cudaFuncSetAttribute(gemm_skinny_kernel<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        attr = true;
      }
      note("gemm_skinny4", dim3((a.N + 31) / 32), smem);
      gemm_skinny_kernel<4><<<(a.N + 31) / 32, 256, smem, st>>>(a);
    } else {
      constexpr size_t smem = sizeof(float) * (8 * SKK * 68 + 8 * SKK * 8);
      note("gemm_skinny1", dim3((a.N + 7) / 8), smem);
      gemm_skinny_kernel<1><<<(a.N + 7) / 8, 256, smem, st>>>(a);
    }
    return cudaGetLastError();
  }
  if (a.M >= 1024 && a.N >= 128) {
    dim3 grid((a.N + LBN - 1) / LBN, (a.M + LBM - 1) / LBM);
    note("gemm_big", grid, 0);
    gemm_big_kernel<<<grid, 256, 0, st>>>(a);
    return cudaGetLastError();
  }
  // small-M (decoder step) problems: narrower N tiles -> more CTAs
  if (a.M <= 128 && a.N >= 512) {
    dim3 grid((a.N + 31) / 32, (a.M + BM - 1) / BM);
    note("gemm32", grid, 0);
    gemm_kernel<32><<<grid, 256, 0, st>>>(a);
  } else {
    dim3 grid((a.N + 63) / 64, (a.M + BM - 1) / BM);
    note("gemm64", grid, 0);
    gemm_kernel<64><<<grid, 256, 0, st>>>(a);
  }
  return cudaGetLastError();
}

cudaError_t launch_gru_cell(const float* gi, int ldgi, const float* gh, float* h, int ldh, float* out2, int ldout2,
                            int M, int H, cudaStream_t st) {
  gru_cell_kernel<<<(M * H + 255) / 256, 256, 0, st>>>(gi, ldgi, gh, h, ldh, out2, ldout2, M, H);
  return cudaGetLastError();
}

cudaError_t launch_lstm_cell(const float* g, float* c, float* h, float* x, int M, int H, cudaStream_t st) {
  lstm_cell_kernel<<<(M * H + 255) / 256, 256, 0, st>>>(g, c, h, x, M, H);
  return cudaGetLastError();
}

cudaError_t launch_highway(const float* x12, float* y, int M, int C, cudaStream_t st) {
  highway_kernel<<<(unsigned)(((size_t)M * C + 255) / 256), 256, 0, st>>>(x12, y, M, C);
  return cudaGetLastError();
}

cudaError_t launch_maxpool2(const float* x, float* y, int B, int T, int C, cudaStream_t st) {
  maxpool2_kernel<<<(unsigned)(((size_t)B * T * C + 255) / 256), 256, 0, st>>>(x, y, B, T, C);
  return cudaGetLastError();
}

cudaError_t launch_embedding(const int32_t* ids, const float* table, float* y, int M, int D, cudaStream_t st) {
  embedding_kernel<<<(unsigned)(((size_t)M * D + 255) / 256), 256, 0, st>>>(ids, table, y, M, D);
  return cudaGetLastError();
}

cudaError_t launch_copy_cols(const float* src, int ldsrc, int rows_per_src, float* dst, int lddst, int off, int M,
                             int n, cudaStream_t st) {
  copy_cols_kernel<<<(unsigned)(((size_t)M * n + 255) / 256), 256, 0, st>>>(src, ldsrc, rows_per_src, dst, lddst, off, M, n);
  return cudaGetLastError();
}

}  // namespace taco
}  // namespace mb
