// FP32 FFMA implementation of the tap-conv op: the parity anchor of the GAN path (MB_PREC_FP32)
// and the executor of the few layers the tensor-core path keeps in FP32 (conv_pre: Cin=80,
// conv_post: Cout=1).  Register-tiled direct convolution, 64(co) x 64(l) output tile per CTA,
// 4x4 per thread, input window and weight slabs staged through shared memory in chunks of 8
// input channels.  Reference semantics: hifigan/models.py:35-42, :134-150;
// fregan/generator.py:137-166.
#include <cstdlib>

#include "gan_kernels.h"

namespace mb {

namespace {

constexpr int CO_T = 64;
constexpr int L_T = 64;
constexpr int CI_T = 8;
constexpr int XW_MAX = L_T + 96;  // window: tile + tap span (70 for k=11,d=7 in Fre-GAN)

__device__ __forceinline__ float lrelu(float v, float slope) { return v > 0.f ? v : v * slope; }

__device__ __forceinline__ float tload(const TRef& t, int b, int c, int l) {
  const size_t i = tref_index(t, b, c, l);
  if (t.layout == LAYOUT_F16B) return __half2float(reinterpret_cast<const __half*>(t.p)[i]);
  return reinterpret_cast<const float*>(t.p)[i];
}

__device__ __forceinline__ void tstore(const TRef& t, int b, int c, int l, float v) {
  const size_t i = tref_index(t, b, c, l);
  if (t.layout == LAYOUT_F16B) {
    const __half h = __float2half_rn(v);
    reinterpret_cast<__half*>(t.p)[i] = h;
    if (t.hilo) reinterpret_cast<__half*>(t.p)[tref_index(t, b, c + (t.C >> 1), l)] = __float2half_rn(v - __half2float(h));
  } else {
    reinterpret_cast<float*>(t.p)[i] = v;
  }
}

// shared epilogue of both FP32 kernels
__device__ __forceinline__ void epilogue_store(const TapConv& p, const TapConvIO& io, int b, int co, int lo,
                                               int valid_out, float v) {
  if (io.res.p) v += tload(io.res, b, co, lo);
  if (p.mode == EPI_ADD) v = tload(io.y32, b, co, lo) + v;
  else if (p.mode == EPI_ADD_DIV) v = (tload(io.y32, b, co, lo) + v) / p.div;
  if (p.act_tanh) v = tanhf(v);
  if (lo >= valid_out) v = 0.f;
  if (io.y32.p) tstore(io.y32, b, co, lo, v);
  if (io.y16.p) tstore(io.y16, b, co, lo, lrelu(v, io.out16_slope));
  if (io.y2_32.p) {
    const float s = (lo >= valid_out) ? 0.f : tload(io.y2_32, b, co, lo) + v;
    tstore(io.y2_32, b, co, lo, s);
    if (io.y2_16.p) tstore(io.y2_16, b, co, lo, lrelu(s, io.y2_16_slope));
  }
}

__global__ void __launch_bounds__(256) tapconv_f32_kernel(TapConv p, TapConvIO io, const float* __restrict__ w,
                                                          const float* __restrict__ bias) {
  __shared__ float xs[CI_T][XW_MAX];
  __shared__ __align__(16) float ws[kMaxTaps][CI_T][CO_T];

  const int tid = threadIdx.x;
  const int tx = tid & 15;   // l lane
  const int ty = tid >> 4;   // co group (4 channels)
  const int q0 = blockIdx.x * L_T;
  const int co0 = blockIdx.y * CO_T;
  const int b = blockIdx.z / p.stride;
  const int r = blockIdx.z % p.stride;

  const int nt = p.ntaps[r];
  int omin = 0x7fffffff, omax = -0x7fffffff;
  for (int t = 0; t < nt; ++t) {
    omin = min(omin, p.off[r][t]);
    omax = max(omax, p.off[r][t]);
  }
  const int XW = L_T + (omax - omin);
  const int valid_in = p.lengths ? min(p.Lin, p.lengths[b] * p.len_mul_in) : p.Lin;
  const int valid_out = p.lengths ? min(p.Lout, p.lengths[b] * p.len_mul_out) : p.Lout;
  const float in_slope = (io.x.layout == LAYOUT_F16B) ? 1.f : p.in_slope;

  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

  for (int ci0 = 0; ci0 < p.Cin; ci0 += CI_T) {
    // stage input window (activation applied once here)
    for (int i = tid; i < CI_T * XW; i += 256) {
      const int ci = i / XW, j = i - ci * XW;
      const int l = q0 + omin + j;
      float v = 0.f;
      if (ci0 + ci < p.Cin && l >= 0 && l < valid_in) v = lrelu(tload(io.x, b, ci0 + ci, l), in_slope);
      xs[ci][j] = v;
    }
    // stage weight slabs
    for (int i = tid; i < nt * CI_T * CO_T; i += 256) {
      const int t = i / (CI_T * CO_T);
      const int rem = i - t * (CI_T * CO_T);
      const int ci = rem / CO_T, co = rem - ci * CO_T;
      float v = 0.f;
      if (ci0 + ci < p.Cin && co0 + co < p.Cout)
        v = w[((size_t)p.slab[r][t] * p.Cin + (ci0 + ci)) * p.Cout + co0 + co];
      ws[t][ci][co] = v;
    }
    __syncthreads();
    for (int t = 0; t < nt; ++t) {
      const int o = p.off[r][t] - omin;
#pragma unroll
      for (int ci = 0; ci < CI_T; ++ci) {
        const float4 wv = *reinterpret_cast<const float4*>(&ws[t][ci][ty * 4]);
        float xv[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) xv[j] = xs[ci][tx + 16 * j + o];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          acc[0][j] = fmaf(wv.x, xv[j], acc[0][j]);
          acc[1][j] = fmaf(wv.y, xv[j], acc[1][j]);
          acc[2][j] = fmaf(wv.z, xv[j], acc[2][j]);
          acc[3][j] = fmaf(wv.w, xv[j], acc[3][j]);
        }
      }
    }
    __syncthreads();
  }

#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int co = co0 + ty * 4 + i;
    if (co >= p.Cout) continue;
    const float bv = bias ? bias[co] : 0.f;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int q = q0 + tx + 16 * j;
      if (q >= p.Lin) continue;
      epilogue_store(p, io, b, co, q * p.stride + r, valid_out, acc[i][j] + bv);
    }
  }
}

// Cout == 1 (conv_post): weights [taps][Cin] in shared memory; a thread produces R consecutive output rows.  R = 1: every
// load of a warp is 32 consecutive 16-byte quads (fully coalesced; the k-fold re-reads of a row by neighbouring threads are L1
// hits); R = 4 (round 1): fewer L1 reads but a 64-byte lane stride.  Per-output accumulation order is the same for every R.
template <int R>
__global__ void __launch_bounds__(256) tapconv_cout1_kernel(TapConv p, TapConvIO io, const float* __restrict__ w,
                                                            const float* __restrict__ bias) {
  extern __shared__ float wsm[];  // [ntaps][Cin]
  const int b = blockIdx.y;
  const int nt = p.ntaps[0];
  for (int i = threadIdx.x; i < nt * p.Cin; i += blockDim.x) {
    const int t = i / p.Cin, ci = i - t * p.Cin;
    wsm[i] = w[((size_t)p.slab[0][t] * p.Cin + ci) * p.Cout];
  }
  __syncthreads();
  const int l0 = (blockIdx.x * blockDim.x + threadIdx.x) * R;
  if (l0 >= p.Lin) return;
  const int valid_in = p.lengths ? min(p.Lin, p.lengths[b] * p.len_mul_in) : p.Lin;
  const int valid_out = p.lengths ? min(p.Lout, p.lengths[b] * p.len_mul_out) : p.Lout;
  const float in_slope = (io.x.layout == LAYOUT_F16B) ? 1.f : p.in_slope;
  float acc[R];
#pragma unroll
  for (int i = 0; i < R; ++i) acc[i] = 0.f;
  // contiguous tap offsets off[t] = t - pad (dilation 1) let us walk input rows once
  const int o0 = p.off[0][0];
  bool contiguous = true;
  for (int t = 1; t < nt; ++t) contiguous = contiguous && (p.off[0][t] == o0 + t);
  if (io.x.layout == LAYOUT_F32B && contiguous) {
    const float4* xp = reinterpret_cast<const float4*>(io.x.p);
    for (int c4 = 0; c4 < (p.Cin >> 2); ++c4) {
      const float4* run = xp + ((size_t)b * (p.Cin >> 2) + c4) * p.Lin;
      for (int j = 0; j < nt + R - 1; ++j) {   // input row l0 + o0 + j feeds output i with tap t = j - i
        const int li = l0 + o0 + j;
        if (li < 0 || li >= valid_in) continue;
        float4 v = run[li];
        v.x = lrelu(v.x, in_slope); v.y = lrelu(v.y, in_slope); v.z = lrelu(v.z, in_slope); v.w = lrelu(v.w, in_slope);
#pragma unroll
        for (int i = 0; i < R; ++i) {
          const int t = j - i;
          if (t < 0 || t >= nt) continue;
          const float* wt = &wsm[t * p.Cin + c4 * 4];
          acc[i] = fmaf(wt[0], v.x, acc[i]);
          acc[i] = fmaf(wt[1], v.y, acc[i]);
          acc[i] = fmaf(wt[2], v.z, acc[i]);
          acc[i] = fmaf(wt[3], v.w, acc[i]);
        }
      }
    }
  } else {
    for (int ci = 0; ci < p.Cin; ++ci)
      for (int t = 0; t < nt; ++t)
        for (int i = 0; i < R; ++i) {
          const int li = l0 + i + p.off[0][t];
          if (li < 0 || li >= valid_in) continue;
          acc[i] = fmaf(wsm[t * p.Cin + ci], lrelu(tload(io.x, b, ci, li), in_slope), acc[i]);
        }
  }
  for (int i = 0; i < R; ++i)
    if (l0 + i < p.Lin) epilogue_store(p, io, b, 0, l0 + i, valid_out, acc[i] + (bias ? bias[0] : 0.f));
}

// Cout == 1, shared-memory tile version (conv_post of the F32B plane, taps contiguous, Cin % 4 == 0).  The R-rows-per-thread kernel
// above applies the input leaky-relu once per (thread, row) - (nt + R - 1) / R times per element - and is bound by those instructions and
// its L1 reads (0.099 ms for 210 MB).  Here a block of 128 threads stages kPostTile + nt - 1 activated rows of all channel quads once
// (coalesced 16-byte loads, leaky-relu applied once, rows outside the utterance = 0), then every thread produces 4 CONSECUTIVE outputs
// from 10 rows per quad.  The tile is stored as four row planes (row r -> plane r & 3, slot r >> 2) so that the lanes of a warp, whose
// first rows are 4 apart, read consecutive 16-byte slots.  Accumulation order per output = the order of the kernel above (channel quad,
// tap, channel), so results are bit-identical; a masked row contributes fma(w, 0, acc) = acc.
constexpr int kPostTile = 512;  // output rows per block (128 threads x 4)
template <int NT, int CQ>  // CQ = Cin / 4 channel quads (compile time: the staging loop keeps CQ independent 16-byte loads in flight per thread)
__global__ void __launch_bounds__(128) convpost_tile_kernel(TapConv p, TapConvIO io, const float* __restrict__ w,
                                                            const float* __restrict__ bias) {
  extern __shared__ __align__(16) float psm[];
  constexpr int C4 = CQ;
  constexpr int SLOTS = kPostTile / 4 + 2;           // slots per plane (rows r >> 2, r < kPostTile + NT - 1 <= kPostTile + 8)
  float* wsm = psm;                                   // [NT][Cin]
  float4* tile = reinterpret_cast<float4*>(psm + ((NT * p.Cin + 3) & ~3));  // [C4][4][SLOTS]
  const int b = blockIdx.y, tid = threadIdx.x;
  for (int i = tid; i < NT * p.Cin; i += 128) {
    const int t = i / p.Cin, ci = i - t * p.Cin;
    wsm[i] = w[((size_t)p.slab[0][t] * p.Cin + ci) * p.Cout];
  }
  const int l_blk = blockIdx.x * kPostTile;
  const int o0 = p.off[0][0];
  const int valid_in = p.lengths ? min(p.Lin, p.lengths[b] * p.len_mul_in) : p.Lin;
  const int valid_out = p.lengths ? min(p.Lout, p.lengths[b] * p.len_mul_out) : p.Lout;
  const float4* xp = reinterpret_cast<const float4*>(io.x.p) + (size_t)b * C4 * p.Lin;
  const int rows = kPostTile + NT - 1;
  for (int r = tid; r < rows; r += 128) {
    const int li = l_blk + o0 + r;
    const bool ok = (li >= 0 && li < valid_in);
    float4 v[CQ];
#pragma unroll
    for (int q = 0; q < CQ; ++q) v[q] = ok ? xp[(size_t)q * p.Lin + li] : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int q = 0; q < CQ; ++q) {
      float4 a = v[q];
      a.x = lrelu(a.x, p.in_slope); a.y = lrelu(a.y, p.in_slope); a.z = lrelu(a.z, p.in_slope); a.w = lrelu(a.w, p.in_slope);
      tile[((size_t)q * 4 + (r & 3)) * SLOTS + (r >> 2)] = a;
    }
  }
  __syncthreads();
  float acc[4] = {0.f, 0.f, 0.f, 0.f};
  for (int q = 0; q < C4; ++q) {
    float4 x[NT + 3];
#pragma unroll
    for (int j = 0; j < NT + 3; ++j) x[j] = tile[((size_t)q * 4 + (j & 3)) * SLOTS + tid + (j >> 2)];  // row 4 * tid + j
    float4 wt[NT];
#pragma unroll
    for (int t = 0; t < NT; ++t) wt[t] = *reinterpret_cast<const float4*>(&wsm[t * p.Cin + q * 4]);
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int t = 0; t < NT; ++t) {
        acc[i] = fmaf(wt[t].x, x[i + t].x, acc[i]);
        acc[i] = fmaf(wt[t].y, x[i + t].y, acc[i]);
        acc[i] = fmaf(wt[t].z, x[i + t].z, acc[i]);
        acc[i] = fmaf(wt[t].w, x[i + t].w, acc[i]);
      }
  }
  const float bv = bias ? bias[0] : 0.f;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int l = l_blk + 4 * tid + i;
    if (l < p.Lin) epilogue_store(p, io, b, 0, l, valid_out, acc[i] + bv);
  }
}

__global__ void add_inplace_kernel(TRef dst32, TRef src32, TRef dst16, float slope, int B) {
  const size_t n = (size_t)B * dst32.C * dst32.L;
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  float* d = reinterpret_cast<float*>(dst32.p);
  const float* s = reinterpret_cast<const float*>(src32.p);
  for (; i < n; i += stride) {
    const float v = d[i] + s[i];
    d[i] = v;
    if (dst16.p) {
      // decode (b, c, l) from the fp32 layout's linear index
      int b, c, l;
      if (dst32.layout == LAYOUT_NCL) {
        l = (int)(i % dst32.L);
        c = (int)((i / dst32.L) % dst32.C);
        b = (int)(i / ((size_t)dst32.L * dst32.C));
      } else {
        const int e = (int)(i & 3);
        const size_t j = i >> 2;
        l = (int)(j % dst32.L);
        const size_t g = j / dst32.L;
        c = (int)(g % (dst32.C >> 2)) * 4 + e;
        b = (int)(g / (dst32.C >> 2));
      }
      tstore(dst16, b, c, l, lrelu(v, slope));
    }
  }
}

__global__ void zero_pads_kernel(TRef plane, int B) {
  // one thread per (run, pad row, 16-byte chunk)
  const int cw = f16_cw(plane.C);
  const int Lp = f16_lp(plane.L);
  const int npad = Lp - plane.L;            // kPadRows in front, the rest behind
  const int cpr = cw >> 3;                  // 16-byte chunks per row
  const size_t runs = (size_t)B * (plane.C / cw);
  const size_t n = runs * npad * cpr;
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int ch = (int)(i % cpr);
  const size_t j = i / cpr;
  const size_t run = j / npad;
  const int pr = (int)(j % npad);
  const int row = pr < kPadRows ? pr : plane.L + pr;
  uint4* ptr = reinterpret_cast<uint4*>(plane.p) + (run * Lp + row) * cpr + ch;
  *ptr = make_uint4(0, 0, 0, 0);
}

__global__ void convert_layout_kernel(TRef src, TRef dst, int B, float slope) {
  const size_t n = (size_t)B * src.C * src.L;
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int l = (int)(i % src.L);
  const int c = (int)((i / src.L) % src.C);
  const int b = (int)(i / ((size_t)src.L * src.C));
  tstore(dst, b, c, l, lrelu(tload(src, b, c, l), slope));
}

// dst slabs are [K][Cin_p][Cout_p] (Cin_p >= Cin, Cout_p >= Cout: zero-padded channels, the caller clears dst first)
__global__ void pack_slabs_kernel(const float* __restrict__ w, float* __restrict__ dst, int Cout, int Cin,
                                  int K, int transposed, int Cout_p, int Cin_p) {
  const size_t n = (size_t)Cout * Cin * K;
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int co = (int)(i % Cout);
  const int ci = (int)((i / Cout) % Cin);
  const int k = (int)(i / ((size_t)Cout * Cin));
  const size_t src = transposed ? ((size_t)ci * Cout + co) * K + k : ((size_t)co * Cin + ci) * K + k;
  dst[((size_t)k * Cin_p + ci) * Cout_p + co] = w[src];
}

}  // namespace

cudaError_t launch_tapconv_f32(const TapConv& p, const TapConvIO& io, const float* w, const float* bias,
                               cudaStream_t stream) {
  dim3 grid((p.Lin + L_T - 1) / L_T, (p.Cout + CO_T - 1) / CO_T, p.B * p.stride);
  tapconv_f32_kernel<<<grid, 256, 0, stream>>>(p, io, w, bias);
  return cudaGetLastError();
}

cudaError_t launch_tapconv_cout1_f32(const TapConv& p, const TapConvIO& io, const float* w, const float* bias,
                                     cudaStream_t stream) {
  if (p.Cout != 1 || p.stride != 1) return cudaErrorInvalidValue;
  {
    // MB_POST_TILE=1: shared-memory tile kernel for the F32B plane with 7 contiguous taps (conv_post of both generators).  Default 0:
    // bit-identical output but MEASURED SLOWER than the R-rows-per-thread kernel (0.123 vs 0.099 ms; 0.191 ms before the staging loads
    // were batched eight per thread): three 67 KB blocks per SM alternate between a load phase and a compute phase and keep fewer bytes in
    // flight than 2048 resident threads that simply re-read their rows through L1.
    static const bool tile_on = [] {
      const char* e = getenv("MB_POST_TILE");
      return e ? atoi(e) != 0 : false;
    }();
    const int nt = p.ntaps[0];
    bool contiguous = true;
    for (int t = 1; t < nt; ++t) contiguous = contiguous && (p.off[0][t] == p.off[0][0] + t);
    if (tile_on && nt == 7 && contiguous && io.x.layout == LAYOUT_F32B && (p.Cin == 32 || p.Cin == 16)) {
      const size_t smem = sizeof(float) * (((size_t)nt * p.Cin + 3) & ~(size_t)3) +
                          sizeof(float4) * (size_t)(p.Cin >> 2) * 4 * (kPostTile / 4 + 2);
      static bool attr = false;
      if (!attr) {
        cudaError_t e = cudaFuncSetAttribute(convpost_tile_kernel<7, 8>, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024);
        if (e == cudaSuccess) e = cudaFuncSetAttribute(convpost_tile_kernel<7, 4>, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024);
        if (e != cudaSuccess) return e;
        attr = true;
      }
      dim3 grid((p.Lin + kPostTile - 1) / kPostTile, p.B);
      if (p.Cin == 32) convpost_tile_kernel<7, 8><<<grid, 128, smem, stream>>>(p, io, w, bias);
      else convpost_tile_kernel<7, 4><<<grid, 128, smem, stream>>>(p, io, w, bias);
      return cudaGetLastError();
    }
  }
  static const int rows = [] {
    const char* e = getenv("MB_POST_ROWS");  // A/B switch: 1, 2 (default: measured fastest, 0.099 vs 0.127 / 0.122 ms) or 4 output rows per thread
    const int r = e ? atoi(e) : 2;
    return (r == 2 || r == 4) ? r : 1;
  }();
  dim3 grid((p.Lin + 256 * rows - 1) / (256 * rows), p.B);
  const size_t smem = sizeof(float) * p.ntaps[0] * p.Cin;
  if (rows == 4) tapconv_cout1_kernel<4><<<grid, 256, smem, stream>>>(p, io, w, bias);
  else if (rows == 2) tapconv_cout1_kernel<2><<<grid, 256, smem, stream>>>(p, io, w, bias);
  else tapconv_cout1_kernel<1><<<grid, 256, smem, stream>>>(p, io, w, bias);
  return cudaGetLastError();
}

cudaError_t launch_add_inplace_f32(const TRef& dst32, const TRef& src32, const TRef& dst16, float slope, int B,
                                   cudaStream_t stream) {
  const size_t n = (size_t)B * dst32.C * dst32.L;
  const int threads = 256;
  size_t blocks = (n + threads - 1) / threads;
  if (blocks > 132 * 16) blocks = 132 * 16;
  if (blocks == 0) return cudaSuccess;
  add_inplace_kernel<<<(unsigned)blocks, threads, 0, stream>>>(dst32, src32, dst16, slope, B);
  return cudaGetLastError();
}

cudaError_t launch_zero_pads_f16(const TRef& plane, int B, cudaStream_t stream) {
  const size_t n = (size_t)B * (plane.C >> 3) * (f16_lp(plane.L) - plane.L);
  if (n == 0) return cudaSuccess;
  zero_pads_kernel<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(plane, B);
  return cudaGetLastError();
}

cudaError_t launch_convert_layout(const TRef& src, const TRef& dst, int B, float slope, cudaStream_t stream) {
  const size_t n = (size_t)B * src.C * src.L;
  if (n == 0) return cudaSuccess;
  convert_layout_kernel<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(src, dst, B, slope);
  return cudaGetLastError();
}

cudaError_t launch_pack_slabs_f32(const float* w, float* dst, int Cout, int Cin, int K, bool transposed,
                                  cudaStream_t stream, int Cout_p, int Cin_p) {
  const size_t n = (size_t)Cout * Cin * K;
  if (Cout_p < Cout) Cout_p = Cout;
  if (Cin_p < Cin) Cin_p = Cin;
  if (Cout_p != Cout || Cin_p != Cin) {
    cudaError_t e = cudaMemsetAsync(dst, 0, sizeof(float) * (size_t)K * Cin_p * Cout_p, stream);
    if (e != cudaSuccess) return e;
  }
  pack_slabs_kernel<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(w, dst, Cout, Cin, K, transposed ? 1 : 0, Cout_p, Cin_p);
  return cudaGetLastError();
}

}  // namespace mb
