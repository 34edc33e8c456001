// Implicit-GEMM Conv2d on the tensor cores (sm_90a wgmma), FP32-equivalent by the 3-term fp16 split: the PPG extractor's
// embed.conv.2 (Conformer Conv2dNoSubsampling / Conv2dSubsampling, 71 % of the extractor's MACs at the stand-in config).
//
//   grid      : blockIdx.x = 128 output pixels (b, t, f), blockIdx.y = NT output channels
//   operands  : per k-block of 64 (8 channels of one tap per 16-byte chunk, C % 8 == 0) every thread gathers 4 pixel rows x
//               1 chunk of the activation hi / lo tiles with zero-filling cp.async, and a slice of the packed weight tiles;
//               shared-memory tiles are K-major SWIZZLE_128B (chunk c of row r at c ^ (r & 7)), as in tacotron_tc.cu
//   pipeline  : kStages-deep cp.async ring, two MMA warpgroups of 64 pixel rows; 12 wgmmas per k-block (4 k16 steps x 3
//               split terms) into one M64 x NT accumulator per warpgroup
//   epilogue  : bias, ReLU, split into the next GEMM's operand tiles straight from the accumulator registers
#include <cuda_fp16.h>

#include "gan_tc_dev.cuh"
#include "ppgx_kernels.cuh"
#include "ppgx_wgmma.cuh"
#include "tacotron_kernels.cuh"

namespace mb {
namespace ppgx {

namespace {

using namespace tcdev;

constexpr int kStages = 3;
constexpr uint32_t kATile = 16384;  // 128 rows x 128 B

__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src, uint32_t src_bytes) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(src_bytes) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }
// cp.async writes are generic-proxy writes; wgmma reads shared memory through the async proxy
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

template <int NT>
__device__ __forceinline__ void mma_nt(float (&d)[NT / 2], uint64_t a, uint64_t b, uint32_t acc) {
  if constexpr (NT == 144) wgmma_m64n144k16(d, a, b, acc);
  else wgmma_f16<NT>(d, a, b, acc);
}

template <int NT>
__host__ __device__ constexpr uint32_t stage_bytes() { return 2 * kATile + 2 * (uint32_t)NT * 128u; }

template <int NT>
__global__ void __launch_bounds__(256, 1) conv2d_tc_kernel(const __grid_constant__ Conv2dTcArgs p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  constexpr uint32_t kW = (uint32_t)NT * 128u, kStage = stage_bytes<NT>();
  const int tid = threadIdx.x;
  const int TF = p.T_out * p.F_out;
  const int M = p.B * TF;
  const int m0 = blockIdx.x * 128;
  const int ntile = blockIdx.y;
  const int j = tid & 7;  // the 16-byte chunk (8 channels) this thread gathers in every k-block

  // the 4 pixel rows this thread gathers: r = (tid >> 3) + 32 i
  int rbase[4], ti0[4], fi0[4], rlen[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int m = m0 + (tid >> 3) + 32 * i;
    rlen[i] = 0;
    rbase[i] = ti0[i] = fi0[i] = 0;
    if (m < M) {
      const int b = m / TF, rem = m - b * TF;
      const int t = rem / p.F_out, f = rem - t * p.F_out;
      rbase[i] = b * p.T_in;
      ti0[i] = t * p.stride - p.pad;
      fi0[i] = f * p.stride - p.pad;
      rlen[i] = p.len_in[b];
    }
  }
  const uint8_t* wimg = reinterpret_cast<const uint8_t*>(p.w) + (size_t)ntile * p.KB * 2 * kW;

  auto load = [&](int kb, int s) {
    const uint32_t st = smem_u32(smem + (size_t)s * kStage);
    const int k0 = kb * 64 + 8 * j;
    const bool kv = k0 < p.K;
    const int tap = kv ? k0 / p.C : 0;
    const int c0 = k0 - tap * p.C;
    const int dt = tap / p.kw, df = tap - dt * p.kw;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int r = (tid >> 3) + 32 * i;
      const int ti = ti0[i] + dt, fi = fi0[i] + df;
      const bool ok = kv && ti >= 0 && ti < rlen[i] && fi >= 0 && fi < p.F_in;
      const size_t off = ok ? ((size_t)(rbase[i] + ti) * p.F_in + fi) * p.C + c0 : 0;
      const uint32_t dst = st + (uint32_t)r * 128u + (uint32_t)((j ^ (r & 7)) * 16);
      cp_async16(dst, p.x_hi + off, ok ? 16u : 0u);
      cp_async16(dst + kATile, p.x_lo + off, ok ? 16u : 0u);
    }
    const uint8_t* ws = wimg + (size_t)kb * 2 * kW;
    for (int c = tid; c < (int)(2 * kW / 16); c += 256) cp_async16(st + 2 * kATile + (uint32_t)c * 16u, ws + (size_t)c * 16, 16u);
  };

#pragma unroll
  for (int s = 0; s < kStages - 1; ++s) {
    if (s < p.KB) load(s, s);
    cp_async_commit();
  }
  const int g = tid >> 7;  // warpgroup: pixel rows [64 g, 64 g + 64)
  const uint64_t desc0 = make_desc(0, 1024u, 1u, 0);
  float acc[NT / 2];
#pragma unroll
  for (int i = 0; i < NT / 2; ++i) acc[i] = 0.f;
  for (int kb = 0; kb < p.KB; ++kb) {
    const int nk = kb + kStages - 1;
    if (nk < p.KB) load(nk, nk % kStages);
    cp_async_commit();
    cp_async_wait<kStages - 1>();
    fence_proxy_async();
    __syncthreads();
    const uint32_t base = smem_u32(smem + (size_t)(kb % kStages) * kStage);
    const uint64_t ah = desc0 + (uint64_t)((base + (uint32_t)g * 8192u) >> 4);
    const uint64_t al = desc0 + (uint64_t)((base + kATile + (uint32_t)g * 8192u) >> 4);
    const uint64_t wh = desc0 + (uint64_t)((base + 2 * kATile) >> 4);
    const uint64_t wl = desc0 + (uint64_t)((base + 2 * kATile + kW) >> 4);
    fence_acc(acc);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      mma_nt<NT>(acc, ah + (uint64_t)(2 * k), wh + (uint64_t)(2 * k), 1u);
      mma_nt<NT>(acc, al + (uint64_t)(2 * k), wh + (uint64_t)(2 * k), 1u);
      mma_nt<NT>(acc, ah + (uint64_t)(2 * k), wl + (uint64_t)(2 * k), 1u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    fence_acc(acc);
    __syncthreads();  // every warpgroup is done with this stage before a later load refills it
  }
  cp_async_wait<0>();

  // epilogue from the accumulator fragment: d[4 jj + e] = row 16 w + l / 4 + 8 (e >> 1), column 8 jj + 2 (l % 4) + (e & 1)
  const int w = (tid >> 5) & 3, l = tid & 31;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int m = m0 + 64 * g + 16 * w + (l >> 2) + 8 * h;
    if (m >= M) continue;
    const int b = m / TF, rem = m - b * TF;
    const int t = rem / p.F_out, f = rem - t * p.F_out;
    const int orow = b * p.T_out + t;
#pragma unroll
    for (int jj = 0; jj < NT / 8; ++jj) {
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int n = ntile * NT + 8 * jj + 2 * (l & 3) + e;
        if (n >= p.N) continue;
        const float v = fmaxf(acc[4 * jj + 2 * h + e] * p.inv_scale + p.bias[n], 0.f);
        taco::store_split_scalar(v, orow, p.rows_total, n * p.F_out + f, p.y_hi, p.y_lo);
      }
    }
  }
}

// w [N][C][kh][kw] -> [N / NT][KB][hi | lo][NT][64] with k = (dt kw + df) C + c; chunk c8 of row n at c8 ^ (n & 7)
__global__ void conv2d_tc_pack_kernel(const float* __restrict__ w, int N, int C, int kh, int kw, int NT, int KB, float scale,
                                      __half* __restrict__ dst) {
  const size_t total = (size_t)((N + NT - 1) / NT) * KB * NT * 8;
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int c8 = (int)(i & 7);
  const int nn = (int)((i >> 3) % NT);
  const int kb = (int)((i / ((size_t)8 * NT)) % KB);
  const int tile = (int)(i / ((size_t)8 * NT * KB));
  const int n = tile * NT + nn;
  const int K = kh * kw * C;
  __align__(16) __half hi[8], lo[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    const int k = kb * 64 + c8 * 8 + e;
    float v = 0.f;
    if (n < N && k < K) {
      const int tap = k / C, c = k - tap * C;
      const int dt = tap / kw, df = tap - dt * kw;
      v = w[(((size_t)n * C + c) * kh + dt) * kw + df] * scale;
    }
    hi[e] = __float2half_rn(v);
    lo[e] = __float2half_rn(v - __half2float(hi[e]));
  }
  const size_t t = ((size_t)tile * KB + kb) * 2;
  const size_t o = (size_t)nn * 8 + (size_t)(c8 ^ (nn & 7));
  reinterpret_cast<uint4*>(dst)[t * NT * 8 + o] = *reinterpret_cast<const uint4*>(hi);
  reinterpret_cast<uint4*>(dst)[(t + 1) * NT * 8 + o] = *reinterpret_cast<const uint4*>(lo);
}

template <int NT>
cudaError_t launch_nt(const Conv2dTcArgs& a, cudaStream_t st) {
  const size_t smem = (size_t)kStages * stage_bytes<NT>() + 1024;
  cudaError_t e = cudaFuncSetAttribute(conv2d_tc_kernel<NT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  const int M = a.B * a.T_out * a.F_out;
  dim3 grid((M + 127) / 128, (a.N + NT - 1) / NT);
  conv2d_tc_kernel<NT><<<grid, 256, smem, st>>>(a);
  return cudaGetLastError();
}

}  // namespace

int conv2d_tc_ntile(int N) {
  if (N % 144 == 0) return 144;
  if (N % 64 == 0) return 64;
  if (N % 32 == 0) return 32;
  return 0;
}

size_t conv2d_tc_weight_bytes(int N, int C, int kh, int kw) {
  const int NT = conv2d_tc_ntile(N);
  if (NT == 0) return 0;
  const size_t KB = ((size_t)kh * kw * C + 63) / 64;
  return (size_t)(N / NT) * KB * 2 * NT * 64 * sizeof(__half);
}

cudaError_t conv2d_tc_pack(const float* w, int N, int C, int kh, int kw, float scale, __half* dst, cudaStream_t st) {
  const int NT = conv2d_tc_ntile(N);
  if (NT == 0 || C % 8) return cudaErrorInvalidValue;
  const int KB = (kh * kw * C + 63) / 64;
  const size_t total = (size_t)(N / NT) * KB * NT * 8;
  conv2d_tc_pack_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(w, N, C, kh, kw, NT, KB, scale, dst);
  return cudaGetLastError();
}

cudaError_t launch_conv2d_tc(const Conv2dTcArgs& a, cudaStream_t st) {
  if (a.C % 8 || a.rows_total % 128 || a.KB != (a.kh * a.kw * a.C + 63) / 64) return cudaErrorInvalidValue;
  switch (conv2d_tc_ntile(a.N)) {
    case 144: return launch_nt<144>(a, st);
    case 64: return launch_nt<64>(a, st);
    case 32: return launch_nt<32>(a, st);
    default: return cudaErrorInvalidValue;
  }
}

}  // namespace ppgx
}  // namespace mb
