// Kernels of the PPG extractor (csrc/ppg_extractor.cu) that live in their own translation unit: the implicit-GEMM
// Conv2d on wgmma (csrc/conv2d_tc.cu).
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <cstddef>

namespace mb {
namespace ppgx {

// embed.conv.2 as an implicit GEMM: Y[pixel][n] = relu(bias[n] + sum_{dt, df, c} W[n][c][dt][df] * X[t s + dt - p][f s + df - p][c])
// M = output pixels (b, t, f), N = out channels, K = kh kw C ordered (dt, df, c).  The 3-term fp16 split (hi hi + lo hi + hi lo,
// FP32 accumulation) of tacotron_tc.cu, so the product is FP32-equivalent.  No im2col: each CTA gathers its 128 pixels x 64 k
// operand tile straight from the channels-last hi / lo input planes with zero-filling 16-byte cp.async (taps outside the
// plane or past the row's own length read zeros).  The epilogue writes relu(.) split into the hi / lo operand tiles of the
// next GEMM (embed.out.0), at row b T_out + t and column n F_out + f: the [t][c F + f] layout of subsampling.py's view.
struct Conv2dTcArgs {
  const __half* x_hi;    // [B][T_in][F_in][C]
  const __half* x_lo;
  const int* len_in;     // [B] valid input frames of each row (device)
  int B, T_in, F_in, C;
  int T_out, F_out, kh, kw, stride, pad;
  const __half* w;       // conv2d_tc_pack image: [N / NT][KB][hi | lo][NT][64], SWIZZLE_128B rows
  const float* bias;     // [N]
  int N, K, KB;
  float inv_scale;
  __half* y_hi;          // operand tiles [ceil(N F_out / 64)][rows_total][64]
  __half* y_lo;
  int rows_total;
};

// n-tile width the kernel uses for N output channels (0: not supported)
int conv2d_tc_ntile(int N);
size_t conv2d_tc_weight_bytes(int N, int C, int kh, int kw);
// w fp32 [N][C][kh][kw] * scale -> the packed image
cudaError_t conv2d_tc_pack(const float* w, int N, int C, int kh, int kw, float scale, __half* dst, cudaStream_t st);
cudaError_t launch_conv2d_tc(const Conv2dTcArgs& a, cudaStream_t st);

}  // namespace ppgx
}  // namespace mb
