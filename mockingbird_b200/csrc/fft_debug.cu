// The shared-memory Stockham FFT of mb_fft.cuh on its own (mb_fft_debug): DESIGN.md section 4j.
//
// Griffin-Lim (float2) and the log-MMSE denoiser (double2) only reach the transform inside their frame kernels; this entry
// runs it on `rows` independent rows so that tests can hold it to a float64 DFT at every size the handles accept.  One CTA
// of 256 threads per row and two n-point buffers in dynamic shared memory, as gl_frame_kernel and lm_frame_kernel use it, over
// the twiddle table the handles build (fft_twiddles).
#include <vector>

#include "mb_common.h"
#include "mb_fft.cuh"

using namespace mb;

namespace {

template <bool INV, class T>
__global__ void __launch_bounds__(256) fft_debug_kernel(const T* __restrict__ x, T* __restrict__ y, const T* __restrict__ tw,
                                                        int n) {
  extern __shared__ __align__(16) unsigned char fft_sm[];
  T* a = (T*)fft_sm;
  const T* xr = x + (size_t)blockIdx.x * n;
  for (int j = threadIdx.x; j < n; j += blockDim.x) a[j] = xr[j];
  __syncthreads();
  const T* z = stockham<INV>(a, a + n, tw, n);
  T* yr = y + (size_t)blockIdx.x * n;
  for (int j = threadIdx.x; j < n; j += blockDim.x) yr[j] = z[j];
}

template <class T, class R>
int run(const T* x, T* y, int n, int rows, bool inverse, cudaStream_t st) {
  std::vector<R> host(2 * (size_t)n);
  fft_twiddles(n, host.data());
  const size_t smem = 2 * sizeof(T) * n;
  const void* k = inverse ? (const void*)fft_debug_kernel<true, T> : (const void*)fft_debug_kernel<false, T>;
  if (smem > 48 * 1024) MB_CUDA_CHECK(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  T* tw = nullptr;
  MB_CUDA_CHECK(cudaMallocAsync((void**)&tw, sizeof(T) * n, st));
  MB_CUDA_CHECK(cudaMemcpyAsync(tw, host.data(), sizeof(T) * n, cudaMemcpyHostToDevice, st));
  if (inverse) fft_debug_kernel<true, T><<<rows, 256, smem, st>>>(x, y, tw, n);
  else fft_debug_kernel<false, T><<<rows, 256, smem, st>>>(x, y, tw, n);
  const cudaError_t launched = cudaGetLastError();
  MB_CUDA_CHECK(cudaFreeAsync(tw, st));
  MB_CUDA_CHECK(cudaStreamSynchronize(st));  // the twiddles came from pageable host memory owned by this call
  if (launched != cudaSuccess)
    return fail(MB_ERR_CUDA, "launch of fft_debug_kernel failed: %s", cudaGetErrorString(launched));
  count_launch();
  return MB_OK;
}

}  // namespace

extern "C" {

int mb_fft_debug(const void* x, void* y, int32_t n, int32_t rows, int32_t dtype, int32_t inverse, void* stream) {
  if (!x || !y) return fail(MB_ERR_INVALID, "mb_fft_debug: null argument");
  if (!fft_supported(n)) return fail(MB_ERR_INVALID, "mb_fft_debug: n = %d is not 2^a or 5 * 2^a in [64, 2048]", n);
  if (rows <= 0) return fail(MB_ERR_INVALID, "mb_fft_debug: rows = %d", rows);
  if (dtype != 0 && dtype != 1) return fail(MB_ERR_INVALID, "mb_fft_debug: dtype = %d (0 float2, 1 double2)", dtype);
  cudaStream_t st = (cudaStream_t)stream;
  if (dtype == 0) return run<float2, float>((const float2*)x, (float2*)y, n, rows, inverse != 0, st);
  return run<double2, double>((const double2*)x, (double2*)y, n, rows, inverse != 0, st);
}

}  // extern "C"
