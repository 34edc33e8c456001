// numpy's pairwise summation (numpy/_core/src/umath/loops_utils.h.src, the order np.add.reduce takes over a contiguous
// float32 or float64 array: the same 8-accumulator, 128-element blocks for both) of an element function f(i), i in [0, n),
// in the element type T (float or double), every addition rounded once.  Shared by the resampler's levelling (f = x * x,
// float32 and float64) and the wav2vec2 feature extractor's normalisation (f = x, then f = (x - mean)^2).
#pragma once
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdint>
#include <vector>

namespace mb {

// rounded arithmetic by element type: never contracted into an FMA
__device__ __forceinline__ float add_rn(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ double add_rn(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ float mul_rn(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ double mul_rn(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ float div_rn(float a, float b) { return __fdiv_rn(a, b); }
__device__ __forceinline__ double div_rn(double a, double b) { return __ddiv_rn(a, b); }

template <class T, class F>
__device__ T pairwise_sum(const F& f, int64_t i0, int64_t n) {
  if (n < 8) {
    T r = (T)-0.0;
    for (int64_t i = 0; i < n; ++i) r = add_rn(r, (T)f(i0 + i));
    return r;
  }
  if (n <= 128) {
    T r[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) r[k] = f(i0 + k);
    int64_t i = 8;
    for (; i < n - (n % 8); i += 8)
#pragma unroll
      for (int k = 0; k < 8; ++k) r[k] = add_rn(r[k], (T)f(i0 + i + k));
    T res = add_rn(add_rn(add_rn(r[0], r[1]), add_rn(r[2], r[3])), add_rn(add_rn(r[4], r[5]), add_rn(r[6], r[7])));
    for (; i < n; ++i) res = add_rn(res, (T)f(i0 + i));
    return res;
  }
  int64_t n2 = n / 2;
  n2 -= n2 % 8;
  return add_rn(pairwise_sum<T>(f, i0, n2), pairwise_sum<T>(f, i0 + n2, n - n2));
}

// The same sum by one CTA: the tree is split into 2^depth subtrees (depth from pairwise_depth), one per thread, and the levels
// above them are added bottom up in shared memory `part` (at least 2^depth elements of T).  Every thread returns the sum.
template <class F, class T>
__device__ T pairwise_sum_block(const F& f, int64_t n, int depth, T* part) {
  const int nsub = 1 << depth;
  if ((int)threadIdx.x < nsub) {
    int64_t off = 0, m = n;
    for (int d = depth - 1; d >= 0; --d) {  // walk down: bit d of the thread index picks the right half
      int64_t n2 = m / 2;
      n2 -= n2 % 8;
      if ((threadIdx.x >> d) & 1) off += n2, m -= n2;
      else m = n2;
    }
    part[threadIdx.x] = pairwise_sum<T>(f, off, m);
  }
  __syncthreads();
  for (int w = nsub >> 1; w >= 1; w >>= 1) {
    T v = 0;
    if ((int)threadIdx.x < w) v = add_rn(part[2 * threadIdx.x], part[2 * threadIdx.x + 1]);
    __syncthreads();
    if ((int)threadIdx.x < w) part[threadIdx.x] = v;
    __syncthreads();
  }
  const T s = part[0];
  __syncthreads();  // part may be reused by the caller's next sum
  return s;
}

// the deepest level (<= 8) whose nodes all sit below internal nodes (more than 128 elements) of numpy's pairwise tree
inline int pairwise_depth(int64_t n) {
  std::vector<int64_t> sizes{n};
  int d = 0;
  while (d < 8) {
    if (*std::min_element(sizes.begin(), sizes.end()) <= 128) break;
    std::vector<int64_t> next;
    for (int64_t s : sizes) {
      int64_t n2 = s / 2;
      n2 -= n2 % 8;
      next.push_back(n2);
      next.push_back(s - n2);
    }
    std::sort(next.begin(), next.end());
    next.erase(std::unique(next.begin(), next.end()), next.end());
    sizes.swap(next);
    ++d;
  }
  return d;
}

}  // namespace mb
