// numpy's float32 pairwise summation (numpy/_core/src/umath/loops_utils.h.src, the order np.add.reduce takes over a contiguous
// float32 array) of an element function f(i), i in [0, n).  Shared by the resampler's levelling (f = x * x) and the wav2vec2
// feature extractor's normalisation (f = x, then f = (x - mean)^2).
#pragma once
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdint>
#include <vector>

namespace mb {

template <class F>
__device__ float pairwise_sum(const F& f, int64_t i0, int64_t n) {
  if (n < 8) {
    float r = -0.0f;
    for (int64_t i = 0; i < n; ++i) r = __fadd_rn(r, f(i0 + i));
    return r;
  }
  if (n <= 128) {
    float r[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) r[k] = f(i0 + k);
    int64_t i = 8;
    for (; i < n - (n % 8); i += 8)
#pragma unroll
      for (int k = 0; k < 8; ++k) r[k] = __fadd_rn(r[k], f(i0 + i + k));
    float res = __fadd_rn(__fadd_rn(__fadd_rn(r[0], r[1]), __fadd_rn(r[2], r[3])),
                          __fadd_rn(__fadd_rn(r[4], r[5]), __fadd_rn(r[6], r[7])));
    for (; i < n; ++i) res = __fadd_rn(res, f(i0 + i));
    return res;
  }
  int64_t n2 = n / 2;
  n2 -= n2 % 8;
  return __fadd_rn(pairwise_sum(f, i0, n2), pairwise_sum(f, i0 + n2, n - n2));
}

// The same sum by one CTA: the tree is split into 2^depth subtrees (depth from pairwise_depth), one per thread, and the levels
// above them are added bottom up in shared memory `part` (at least 2^depth floats).  Every thread returns the sum.
template <class F>
__device__ float pairwise_sum_block(const F& f, int64_t n, int depth, float* part) {
  const int nsub = 1 << depth;
  if ((int)threadIdx.x < nsub) {
    int64_t off = 0, m = n;
    for (int d = depth - 1; d >= 0; --d) {  // walk down: bit d of the thread index picks the right half
      int64_t n2 = m / 2;
      n2 -= n2 % 8;
      if ((threadIdx.x >> d) & 1) off += n2, m -= n2;
      else m = n2;
    }
    part[threadIdx.x] = pairwise_sum(f, off, m);
  }
  __syncthreads();
  for (int w = nsub >> 1; w >= 1; w >>= 1) {
    float v = 0.0f;
    if ((int)threadIdx.x < w) v = __fadd_rn(part[2 * threadIdx.x], part[2 * threadIdx.x + 1]);
    __syncthreads();
    if ((int)threadIdx.x < w) part[threadIdx.x] = v;
    __syncthreads();
  }
  const float s = part[0];
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
