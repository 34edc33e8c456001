// Shared-memory Stockham FFT shared by Griffin-Lim (float2, csrc/griffinlim.cu) and the log-MMSE denoiser (double2,
// csrc/logmmse.cu): DESIGN.md sections 4i and 4j.
//
// N = 2^a or 5 * 2^a complex points.  Stages run with Ns = 1, R, R R', ... and take radix 4 while 4 divides N / Ns, then
// radix 2 while 2 does, then radix 5; a power of two therefore runs exactly the radix-4 stages (and one final radix-2
// stage for odd log2 N) it always ran.  The twiddle table tw[m] = exp(-2 pi i m / N) is computed on the host in float64
// (rounded to float for the float2 instance); INV conjugates it and the butterfly's +-i, unscaled.
#pragma once
#include <cuda_runtime.h>

#include <cmath>

namespace mb {

// the twiddle table of an N-point transform, tw[2 m] + i tw[2 m + 1] = exp(-2 pi i m / N), computed in float64 and rounded
// once to R (float for the float2 instance); every user of stockham() builds its table here
template <class R>
inline void fft_twiddles(int N, R* tw) {
  const double PI = 3.14159265358979323846;
  for (int k = 0; k < N; ++k) {
    tw[2 * k] = (R)std::cos(2.0 * PI * k / N);
    tw[2 * k + 1] = (R)(-std::sin(2.0 * PI * k / N));
  }
}

// 2^a or 5 * 2^a in [64, 2048]: the sizes stockham() is built and tested for
inline bool fft_supported(int n) {
  if (n < 64 || n > 2048) return false;
  if (n % 5 == 0) n /= 5;
  return (n & (n - 1)) == 0;
}

__device__ __forceinline__ float2 cmul(float2 a, float2 b) {
  return make_float2(fmaf(a.x, b.x, -(a.y * b.y)), fmaf(a.x, b.y, a.y * b.x));
}
__device__ __forceinline__ float2 cadd(float2 a, float2 b) { return make_float2(a.x + b.x, a.y + b.y); }
__device__ __forceinline__ float2 csub(float2 a, float2 b) { return make_float2(a.x - b.x, a.y - b.y); }
__device__ __forceinline__ float2 cscale(float2 a, float s) { return make_float2(a.x * s, a.y * s); }

__device__ __forceinline__ double2 cmul(double2 a, double2 b) {
  return make_double2(fma(a.x, b.x, -(a.y * b.y)), fma(a.x, b.y, a.y * b.x));
}
__device__ __forceinline__ double2 cadd(double2 a, double2 b) { return make_double2(a.x + b.x, a.y + b.y); }
__device__ __forceinline__ double2 csub(double2 a, double2 b) { return make_double2(a.x - b.x, a.y - b.y); }
__device__ __forceinline__ double2 cscale(double2 a, double s) { return make_double2(a.x * s, a.y * s); }

// e * (-i) (forward) or e * (+i) (inverse)
template <bool INV, class T>
__device__ __forceinline__ T rot_i(T e) {
  return INV ? T{-e.y, e.x} : T{e.y, -e.x};
}

// Stockham autosort FFT of N complex points in shared memory (a -> b -> a ...); returns the buffer holding the result.
template <bool INV, class T>
__device__ T* stockham(T* a, T* b, const T* __restrict__ tw, int N) {
  using R_t = decltype(T::x);
  for (int Ns = 1; Ns < N;) {
    const int rest = N / Ns;
    const int R = (rest & 3) == 0 ? 4 : (rest & 1) == 0 ? 2 : 5;
    const int nr = N / R, step = N / (Ns * R);
    for (int j = threadIdx.x; j < nr; j += blockDim.x) {
      const int k = j & (Ns - 1);
      const int d = (j - k) * R + k;
      if (R == 4) {
        T t1 = __ldg(tw + k * step), t2 = __ldg(tw + 2 * k * step), t3 = __ldg(tw + 3 * k * step);
        if (INV) t1.y = -t1.y, t2.y = -t2.y, t3.y = -t3.y;
        const T v0 = a[j], v1 = cmul(a[j + nr], t1), v2 = cmul(a[j + 2 * nr], t2), v3 = cmul(a[j + 3 * nr], t3);
        const T b0 = cadd(v0, v2), b1 = csub(v0, v2), b2 = cadd(v1, v3);
        const T b3 = rot_i<INV>(csub(v1, v3));  // (v1 - v3) * (-+i)
        b[d] = cadd(b0, b2);
        b[d + Ns] = cadd(b1, b3);
        b[d + 2 * Ns] = csub(b0, b2);
        b[d + 3 * Ns] = csub(b1, b3);
      } else if (R == 2) {
        T t1 = __ldg(tw + k * step);
        if (INV) t1.y = -t1.y;
        const T v0 = a[j], v1 = cmul(a[j + nr], t1);
        b[d] = cadd(v0, v1);
        b[d + Ns] = csub(v0, v1);
      } else {  // radix 5: y_q = sum_r v_r exp(-+2 pi i q r / 5)
        // Ns is not a power of two here only when the radix-5 stage is the last one (Ns = N / 5 = 2^a), so k = j & (Ns - 1)
        // stays exact
        const R_t c1 = (R_t)0.30901699437494742410, c2 = (R_t)-0.80901699437494742410;  // cos(2 pi / 5), cos(4 pi / 5)
        const R_t s1 = (R_t)0.95105651629515357212, s2 = (R_t)0.58778525229247312917;   // sin(2 pi / 5), sin(4 pi / 5)
        T t1 = __ldg(tw + k * step), t2 = __ldg(tw + 2 * k * step), t3 = __ldg(tw + 3 * k * step),
          t4 = __ldg(tw + 4 * k * step);
        if (INV) t1.y = -t1.y, t2.y = -t2.y, t3.y = -t3.y, t4.y = -t4.y;
        const T v0 = a[j], v1 = cmul(a[j + nr], t1), v2 = cmul(a[j + 2 * nr], t2), v3 = cmul(a[j + 3 * nr], t3),
                v4 = cmul(a[j + 4 * nr], t4);
        const T s14 = cadd(v1, v4), d14 = csub(v1, v4), s23 = cadd(v2, v3), d23 = csub(v2, v3);
        const T A1 = cadd(v0, cadd(cscale(s14, c1), cscale(s23, c2)));
        const T A2 = cadd(v0, cadd(cscale(s14, c2), cscale(s23, c1)));
        const T B1 = rot_i<INV>(cadd(cscale(d14, s1), cscale(d23, s2)));
        const T B2 = rot_i<INV>(csub(cscale(d14, s2), cscale(d23, s1)));
        b[d] = cadd(v0, cadd(s14, s23));
        b[d + Ns] = cadd(A1, B1);
        b[d + 2 * Ns] = cadd(A2, B2);
        b[d + 3 * Ns] = csub(A2, B2);
        b[d + 4 * Ns] = csub(A1, B1);
      }
    }
    __syncthreads();
    T* t = a;
    a = b;
    b = t;
    Ns *= R;
  }
  return a;
}

}  // namespace mb
