// Polyphase resampling and per-clip levelling on H100 (mb_resample_*): DESIGN.md section 4k.
//
//   replaces  scipy.signal.resample_poly(x, up, down) (window ('kaiser', 5.0), padtype 'constant') as
//             synthesizer/audio_host.py load_wav / preprocess_wav call it, normalize_volume(wav, -30, increase_only=True)
//             and load_preprocess_wav's rescale wav / max|wav| * rescaling_max
//
// The arithmetic is scipy's float32 upfirdn, so that every output sample is bitwise the host's:
//   y[j] = sum over input samples n ascending of h[j down + half_len - n up] * x[n]
// i.e. the polyphase taps of phase (j down + half_len) mod up in DESCENDING tap index, one rounded float32 multiply and one
// rounded float32 add per tap (__fmul_rn / __fadd_rn: never contracted to an FMA, and the library is built with
// -fmad=false as well), from a zero accumulator.  The zero taps scipy's padding adds are skipped: for finite input they
// add +0 or -0 to an accumulator that can never be -0, which changes nothing.
//
// rs_resample_kernel   one CTA per work item (clip, tile of kTile output samples), one output per thread; the input window
//                      of the tile plus the filter halo is staged in shared memory by a bulk copy (the 16-byte aligned
//                      interior) and plain loads (the unaligned ends); the polyphase table [up][taps] is staged the same way
//                      when it fits under the handle's limit, else read through L2
// rs_sumsq_kernel      one CTA per clip: the sum of x * x in numpy's pairwise order (np.add.reduce on float32 or float64)
// rs_scale_kernel      y = x * gain[b] (one rounded multiply)
// rs_rescale_kernel    one CTA per clip: m = max |x| (exact), y = (x / m) * peak (two rounded operations)
// The three levelling kernels are instantiated for float (mb_resample_sumsq / _scale / _rescale) and for double (the _f64
// entries, the text-to-speech chain's float64 post-processing, gen_voice.py).
#include <algorithm>
#include <cmath>
#include <cstring>
#include <vector>

#include "gan_tc_dev.cuh"
#include "mb_common.h"
#include "mb_pairwise.cuh"

using namespace mb;
using namespace mb::tcdev;

namespace {

constexpr int kTile = 512;  // output samples per work item = threads per CTA
constexpr int kLevelThreads = 256;
constexpr int kDefaultFilterSmem = 64 * 1024;  // 11025 -> 16000 (640 phases x 21 taps) is 52 KB
constexpr int kMaxSmem = 200 * 1024;

struct RsClip {
  int64_t in_off, out_off;  // first input / output sample of the clip in the flat buffers
  int32_t n_in, n_out;
  int32_t up, down, half_len, taps;  // up == down == 1: a copy (taps = 0)
  int64_t filt;                      // first float of the polyphase table [up][taps] in the arena
  int32_t smem_filter;               // 1: the table is staged in shared memory
  int32_t tile0;                     // first work item of the clip
};

struct RsParams {
  const void* x;
  float* out;
  const RsClip* clips;
  const float* arena;
  int32_t batch;
  int32_t win_bytes;  // shared-memory bytes of the staged input window (a multiple of 16)
};

template <typename T>
__device__ __forceinline__ float sample(T v) {
  if constexpr (sizeof(T) == 2) return __fdiv_rn((float)v, 32768.0f);  // exact: load_wav's int16 / 32768
  else return v;
}

// elements [g_lo, g_hi) of src into dst, where dst[0] is element a_lo (a multiple of 16 bytes): the aligned interior by one
// bulk copy on `bar` (thread 0 issues it), the ends by plain loads.  Returns the bytes the bulk copy will complete.
template <typename T>
__device__ __forceinline__ uint32_t stage(T* dst, const T* src, int64_t a_lo, int64_t g_lo, int64_t g_hi, uint64_t* bar) {
  constexpr int64_t epv = 16 / sizeof(T);
  const int64_t b0 = (g_lo + epv - 1) / epv * epv, b1 = g_hi / epv * epv;
  uint32_t bytes = 0;
  if (b1 > b0) {
    bytes = (uint32_t)((b1 - b0) * sizeof(T));
    if (threadIdx.x == 0) bulk_g2s(smem_u32(dst + (b0 - a_lo)), src + b0, bytes, bar);
    for (int64_t g = g_lo + threadIdx.x; g < b0; g += blockDim.x) dst[g - a_lo] = src[g];
    for (int64_t g = b1 + threadIdx.x; g < g_hi; g += blockDim.x) dst[g - a_lo] = src[g];
  } else {
    for (int64_t g = g_lo + threadIdx.x; g < g_hi; g += blockDim.x) dst[g - a_lo] = src[g];
  }
  return bytes;
}

template <typename T>
__global__ void __launch_bounds__(kTile) rs_resample_kernel(const RsParams p) {
  extern __shared__ __align__(16) unsigned char sm[];
  __shared__ __align__(8) uint64_t bar;
  int lo = 0, hi = p.batch - 1;  // the clip of this work item: the last with tile0 <= blockIdx.x
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (p.clips[mid].tile0 <= (int)blockIdx.x) lo = mid;
    else hi = mid - 1;
  }
  const RsClip c = p.clips[lo];
  const int64_t j0 = (int64_t)(blockIdx.x - c.tile0) * kTile;
  const int64_t j = j0 + threadIdx.x;
  const int64_t j1 = min(j0 + kTile, (int64_t)c.n_out);  // uniform across the CTA
  const T* x = (const T*)p.x;
  if (c.taps == 0) {
    if (j < j1) p.out[c.out_off + j] = sample(x[c.in_off + j]);
    return;
  }
  // input samples the tile reads: ceil((j0 down - half_len) / up) .. floor(((j1 - 1) down + half_len) / up), in the clip
  const int64_t up = c.up, down = c.down, hl = c.half_len;
  const int64_t num_lo = j0 * down - hl;
  const int64_t w_lo = max((int64_t)0, num_lo >= 0 ? (num_lo + up - 1) / up : -((-num_lo) / up));
  const int64_t w_hi = min((int64_t)c.n_in, ((j1 - 1) * down + hl) / up + 1);
  constexpr int64_t epv = 16 / sizeof(T);
  const int64_t g_lo = c.in_off + w_lo, g_hi = c.in_off + w_hi, a_lo = g_lo / epv * epv;
  T* win = (T*)sm;
  float* filt_s = (float*)(sm + p.win_bytes);
  const int64_t fsize = (int64_t)c.up * c.taps;
  if (threadIdx.x == 0) {
    mbar_init(&bar, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  uint32_t tx = stage(win, x, a_lo, g_lo, g_hi, &bar);
  if (c.smem_filter) tx += stage(filt_s, p.arena, c.filt, c.filt, c.filt + fsize, &bar);
  if (threadIdx.x == 0) mbar_expect_tx(&bar, tx);  // arrives once: completes when the bulk bytes have landed
  __syncthreads();
  mbar_wait(&bar, 0);
  if (j >= j1) return;
  const float* filt = c.smem_filter ? filt_s : p.arena + c.filt;
  const int64_t cj = j * down + hl;
  const int phase = (int)(cj % up);
  const int64_t ntop = cj / up;  // the input sample under tap `phase` (q = 0)
  const int qmax = (int)min((int64_t)(2 * c.half_len - phase) / up, ntop);
  const int qmin = (int)max((int64_t)0, ntop - (c.n_in - 1));
  const float* fp = filt + (int64_t)phase * c.taps;
  const T* xs = win + (c.in_off + ntop - a_lo);
  float acc = 0.0f;
  // scipy's order: ascending input index = descending tap index; separate rounded multiply and add (no contraction)
  for (int q = qmax; q >= qmin; --q) acc = __fadd_rn(acc, __fmul_rn(fp[q], sample(xs[-q])));
  p.out[c.out_off + j] = acc;
}

struct LvClip {
  int64_t off;
  int32_t n;
  int32_t depth;  // the pairwise tree is split into 2^depth subtrees, one per thread; every node above them is internal
};

// numpy's max of |x| as the levelling reads it: the float32 kernels keep fmaxf (a NaN sample is skipped); the float64 kernel
// propagates NaN as np.abs(x).max() does, so a NaN anywhere makes the clip all NaN
__device__ __forceinline__ float max_abs(float m, float v) { return fmaxf(m, fabsf(v)); }
__device__ __forceinline__ double max_abs(double m, double v) {
  const double a = fabs(v);
  return (a > m || a != a) ? a : m;
}

template <typename T>
__global__ void __launch_bounds__(kLevelThreads) rs_sumsq_kernel(const T* __restrict__ x, const LvClip* clips,
                                                                 T* __restrict__ sumsq) {
  __shared__ T part[kLevelThreads];
  const LvClip c = clips[blockIdx.x];
  const T* a = x + c.off;
  const T s = pairwise_sum_block([a](int64_t i) { return mul_rn(a[i], a[i]); }, c.n, c.depth, part);
  if (threadIdx.x == 0) sumsq[blockIdx.x] = s;
}

template <typename T>
__global__ void __launch_bounds__(kLevelThreads) rs_scale_kernel(const T* __restrict__ x, const LvClip* clips,
                                                                 const T* __restrict__ gains, T* __restrict__ y) {
  const LvClip c = clips[blockIdx.y];
  const T g = gains[blockIdx.y];
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < c.n; i += (int64_t)gridDim.x * blockDim.x)
    y[c.off + i] = mul_rn(x[c.off + i], g);
}

template <typename T>
__global__ void __launch_bounds__(kLevelThreads) rs_rescale_kernel(const T* __restrict__ x, const LvClip* clips, T peak,
                                                                   T* __restrict__ y) {
  __shared__ T red[kLevelThreads / 32];
  const LvClip c = clips[blockIdx.x];
  const T* xc = x + c.off;
  T m = 0;
  for (int64_t i = threadIdx.x; i < c.n; i += blockDim.x) m = max_abs(m, xc[i]);
  for (int o = 16; o > 0; o >>= 1) m = max_abs(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
  __syncthreads();
  m = red[0];
  for (int w = 1; w < kLevelThreads / 32; ++w) m = max_abs(m, red[w]);
  for (int64_t i = threadIdx.x; i < c.n; i += blockDim.x) y[c.off + i] = mul_rn(div_rn(xc[i], m), peak);
}


struct Filter {
  int32_t up, down, half_len, taps;
  std::vector<float> table;  // [up][taps]
  int64_t off;               // floats from the arena start (a multiple of 4)
};

}  // namespace

struct mb_resample {
  int32_t smem_limit = kDefaultFilterSmem;
  std::vector<Filter> filters;
  float* arena = nullptr;
  bool finalized = false;
};

extern "C" {

int mb_resample_create(int32_t filter_smem_bytes, mb_resample** out) {
  if (!out) return fail(MB_ERR_INVALID, "mb_resample_create: null argument");
  if (filter_smem_bytes > kDefaultFilterSmem * 2)
    return fail(MB_ERR_INVALID, "mb_resample_create: filter_smem_bytes = %d exceeds %d", (int)filter_smem_bytes,
                kDefaultFilterSmem * 2);
  mb_resample* h = new mb_resample();
  if (filter_smem_bytes >= 0) h->smem_limit = filter_smem_bytes;
  *out = h;
  return MB_OK;
}

void mb_resample_destroy(mb_resample* h) { delete h; }

int mb_resample_add_filter(mb_resample* h, int32_t up, int32_t down, const float* taps_host, int32_t n_taps,
                           int32_t* index_out) {
  if (!h || !taps_host || !index_out) return fail(MB_ERR_INVALID, "mb_resample_add_filter: null argument");
  if (up < 1 || down < 1 || (up == 1 && down == 1))
    return fail(MB_ERR_INVALID, "mb_resample_add_filter: up = %d, down = %d (a ratio other than 1, both >= 1)", (int)up,
                (int)down);
  int32_t a = up, b = down;
  while (b) std::swap(a %= b, b);
  if (a != 1) return fail(MB_ERR_INVALID, "mb_resample_add_filter: up = %d and down = %d share the factor %d", (int)up, (int)down, (int)a);
  const int64_t half_len = 10 * (int64_t)std::max(up, down);
  if (half_len > (1 << 26) || n_taps != 2 * half_len + 1)
    return fail(MB_ERR_INVALID, "mb_resample_add_filter: n_taps = %d; resample_poly's filter has 20 max(up, down) + 1 = %lld",
                (int)n_taps, (long long)(2 * half_len + 1));
  // a tile reads about (kTile down + 2 half_len) / up input samples; refuse ratios whose window would not fit
  const int64_t win = ((int64_t)(kTile - 1) * down + 2 * half_len) / up + 2;
  if (win * 4 + 32 > kMaxSmem - kDefaultFilterSmem * 2)
    return fail(MB_ERR_INVALID, "mb_resample_add_filter: down / up = %d / %d reads %lld input samples per tile; too many",
                (int)down, (int)up, (long long)win);
  for (size_t i = 0; i < h->filters.size(); ++i)
    if (h->filters[i].up == up && h->filters[i].down == down) {
      *index_out = (int32_t)i;
      return MB_OK;
    }
  Filter f{up, down, (int32_t)half_len, (int32_t)((n_taps + up - 1) / up), {}, 0};
  f.table.assign((size_t)up * f.taps, 0.0f);
  for (int p = 0; p < up; ++p)
    for (int q = 0; q < f.taps && p + (int64_t)q * up < n_taps; ++q) f.table[(size_t)p * f.taps + q] = taps_host[p + (int64_t)q * up];
  int64_t off = 0;
  for (const Filter& g : h->filters) off += align_up(g.table.size(), 4);
  f.off = off;
  h->filters.push_back(std::move(f));
  h->arena = nullptr;  // the table grew: a new arena and finalize are needed
  h->finalized = false;
  *index_out = (int32_t)(h->filters.size() - 1);
  return MB_OK;
}

size_t mb_resample_arena_bytes(const mb_resample* h) {
  if (!h) return 0;
  size_t n = 0;
  for (const Filter& f : h->filters) n += align_up(f.table.size(), 4);
  return std::max<size_t>(n, 4) * sizeof(float);
}

int mb_resample_set_arena(mb_resample* h, void* arena, size_t bytes) {
  if (int rc = check_arena("mb_resample_set_arena", h, arena, bytes, mb_resample_arena_bytes(h), 16)) return rc;
  h->arena = (float*)arena;
  h->finalized = false;
  return MB_OK;
}

int mb_resample_finalize(mb_resample* h, void* stream) {
  if (!h || !h->arena) return fail(MB_ERR_STATE, "mb_resample_finalize: no arena");
  cudaStream_t st = (cudaStream_t)stream;
  for (const Filter& f : h->filters)
    MB_CUDA_CHECK(cudaMemcpyAsync(h->arena + f.off, f.table.data(), sizeof(float) * f.table.size(), cudaMemcpyHostToDevice, st));
  MB_CUDA_CHECK(cudaStreamSynchronize(st));  // the sources are pageable host memory owned by the handle
  h->finalized = true;
  return MB_OK;
}

int mb_resample_filter_in_smem(const mb_resample* h, int32_t index) {
  if (!h || index < 0 || index >= (int32_t)h->filters.size()) return -1;
  return h->filters[index].table.size() * sizeof(float) <= (size_t)h->smem_limit ? 1 : 0;
}

int64_t mb_resample_output_length(int32_t up, int32_t down, int64_t n) {
  if (up < 1 || down < 1 || n < 0) return -1;
  return (n * up + down - 1) / down;
}

size_t mb_resample_workspace_bytes(const mb_resample* h, int32_t batch) {
  if (!h || batch < 1) return 0;
  return align_up(sizeof(RsClip) * (size_t)batch, 256) + 256;
}

// the clip table of a forward call: offsets, ratio, filter placement and first work item of every clip, the number of
// work items, and the shared-memory bytes of the largest input window and of the largest staged filter
static int plan(const mb_resample* h, const char* fn, int32_t dtype, const int32_t* lengths_host, const int32_t* filters_host,
                int32_t batch, std::vector<RsClip>& clips, int64_t& tiles, int64_t& win_max, int64_t& filt_max) {
  if (batch < 1) return fail(MB_ERR_INVALID, "%s: batch = %d", fn, (int)batch);
  clips.assign(batch, RsClip{});
  int64_t in_off = 0, out_off = 0;
  tiles = 0, win_max = 16, filt_max = 0;
  for (int b = 0; b < batch; ++b) {
    const int32_t n = lengths_host[b], fi = filters_host[b];
    if (n < 1) return fail(MB_ERR_INVALID, "%s: clip %d has %d samples", fn, b, (int)n);
    if (fi < -1 || fi >= (int32_t)h->filters.size())
      return fail(MB_ERR_INVALID, "%s: clip %d names filter %d of %d", fn, b, (int)fi, (int)h->filters.size());
    RsClip& c = clips[b];
    c.in_off = in_off;
    c.out_off = out_off;
    c.n_in = n;
    c.up = c.down = 1;
    c.n_out = n;
    if (fi >= 0) {
      const Filter& f = h->filters[fi];
      const int64_t n_out = mb_resample_output_length(f.up, f.down, n);
      if (n_out > INT32_MAX) return fail(MB_ERR_INVALID, "%s: clip %d gives %lld samples", fn, b, (long long)n_out);
      c.n_out = (int32_t)n_out;
      c.up = f.up, c.down = f.down, c.half_len = f.half_len, c.taps = f.taps;
      c.filt = f.off;
      c.smem_filter = mb_resample_filter_in_smem(h, fi);
      const int64_t win = ((int64_t)(kTile - 1) * f.down + 2 * (int64_t)f.half_len) / f.up + 2;
      win_max = std::max(win_max, win * (dtype == MB_RESAMPLE_I16 ? 2 : 4) + 32);
      if (c.smem_filter) filt_max = std::max<int64_t>(filt_max, (int64_t)f.table.size() * 4 + 32);
    }
    c.tile0 = (int32_t)tiles;
    tiles += (c.n_out + kTile - 1) / kTile;
    if (tiles > INT32_MAX) return fail(MB_ERR_INVALID, "%s: too many output samples for one call", fn);
    in_off += n;
    out_off += c.n_out;
  }
  return MB_OK;
}

int mb_resample_work_items(const mb_resample* h, const int32_t* lengths_host, const int32_t* filters_host, int32_t batch,
                           int32_t* tile0_host, int64_t* out_offsets_host) {
  if (!h || !lengths_host || !filters_host || !tile0_host || !out_offsets_host)
    return fail(MB_ERR_INVALID, "mb_resample_work_items: null argument");
  std::vector<RsClip> clips;
  int64_t tiles, win_max, filt_max;
  if (int rc = plan(h, "mb_resample_work_items", MB_RESAMPLE_F32, lengths_host, filters_host, batch, clips, tiles, win_max,
                    filt_max))
    return rc;
  for (int b = 0; b < batch; ++b) tile0_host[b] = clips[b].tile0, out_offsets_host[b] = clips[b].out_off;
  tile0_host[batch] = (int32_t)tiles;
  out_offsets_host[batch] = clips[batch - 1].out_off + clips[batch - 1].n_out;
  return MB_OK;
}

int mb_resample_forward(mb_resample* h, const void* x, int32_t dtype, const int32_t* lengths_host, const int32_t* filters_host,
                        int32_t batch, float* out, void* workspace, size_t workspace_bytes, void* stream) {
  if (!h || !x || !lengths_host || !filters_host || !out) return fail(MB_ERR_INVALID, "mb_resample_forward: null argument");
  if (dtype != MB_RESAMPLE_F32 && dtype != MB_RESAMPLE_I16)
    return fail(MB_ERR_INVALID, "mb_resample_forward: dtype = %d", (int)dtype);
  if ((uintptr_t)x % 16) return fail(MB_ERR_INVALID, "mb_resample_forward: x must be 16-byte aligned");
  char* ws;
  if (int rc = bind("mb_resample_forward", workspace, workspace_bytes, mb_resample_workspace_bytes(h, batch), &ws)) return rc;
  std::vector<RsClip> clips;
  int64_t tiles = 0, win_max = 0, filt_max = 0;
  if (int rc = plan(h, "mb_resample_forward", dtype, lengths_host, filters_host, batch, clips, tiles, win_max, filt_max))
    return rc;
  for (int b = 0; b < batch && !h->finalized; ++b)
    if (filters_host[b] >= 0) return fail(MB_ERR_STATE, "mb_resample_forward: clip %d: filters not finalized", b);
  cudaStream_t st = (cudaStream_t)stream;
  MB_CUDA_CHECK(cudaMemcpyAsync(ws, clips.data(), sizeof(RsClip) * clips.size(), cudaMemcpyHostToDevice, st));
  RsParams p{x, out, (const RsClip*)ws, h->arena, batch, (int32_t)align_up((size_t)win_max, 16)};
  const size_t smem = (size_t)p.win_bytes + align_up((size_t)filt_max, 16);
  const void* k = dtype == MB_RESAMPLE_I16 ? (const void*)rs_resample_kernel<int16_t> : (const void*)rs_resample_kernel<float>;
  if (smem > 48 * 1024) MB_CUDA_CHECK(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  if (dtype == MB_RESAMPLE_I16) rs_resample_kernel<int16_t><<<(unsigned)tiles, kTile, smem, st>>>(p);
  else rs_resample_kernel<float><<<(unsigned)tiles, kTile, smem, st>>>(p);
  MB_LAUNCH_CHECK("rs_resample_kernel");
  return MB_OK;
}

size_t mb_resample_level_workspace_bytes(int32_t batch) {
  return batch < 1 ? 0 : align_up(sizeof(LvClip) * (size_t)batch, 256) + 256;
}

static int level_table(const char* fn, const int32_t* lengths_host, int32_t batch, void* workspace, size_t workspace_bytes,
                       cudaStream_t st, const LvClip** table, int32_t* max_len) {
  if (batch < 1) return fail(MB_ERR_INVALID, "%s: batch = %d", fn, (int)batch);
  LvClip* ws;
  if (int rc = bind(fn, workspace, workspace_bytes, mb_resample_level_workspace_bytes(batch), &ws)) return rc;
  std::vector<LvClip> clips(batch);
  int64_t off = 0;
  *max_len = 0;
  for (int b = 0; b < batch; ++b) {
    if (lengths_host[b] < 1) return fail(MB_ERR_INVALID, "%s: clip %d has %d samples", fn, b, (int)lengths_host[b]);
    clips[b] = LvClip{off, lengths_host[b], pairwise_depth(lengths_host[b])};
    off += lengths_host[b];
    *max_len = std::max(*max_len, lengths_host[b]);
  }
  MB_CUDA_CHECK(cudaMemcpyAsync(ws, clips.data(), sizeof(LvClip) * clips.size(), cudaMemcpyHostToDevice, st));
  *table = ws;
  return MB_OK;
}

}  // extern "C"

template <typename T>
static int level_sumsq(const char* fn, const T* x, const int32_t* lengths_host, int32_t batch, T* sumsq, void* workspace,
                       size_t workspace_bytes, void* stream) {
  if (!x || !lengths_host || !sumsq) return fail(MB_ERR_INVALID, "%s: null argument", fn);
  cudaStream_t st = (cudaStream_t)stream;
  const LvClip* t;
  int32_t n_max;
  if (int rc = level_table(fn, lengths_host, batch, workspace, workspace_bytes, st, &t, &n_max)) return rc;
  rs_sumsq_kernel<T><<<batch, kLevelThreads, 0, st>>>(x, t, sumsq);
  MB_LAUNCH_CHECK("rs_sumsq_kernel");
  return MB_OK;
}

template <typename T>
static int level_scale(const char* fn, const T* x, const int32_t* lengths_host, int32_t batch, const T* gains, T* y,
                       void* workspace, size_t workspace_bytes, void* stream) {
  if (!x || !lengths_host || !gains || !y) return fail(MB_ERR_INVALID, "%s: null argument", fn);
  cudaStream_t st = (cudaStream_t)stream;
  const LvClip* t;
  int32_t n_max;
  if (int rc = level_table(fn, lengths_host, batch, workspace, workspace_bytes, st, &t, &n_max)) return rc;
  const dim3 grid((unsigned)std::min<int64_t>(64, ((int64_t)n_max + kLevelThreads - 1) / kLevelThreads), (unsigned)batch);
  rs_scale_kernel<T><<<grid, kLevelThreads, 0, st>>>(x, t, gains, y);
  MB_LAUNCH_CHECK("rs_scale_kernel");
  return MB_OK;
}

template <typename T>
static int level_rescale(const char* fn, const T* x, const int32_t* lengths_host, int32_t batch, T peak, T* y, void* workspace,
                         size_t workspace_bytes, void* stream) {
  if (!x || !lengths_host || !y) return fail(MB_ERR_INVALID, "%s: null argument", fn);
  cudaStream_t st = (cudaStream_t)stream;
  const LvClip* t;
  int32_t n_max;
  if (int rc = level_table(fn, lengths_host, batch, workspace, workspace_bytes, st, &t, &n_max)) return rc;
  rs_rescale_kernel<T><<<batch, kLevelThreads, 0, st>>>(x, t, peak, y);
  MB_LAUNCH_CHECK("rs_rescale_kernel");
  return MB_OK;
}

extern "C" {

int mb_resample_sumsq(const float* x, const int32_t* lengths_host, int32_t batch, float* sumsq, void* workspace,
                      size_t workspace_bytes, void* stream) {
  return level_sumsq("mb_resample_sumsq", x, lengths_host, batch, sumsq, workspace, workspace_bytes, stream);
}

int mb_resample_scale(const float* x, const int32_t* lengths_host, int32_t batch, const float* gains, float* y, void* workspace,
                      size_t workspace_bytes, void* stream) {
  return level_scale("mb_resample_scale", x, lengths_host, batch, gains, y, workspace, workspace_bytes, stream);
}

int mb_resample_rescale(const float* x, const int32_t* lengths_host, int32_t batch, float peak, float* y, void* workspace,
                        size_t workspace_bytes, void* stream) {
  return level_rescale("mb_resample_rescale", x, lengths_host, batch, peak, y, workspace, workspace_bytes, stream);
}

int mb_resample_sumsq_f64(const double* x, const int32_t* lengths_host, int32_t batch, double* sumsq, void* workspace,
                          size_t workspace_bytes, void* stream) {
  return level_sumsq("mb_resample_sumsq_f64", x, lengths_host, batch, sumsq, workspace, workspace_bytes, stream);
}

int mb_resample_scale_f64(const double* x, const int32_t* lengths_host, int32_t batch, const double* gains, double* y,
                          void* workspace, size_t workspace_bytes, void* stream) {
  return level_scale("mb_resample_scale_f64", x, lengths_host, batch, gains, y, workspace, workspace_bytes, stream);
}

int mb_resample_rescale_f64(const double* x, const int32_t* lengths_host, int32_t batch, double peak, double* y,
                            void* workspace, size_t workspace_bytes, void* stream) {
  return level_rescale("mb_resample_rescale_f64", x, lengths_host, batch, peak, y, workspace, workspace_bytes, stream);
}

}  // extern "C"
