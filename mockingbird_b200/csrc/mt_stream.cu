// Reference-identical sampling noise at kernel speed (mb_mtstream_*).
//
// WaveRNN.generate draws `Categorical(p).sample()` = argmax(p / q), q = empty_like(p).exponential_(1)
// from the GLOBAL torch CPU generator (fatchord_version.py:223-226; SURVEY.md fact 5).  ATen's CPU
// exponential_ is serial per element:  r64 = (mt19937() << 32) | mt19937();  u = (r64 & (2^53-1)) * 2^-53;
// q = (float)(-log1p(-u))  (double arithmetic) - 25 ns per element on one core, i.e. 6.6 s for the 261 M
// elements of BASELINE configs[2], 15x the time of the sample-loop kernel.
//
// This component reproduces that stream bit for bit without the host bottleneck:
//   * a host worker thread runs MT19937 from the generator's exact state (624 words + position) with a
//     vectorisable block twist (AVX2 / AVX-512 clones) and ships the UNTEMPERED state words into a ring of pinned host buffers
//     (the tempering is elementwise and moves to the device: half the host work per draw),
//   * each chunk's raw draws are copied H2D on a side stream and converted on the device
//     (mt_to_exp_kernel: the same double-precision formula) into the fp32 noise tensor the sample kernel
//     consumes, overlapped with the sample kernel of the previous chunk,
//   * the generator state after the call is handed back so the host can store it into torch's generator
//     (subsequent torch draws continue exactly as after the reference's own generate()).
// Equality with ATen's stream is asserted by tests/test_mtstream.py (host draws) and the cfg-1 / cfg-3
// golden tests (510 400 integer samples identical to the reference).
#include <atomic>
#include <condition_variable>
#include <cstring>
#include <mutex>
#include <thread>
#include <vector>

#include "../../include/mb_wavernn_math.h"
#include "mb_common.h"
#include "mt19937_host.h"

namespace {

constexpr int kN = 624;
using mb::MtPos;
using mb::mt_fill;

// raw draws (hi, lo) -> q = (float)(-log1p(-u)), u = ((hi<<32|lo) & (2^53-1)) * 2^-53   (ATen: uniform_real_distribution<double>
// + transformation::exponential, aten/src/ATen/core/TransformationHelper.h, CPU branch)
__device__ __forceinline__ uint32_t mt_temper_dev(uint32_t y) {
  y ^= (y >> 11);
  y ^= (y << 7) & 0x9d2c5680u;
  y ^= (y << 15) & 0xefc60000u;
  y ^= (y >> 18);
  return y;
}

// TEMPER: the host sent untempered MT19937 state words (mb_mtstream path); otherwise finished 32-bit outputs
template <bool TEMPER>
__global__ void mt_to_exp_kernel(const uint2* __restrict__ raw, float* __restrict__ out, size_t n) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  uint2 r = raw[i];
  if (TEMPER) {
    r.x = mt_temper_dev(r.x);
    r.y = mt_temper_dev(r.y);
  }
  const unsigned long long r64 = ((unsigned long long)r.x << 32) | (unsigned long long)r.y;
  const double u = (double)(r64 & ((1ULL << 53) - 1ULL)) * 1.1102230246251565e-16;  // 2^-53
  out[i] = (float)(-log1p(-u));
}

// one word per element -> ATen's CPU float uniform_(1e-5, 1 - 1e-5) (the MOL sampler's draws; mb_torch_uniform)
template <bool TEMPER>
__global__ void mt_to_uniform_kernel(const uint32_t* __restrict__ raw, float* __restrict__ out, size_t n) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint32_t w = TEMPER ? mt_temper_dev(raw[i]) : raw[i];
  out[i] = mb_torch_uniform(w);
}

}  // namespace

struct mb_mtstream {
  int nslots = 0;
  size_t slot_words = 0;  // capacity of one pinned slot in 32-bit draws
  std::vector<uint32_t*> slots;
  std::vector<cudaEvent_t> copied;  // H2D of the slot's last use finished
  std::vector<char> copy_pending;
  cudaStream_t side = nullptr;
  cudaEvent_t ready[2] = {nullptr, nullptr};     // convert of chunk k finished (side stream)
  cudaEvent_t consumed[2] = {nullptr, nullptr};  // sample kernel of chunk k launched-and-done marker (main stream)
  char consumed_set[2] = {0, 0};
  int device = 0;
  // per call
  MtPos gen{};
  std::thread worker;
  std::mutex mu;
  std::condition_variable cv;
  uint64_t produced = 0, taken = 0;  // slots filled / slots handed to the device
  uint64_t total_words = 0, words_per_chunk = 0, n_chunks = 0;
  bool running = false;
  std::atomic<int> error{0};
};

namespace {

void worker_main(mb_mtstream* ms) {
  cudaSetDevice(ms->device);
  for (uint64_t c = 0; c < ms->n_chunks; ++c) {
    const int slot = (int)(c % (uint64_t)ms->nslots);
    {
      std::unique_lock<std::mutex> lk(ms->mu);
      ms->cv.wait(lk, [&] { return c < ms->taken + (uint64_t)ms->nslots; });
    }
    if (ms->copy_pending[slot]) {
      if (cudaEventSynchronize(ms->copied[slot]) != cudaSuccess) ms->error = 1;
      ms->copy_pending[slot] = 0;
    }
    const uint64_t done = c * ms->words_per_chunk;
    const uint64_t n = ms->total_words - done < ms->words_per_chunk ? ms->total_words - done : ms->words_per_chunk;
    mt_fill(ms->gen, ms->slots[slot], (size_t)n, /*temper=*/false);  // tempering happens in mt_to_exp_kernel<true>
    {
      std::lock_guard<std::mutex> lk(ms->mu);
      ms->produced = c + 1;
    }
    ms->cv.notify_all();
  }
}

}  // namespace

extern "C" {

int mb_mtstream_create(uint64_t slot_words, int32_t nslots, mb_mtstream** out) {
  if (!out || slot_words == 0 || nslots < 2 || nslots > 8) return mb::fail(MB_ERR_INVALID, "mb_mtstream_create: bad argument");
  mb_mtstream* ms = new mb_mtstream();
  ms->nslots = nslots;
  ms->slot_words = slot_words;
  cudaGetDevice(&ms->device);
  ms->slots.assign(nslots, nullptr);
  ms->copied.assign(nslots, nullptr);
  ms->copy_pending.assign(nslots, 0);
  for (int i = 0; i < nslots; ++i) {
    if (cudaHostAlloc((void**)&ms->slots[i], slot_words * 4, cudaHostAllocDefault) != cudaSuccess ||
        cudaEventCreateWithFlags(&ms->copied[i], cudaEventDisableTiming) != cudaSuccess) {
      mb_mtstream_destroy(ms);
      return mb::fail(MB_ERR_CUDA, "mb_mtstream_create: pinned allocation of %zu bytes failed", (size_t)slot_words * 4);
    }
  }
  for (int i = 0; i < 2; ++i) {
    cudaEventCreateWithFlags(&ms->ready[i], cudaEventDisableTiming);
    cudaEventCreateWithFlags(&ms->consumed[i], cudaEventDisableTiming);
  }
  if (cudaStreamCreateWithFlags(&ms->side, cudaStreamNonBlocking) != cudaSuccess) {
    mb_mtstream_destroy(ms);
    return mb::fail(MB_ERR_CUDA, "mb_mtstream_create: side stream");
  }
  *out = ms;
  return MB_OK;
}

void mb_mtstream_destroy(mb_mtstream* ms) {
  if (!ms) return;
  if (ms->running && ms->worker.joinable()) {
    {
      std::lock_guard<std::mutex> lk(ms->mu);
      ms->taken = ms->n_chunks + 64;  // release the producer
    }
    ms->cv.notify_all();
    ms->worker.join();
  }
  if (ms->side) {
    cudaStreamSynchronize(ms->side);
    cudaStreamDestroy(ms->side);
  }
  for (auto p : ms->slots)
    if (p) cudaFreeHost(p);
  for (auto e : ms->copied)
    if (e) cudaEventDestroy(e);
  for (int i = 0; i < 2; ++i) {
    if (ms->ready[i]) cudaEventDestroy(ms->ready[i]);
    if (ms->consumed[i]) cudaEventDestroy(ms->consumed[i]);
  }
  delete ms;
}

int mb_mtstream_begin(mb_mtstream* ms, const uint32_t* state624, int32_t left, int32_t next, uint64_t total_words,
                      uint64_t words_per_chunk) {
  if (!ms || !state624) return mb::fail(MB_ERR_INVALID, "mb_mtstream_begin: null argument");
  if (ms->running) return mb::fail(MB_ERR_STATE, "mb_mtstream_begin: a stream is already running (call mb_mtstream_finish)");
  if (words_per_chunk == 0 || words_per_chunk > ms->slot_words)
    return mb::fail(MB_ERR_INVALID, "mb_mtstream_begin: chunk of %llu draws exceeds the slot capacity %zu",
                    (unsigned long long)words_per_chunk, ms->slot_words);
  if (left < 1 || left > kN || next < 0 || next > kN || (left > 1 && next + (left - 1) != kN))
    return mb::fail(MB_ERR_INVALID, "mb_mtstream_begin: inconsistent generator position (left=%d next=%d)", left, next);
  memcpy(ms->gen.s, state624, sizeof(uint32_t) * kN);
  ms->gen.avail = left - 1;
  ms->gen.idx = next;
  ms->total_words = total_words;
  ms->words_per_chunk = words_per_chunk;
  ms->n_chunks = (total_words + words_per_chunk - 1) / words_per_chunk;
  ms->produced = ms->taken = 0;
  ms->consumed_set[0] = ms->consumed_set[1] = 0;
  ms->error = 0;
  ms->running = true;
  ms->worker = std::thread(worker_main, ms);
  return MB_OK;
}

}  // extern "C"

namespace {

// Chunk k (in call order): wait for the host draws, copy them to `dev_raw` on the side stream, convert `n_elems`
// (= words / 2 for Exp(1), = words for uniforms) of them into `dev_noise` (fp32), and make `main_stream` wait for the
// result.  The device buffers are the caller's (double-buffered by the caller: chunk k and k+2 may share storage).
int mtstream_next(mb_mtstream* ms, uint64_t n_elems, bool uniform, void* dev_raw, float* dev_noise, void* main_stream) {
  if (!ms || !dev_raw || !dev_noise) return mb::fail(MB_ERR_INVALID, "mb_mtstream_next: null argument");
  if (!ms->running || ms->taken >= ms->n_chunks) return mb::fail(MB_ERR_STATE, "mb_mtstream_next: no chunk left");
  const uint64_t c = ms->taken;
  const uint64_t done = c * ms->words_per_chunk;
  const uint64_t words = ms->total_words - done < ms->words_per_chunk ? ms->total_words - done : ms->words_per_chunk;
  const uint64_t want = uniform ? n_elems : 2 * n_elems;
  if (want != words) return mb::fail(MB_ERR_INVALID, "mb_mtstream_next: chunk %llu holds %llu draws, caller asked for %llu",
                                     (unsigned long long)c, (unsigned long long)words, (unsigned long long)want);
  {
    std::unique_lock<std::mutex> lk(ms->mu);
    ms->cv.wait(lk, [&] { return ms->produced > c; });
  }
  if (ms->error) return mb::fail(MB_ERR_CUDA, "mb_mtstream: worker failed");
  const int slot = (int)(c % (uint64_t)ms->nslots);
  const int par = (int)(c & 1);
  cudaStream_t st = (cudaStream_t)main_stream;
  if (ms->consumed_set[par]) MB_CUDA_CHECK(cudaStreamWaitEvent(ms->side, ms->consumed[par], 0));  // buffers of chunk k-2 are free
  MB_CUDA_CHECK(cudaMemcpyAsync(dev_raw, ms->slots[slot], words * 4, cudaMemcpyHostToDevice, ms->side));
  MB_CUDA_CHECK(cudaEventRecord(ms->copied[slot], ms->side));
  ms->copy_pending[slot] = 1;
  if (uniform) {
    mt_to_uniform_kernel<true><<<(unsigned)((n_elems + 255) / 256), 256, 0, ms->side>>>(reinterpret_cast<const uint32_t*>(dev_raw),
                                                                                        dev_noise, (size_t)n_elems);
    MB_LAUNCH_CHECK("mt_to_uniform_kernel");
  } else {
    mt_to_exp_kernel<true><<<(unsigned)((n_elems + 255) / 256), 256, 0, ms->side>>>(reinterpret_cast<const uint2*>(dev_raw), dev_noise,
                                                                                    (size_t)n_elems);
    MB_LAUNCH_CHECK("mt_to_exp_kernel");
  }
  MB_CUDA_CHECK(cudaEventRecord(ms->ready[par], ms->side));
  MB_CUDA_CHECK(cudaStreamWaitEvent(st, ms->ready[par], 0));
  {
    std::lock_guard<std::mutex> lk(ms->mu);
    ms->taken = c + 1;
  }
  ms->cv.notify_all();
  return MB_OK;
}

}  // namespace

extern "C" {

int mb_mtstream_next(mb_mtstream* ms, uint64_t n_elems, void* dev_raw, float* dev_noise, void* main_stream) {
  return mtstream_next(ms, n_elems, false, dev_raw, dev_noise, main_stream);
}

int mb_mtstream_next_uniform(mb_mtstream* ms, uint64_t n_elems, void* dev_raw, float* dev_noise, void* main_stream) {
  return mtstream_next(ms, n_elems, true, dev_raw, dev_noise, main_stream);
}

// call right after the consumer kernel of the chunk handed out by the last mb_mtstream_next was launched
int mb_mtstream_consumed(mb_mtstream* ms, void* main_stream) {
  if (!ms || ms->taken == 0) return mb::fail(MB_ERR_STATE, "mb_mtstream_consumed: nothing handed out");
  const int par = (int)((ms->taken - 1) & 1);
  MB_CUDA_CHECK(cudaEventRecord(ms->consumed[par], (cudaStream_t)main_stream));
  ms->consumed_set[par] = 1;
  return MB_OK;
}

// joins the worker; returns the generator state after exactly total_words draws (at::mt19937 layout: 624 words,
// left_, next_) so that the host can store it back into torch's generator
int mb_mtstream_finish(mb_mtstream* ms, uint32_t* state624, int32_t* left, int32_t* next) {
  if (!ms) return mb::fail(MB_ERR_INVALID, "mb_mtstream_finish: null handle");
  if (!ms->running) return mb::fail(MB_ERR_STATE, "mb_mtstream_finish: not running");
  {
    std::lock_guard<std::mutex> lk(ms->mu);
    if (ms->taken < ms->n_chunks) ms->taken = ms->n_chunks + 64;  // abandoned call: let the producer run to the end
  }
  ms->cv.notify_all();
  if (ms->worker.joinable()) ms->worker.join();
  ms->running = false;
  if (state624) memcpy(state624, ms->gen.s, sizeof(uint32_t) * kN);
  if (left) *left = ms->gen.avail + 1;
  if (next) *next = ms->gen.idx;
  return ms->error ? mb::fail(MB_ERR_CUDA, "mb_mtstream: worker failed") : MB_OK;
}

// host-only test / measurement hook: n raw draws from (state, left, next); returns the advanced position
int mb_mt19937_fill(uint32_t* state624, int32_t* left, int32_t* next, uint32_t* out, uint64_t n) {
  if (!state624 || !left || !next || !out) return mb::fail(MB_ERR_INVALID, "mb_mt19937_fill: null argument");
  MtPos g;
  memcpy(g.s, state624, sizeof(uint32_t) * kN);
  g.avail = *left - 1;
  g.idx = *next;
  mt_fill(g, out, (size_t)n);
  memcpy(state624, g.s, sizeof(uint32_t) * kN);
  *left = g.avail + 1;
  *next = g.idx;
  return MB_OK;
}

// Several independent streams into one chunk of noise (the multi-utterance sample loop: one generator position per
// utterance).  Source s continues from (states[s], left[s], next[s]) and writes, for each of the first steps[s] steps j of the
// chunk, its words_per_step[s] draws at out[j * stride + col[s]]; the positions are advanced in place.  The sources are
// independent, so n_threads host threads take them one at a time from a shared counter.
int mb_mt19937_fill_sources(int32_t n_src, uint32_t* states, int32_t* left, int32_t* next, const uint64_t* words_per_step,
                            const uint64_t* col, const int32_t* steps, uint32_t* out, uint64_t stride, int32_t n_threads) {
  if (n_src <= 0 || !states || !left || !next || !words_per_step || !col || !steps || !out || n_threads <= 0)
    return mb::fail(MB_ERR_INVALID, "mb_mt19937_fill_sources: bad argument");
  for (int s = 0; s < n_src; ++s) {
    if (steps[s] < 0 || col[s] + words_per_step[s] > stride)
      return mb::fail(MB_ERR_INVALID, "mb_mt19937_fill_sources: source %d (columns [%llu, %llu)) outside the step of %llu words", s,
                      (unsigned long long)col[s], (unsigned long long)(col[s] + words_per_step[s]), (unsigned long long)stride);
    if (left[s] < 1 || left[s] > kN || next[s] < 0 || next[s] > kN || (left[s] > 1 && next[s] + (left[s] - 1) != kN))
      return mb::fail(MB_ERR_INVALID, "mb_mt19937_fill_sources: inconsistent generator position of source %d (left=%d next=%d)", s,
                      left[s], next[s]);
  }
  std::atomic<int> cursor{0};
  auto run = [&] {
    for (int s = cursor.fetch_add(1); s < n_src; s = cursor.fetch_add(1)) {
      MtPos g;
      memcpy(g.s, states + (size_t)s * kN, sizeof(uint32_t) * kN);
      g.avail = left[s] - 1;
      g.idx = next[s];
      for (int j = 0; j < steps[s]; ++j) mt_fill(g, out + (size_t)j * stride + col[s], (size_t)words_per_step[s]);
      memcpy(states + (size_t)s * kN, g.s, sizeof(uint32_t) * kN);
      left[s] = g.avail + 1;
      next[s] = g.idx;
    }
  };
  const int nt = n_threads < n_src ? n_threads : n_src;
  std::vector<std::thread> pool;
  for (int t = 1; t < nt; ++t) pool.emplace_back(run);
  run();
  for (auto& t : pool) t.join();
  return MB_OK;
}

// device conversion alone (test hook / callers that bring their own raw draws)
int mb_mt_to_exp(const void* dev_raw, float* dev_noise, uint64_t n_elems, void* stream) {
  if (!dev_raw || !dev_noise) return mb::fail(MB_ERR_INVALID, "mb_mt_to_exp: null argument");
  if (n_elems == 0) return MB_OK;
  mt_to_exp_kernel<false><<<(unsigned)((n_elems + 255) / 256), 256, 0, (cudaStream_t)stream>>>(reinterpret_cast<const uint2*>(dev_raw),
                                                                                              dev_noise, (size_t)n_elems);
  MB_LAUNCH_CHECK("mt_to_exp_kernel");
  return MB_OK;
}

int mb_mt_to_uniform(const void* dev_raw, float* dev_noise, uint64_t n_elems, void* stream) {
  if (!dev_raw || !dev_noise) return mb::fail(MB_ERR_INVALID, "mb_mt_to_uniform: null argument");
  if (n_elems == 0) return MB_OK;
  mt_to_uniform_kernel<false><<<(unsigned)((n_elems + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
      reinterpret_cast<const uint32_t*>(dev_raw), dev_noise, (size_t)n_elems);
  MB_LAUNCH_CHECK("mt_to_uniform_kernel");
  return MB_OK;
}

}  // extern "C"
