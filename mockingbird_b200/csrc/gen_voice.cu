// The text-to-speech chain's device steps between Tacotron and the levelling (gen_voice.py): DESIGN.md section 4p.
//
//   replaces  the trailing-silence trim of every synthesized spectrogram (synthesizer/inference.py:135-138) and gen_one_wav's
//             break assembly (gen_voice.py:30-34): the vocoded document cut at cumsum(frames) * hop_size with numpy's clamped
//             slicing, each piece followed by int(0.15 * sample_rate) zeros, the whole widened to float64
//
// tts_trim_kernel   one CTA per Tacotron row: the largest t <= row_frames[b] whose frame t - 1 is not silent, a frame being
//                   silent when every channel is < threshold (a NaN channel makes it not silent: numpy's max propagates NaN)
// tts_join_kernel   one CTA per work item (piece, tile of kJoinTile output samples): the piece's float32 samples widened to
//                   float64 (exact), then its zeros
#include <algorithm>
#include <vector>

#include "mb_common.h"

using namespace mb;

namespace {

constexpr int kTrimThreads = 256;
constexpr int kJoinThreads = 256;
constexpr int kJoinTile = 4 * kJoinThreads;  // output samples per work item

__global__ void __launch_bounds__(kTrimThreads) tts_trim_kernel(const float* __restrict__ lin, int32_t n_mels, int32_t frames,
                                                                const int32_t* __restrict__ row_frames, float threshold,
                                                                int32_t* __restrict__ trimmed) {
  __shared__ int32_t last;
  if (threadIdx.x == 0) last = 0;
  __syncthreads();
  const int32_t f = row_frames[blockIdx.x];
  const float* row = lin + (int64_t)blockIdx.x * n_mels * frames;
  int32_t mine = 0;  // 1 + the last loud frame this thread saw
  for (int32_t t = threadIdx.x; t < f; t += blockDim.x) {
    bool loud = false;
    for (int c = 0; c < n_mels && !loud; ++c) loud = !(row[(int64_t)c * frames + t] < threshold);
    if (loud) mine = t + 1;
  }
  if (mine) atomicMax(&last, mine);
  __syncthreads();
  if (threadIdx.x == 0) trimmed[blockIdx.x] = last;
}

struct JoinItem {
  const float* src;  // first sample of the piece (its clamped start in the vocoder row)
  int64_t dst;       // first output sample of the piece
  int32_t n, zeros;  // samples copied, zeros after them
  int32_t tile0;     // first work item of the piece
  int32_t pad;
};

__global__ void __launch_bounds__(kJoinThreads) tts_join_kernel(const JoinItem* __restrict__ items, int32_t n_items,
                                                                double* __restrict__ out) {
  int lo = 0, hi = n_items - 1;  // the piece of this work item: the last with tile0 <= blockIdx.x
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (items[mid].tile0 <= (int)blockIdx.x) lo = mid;
    else hi = mid - 1;
  }
  const JoinItem it = items[lo];
  const int64_t k0 = (int64_t)(blockIdx.x - it.tile0) * kJoinTile;
  const int64_t k1 = min(k0 + kJoinTile, (int64_t)it.n + it.zeros);
  for (int64_t k = k0 + threadIdx.x; k < k1; k += blockDim.x) out[it.dst + k] = k < it.n ? (double)it.src[k] : 0.0;
}

WsLayout trim_layout(int32_t batch) {
  WsLayout L;
  L.take<int32_t>(batch);  // row_frames
  return L;
}

WsLayout join_layout(int32_t n_pieces) {
  WsLayout L;
  L.take<JoinItem>(n_pieces);
  return L;
}

// the clamped cut of every piece and its place in the output: numpy's x[start:end] on a row of src_len samples
int join_plan(const char* fn, const mb_tts_piece* pieces, int32_t n_pieces, std::vector<JoinItem>* items, int64_t* tiles,
              int64_t* total) {
  if (!pieces) return fail(MB_ERR_INVALID, "%s: null piece table", fn);
  if (n_pieces < 1) return fail(MB_ERR_INVALID, "%s: n_pieces = %d", fn, (int)n_pieces);
  items->assign(n_pieces, JoinItem{});
  int64_t dst = 0, t = 0;
  for (int i = 0; i < n_pieces; ++i) {
    const mb_tts_piece& p = pieces[i];
    if (p.src_len < 0 || p.start < 0 || p.end < p.start || p.zeros < 0)
      return fail(MB_ERR_INVALID, "%s: piece %d: src_len = %lld, cut [%lld, %lld), zeros = %d (need 0 <= start <= end)", fn, i,
                  (long long)p.src_len, (long long)p.start, (long long)p.end, (int)p.zeros);
    if (p.src_len > 0 && !p.src) return fail(MB_ERR_INVALID, "%s: piece %d: null source row", fn, i);
    const int64_t a = std::min(p.start, p.src_len), b = std::min(p.end, p.src_len);
    if (b - a + p.zeros > INT32_MAX) return fail(MB_ERR_INVALID, "%s: piece %d is too long", fn, i);
    JoinItem& it = (*items)[i];
    it.src = p.src ? p.src + a : nullptr;
    it.n = (int32_t)(b - a);
    it.zeros = p.zeros;
    it.dst = dst;
    it.tile0 = (int32_t)t;
    dst += it.n + (int64_t)it.zeros;
    t += ((int64_t)it.n + it.zeros + kJoinTile - 1) / kJoinTile;
    if (t > INT32_MAX) return fail(MB_ERR_INVALID, "%s: too many output samples for one call", fn);
  }
  *tiles = t;
  *total = dst;
  return MB_OK;
}

}  // namespace

extern "C" {

size_t mb_tacotron_trim_workspace_bytes(int32_t batch) { return batch < 1 ? 0 : trim_layout(batch).total(); }

int mb_tacotron_trim_frames(const float* linear, int32_t batch, int32_t n_mels, int32_t frames, const int32_t* row_frames_host,
                            float threshold, int32_t* trimmed, void* workspace, size_t workspace_bytes, void* stream) {
  const char* fn = "mb_tacotron_trim_frames";
  if (!linear || !row_frames_host || !trimmed) return fail(MB_ERR_INVALID, "%s: null argument", fn);
  if (batch < 1 || n_mels < 1 || frames < 0)
    return fail(MB_ERR_INVALID, "%s: batch = %d, n_mels = %d, frames = %d", fn, (int)batch, (int)n_mels, (int)frames);
  for (int b = 0; b < batch; ++b)
    if (row_frames_host[b] < 0 || row_frames_host[b] > frames)
      return fail(MB_ERR_INVALID, "%s: row %d has %d frames of %d", fn, b, (int)row_frames_host[b], (int)frames);
  char* ws;
  if (int rc = bind(fn, workspace, workspace_bytes, mb_tacotron_trim_workspace_bytes(batch), &ws)) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  int32_t* rf = (int32_t*)ws;
  MB_CUDA_CHECK(cudaMemcpyAsync(rf, row_frames_host, sizeof(int32_t) * batch, cudaMemcpyHostToDevice, st));
  tts_trim_kernel<<<batch, kTrimThreads, 0, st>>>(linear, n_mels, frames, rf, threshold, trimmed);
  MB_LAUNCH_CHECK("tts_trim_kernel");
  return MB_OK;
}

int mb_tts_join_plan(const mb_tts_piece* pieces_host, int32_t n_pieces, int64_t* offsets_host) {
  if (!offsets_host) return fail(MB_ERR_INVALID, "mb_tts_join_plan: null argument");
  std::vector<JoinItem> items;
  int64_t tiles, total;
  if (int rc = join_plan("mb_tts_join_plan", pieces_host, n_pieces, &items, &tiles, &total)) return rc;
  for (int i = 0; i < n_pieces; ++i) offsets_host[i] = items[i].dst;
  offsets_host[n_pieces] = total;
  return MB_OK;
}

size_t mb_tts_join_workspace_bytes(int32_t n_pieces) { return n_pieces < 1 ? 0 : join_layout(n_pieces).total(); }

int mb_tts_join(const mb_tts_piece* pieces_host, int32_t n_pieces, double* out, void* workspace, size_t workspace_bytes,
                void* stream) {
  const char* fn = "mb_tts_join";
  if (!out) return fail(MB_ERR_INVALID, "%s: null argument", fn);
  std::vector<JoinItem> items;
  int64_t tiles, total;
  if (int rc = join_plan(fn, pieces_host, n_pieces, &items, &tiles, &total)) return rc;
  char* ws;
  if (int rc = bind(fn, workspace, workspace_bytes, mb_tts_join_workspace_bytes(n_pieces), &ws)) return rc;
  if (tiles == 0) return MB_OK;
  cudaStream_t st = (cudaStream_t)stream;
  MB_CUDA_CHECK(cudaMemcpyAsync(ws, items.data(), sizeof(JoinItem) * items.size(), cudaMemcpyHostToDevice, st));
  tts_join_kernel<<<(unsigned)tiles, kJoinThreads, 0, st>>>((const JoinItem*)ws, n_pieces, out);
  MB_LAUNCH_CHECK("tts_join_kernel");
  return MB_OK;
}

}  // extern "C"
