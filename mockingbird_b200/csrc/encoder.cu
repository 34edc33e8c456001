// Speaker encoder inference on H100 (mb_encoder_*): 3-layer LSTM over partial-utterance mel frames,
// last hidden state -> Linear -> ReLU -> L2 normalise; utterance embedding = L2(mean of partials).
//
// reference: models/encoder/model.py:41-61 (SpeakerEncoder.forward),
//            models/encoder/inference.py:51-64 (embed_frames_batch), :128-172 (embed_utterance)
//
// Layout: frames are [rows][T][C] (batch_first like nn.LSTM(batch_first=True)).  Per layer the input
// projection of the WHOLE sequence is one GEMM (M = rows*T); the recurrence then needs one
// [rows x H] x [H x 4H] GEMM per time step whose epilogue adds that step's projected input row, followed
// by the fused gate kernel that writes h_t straight into the layer's output sequence (the next step's
// GEMM operand, and the next layer's input).  When hidden_size % 64 == 0 the recurrent step is ONE launch of
// the tensor-core kernel tc_lstm_seq_kernel (tacotron_tc.cu: 3-term fp16 split, FP32-equivalent; cell update
// in the epilogue; h_t written as the next step's operand tiles); MB_ENC_TC=0 keeps the FFMA path.
// mb_encoder_embed_rows (many utterances, DESIGN.md section 4c): rows gathered on the device from a ragged frame buffer through
// a row table, each row's embedding taken at its own last step, and routes that never depend on the row count.
#include <climits>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include "../../include/mockingbird_b200.h"
#include "mb_common.h"
#include "tacotron_kernels.cuh"

using namespace mb;
using namespace mb::taco;

struct mb_encoder {
  mb_encoder_config cfg{};
  WeightTable w;
  bool finalized = false;
  float tc_inv_scale[8] = {1.f, 1.f, 1.f, 1.f, 1.f, 1.f, 1.f, 1.f};
  float big_inv_scale[8] = {1.f, 1.f, 1.f, 1.f, 1.f, 1.f, 1.f, 1.f};  // input-projection images (packed on first use)
  bool big_packed[8] = {false, false, false, false, false, false, false, false};
};

namespace {

float* P(const mb_encoder* h, const std::string& name) { return h->w.ptr(name); }

#define TK(expr)                                                                                          \
  do {                                                                                                    \
    cudaError_t _e = (expr);                                                                              \
    if (_e != cudaSuccess) return fail(MB_ERR_CUDA, "%s: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
    count_launch();                                                                                       \
  } while (0)

__device__ __forceinline__ float sigm(float x) { return 1.f / (1.f + expf(-x)); }

// ATen lstm_cell gate order [i, f, g, o]: c' = f*c + i*g, h' = o*tanh(c').  g: [M][4H] pre-activations
// (W_ih x + b_ih + W_hh h + b_hh); c: [M][H] in/out; h_out row m at h_out + m*ldh.
__global__ void enc_lstm_cell_kernel(const float* __restrict__ g, float* __restrict__ c, float* __restrict__ h_out,
                                     size_t ldh, int M, int H, int first) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= M * H) return;
  const int m = idx / H, j = idx - m * H;
  const float* gr = g + (size_t)m * 4 * H;
  const float ig = sigm(gr[j]), fg = sigm(gr[H + j]), gg = tanhf(gr[2 * H + j]), og = sigm(gr[3 * H + j]);
  const float cp = first ? 0.f : c[idx];
  const float cn = fg * cp + ig * gg;
  c[idx] = cn;
  h_out[(size_t)m * ldh + j] = og * tanhf(cn);
}

__global__ void add_vec_kernel(const float* a, const float* b, float* y, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) y[i] = a[i] + b[i];
}

// embeds[m] = raw[m] / (||raw[m]||_2 + 1e-5)   (model.py:58); one warp per row
__global__ void enc_l2norm_kernel(const float* __restrict__ raw, float* __restrict__ out, int M, int E) {
  const int m = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (m >= M) return;
  float s = 0.f;
  for (int j = lane; j < E; j += 32) {
    const float v = raw[(size_t)m * E + j];
    s = fmaf(v, v, s);
  }
  for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  const float inv = 1.f / (sqrtf(s) + 1e-5f);
  for (int j = lane; j < E; j += 32) out[(size_t)m * E + j] = raw[(size_t)m * E + j] * inv;
}

// utterance embedding (inference.py:164-166): raw = mean over the utterance's partial embeddings,
// embed = raw / ||raw||_2.  offsets: CSR [U+1] into the partial rows.  One warp per utterance.
__global__ void enc_reduce_kernel(const float* __restrict__ partial, const int32_t* __restrict__ offsets,
                                  float* __restrict__ out, int U, int E) {
  const int u = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (u >= U) return;
  const int p0 = offsets[u], p1 = offsets[u + 1];
  const float invn = 1.f / (float)(p1 - p0);
  float s = 0.f;
  for (int j = lane; j < E; j += 32) {
    float a = 0.f;
    for (int p = p0; p < p1; ++p) a += partial[(size_t)p * E + j];
    a *= invn;
    out[(size_t)u * E + j] = a;
    s = fmaf(a, a, s);
  }
  for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  const float inv = 1.f / sqrtf(s);
  for (int j = lane; j < E; j += 32) out[(size_t)u * E + j] *= inv;
}

// mb_encoder_embed_rows: tab = row_start [R] | row_len [R].  x[r][t] = frames[row_start[r] + t] for t < row_len[r], else 0
__global__ void enc_gather_rows_kernel(const float* __restrict__ frames, const int32_t* __restrict__ tab, float* __restrict__ x,
                                       int R, int T, int C) {
  const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (size_t)R * T * C) return;
  const int r = (int)(idx / ((size_t)T * C));
  const int rem = (int)(idx - (size_t)r * T * C), t = rem / C, k = rem - t * C;
  x[idx] = t < tab[R + r] ? frames[((size_t)tab[r] + t) * C + k] : 0.f;
}

// last[r] = seq[r][row_len[r] - 1]: each row's top-layer hidden state at its own last step (the LSTM is causal, so the steps
// past a row's end do not reach it)
__global__ void enc_gather_last_kernel(const float* __restrict__ seq, const int32_t* __restrict__ tab, float* __restrict__ last,
                                       int R, int T, int H) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= R * H) return;
  const int r = idx / H, j = idx - r * H;
  last[idx] = seq[((size_t)r * T + tab[R + r] - 1) * H + j];
}

GemmArgs gemm1(const float* x, int K, int ld, const float* W, int ldw, const float* bias, int M, int N, float* Y,
               int ldy, int act = ACT_NONE) {
  GemmArgs a;
  memset(&a, 0, sizeof(a));
  a.nseg = 1;
  a.seg[0] = {x, K, ld, 0, 0, 1};
  a.W = W;
  a.ldw = ldw;
  a.bias = bias;
  a.M = M;
  a.N = N;
  a.T = 1;
  a.act = act;
  a.Y = Y;
  a.ldy = ldy;
  return a;
}

struct Ws {
  size_t xproj, seq0, seq1, gates, c, raw, t_hi, t_lo, big_hi, big_lo;  // float offsets
  size_t total;                                                         // bytes
  size_t in, last, tab;  // mb_encoder_embed_rows only: gathered input [R][T][C], last hidden rows [R][H], row table [2][R]
};

bool enc_use_tc(const mb_encoder_config& c) {
  static const bool env = [] {
    const char* e = getenv("MB_ENC_TC");
    return e ? atoi(e) != 0 : true;
  }();
  return env && c.hidden_size % 64 == 0;
}

Ws ws_layout(const mb_encoder_config& c, size_t R, size_t T, bool rows = false) {
  Ws L;
  L.in = L.last = L.tab = 0;
  WsLayout W;
  const size_t H = c.hidden_size;
  L.xproj = W.take<float>(R * T * 4 * H);
  L.seq0 = W.take<float>(R * T * H);
  L.seq1 = W.take<float>(R * T * H);
  L.gates = W.take<float>(R * 4 * H);
  L.c = W.take<float>(R * H);
  L.raw = W.take<float>(R * (size_t)c.embedding_size);
  const size_t rows_total = (R + 127) / 128 * 128;
  const size_t tile_floats = (H / 64) * rows_total * 128 / 4;  // one operand plane (hi or lo) of h, in floats
  L.t_hi = W.take<float>(2 * tile_floats);  // two parities
  L.t_lo = W.take<float>(2 * tile_floats);
  const int kmax = c.hidden_size > c.mel_n_channels ? c.hidden_size : c.mel_n_channels;
  // operand tiles of the whole-sequence input projection
  L.big_hi = W.take<float>(tc_big_act_bytes((int)(R * T), 1, kmax) / 4);
  L.big_lo = W.take<float>(tc_big_act_bytes((int)(R * T), 1, kmax) / 4);
  if (rows) {
    L.in = W.take<float>(R * T * (size_t)c.mel_n_channels);
    L.last = W.take<float>(R * H);
    L.tab = W.take<float>(2 * R);
  }
  L.total = W.total();
  return L;
}

// The LSTM stack over frames [R][T][C]; *top = the last layer's output sequence [R][T][H].  fixed_route: every launch takes a
// route chosen without looking at R or T (tc_big input projections and tc_lstm_seq steps, or with MB_ENC_TC=0 fma_chain
// GEMMs), so a row's bits do not depend on how many rows share the call; otherwise the input projection takes tc_big only
// from 512 rows*frames and launch_gemm picks its kernel by M.
int run_layers(mb_encoder* h, const float* frames, int R, int T, const Ws& L, float* ws, bool fixed_route, const float** top,
               cudaStream_t st) {
  const mb_encoder_config& c = h->cfg;
  const int H = c.hidden_size, C = c.mel_n_channels;
  const float* in = frames;
  int in_dim = C;
  float* seq[2] = {ws + L.seq0, ws + L.seq1};
  for (int l = 0; l < c.num_layers; ++l) {
    const std::string s = std::to_string(l);
    float* outseq = seq[l & 1];
    // input projection of the whole sequence: xproj[r*T + t] = W_ih x_t + (b_ih + b_hh)
    if (enc_use_tc(c) && (fixed_route || (size_t)R * T >= 512)) {
      // whole-sequence input projection on the 128x128-tile tensor-core GEMM (3-term split; images packed on first use)
      __half* wimg = reinterpret_cast<__half*>(P(h, "lstm.ih_bigw_l" + s));
      const int KBs = (in_dim + 63) / 64;
      if (!h->big_packed[l]) {
        unsigned int* dmax = reinterpret_cast<unsigned int*>(P(h, "scratch.absmax.bias_sum"));
        MB_CUDA_CHECK(cudaMemsetAsync(dmax, 0, sizeof(unsigned int), st));
        TK(tc_skinny_absmax(P(h, "lstm.weight_ih_l" + s), (size_t)4 * H * in_dim, dmax, st));
        unsigned int hmax = 0;
        MB_CUDA_CHECK(cudaMemcpyAsync(&hmax, dmax, sizeof(hmax), cudaMemcpyDeviceToHost, st));
        MB_CUDA_CHECK(cudaStreamSynchronize(st));
        TcBigPack q;
        memset(&q, 0, sizeof(q));
        q.W = P(h, "lstm.weight_ih_l" + s);
        q.ldw = in_dim;
        q.N = 4 * H;
        q.nseg = 1;
        q.K = in_dim;
        q.KBs = KBs;
        q.w_off[0] = 0;
        q.w_stride[0] = 1;
        q.scale = tc_weight_scale(hmax);
        h->big_inv_scale[l] = 1.f / q.scale;
        TK(launch_pack_big_w(q, wimg, st));
        h->big_packed[l] = true;
      }
      TcIm2col q;
      memset(&q, 0, sizeof(q));
      q.x[0] = in;
      q.ld[0] = in_dim;
      q.nseg = 1;
      q.K = in_dim;
      q.KBs = KBs;
      q.M = R * T;
      q.T = 1;
      q.rows_total = (R * T + 127) / 128 * 128;
      TK(launch_im2col_split(q, reinterpret_cast<__half*>(ws + L.big_hi), reinterpret_cast<__half*>(ws + L.big_lo), st));
      TcBigArgs t;
      memset(&t, 0, sizeof(t));
      t.a_hi = reinterpret_cast<const __half*>(ws + L.big_hi);
      t.a_lo = reinterpret_cast<const __half*>(ws + L.big_lo);
      t.w = wimg;
      t.bias = P(h, "lstm.bias_sum_l" + s);
      t.KB = KBs;
      t.M = R * T;
      t.N = 4 * H;
      t.rows_total = q.rows_total;
      t.act = ACT_NONE;
      t.inv_scale = h->big_inv_scale[l];
      t.y = ws + L.xproj;
      t.ldy = 4 * H;
      TK(launch_tc_big(t, st));
    } else {
      GemmArgs a = gemm1(in, in_dim, in_dim, P(h, "lstm.weight_ih_l" + s), in_dim, P(h, "lstm.bias_sum_l" + s), R * T, 4 * H,
                         ws + L.xproj, 4 * H);
      a.fma_chain = fixed_route;
      TK(launch_gemm(a, st));
    }
    const float* whh = P(h, "lstm.weight_hh_l" + s);
    if (enc_use_tc(c)) {
      const size_t rows_total = ((size_t)R + 127) / 128 * 128;
      const size_t tile_bytes = (size_t)(H / 64) * rows_total * 128;
      MB_CUDA_CHECK(cudaMemsetAsync(ws + L.t_hi, 0, 2 * tile_bytes, st));  // h_{-1} = 0 (and the rows past R)
      MB_CUDA_CHECK(cudaMemsetAsync(ws + L.t_lo, 0, 2 * tile_bytes, st));
      MB_CUDA_CHECK(cudaMemsetAsync(ws + L.c, 0, sizeof(float) * (size_t)R * H, st));
      TcLstmSeqArgs ta;
      memset(&ta, 0, sizeof(ta));
      ta.w = reinterpret_cast<const __half*>(P(h, "lstm.hh_tcw_l" + s));
      ta.c = ws + L.c;
      ta.inv_scale = h->tc_inv_scale[l];
      ta.ldgi = T * 4 * H;
      ta.ldout = T * H;
      ta.KB = H / 64;
      ta.M = R;
      ta.H = H;
      ta.rows_total = (int)rows_total;
      for (int t = 0; t < T; ++t) {
        const int par = t & 1;
        ta.a_hi = reinterpret_cast<const __half*>(reinterpret_cast<const char*>(ws + L.t_hi) + par * tile_bytes);
        ta.a_lo = reinterpret_cast<const __half*>(reinterpret_cast<const char*>(ws + L.t_lo) + par * tile_bytes);
        ta.nxt_hi = reinterpret_cast<__half*>(reinterpret_cast<char*>(ws + L.t_hi) + (par ^ 1) * tile_bytes);
        ta.nxt_lo = reinterpret_cast<__half*>(reinterpret_cast<char*>(ws + L.t_lo) + (par ^ 1) * tile_bytes);
        ta.gi = ws + L.xproj + (size_t)t * 4 * H;
        ta.out = outseq + (size_t)t * H;
        TK(launch_tc_lstm_seq(ta, st));
      }
      in = outseq;
      in_dim = H;
      continue;
    }
    for (int t = 0; t < T; ++t) {
      const float* g = ws + L.xproj + (size_t)t * 4 * H;  // row r of step t at + r*T*4H
      size_t ldg = (size_t)T * 4 * H;
      if (t > 0) {
        GemmArgs b = gemm1(outseq + (size_t)(t - 1) * H, H, T * H, whh, H, nullptr, R, 4 * H, ws + L.gates, 4 * H);
        b.res = g;
        b.ldres = (int)ldg;
        b.fma_chain = fixed_route;
        TK(launch_gemm(b, st));
        g = ws + L.gates;
        ldg = 4 * H;
      }
      if (ldg == (size_t)4 * H) {
        enc_lstm_cell_kernel<<<(R * H + 255) / 256, 256, 0, st>>>(g, ws + L.c, outseq + (size_t)t * H, (size_t)T * H, R, H, 0);
      } else {
        // t == 0: h_{-1} = 0, the gates are the projected input alone; copy rows into the dense gate buffer
        MB_CUDA_CHECK(cudaMemcpy2DAsync(ws + L.gates, (size_t)4 * H * 4, g, ldg * 4, (size_t)4 * H * 4, R,
                                        cudaMemcpyDeviceToDevice, st));
        enc_lstm_cell_kernel<<<(R * H + 255) / 256, 256, 0, st>>>(ws + L.gates, ws + L.c, outseq, (size_t)T * H, R, H, 1);
      }
      MB_LAUNCH_CHECK("enc_lstm_cell_kernel");
    }
    in = outseq;
    in_dim = H;
  }
  *top = in;
  return MB_OK;
}

}  // namespace

extern "C" {

int mb_encoder_create(const mb_encoder_config* cfg, mb_encoder** out) {
  if (!cfg || !out) return fail(MB_ERR_INVALID, "mb_encoder_create: null argument");
  const mb_encoder_config& c = *cfg;
  if (c.mel_n_channels <= 0 || c.hidden_size <= 0 || c.num_layers <= 0 || c.num_layers > 8 || c.embedding_size <= 0)
    return fail(MB_ERR_INVALID, "mb_encoder_create: unsupported hyper-parameters");
  mb_encoder* h = new mb_encoder();
  h->cfg = c;
  const int H = c.hidden_size;
  WeightTable& w = h->w;
  w.add_derived("scratch.absmax.bias_sum", 64);  // device scratch of the weight-image packers (no cudaMalloc after create)
  for (int l = 0; l < c.num_layers; ++l) {
    const int in = l == 0 ? c.mel_n_channels : H;
    const std::string s = std::to_string(l);
    w.add("lstm.weight_ih_l" + s, {4 * H, in});
    w.add("lstm.weight_hh_l" + s, {4 * H, H});
    w.add("lstm.bias_ih_l" + s, {4 * H});
    w.add("lstm.bias_hh_l" + s, {4 * H});
    w.add_derived("lstm.bias_sum_l" + s, 4 * H);                          // b_ih + b_hh
    w.add_derived("lstm.hh_tcw_l" + s, tc_gated_weight_bytes(H, H) / 4);  // tensor-core images of W_hh
    w.add_derived("lstm.hh_tcb_l" + s, 4 * H);                            // (unused zero bias of the images)
    w.add_derived("lstm.ih_bigw_l" + s, tc_big_weight_bytes(4 * H, 1, in) / 4);  // images of W_ih
  }
  w.add("linear.weight", {c.embedding_size, H});
  w.add("linear.bias", {c.embedding_size});
  *out = h;
  return MB_OK;
}

void mb_encoder_destroy(mb_encoder* h) { delete h; }

size_t mb_encoder_arena_bytes(const mb_encoder* h) { return h ? h->w.floats() * sizeof(float) : 0; }

int mb_encoder_set_arena(mb_encoder* h, void* arena, size_t bytes) {
  if (int rc = check_arena("mb_encoder_set_arena", h, arena, bytes, mb_encoder_arena_bytes(h), 256)) return rc;
  h->w.attach((float*)arena);
  h->finalized = false;
  for (bool& b : h->big_packed) b = false;  // a new arena holds none of the lazily packed images
  return MB_OK;
}

int mb_encoder_set_weight(mb_encoder* h, const char* name, const float* w, const int64_t* dims, int32_t ndim,
                          void* stream) {
  if (!h) return fail(MB_ERR_INVALID, "mb_encoder_set_weight: null argument");
  if (int rc = h->w.set("mb_encoder_set_weight", name, w, dims, ndim, stream)) return rc;
  h->finalized = false;
  for (bool& b : h->big_packed) b = false;  // images packed from the previous weights are stale
  return MB_OK;
}

int mb_encoder_finalize(mb_encoder* h, void* stream) {
  if (!h) return fail(MB_ERR_INVALID, "mb_encoder_finalize: null handle");
  cudaStream_t st = (cudaStream_t)stream;
  if (int rc = h->w.check_all_set("mb_encoder_finalize")) return rc;
  const int n = 4 * h->cfg.hidden_size;
  for (int l = 0; l < h->cfg.num_layers; ++l) {
    const std::string s = std::to_string(l);
    add_vec_kernel<<<(n + 255) / 256, 256, 0, st>>>(P(h, "lstm.bias_ih_l" + s), P(h, "lstm.bias_hh_l" + s),
                                                    P(h, "lstm.bias_sum_l" + s), n);
    MB_LAUNCH_CHECK("add_vec_kernel");
  }
  if (enc_use_tc(h->cfg)) {
    // tensor-core images of every W_hh (power-of-two scale from max |w|, tc_weight_scale)
    const int H = h->cfg.hidden_size;
    unsigned int* dmax = reinterpret_cast<unsigned int*>(P(h, "scratch.absmax.bias_sum"));
    MB_CUDA_CHECK(cudaMemsetAsync(dmax, 0, 8 * sizeof(unsigned int), st));
    for (int l = 0; l < h->cfg.num_layers; ++l)
      TK(tc_skinny_absmax(P(h, "lstm.weight_hh_l" + std::to_string(l)), (size_t)4 * H * H, dmax + l, st));
    unsigned int hmax[8] = {0};
    MB_CUDA_CHECK(cudaMemcpyAsync(hmax, dmax, sizeof(hmax), cudaMemcpyDeviceToHost, st));
    MB_CUDA_CHECK(cudaStreamSynchronize(st));
    for (int l = 0; l < h->cfg.num_layers; ++l) {
      const float scale = tc_weight_scale(hmax[l]);
      h->tc_inv_scale[l] = 1.f / scale;
      const std::string s = std::to_string(l);
      TK(tc_skinny_pack(P(h, "lstm.weight_hh_l" + s), H, nullptr, 0, nullptr, nullptr, 4 * H, H, scale,
                        reinterpret_cast<__half*>(P(h, "lstm.hh_tcw_l" + s)), P(h, "lstm.hh_tcb_l" + s), st));
    }
  }
  h->finalized = true;
  return MB_OK;
}

size_t mb_encoder_workspace_bytes(const mb_encoder* h, int32_t rows, int32_t n_frames) {
  if (!h || rows <= 0 || n_frames <= 0) return 0;
  return ws_layout(h->cfg, rows, n_frames).total;
}

int mb_encoder_embed_frames(mb_encoder* h, const float* frames, int32_t rows, int32_t n_frames, float* embeds,
                            void* workspace, size_t workspace_bytes, void* stream) {
  if (!h || !frames || !embeds) return fail(MB_ERR_INVALID, "mb_encoder_embed_frames: null argument");
  if (!h->finalized) return fail(MB_ERR_STATE, "mb_encoder_embed_frames: weights not finalized");
  if (rows <= 0 || n_frames <= 0) return fail(MB_ERR_INVALID, "mb_encoder_embed_frames: bad shape");
  const mb_encoder_config& c = h->cfg;
  const Ws L = ws_layout(c, rows, n_frames);
  float* ws;
  if (int rc = bind("mb_encoder_embed_frames", workspace, workspace_bytes, L.total, &ws)) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  const int R = rows, T = n_frames, H = c.hidden_size, E = c.embedding_size;
  const float* top = nullptr;
  if (int rc = run_layers(h, frames, R, T, L, ws, false, &top, st)) return rc;
  // hidden[-1] = last layer's h at t = T-1 -> relu(linear) -> L2 normalise
  GemmArgs e = gemm1(top + (size_t)(T - 1) * H, H, T * H, P(h, "linear.weight"), H, P(h, "linear.bias"), R, E, ws + L.raw, E,
                     ACT_RELU);
  TK(launch_gemm(e, st));
  enc_l2norm_kernel<<<(R + 7) / 8, 256, 0, st>>>(ws + L.raw, embeds, R, E);
  MB_LAUNCH_CHECK("enc_l2norm_kernel");
  return MB_OK;
}

size_t mb_encoder_rows_workspace_bytes(const mb_encoder* h, int32_t rows, int32_t max_len) {
  if (!h || rows <= 0 || max_len <= 0) return 0;
  return ws_layout(h->cfg, rows, max_len, true).total;
}

int mb_encoder_embed_rows(mb_encoder* h, const float* frames, int64_t n_frames, const int32_t* row_start_host,
                          const int32_t* row_len_host, int32_t rows, float* embeds, void* workspace, size_t workspace_bytes,
                          void* stream) {
  const char* fn = "mb_encoder_embed_rows";
  if (!h || !frames || !row_start_host || !row_len_host || !embeds) return fail(MB_ERR_INVALID, "%s: null argument", fn);
  if (!h->finalized) return fail(MB_ERR_STATE, "%s: weights not finalized", fn);
  if (rows <= 0) return fail(MB_ERR_INVALID, "%s: rows = %d", fn, (int)rows);
  const mb_encoder_config& c = h->cfg;
  const int R = rows, H = c.hidden_size, C = c.mel_n_channels, E = c.embedding_size;
  int T = 0;
  std::vector<int32_t> tab(2 * (size_t)R);
  for (int r = 0; r < R; ++r) {
    const int32_t s0 = row_start_host[r], n = row_len_host[r];
    if (n <= 0 || s0 < 0 || (int64_t)s0 + n > n_frames)
      return fail(MB_ERR_INVALID, "%s: row %d = frames [%d, %d + %d) is empty or outside the %lld frames", fn, r, (int)s0,
                  (int)s0, (int)n, (long long)n_frames);
    tab[r] = s0;
    tab[R + r] = n;
    T = n > T ? n : T;
  }
  if ((int64_t)R * T * 4 * H > INT32_MAX) return fail(MB_ERR_INVALID, "%s: %d rows of up to %d frames are too many for one call", fn, R, T);
  const Ws L = ws_layout(c, R, T, true);
  float* ws;
  if (int rc = bind(fn, workspace, workspace_bytes, L.total, &ws)) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  int32_t* dtab = reinterpret_cast<int32_t*>(ws + L.tab);
  MB_CUDA_CHECK(cudaMemcpyAsync(dtab, tab.data(), tab.size() * sizeof(int32_t), cudaMemcpyHostToDevice, st));
  const size_t n_in = (size_t)R * T * C;
  enc_gather_rows_kernel<<<(unsigned)((n_in + 255) / 256), 256, 0, st>>>(frames, dtab, ws + L.in, R, T, C);
  MB_LAUNCH_CHECK("enc_gather_rows_kernel");
  const float* top = nullptr;
  if (int rc = run_layers(h, ws + L.in, R, T, L, ws, true, &top, st)) return rc;
  enc_gather_last_kernel<<<(R * H + 255) / 256, 256, 0, st>>>(top, dtab, ws + L.last, R, T, H);
  MB_LAUNCH_CHECK("enc_gather_last_kernel");
  GemmArgs e = gemm1(ws + L.last, H, H, P(h, "linear.weight"), H, P(h, "linear.bias"), R, E, ws + L.raw, E, ACT_RELU);
  e.fma_chain = 1;
  TK(launch_gemm(e, st));
  enc_l2norm_kernel<<<(R + 7) / 8, 256, 0, st>>>(ws + L.raw, embeds, R, E);
  MB_LAUNCH_CHECK("enc_l2norm_kernel");
  return MB_OK;
}

int mb_encoder_reduce_partials(mb_encoder* h, const float* partial_embeds, const int32_t* offsets, int32_t n_utterances,
                               float* utterance_embeds, void* stream) {
  if (!h || !partial_embeds || !offsets || !utterance_embeds)
    return fail(MB_ERR_INVALID, "mb_encoder_reduce_partials: null argument");
  if (n_utterances <= 0) return fail(MB_ERR_INVALID, "mb_encoder_reduce_partials: bad shape");
  enc_reduce_kernel<<<(n_utterances + 7) / 8, 256, 0, (cudaStream_t)stream>>>(partial_embeds, offsets, utterance_embeds,
                                                                             n_utterances, h->cfg.embedding_size);
  MB_LAUNCH_CHECK("enc_reduce_kernel");
  return MB_OK;
}

}  // extern "C"
