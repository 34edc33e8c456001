// mb_taco_tc_debug: one launch of a 3-term-split tensor-core GEMM (tacotron_tc.cu) on caller-provided fp32 tensors, prepared by the
// same functions and in the same order as the forward: absmax -> tc_weight_scale -> weight pack -> operand split -> launch.  Lets
// the tests compare each kernel, at shapes and launch variants the models never reach, with a float64 reference of its operation.
#include <cuda_fp16.h>

#include <cstdio>
#include <cstring>

#include "mb_common.h"
#include "tacotron_kernels.cuh"

namespace mb {
namespace taco {
namespace {

#define TK(expr)                                                                                                           \
  do {                                                                                                                     \
    cudaError_t _e = (expr);                                                                                               \
    if (_e != cudaSuccess) return fail(MB_ERR_CUDA, "%s: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
    count_launch();                                                                                                        \
  } while (0)

struct DebugWs {      // byte offsets into the workspace (256-byte aligned)
  size_t absmax;      // 2 x uint
  size_t w[2], bias[2], a_hi[2], a_lo[2], nxt_hi[2], nxt_lo[2];
  size_t w_bytes, bias_bytes, a_bytes;  // per direction
  size_t total;
};

int spec_K(const mb_taco_tc_debug_spec& s) { return s.kind <= MB_TACO_TC_SKINNY_LSTM ? s.K0 + s.K1 : s.K0; }

DebugWs debug_layout(const mb_taco_tc_debug_spec& s) {
  DebugWs L;
  memset(&L, 0, sizeof(L));
  const int K = spec_K(s);
  const int ndir = s.kind == MB_TACO_TC_GRU ? s.ndir : 1;
  switch (s.kind) {
    case MB_TACO_TC_SKINNY_PLAIN:
      L.w_bytes = tc_skinny_weight_bytes(s.N, K);
      L.bias_bytes = (size_t)(s.N + 31) / 32 * 32 * 4;
      L.a_bytes = tc_skinny_act_bytes(s.M, K);
      break;
    case MB_TACO_TC_SKINNY_LSTM:
    case MB_TACO_TC_GRU:
      L.w_bytes = tc_gated_weight_bytes(s.H, K);
      L.bias_bytes = (size_t)4 * s.H * 4;
      L.a_bytes = tc_skinny_act_bytes(s.M, K);
      break;
    case MB_TACO_TC_LSTM_SEQ:
      L.w_bytes = tc_gated_weight_bytes(s.H, K);
      L.bias_bytes = (size_t)4 * s.H * 4;
      L.a_bytes = tc_big_act_bytes(s.M, 1, K);
      break;
    default:
      L.w_bytes = tc_big_weight_bytes(s.N, s.nseg, K);
      L.a_bytes = tc_big_act_bytes(s.M, s.nseg, K);
      break;
  }
  size_t off = 0;
  auto take = [&](size_t bytes) {
    const size_t o = off;
    off += align_up(bytes > 0 ? bytes : 1, 256);
    return o;
  };
  L.absmax = take(2 * sizeof(unsigned int));
  for (int d = 0; d < ndir; ++d) {
    L.w[d] = take(L.w_bytes);
    L.bias[d] = take(L.bias_bytes);
    L.a_hi[d] = take(L.a_bytes);
    L.a_lo[d] = take(L.a_bytes);
    L.nxt_hi[d] = take(L.a_bytes);
    L.nxt_lo[d] = take(L.a_bytes);
  }
  L.total = off + 256;
  return L;
}

int check_spec(const mb_taco_tc_debug_spec& s) {
  const char* me = "mb_taco_tc_debug";
  if (s.kind < MB_TACO_TC_SKINNY_PLAIN || s.kind > MB_TACO_TC_BIG) return fail(MB_ERR_INVALID, "%s: bad kind %d", me, s.kind);
  if (s.M <= 0 || s.K0 <= 0 || s.K1 < 0 || !s.w[0] || !s.x[0]) return fail(MB_ERR_INVALID, "%s: empty shape or null operand", me);
  const bool gated = s.kind != MB_TACO_TC_SKINNY_PLAIN && s.kind != MB_TACO_TC_BIG;
  if (gated && (s.H <= 0 || s.H % 8)) return fail(MB_ERR_INVALID, "%s: H = %d must be a positive multiple of 8", me, s.H);
  if (!gated && s.N <= 0) return fail(MB_ERR_INVALID, "%s: N = %d", me, s.N);
  if (s.kind == MB_TACO_TC_GRU || s.kind == MB_TACO_TC_LSTM_SEQ) {
    if (s.K0 != s.H || s.K1 != 0 || s.H % 64) return fail(MB_ERR_INVALID, "%s: recurrent K must be H (a multiple of 64)", me);
  }
  if (s.kind == MB_TACO_TC_GRU && (s.ndir < 1 || s.ndir > 2 || (s.ndir == 2 && (!s.w[1] || !s.x[1]))))
    return fail(MB_ERR_INVALID, "%s: ndir %d", me, s.ndir);
  if (s.kind == MB_TACO_TC_BIG && (s.nseg < 1 || s.nseg > kMaxSeg || s.T < 1))
    return fail(MB_ERR_INVALID, "%s: nseg %d / T %d", me, s.nseg, s.T);
  if (s.kind <= MB_TACO_TC_GRU && s.M > 128) return fail(MB_ERR_INVALID, "%s: M = %d > 128 for a skinny kernel", me, s.M);
  if (s.cluster != 0 && s.cluster != 1 && s.cluster != 2 && s.cluster != 4 && s.cluster != 8)
    return fail(MB_ERR_INVALID, "%s: cluster %d", me, s.cluster);
  return MB_OK;
}

int env_flag(const char* name, int dflt) {
  const char* e = getenv(name);
  return e ? (atoi(e) != 0) : dflt;
}

}  // namespace
}  // namespace taco
}  // namespace mb

using namespace mb;
using namespace mb::taco;

extern "C" {

size_t mb_taco_tc_debug_workspace_bytes(const mb_taco_tc_debug_spec* spec) {
  if (!spec || check_spec(*spec) != MB_OK) return 0;
  return debug_layout(*spec).total;
}

int mb_taco_tc_debug(const mb_taco_tc_debug_spec* spec, void* workspace, size_t workspace_bytes, void* stream, char* report,
                     size_t report_len) {
  if (!spec || !workspace) return fail(MB_ERR_INVALID, "mb_taco_tc_debug: null argument");
  const mb_taco_tc_debug_spec& s = *spec;
  int rc = check_spec(s);
  if (rc != MB_OK) return rc;
  const DebugWs L = debug_layout(s);
  if (workspace_bytes < L.total) return fail(MB_ERR_WORKSPACE, "mb_taco_tc_debug: workspace %zu < %zu bytes", workspace_bytes, L.total);
  char* ws = (char*)(((uintptr_t)workspace + 255) & ~(uintptr_t)255);
  cudaStream_t st = (cudaStream_t)stream;
  auto half_at = [&](size_t off) { return reinterpret_cast<__half*>(ws + off); };
  const int K = spec_K(s);
  const int KB = (K + 63) / 64;
  const int ndir = s.kind == MB_TACO_TC_GRU ? s.ndir : 1;
  const int rows_w = s.kind == MB_TACO_TC_SKINNY_PLAIN || s.kind == MB_TACO_TC_BIG ? s.N
                     : s.kind == MB_TACO_TC_GRU                                    ? 3 * s.H
                                                                                   : 4 * s.H;

  // 1. max |w| of every weight image, 2. its power-of-two scale (one host read-back, as at finalize / first use)
  unsigned int* dmax = reinterpret_cast<unsigned int*>(ws + L.absmax);
  MB_CUDA_CHECK(cudaMemsetAsync(dmax, 0, 2 * sizeof(unsigned int), st));
  for (int d = 0; d < ndir; ++d) {
    if (s.kind == MB_TACO_TC_BIG) {
      TK(tc_skinny_absmax(s.w[0], (size_t)s.N * s.ldw, dmax, st));
    } else if (s.kind == MB_TACO_TC_GRU) {
      TK(tc_skinny_absmax(s.w[d], (size_t)rows_w * K, dmax + d, st));
    } else {
      TK(tc_skinny_absmax(s.w[0], (size_t)rows_w * s.K0, dmax, st));
      if (s.w[1] && s.K1 > 0) TK(tc_skinny_absmax(s.w[1], (size_t)rows_w * s.K1, dmax, st));
    }
  }
  unsigned int hmax[2] = {0, 0};
  MB_CUDA_CHECK(cudaMemcpyAsync(hmax, dmax, sizeof(hmax), cudaMemcpyDeviceToHost, st));
  MB_CUDA_CHECK(cudaStreamSynchronize(st));
  float scale[2];
  for (int d = 0; d < 2; ++d) scale[d] = tc_weight_scale(hmax[d]);

  // 3. weight images, 4. operand tiles, 5. the launch
  const int pdl = s.pdl < 0 ? -1 : s.pdl;
  TcLaunchInfo info;
  memset(&info, 0, sizeof(info));
  const char* kname = "";
  if (s.kind == MB_TACO_TC_BIG) {
    TcBigPack q;
    memset(&q, 0, sizeof(q));
    q.W = s.w[0];
    q.ldw = s.ldw;
    q.N = s.N;
    q.nseg = s.nseg;
    q.K = K;
    q.KBs = KB;
    for (int g = 0; g < s.nseg; ++g) {
      q.w_off[g] = s.w_off[g];
      q.w_stride[g] = s.w_stride[g];
    }
    q.scale = scale[0];
    TK(launch_pack_big_w(q, half_at(L.w[0]), st));
    TcIm2col c;
    memset(&c, 0, sizeof(c));
    for (int g = 0; g < s.nseg; ++g) {
      c.x[g] = s.x[g];
      c.ld[g] = s.ldx[g];
      c.shift[g] = s.shift[g];
    }
    c.nseg = s.nseg;
    c.K = K;
    c.KBs = KB;
    c.M = s.M;
    c.T = s.T;
    c.rows_total = (s.M + 127) / 128 * 128;
    TK(launch_im2col_split(c, half_at(L.a_hi[0]), half_at(L.a_lo[0]), st));
    TcBigArgs t;
    memset(&t, 0, sizeof(t));
    t.a_hi = half_at(L.a_hi[0]);
    t.a_lo = half_at(L.a_lo[0]);
    t.w = half_at(L.w[0]);
    t.bias = s.b[0];
    t.KB = s.nseg * KB;
    t.M = s.M;
    t.N = s.N;
    t.rows_total = c.rows_total;
    t.act = s.act;
    t.inv_scale = 1.f / scale[0];
    t.bn_scale = s.bn_scale;
    t.bn_shift = s.bn_shift;
    t.res = s.res;
    t.ldres = s.ldres;
    t.y = s.y;
    t.ldy = s.ldy;
    TK(launch_tc_big(t, st, pdl, &info));
    kname = "tc_big";
  } else if (s.kind == MB_TACO_TC_LSTM_SEQ) {
    TK(tc_skinny_pack(s.w[0], K, nullptr, 0, nullptr, nullptr, 4 * s.H, s.H, scale[0], half_at(L.w[0]),
                      reinterpret_cast<float*>(ws + L.bias[0]), st));
    // h_{t-1} as the [KB][ceil128(M)][64] tiles a previous step's epilogue leaves (an im2col with one unshifted segment)
    TcIm2col c;
    memset(&c, 0, sizeof(c));
    c.x[0] = s.x[0];
    c.ld[0] = s.ldx[0];
    c.nseg = 1;
    c.K = K;
    c.KBs = KB;
    c.M = s.M;
    c.T = 1;
    c.rows_total = (s.M + 127) / 128 * 128;
    TK(launch_im2col_split(c, half_at(L.a_hi[0]), half_at(L.a_lo[0]), st));
    TcLstmSeqArgs t;
    memset(&t, 0, sizeof(t));
    t.a_hi = half_at(L.a_hi[0]);
    t.a_lo = half_at(L.a_lo[0]);
    t.nxt_hi = s.nxt_hi[0] ? (__half*)s.nxt_hi[0] : half_at(L.nxt_hi[0]);
    t.nxt_lo = s.nxt_lo[0] ? (__half*)s.nxt_lo[0] : half_at(L.nxt_lo[0]);
    t.w = half_at(L.w[0]);
    t.gi = s.gi[0];
    t.c = s.c;
    t.out = s.out[0];
    t.inv_scale = 1.f / scale[0];
    t.ldgi = s.ldgi;
    t.ldout = s.ldout;
    t.KB = KB;
    t.M = s.M;
    t.H = s.H;
    t.rows_total = c.rows_total;
    TK(launch_tc_lstm_seq(t, st, pdl, &info));
    kname = "tc_lstm_seq";
  } else if (s.kind == MB_TACO_TC_GRU) {
    TcGruArgs g;
    memset(&g, 0, sizeof(g));
    for (int d = 0; d < ndir; ++d) {
      TK(tc_skinny_pack(s.w[d], K, nullptr, 0, s.b[d], nullptr, 3 * s.H, s.H, scale[d], half_at(L.w[d]),
                        reinterpret_cast<float*>(ws + L.bias[d]), st));
      TK(launch_act_split(s.x[d], K, s.ldx[d] > 0 ? s.ldx[d] : K, nullptr, 0, 0, s.M, half_at(L.a_hi[d]), half_at(L.a_lo[d]), st));
      g.a_hi[d] = half_at(L.a_hi[d]);
      g.a_lo[d] = half_at(L.a_lo[d]);
      g.nxt_hi[d] = s.nxt_hi[d] ? (__half*)s.nxt_hi[d] : half_at(L.nxt_hi[d]);
      g.nxt_lo[d] = s.nxt_lo[d] ? (__half*)s.nxt_lo[d] : half_at(L.nxt_lo[d]);
      g.w[d] = half_at(L.w[d]);
      g.bias[d] = reinterpret_cast<const float*>(ws + L.bias[d]);
      g.gi[d] = s.gi[d];
      g.h[d] = s.hst[d];
      g.out[d] = s.out[d];
      g.inv_scale[d] = 1.f / scale[d];
    }
    g.ldgi = s.ldgi;
    g.ldout = s.ldout;
    g.KB = KB;
    g.M = s.M;
    g.H = s.H;
    g.ndir = ndir;
    g.s_hi = (__half*)s.s_hi[0];
    g.s_lo = (__half*)s.s_lo[0];
    g.s_k0 = s.s_k0[0];
    TK(launch_tc_gru(g, st, pdl, &info));
    kname = "tc_gru";
  } else {
    const bool lstm = s.kind == MB_TACO_TC_SKINNY_LSTM;
    TK(tc_skinny_pack(s.w[0], s.K0, s.w[1], s.K1, s.b[0], s.b[1], rows_w, lstm ? s.H : 0, scale[0], half_at(L.w[0]),
                      reinterpret_cast<float*>(ws + L.bias[0]), st));
    TK(launch_act_split(s.x[0], s.K0, s.ldx[0], s.x[1], s.K1, s.ldx[1], s.M, half_at(L.a_hi[0]), half_at(L.a_lo[0]), st));
    TcSkinnyArgs t;
    memset(&t, 0, sizeof(t));
    t.a_hi = half_at(L.a_hi[0]);
    t.a_lo = half_at(L.a_lo[0]);
    t.w = half_at(L.w[0]);
    t.bias = (s.b[0] || s.b[1]) ? reinterpret_cast<const float*>(ws + L.bias[0]) : nullptr;
    t.kb0 = s.kb0;
    t.KB = s.kb_count > 0 ? s.kb_count : KB;
    t.KBw = s.kb_count > 0 ? KB : 0;
    if (s.kb0 < 0 || s.kb0 + t.KB > KB) return fail(MB_ERR_INVALID, "mb_taco_tc_debug: k-blocks [%d, %d) of %d", s.kb0, s.kb0 + t.KB, KB);
    t.M = s.M;
    t.N = lstm ? 4 * s.H : s.N;
    t.mode = lstm ? TCS_LSTM : TCS_PLAIN;
    t.inv_scale = 1.f / scale[0];
    t.y = s.y;
    t.ldy = s.ldy;
    t.step_ptr = s.step_ptr;
    t.step_j = s.step_j;
    t.y_step = s.y_step;
    t.c = s.c;
    t.h = s.h;
    t.x = s.xres;
    t.H = s.H;
    for (int k = 0; k < 2; ++k) {
      t.s_hi[k] = (__half*)s.s_hi[k];
      t.s_lo[k] = (__half*)s.s_lo[k];
      t.s_k0[k] = s.s_k0[k];
    }
    t.pre = s.pre;
    t.ldpre = s.ldpre;
    const int ring8 = s.compact < 0 ? env_flag("MB_TACO_RING8", 1) : s.compact;
    int mc = s.cluster;
    if (mc == 0) {
      const char* e = getenv("MB_TACO_MC");
      mc = e ? atoi(e) : 1;
      if (mc != 2 && mc != 4 && mc != 8) mc = 1;
    }
    TK(launch_tc_skinny(t, st, ring8, mc, pdl, &info));
    kname = lstm ? "tc_skinny_lstm" : "tc_skinny_plain";
  }
  if (s.a_tiles) {
    MB_CUDA_CHECK(cudaMemcpyAsync(s.a_tiles, ws + L.a_hi[0], L.a_bytes, cudaMemcpyDeviceToDevice, st));
    MB_CUDA_CHECK(cudaMemcpyAsync((char*)s.a_tiles + L.a_bytes, ws + L.a_lo[0], L.a_bytes, cudaMemcpyDeviceToDevice, st));
  }
  if (s.w_tiles) MB_CUDA_CHECK(cudaMemcpyAsync(s.w_tiles, ws + L.w[0], L.w_bytes, cudaMemcpyDeviceToDevice, st));
  if (report && report_len)
    snprintf(report, report_len, "kernel=%s grid=%d,%d cluster=%d compact=%d rows_pad=%d mma_groups=%d,%d inv_scale=%.9e a_bytes=%zu w_bytes=%zu\n",
             kname, info.grid_x, info.grid_y, info.cluster, info.compact, info.rows_pad, info.mma_groups, info.mma_groups_last,
             (double)(1.f / scale[0]), L.a_bytes, L.w_bytes);
  return MB_OK;
}

}  // extern "C"
