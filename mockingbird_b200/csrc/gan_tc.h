// Tensor-core (wgmma / bulk-TMA) execution of the GAN generator plan (MB_PREC_F16TC).
// Host-side interface used by gan_api.cu; the kernels live in gan_tc.cu.
#pragma once
#include <cuda_runtime.h>
#include <cstddef>
#include <cstdint>
#include <vector>

#include "gan_kernels.h"

namespace mb {

// per-layer packing decision, filled by tc_plan_layers
struct TcLayer {
  int use_tc = 0;        // 1: tensor-core kernel, 0: FP32 kernel on blocked layouts
  int kc = 0;            // input channels per K-chunk (<= 64, multiple of 16)
  int n_cchunks = 0;     // Cin / kc
  int mt = 1;            // 128-row tiles per work item
  size_t slab_bytes = 0; // one (kernel index, chunk) weight image: [kc/8][Cout][8] fp16
  size_t w16_off = 0;    // byte offset of this layer's images in the tensor-core arena section
  int x3 = 0;            // 1: FP32-equivalent 3-term fp16 split of a layer whose input is an internal "hi/lo" plane
                         //    (TRef::hilo): K-chunks [hi | lo | hi] of the plane x weight images [hi(w) | hi(w) | lo(w)], weights
                         //    pre-scaled by kX3WScale (a power of two) so that lo(w) stays a normal fp16; n_cchunks counts K-chunks
  int x_pchunks = 0;     //    64-channel chunks of the input plane per utterance (x3: 2*Cin/64, or 1 when Cin == 32)
  int split3 = 0;        // 1: fp32-accurate 3-term fp16 split (x_hi*w_hi + x_lo*w_hi + x_hi*w_lo) of a layer whose
                         //    input is the external fp32 tensor (conv_pre): K = 3*Cin padded to 256 channels
};

constexpr float kX3WScale = 256.f;

struct TcLayerDesc {
  bool is_conv;
  bool want_x3 = false;  // run the layer with the 3-term split if the tensor-core kernel covers its shape
  bool force_f32;  // layer shapes the tensor-core kernel does not cover (second destination, nearest-upsample)
  const TapConv* taps;
  int k;
  TcLayer* tc;
};

int tc_plan_layers(std::vector<TcLayerDesc>& layers, size_t* tc_arena_bytes);

// pack one layer's fp16 weight images from the fp32 slabs [K][Cin][Cout]
int tc_pack_weights(const TcLayer& tc, const TapConv& taps, const float* w32_slabs, char* tc_arena,
                    cudaStream_t stream);

struct TcBufReq {
  size_t cr;  // max channels * rows-per-frame of plan buffer i
};

size_t tc_workspace_bytes(const std::vector<TcBufReq>& bufs, int B, int T, int num_mels, int hop);

struct TcOp {
  bool is_conv;
  TapConv taps;
  TcLayer tc;
  const char* name;
  int src, dst, res, dst2;
  int cin, cout, rate_in, rate_out;
  const float* w32;  // fp32 slabs (FP32-kernel layers)
  const float* b32;
};

int tc_forward(const std::vector<TcOp>& ops, const std::vector<TcBufReq>& bufs, const char* tc_arena,
               const float* mel, const int32_t* lengths, int B, int T, int num_mels, int hop, float* wav,
               void* workspace, cudaStream_t stream, cudaEvent_t* events /* nullptr or [ops+1] */);

// MB_TC_RED_ADD=0: accumulate-mode epilogues read, add and store the running sum themselves
bool tc_red_add_enabled();

int tc_debug_layer(const TcOp& op, const char* tc_arena, const float* x, const float* residual, int B, int Lin,
                   float* y, void* workspace, size_t workspace_bytes, cudaStream_t stream);

// which (c1, c2) op pairs tc_forward runs as ONE fused launch (tc_conv_kernel<..., PAIR = true>): fuse_next[i] = 1 for ops
// (i, i + 1).  nbufs = number of plan buffers.
std::vector<char> tc_fusion_plan(const std::vector<TcOp>& ops, int nbufs);

// how tc_forward runs op i (host-only)
struct TcOpPlan {
  int use_tc, x3, split3;
  int kc, n_cchunks, mt, rows_item, resident, wstages, omin, omax;  // the op launched on its own
  int fuse_next, fused_prev;                                         // first / second op of a fused pair
  int pair_mt, pair_rows_item, pair_resident, pair_wstages, pair_omin;  // fuse_next: the pair's launch
  int kn, kmt, kcw, kpair;  // kernel instance <N, MT, CW, PAIR> this op launches (kn = 0: none of its own)
};
int tc_op_plan(const std::vector<TcOp>& ops, const std::vector<char>& fuse_next, int i, TcOpPlan* out);

// what one tc_conv launch ran
struct TcLaunchInfo {
  int n, mt, cw, pair, rows_item, resident, wstages, n_work, grid, red_add;
};

// test hook: one tensor-core layer, or a resblock pair (c2 != nullptr) fused or as two launches, with the epilogue inputs and
// outputs chosen by the caller.  The accumulate mode is op's (c2's) taps.mode / div.
struct TcDebugSpec {
  int B = 0, Lin = 0;
  const float* x = nullptr;           // NCL [B][Cin][Lin] (not activated)
  const float* res = nullptr;         // NCL [B][Cout][Lout]
  int res_kind = 0;                   // 0 none, 1 fp32 plane, 2 activated fp16 plane, 3 hi/lo plane
  float res_slope = 1.f;              // slope the fp16 residual planes are activated with
  const int32_t* lengths = nullptr;   // device [B], in input rows
  bool red_add = false;               // EPI_ADD by red.global.add where the epilogue allows it
  float* y = nullptr;                 // NCL [B][Cout][Lout]: running sum in (accumulate modes), fp32 result out
  int out16 = 0;                      // 0 none, 1 plain fp16 plane, 2 hi/lo plane
  float out_slope = 1.f;
  float* y16 = nullptr;               // NCL [B][C16][Lout]: the fp16 plane read back (hi channels, then lo channels)
  bool two_launches = false;          // pair: c1 into an fp16 plane, then c2 (what an unfused pair does)
};
int tc_debug_launch(const TcOp& op, const TcOp* c2, const TcDebugSpec& spec, const char* tc_arena, void* workspace,
                    size_t workspace_bytes, cudaStream_t stream, TcLaunchInfo* info /* [2] */, int* n_launches);

}  // namespace mb
