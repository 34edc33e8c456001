// FP32 building blocks of the Tacotron path (csrc/tacotron.cu).  Activations are row-major
// [rows][features] ("channels last"), so Linear layers, Conv1d over time (as shifted-row segments),
// GRU/LSTM gate projections and the CBHG convolution bank are all ONE kernel shape:
//
//   Y[m][n] = epi( sum_j sum_kk  X_j[row_j(m)][kk] * W[n*ldw + w_off_j + kk*w_stride_j] )
//
// row_j(m) = m + shift_j inside the same length-T sequence (zero outside) - a tap of a "same" conv -
// and epi = bias, activation, eval-BatchNorm affine (applied AFTER the ReLU like
// common/batch_norm_conv.py:11-14), PreNet dropout mask, residual.
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <cstdint>

namespace mb {
namespace taco {

// ---- fp16 hi / lo operand tiles [KB][rows_pad][64] (16-byte chunks XOR (row & 7)): element (m, k) of the K-major
// SWIZZLE_128B layout the tensor-core GEMMs read (written by launch_act_split or directly by the producing kernels)
__device__ __forceinline__ size_t split_tile_index(int m, int rows_pad, int k) {  // in halves
  const int kb = k >> 6, c8 = (k & 63) >> 3, e = k & 7;
  return (((size_t)kb * rows_pad + m) * 8 + (size_t)(c8 ^ (m & 7))) * 8 + (size_t)e;
}
__device__ __forceinline__ void store_split_scalar(float v, int m, int rows_pad, int k, __half* t_hi, __half* t_lo) {
  const __half hi = __float2half_rn(v);
  const size_t o = split_tile_index(m, rows_pad, k);
  t_hi[o] = hi;
  t_lo[o] = __float2half_rn(v - __half2float(hi));
}
// four consecutive k (k % 4 == 0)
__device__ __forceinline__ void store_split_quad(const float4& v, int m, int rows_pad, int k, __half* t_hi, __half* t_lo) {
  const __half2 h01 = __floats2half2_rn(v.x, v.y), h23 = __floats2half2_rn(v.z, v.w);
  const float2 f01 = __half22float2(h01), f23 = __half22float2(h23);
  const __half2 l01 = __floats2half2_rn(v.x - f01.x, v.y - f01.y), l23 = __floats2half2_rn(v.z - f23.x, v.w - f23.y);
  const size_t o = split_tile_index(m, rows_pad, k);
  uint2 ph, pl;
  ph.x = *reinterpret_cast<const uint32_t*>(&h01);
  ph.y = *reinterpret_cast<const uint32_t*>(&h23);
  pl.x = *reinterpret_cast<const uint32_t*>(&l01);
  pl.y = *reinterpret_cast<const uint32_t*>(&l23);
  *reinterpret_cast<uint2*>(t_hi + o) = ph;
  *reinterpret_cast<uint2*>(t_lo + o) = pl;
}


constexpr int kMaxSeg = 5;

enum Act : int { ACT_NONE = 0, ACT_RELU = 1, ACT_SIGMOID = 2, ACT_TANH = 3 };

struct Seg {
  const float* x;   // [M][ld]
  int K;            // features taken from this segment
  int ld;           // row stride of x
  int shift;        // time shift (conv tap) - 0 for plain Linear inputs
  int w_off;        // first weight column of this segment
  int w_stride;     // weight column stride (Conv1d weight [co][ci][k]: stride k)
};

struct GemmArgs {
  Seg seg[kMaxSeg];
  int nseg;
  const float* W;
  int ldw;
  const float* bias;       // [N] or nullptr
  int M, N, T;             // T: rows per sequence (shift bounds); T <= 1: no sequence structure
  int act;
  const float* bn_scale;   // [N] or nullptr: y = act(.) * scale + shift
  const float* bn_shift;
  const uint8_t* mask;     // [M][N] keep flags (PreNet dropout, p = 0.5 -> x2) or nullptr
  const float* res;        // residual [M][ldres] or nullptr
  int ldres;
  float* Y;
  int ldy;
  // decoder-step indirection (CUDA-graph replay): step = (step_ptr ? *step_ptr : 0) + step_j.  When step_mode != 0
  // segment 0 reads x + step * x_step (or x_first with row stride 0 at step 0: the all-zero go frame) and the
  // dropout mask is mask + step * mask_step.
  int step_mode;
  const int* step_ptr;
  int step_j;
  long long x_step;
  const float* x_first;
  long long mask_step;
};

__device__ __forceinline__ int step_index(const int* step_ptr, int step_j) { return (step_ptr ? *step_ptr : 0) + step_j; }

cudaError_t launch_gemm(const GemmArgs& a, cudaStream_t st);

// Decoder PreNet (sublayer/pre_net.py:11-27) as ONE launch: y = drop2(relu(W2 drop1(relu(W1 x + b1)) + b2)), dropout p = 0.5 with
// injected / device-drawn keep masks (x2).  The intermediate never leaves shared memory; replaces two skinny GEMM launches
// (12 us each, latency-bound) per decoder step.  Same step indirection as GemmArgs (CUDA-graph replay).
struct PrenetArgs {
  const float* x;          // frame (step*r - 1) of row b: x + b * x_ld + step * x_step (step 0: x_first, the zero go frame)
  long long x_ld, x_step;
  const float* x_first;
  const float* W1;         // [H][K] row-major
  const float* b1;
  const float* W2;         // [H][H]
  const float* b2;
  const uint8_t* m1;       // [B][H] keep flags (+ step * mask_step)
  const uint8_t* m2;
  long long mask_step;
  const int* step_ptr;
  int step_j;
  int B, K, H;             // K <= 128, H <= 256
  float* y;                // [B][ldy]
  int ldy;
  __half* s_hi;            // optional: y also goes, split into fp16 hi / lo, into the operand tiles of the next tensor-core GEMM
  __half* s_lo;            //   (columns [s_k0, s_k0 + H) of tiles [KB][s_rows_pad][64], the layout of launch_act_split)
  int s_k0, s_rows_pad;
};
cudaError_t launch_prenet_fused(const PrenetArgs& a, cudaStream_t st);

// h' = GRU cell (ATen gru_cell): gi, gh [M][3H] pre-activations incl. biases; h in/out [M][ldh]
cudaError_t launch_gru_cell(const float* gi, int ldgi, const float* gh, float* h, int ldh, float* out2, int ldout2,
                            int M, int H, cudaStream_t st);
// LSTM cell (ATen lstm_cell): g = gates [M][4H] (ih + hh + biases); c in/out; h out; xres: x += h (residual)
cudaError_t launch_lstm_cell(const float* g, float* c, float* h, float* x, int M, int H, cudaStream_t st);
// y = g*relu(x1) + (1-g)*y, g = sigmoid(x2); x12 = [M][2C] (x1 | x2)
cudaError_t launch_highway(const float* x12, float* y, int M, int C, cudaStream_t st);
// out[b][t][c] = max(x[b][t-1][c], x[b][t][c])   (MaxPool1d(2,1,1)[:T])
cudaError_t launch_maxpool2(const float* x, float* y, int B, int T, int C, cudaStream_t st);
// embedding rows
cudaError_t launch_embedding(const int32_t* ids, const float* table, float* y, int M, int D, cudaStream_t st);
// dst[m][off + j] = src[(m / rows_per_src)][j]  (broadcast a per-sequence vector along time) or row copy
cudaError_t launch_copy_cols(const float* src, int ldsrc, int rows_per_src, float* dst, int lddst, int off, int M,
                             int n, cudaStream_t st);

// ---- tensor-core skinny GEMM (tacotron_tc.cu): Y[M <= 128][N] = A[M][K] . W[N][K]^T as a 3-term fp16 split with
// FP32 accumulation (FP32-equivalent), one CTA per 32 output columns ------------------------------------
enum TcSkinnyMode : int { TCS_PLAIN = 0, TCS_LSTM = 1 };
struct TcSkinnyArgs {
  const __half* a_hi;   // activation tiles [K/64][rows_pad][64] (launch_act_split)
  const __half* a_lo;
  const __half* w;      // packed weight tiles (tc_skinny_pack)
  const float* bias;    // packed bias [ceil32(N)] or nullptr
  int KB, M, N, rows_pad, mode;
  float inv_scale;      // 1 / (power-of-two weight scale used at pack time)
  float* y;             // TCS_PLAIN: out [M][ldy] (+ step * y_step, step = (step_ptr ? *step_ptr : 0) + step_j)
  int ldy;
  const int* step_ptr;
  int step_j;
  long long y_step;
  float* c;             // TCS_LSTM: cell state [M][H] in/out, h [M][H] out, x [M][H] += h (residual, tacotron.py:121,126)
  float* h;
  float* x;
  int H;
  // optional split outputs (hi / lo operand tiles [KB][rows_pad][64] of the NEXT GEMMs, so that no act_split launch is needed):
  //   slot 0: TCS_PLAIN y / TCS_LSTM x' (the residual stream) at columns s_k0[0] + n;  slot 1: TCS_LSTM h' at columns s_k0[1] + n
  __half* s_hi[2];
  __half* s_lo[2];
  int s_k0[2];
  // optional K range: only k-blocks [kb0, kb0 + KB) of a weight image packed with KBw k-blocks per tile (KBw = 0: KB) and of the
  // activation tiles; `pre` [M][ldpre] (tile column order, i.e. what a TCS_PLAIN launch over the other k-blocks wrote) is added to
  // the accumulator before the epilogue.  Lets the part of a GEMM whose input is known early run off the critical path.
  int kb0, KBw;
  const float* pre;
  int ldpre;
  int compact;          // set by launch_tc_skinny: 8 KB activation slots, 8-stage ring (rows_pad == 64)
};
// one recurrent GRU step for 1 or 2 directions (blockIdx.y); pointers per direction
struct TcGruArgs {
  const __half* a_hi[2];  // h_{t-1} operand tiles [H/64][rows_pad][64]
  const __half* a_lo[2];
  __half* nxt_hi[2];      // h_t operand tiles for the next step (ping-pong with a_hi / a_lo)
  __half* nxt_lo[2];
  const __half* w[2];     // W_hh images, gates r|z|n interleaved per 8 units (tc_skinny_pack with lstm_H = H, N = 3H)
  const float* bias[2];   // tile-order b_hh
  const float* gi[2];     // W_ih x_t + b_ih for this step: row m at gi + m * ldgi, [r | z | n] each H wide
  float* h[2];            // state [M][H] in/out
  float* out[2];          // output sequence slot of this step: row m at out + m * ldout
  float inv_scale[2];
  int ldgi, ldout, KB, M, H, rows_pad, ndir;
  __half* s_hi;           // optional (direction 0): h_t also into columns [s_k0, s_k0 + H) of another GEMM's operand tiles
  __half* s_lo;
  int s_k0;
};
cudaError_t launch_tc_gru(const TcGruArgs& a, cudaStream_t st);
// ---- large-M tensor-core GEMM / conv over time (CBHG stacks), 128 x 128 output tiles ---------------------------
struct TcIm2col {       // im2col of the layer input into hi/lo operand tiles (one K segment per conv tap)
  const float* x[kMaxSeg];
  int ld[kMaxSeg];
  int shift[kMaxSeg];
  int nseg, K, KBs;     // K features per segment, KBs = ceil(K / 64) k-blocks per segment
  int M, T, rows_total;
};
struct TcBigPack {      // weights as GemmArgs describes them: W[n * ldw + w_off_s + k * w_stride_s]
  const float* W;
  int ldw, N, nseg, K, KBs;
  int w_off[kMaxSeg];
  int w_stride[kMaxSeg];
  float scale;
};
struct TcBigArgs {
  const __half* a_hi;   // [nseg * KBs][rows_total][64]
  const __half* a_lo;
  const __half* w;      // [ceil(N / 128)][nseg * KBs][hi|lo][128][64]
  const float* bias;    // [N] or nullptr (natural order)
  int KB, M, N, rows_total, act;
  float inv_scale;
  const float* bn_scale;
  const float* bn_shift;
  const float* res;
  int ldres;
  float* y;
  int ldy;
};
size_t tc_big_weight_bytes(int N, int nseg, int K);
size_t tc_big_act_bytes(int M, int nseg, int K);
// what a tensor-core launch ran with (filled by the launchers when asked; mb_taco_tc_debug reports it)
struct TcLaunchInfo {
  int grid_x, grid_y, cluster, compact, rows_pad, mma_groups, mma_groups_last;  // mma_groups(_last): first / last row block
};
// pdl: -1 = MB_TACO_PDL (read once per process), 0 = plain launch, 1 = programmatic dependent launch
cudaError_t launch_im2col_split(const TcIm2col& q, __half* a_hi, __half* a_lo, cudaStream_t st);
cudaError_t launch_pack_big_w(const TcBigPack& q, __half* dst, cudaStream_t st);
cudaError_t launch_tc_big(const TcBigArgs& a, cudaStream_t st, int pdl = -1, TcLaunchInfo* info = nullptr);

// one time step of an LSTM layer over M rows (any M; operand tiles hold rows_total = ceil128(M) rows per k-block)
struct TcLstmSeqArgs {
  const __half* a_hi;   // h_{t-1} tiles [H/64][rows_total][64]
  const __half* a_lo;
  __half* nxt_hi;       // h_t tiles (ping-pong)
  __half* nxt_lo;
  const __half* w;      // W_hh images, gates i|f|g|o interleaved per 8 units (tc_skinny_pack, lstm_H = H, N = 4H)
  const float* gi;      // W_ih x_t + b_ih + b_hh for this step: row m at gi + m * ldgi
  float* c;             // cell state [M][H] in/out
  float* out;           // h_t destination: row m at out + m * ldout
  float inv_scale;
  int ldgi, ldout, KB, M, H, rows_total;
};
cudaError_t launch_tc_lstm_seq(const TcLstmSeqArgs& a, cudaStream_t st, int pdl = -1, TcLaunchInfo* info = nullptr);
size_t tc_gated_weight_bytes(int H, int K);
size_t tc_skinny_weight_bytes(int N, int K);
size_t tc_skinny_act_bytes(int M, int K);
// max |w| into *dev_out (uint bit pattern of a non-negative float; caller zeroes it first)
cudaError_t tc_skinny_absmax(const float* w, size_t n, unsigned int* dev_out, cudaStream_t st);
// power-of-two pack scale of a weight whose max |w| is `absmax_bits` (the bit pattern tc_skinny_absmax leaves): max |w| * scale
// lands in [2^11, 2^12), so the lo parts of the fp16 split stay clear of the subnormal range; a zero, inf or NaN max gives 2^12.
// Every weight image of the tensor-core GEMMs is packed with this scale and read back with 1 / scale.
float tc_weight_scale(unsigned int absmax_bits);
// weights [N][K0 | K1] (two row-major sources) * scale -> hi/lo tiles; lstm_H > 0: gate-interleaved rows
cudaError_t tc_skinny_pack(const float* w0, int K0, const float* w1, int K1, const float* b0, const float* b1, int N,
                           int lstm_H, float scale, __half* w_dst, float* bias_dst, cudaStream_t st);
cudaError_t launch_act_split(const float* s0, int K0, int ld0, const float* s1, int K1, int ld1, int M, __half* a_hi,
                             __half* a_lo, cudaStream_t st);
// Launch variants are arguments: ring8 (compact 8-stage ring for <= 64 rows) 0 / 1, mc = cluster size of the activation multicast
// 1 / 2 / 4 / 8 (used only where it divides the tile count), pdl as above.  The two-argument form takes all three from the
// environment (MB_TACO_RING8, MB_TACO_MC, MB_TACO_PDL), as the forward does.
cudaError_t launch_tc_skinny(const TcSkinnyArgs& a, cudaStream_t st, int ring8, int mc, int pdl, TcLaunchInfo* info = nullptr);
cudaError_t launch_tc_skinny(const TcSkinnyArgs& a, cudaStream_t st);
cudaError_t launch_tc_gru(const TcGruArgs& a, cudaStream_t st, int pdl, TcLaunchInfo* info = nullptr);

}  // namespace taco
}  // namespace mb
