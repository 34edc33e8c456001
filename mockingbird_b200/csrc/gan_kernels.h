// Kernel-launch interface of the GAN generator path (HiFi-GAN / Fre-GAN).
//
// Every channel-mixing layer of the generators (Conv1d, dilated Conv1d, ConvTranspose1d as a
// polyphase bank, nearest-upsample + 1x1) is expressed as ONE op shape, the "tap conv":
//
//   v[b, co, q*stride + r] = bias[co] + sum_{t < ntaps[r]} sum_ci  W[slab[r][t]][ci][co] *
//                                        act_in( x[b, ci, q + off[r][t]] )          r < stride
//   act_in = leaky_relu(., in_slope)   (in_slope == 1 -> identity); x outside [0, valid_in) == 0
//
// followed by a fused epilogue (residual add, MRF accumulate / mean, tanh, length mask).
// reference: hifigan/models.py:35-42 (ResBlock1), :134-150 (Generator.forward).
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <cstdint>

namespace mb {

constexpr int kMaxTaps = 11;    // resblock kernel sizes are (3,7,11)
constexpr int kMaxPhases = 8;   // upsample rates are (5,5,4,2) / (5,5,2,2,2)
constexpr int kPadRows = 40;    // zero rows on both sides of every run of an fp16 activation plane

enum EpiMode : int {
  EPI_STORE = 0,     // y = v
  EPI_ADD = 1,       // y = y + v          (MRF: xs += resblock_j(x), models.py:143)
  EPI_ADD_DIV = 2,   // y = (y + v) / div  (MRF: x = xs / num_kernels, models.py:144)
};

struct TapConv {
  // problem
  int B, Cin, Cout, Lin, Lout;   // Lout == Lin * stride
  int stride;                    // number of output phases
  int ntaps[kMaxPhases];
  int off[kMaxPhases][kMaxTaps];   // input offset of tap t in phase r
  int slab[kMaxPhases][kMaxTaps];  // weight slab (kernel index) of tap t in phase r
  float in_slope;                // leaky-relu slope applied to x on load (1 = none)
  // epilogue
  int mode;                      // EpiMode
  float div;                     // for EPI_ADD_DIV
  int act_tanh;                  // y = tanh(v)
  // valid lengths: utterance b has lengths[b]*len_mul_in valid input rows and
  // lengths[b]*len_mul_out valid output rows (lengths == nullptr -> all valid)
  const int32_t* lengths;
  int len_mul_in, len_mul_out;
};

// Activation tensor layouts ------------------------------------------------------------------
//   LAYOUT_NCL : fp32 [B][C][L]                      (the reference's layout; API boundary)
//   LAYOUT_F32B: fp32 [B][C/4][L][4]                 (residual streams of the tensor-core path)
//   LAYOUT_F16B: fp16 [B][C/CW][Lp][CW], CW = min(C,64), Lp = ceil8(L + 2*kPadRows)
//                 (MMA operand planes: already activated; rows [kPadRows, kPadRows+L) hold data, pad
//                 rows are zero.  Each row of a run is CW*2 = 128 (or 64) bytes and its 16-byte chunks
//                 are stored XOR-swizzled by the row index exactly like the UMMA SWIZZLE_128B
//                 (SWIZZLE_64B) shared-memory layouts, so a conv window is ONE contiguous bulk copy
//                 per 64-channel chunk that lands in shared memory already in tensor-core layout.)
enum Layout : int { LAYOUT_NONE = 0, LAYOUT_NCL = 1, LAYOUT_F32B = 2, LAYOUT_F16B = 3 };

struct TRef {
  void* p = nullptr;
  int layout = LAYOUT_NONE;
  int C = 0, L = 0;
  // F16B planes only: 1 = "hi/lo" operand plane of a 3-term-split consumer.  The plane has C = 2 x logical channels:
  // channel c holds hi = fp16(v), channel c + C/2 holds lo = fp16(v - hi); writers store both, readers see 2C channels.
  int hilo = 0;
};

__host__ __device__ inline int f16_cw(int C) { return C >= 64 ? 64 : C; }
__host__ __device__ inline int f16_lp(int L) { return (L + 2 * kPadRows + 7) & ~7; }
// swizzle phase of padded row r for a row of cw channels (128-byte rows: r & 7, 64-byte rows: (r>>1) & 3)
__host__ __device__ inline int f16_swz(int cw, int r) { return cw == 64 ? (r & 7) : (cw == 32 ? ((r >> 1) & 3) : 0); }

__host__ __device__ inline size_t tref_index(const TRef& t, int b, int c, int l) {
  if (t.layout == LAYOUT_NCL) return ((size_t)b * t.C + c) * t.L + l;
  if (t.layout == LAYOUT_F32B) return (((size_t)b * (t.C >> 2) + (c >> 2)) * t.L + l) * 4 + (c & 3);
  const int cw = f16_cw(t.C);
  const int r = kPadRows + l;
  const int chunk = c / cw, cc = c - chunk * cw;
  return (((size_t)b * (t.C / cw) + chunk) * f16_lp(t.L) + r) * cw + (size_t)((((cc >> 3) ^ f16_swz(cw, r)) << 3) + (cc & 7));
}

// ---- FP32 FFMA kernels ------------------------------------------------------------------------
// w: [kernel_size slabs][Cin][Cout] fp32 ; bias [Cout] or nullptr.
//   x      input (any layout; an F16B input is already activated: in_slope is ignored for it)
//   res    residual (fp32 layouts) or none
//   y32    fp32 destination (NCL / F32B) or none: receives v per the epilogue mode
//   y16    fp16 destination plane or none: receives leaky_relu(v_final, out16_slope)
//   y2_32 / y2_16: second destination (Fre-GAN "x += cond_up(mel)"): y2 += v, y2_16 = lrelu(y2)
struct TapConvIO {
  TRef x, res, y32, y16, y2_32, y2_16;
  float out16_slope = 1.f;
  float y2_16_slope = 1.f;
};
cudaError_t launch_tapconv_f32(const TapConv& p, const TapConvIO& io, const float* w, const float* bias,
                               cudaStream_t stream);

// Cout == 1 special case (conv_post, models.py:146-148).  variant: kCout1Default (the MB_POST_TILE / MB_POST_ROWS switches),
// 1 / 2 / 4 output rows per thread, or kCout1Tile (the shared-memory tile kernel; cudaErrorInvalidValue where it does not apply).
// All variants accumulate in the same order and give bit-identical results.  *kernel (if given) names the instance launched.
constexpr int kCout1Default = 0;
constexpr int kCout1Tile = -1;
cudaError_t launch_tapconv_cout1_f32(const TapConv& p, const TapConvIO& io, const float* w, const float* bias,
                                     cudaStream_t stream, int variant = kCout1Default, const char** kernel = nullptr);

// dst32 += src32 (same layout), optionally refresh dst16 = lrelu(dst32, slope)
cudaError_t launch_add_inplace_f32(const TRef& dst32, const TRef& src32, const TRef& dst16, float slope, int B,
                                   cudaStream_t stream);

// zero the pad rows of an fp16 plane of geometry (B, C, L)
cudaError_t launch_zero_pads_f16(const TRef& plane, int B, cudaStream_t stream);

// layout conversion (debug/test hook only): NCL fp32 <-> blocked planes
cudaError_t launch_convert_layout(const TRef& src, const TRef& dst, int B, float slope, cudaStream_t stream);

// weight repack: Conv1d weight [Cout][Cin][K] or ConvTranspose1d weight [Cin][Cout][K]
//   -> slabs [K][Cin_p][Cout_p] (zero-padded channels when Cin_p / Cout_p exceed the checkpoint's)
cudaError_t launch_pack_slabs_f32(const float* w, float* dst, int Cout, int Cin, int K, bool transposed,
                                  cudaStream_t stream, int Cout_p = 0, int Cin_p = 0);

// Nearest-neighbour upsample by u followed by Conv1d(k, padding=(k-1)/2), folded into a polyphase tap conv: slab s of the
// layer is the sum of the kernel taps W_j, j = jlo[s] .. jhi[s] (one run of consecutive j that all read the same input row).
constexpr int kMaxSlabs = kMaxPhases * kMaxTaps;
struct FoldTable {
  int nslabs;
  int jlo[kMaxSlabs], jhi[kMaxSlabs];
};

// weight fold + repack: Conv1d weight [Cout][Cin][K] -> slabs [nslabs][Cin_p][Cout_p], slab s = sum_{j = jlo[s]}^{jhi[s]} w[:, :, j]
// accumulated in fp32 in ascending j; every element of dst is written (padded channels = 0)
cudaError_t launch_fold_slabs_f32(const float* w, float* dst, int Cout, int Cin, int K, const FoldTable& fold, int Cout_p,
                                  int Cin_p, cudaStream_t stream);

}  // namespace mb
