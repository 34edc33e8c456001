// Tensor-core execution of the GAN generator plan (MB_PREC_F16TC), sm_90a (Hopper warpgroup MMA).
//
// tc_conv_kernel: the tap conv (gan_kernels.h) as an implicit GEMM on the tensor cores (wgmma).
//   D[64 rows x Cout] (fp32, registers) += A[64 rows x 16 ci] (fp16, smem) * B[Cout x 16 ci]^T (fp16, smem)
//   * M = MT x 128 consecutive time rows per work item, N = Cout, K = (tap, input channel).
//   * activations live in HBM as "F16B" planes [B][C/64][Lp][64] (already leaky-relu'd by the
//     producer's epilogue) whose rows are stored PRE-SWIZZLED: the 16-byte chunks of every 128-byte
//     row are XOR-permuted by (row & 7) exactly like the GMMA SWIZZLE_128B shared-memory layout
//     (64-byte rows / SWIZZLE_64B when C = 32).  One bulk-TMA copy (cp.async.bulk) per 64-channel
//     chunk fetches the rows [floor8(m0 + omin), ... + W) of a work item; because the copy starts at
//     a row that is a multiple of 8 and lands 1024-byte aligned, it arrives in shared memory already
//     in the canonical K-major swizzled operand layout (SBO = 1024 B) - no tensor map, no repack.
//     The operand of tap t is the SAME buffer with the descriptor start address advanced by off_t
//     rows (the swizzle is a function of absolute smem address bits, so no base-offset fix-up is needed): every tap, every dilation and every phase of a
//     transposed conv reuse one window; zero padding comes from the zero pad rows of the plane.
//   * weights: per (kernel index, 64-channel chunk) an fp16 image [Cout][64] with the same swizzle,
//     streamed through a ring of shared-memory stages by bulk copies, or kept resident when the
//     layer's whole weight set fits (all C<=64 layers).
//   * warp roles: warpgroup 0 = copy producer (one thread), warpgroups 1-2 = MMA and epilogue, each on half of the rows
//     (registers -> shared-memory staging -> bias/residual/MRF/leaky-relu -> fp32 F32B plane and/or fp16 F16B plane,
//     16 B per thread per 8 channels).  Persistent CTAs, one per SM, static round-robin.
// reference semantics: hifigan/models.py:35-42 (ResBlock1), :134-150 (Generator.forward)
#include "gan_tc.h"

#include <cuda_fp16.h>

#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <map>

#include "gan_tc_dev.cuh"
#include "mb_common.h"

namespace mb {

namespace {

constexpr int kMmaGroups = 2;                      // MMA + epilogue warpgroups
constexpr int kTcThreads = 128 * (1 + kMmaGroups);  // + the copy-producer warpgroup
constexpr int kAStages = 2;
constexpr int kMaxWStages = 16;
constexpr uint32_t kStageBytes = kMmaGroups * 64 * tcdev::kStageLd * 4;  // epilogue staging: 64 rows x 32 columns per warpgroup
constexpr uint32_t kSmemMax = 227 * 1024;
constexpr size_t kPlaneSlack = 128 * 1024;

struct TcParams {
  int B, Lin, Lout, Cin, Cout;
  int stride;
  int ntaps[kMaxPhases];
  int off[kMaxPhases][kMaxTaps];
  int slab[kMaxPhases][kMaxTaps];
  int omin, W, MT;
  int cw, row_bytes, nk16, n_cchunks;   // channels per K-chunk (64 or 32), bytes per operand row
  int baseoff_mode;                    // 1: descriptor base_offset = start address bits 7..9
  int slab_bytes, wstages, resident;
  int tiles_per_utt, n_work;
  uint32_t a_stage_bytes, a_off, w_off, bias_off, bar_off, stage_off;
  const __half* x16;
  int x_Lp;
  const __half* w16;
  const float* bias;
  const float* res32;
  const __half* res16;                 // residual taken from an (activated) fp16 plane instead: x = y >= 0 ? y : y * res_inv
  int res_Lp;
  int res_hilo;                        // 1: the residual plane is a hi/lo plane (2 x Cout channels, 64-channel row chunks): x = inv_lrelu(hi + lo)
  float res_inv;
  float* y32;
  __half* y16;
  int y_Lp;
  int y_nchunks, y_cw, y_c0;           // fp16 destination plane: row chunks per utterance, channels per row chunk, first channel
                                       // this launch writes
  int y_lo_c;                          // >= 0: hi/lo destination plane - lo = fp16(v - fp16(v)) goes to channel + y_lo_c
  int x_pchunks;                       // 64-channel chunks of the INPUT plane per utterance (K-chunk c reads chunk c % x_pchunks)
  float acc_scale;                     // accumulator -> value (1, or 1/kX3WScale for 3-term-split layers)
  float out_slope;
  int mode;
  int red_add;                         // EPI_ADD without fp16 output: S += v by red.global.add.v4.f32
  float div;
  const int32_t* lengths;
  int len_mul_out;
  int rows_item;                       // output rows per work item (MT x 128, or MT x 128 - 2 h2 for a fused pair)
  // fused resblock pair (PAIR kernels): this launch's taps / weights are c1's, shifted by -h2 rows; c2 (k2 taps, dilation 1)
  // reads c1's leaky-relu'd fp16 output from shared memory and owns bias / residual / outputs above
  int k2, h2;
  int off2[kMaxTaps];
  const __half* w2;                    // c2's resident weight images [k2][Cout][cw]
  const float* bias1;
  float slope_mid;                     // leaky-relu between c1 and c2 (c2's in_slope)
  int len_mul_mid;
  uint32_t w2_off, mid_off, slab2_bytes;
};

using namespace tcdev;

struct WorkItem {
  int b, m0, r;
};
__device__ __forceinline__ WorkItem decode_work(const TcParams& p, int work) {
  WorkItem w;
  w.r = work % p.stride;
  const int t = work / p.stride;
  w.m0 = (t % p.tiles_per_utt) * p.rows_item;
  w.b = t / p.tiles_per_utt;
  return w;
}

// N = Cout, MT = 128-row tiles per work item, CW = channels per operand row (64: SWIZZLE_128B, 32: SWIZZLE_64B).
// They are compile-time so that the accumulators are register arrays and every descriptor is "base + immediate".
// PAIR: fused resblock pair (see TcParams); c1's accumulators go through the bias / mask / leaky-relu epilogue into a swizzled fp16
// operand in shared memory ("mid": row j = sequence row m0 - h2 + j) that c2's wgmmas read with a row shift per tap, so the
// intermediate activation never reaches HBM.
template <int N, int MT, int CW, bool PAIR = false>
__global__ void __launch_bounds__(kTcThreads, 1) tc_conv_kernel(const __grid_constant__ TcParams p) {
  constexpr int UC = 16;  // columns per epilogue thread and unit
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);  // swizzle atoms need 1024 B alignment
  uint8_t* a_base = smem + p.a_off;
  uint8_t* w_base = smem + p.w_off;
  float* bias_s = reinterpret_cast<float*>(smem + p.bias_off);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + p.bar_off);
  uint64_t* a_full = bars;
  uint64_t* a_empty = a_full + kAStages;
  uint64_t* w_full = a_empty + kAStages;
  uint64_t* w_empty = w_full + kMaxWStages;
  uint64_t* w2_full = w_empty + kMaxWStages;
  float* stage_s = reinterpret_cast<float*>(smem + p.stage_off);

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    for (int i = 0; i < kAStages; ++i) {
      mbar_init(&a_full[i], 1);
      mbar_init(&a_empty[i], kMmaGroups);
    }
    for (int i = 0; i < kMaxWStages; ++i) {
      mbar_init(&w_full[i], 1);
      mbar_init(&w_empty[i], kMmaGroups);
    }
    mbar_init(w2_full, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  for (int i = threadIdx.x; i < p.Cout; i += kTcThreads) bias_s[i] = p.bias ? p.bias[i] : 0.f;  // weights: never written by a kernel
  __syncthreads();
  // Programmatic dependent launch: everything above (barrier init, bias) overlapped the tail of the previous layer's kernel;
  // activations written by it may only be touched after this wait.  Dependents of THIS kernel may begin their own prologue
  // as soon as SMs free up.
  asm volatile("griddepcontrol.wait;" ::: "memory");
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");

  if (warp < 4) {
    // ===================== copy producer (warpgroup 0, one thread) =====================
    regs_dec<40>();
    if (warp == 0 && lane == 0) {
      int a_stage = 0, a_phase = 0, w_stage = 0, w_phase = 0;
      uint32_t resident_loaded = 0;
      if constexpr (PAIR) {
        mbar_expect_tx(w2_full, (uint32_t)p.k2 * p.slab2_bytes);
        for (int t = 0; t < p.k2; ++t)
          bulk_g2s(smem_u32(smem + p.w2_off + (size_t)t * p.slab2_bytes), p.w2 + (size_t)t * (p.slab2_bytes >> 1), p.slab2_bytes, w2_full);
      }
      for (int work = blockIdx.x; work < p.n_work; work += gridDim.x) {
        const WorkItem wi = decode_work(p, work);
        for (int c = 0; c < p.n_cchunks; ++c) {
          mbar_wait(&a_empty[a_stage], a_phase ^ 1);
          const uint32_t bytes = (uint32_t)(p.W * p.row_bytes);
          mbar_expect_tx(&a_full[a_stage], bytes);
          const int row0 = (kPadRows + wi.m0 + p.omin) & ~7;  // multiple of 8: swizzle phases line up
          const __half* src = p.x16 + (((size_t)wi.b * p.x_pchunks + (c % p.x_pchunks)) * p.x_Lp + (size_t)row0) * p.cw;
          bulk_g2s(smem_u32(a_base + (size_t)a_stage * p.a_stage_bytes), src, bytes, &a_full[a_stage]);
          if (++a_stage == kAStages) { a_stage = 0; a_phase ^= 1; }
          for (int t = 0; t < p.ntaps[wi.r]; ++t) {
            const int sid = p.slab[wi.r][t] * p.n_cchunks + c;
            const __half* src = p.w16 + (size_t)sid * (p.slab_bytes >> 1);
            if (p.resident) {
              if (!(resident_loaded & (1u << sid))) {
                resident_loaded |= (1u << sid);
                mbar_expect_tx(&w_full[sid], (uint32_t)p.slab_bytes);
                bulk_g2s(smem_u32(w_base + (size_t)sid * p.slab_bytes), src, (uint32_t)p.slab_bytes, &w_full[sid]);
              }
            } else {
              mbar_wait(&w_empty[w_stage], w_phase ^ 1);
              mbar_expect_tx(&w_full[w_stage], (uint32_t)p.slab_bytes);
              bulk_g2s(smem_u32(w_base + (size_t)w_stage * p.slab_bytes), src, (uint32_t)p.slab_bytes,
                       &w_full[w_stage]);
              if (++w_stage == p.wstages) { w_stage = 0; w_phase ^= 1; }
            }
          }
        }
      }
    }
  } else {
    // ===================== MMA + epilogue (warpgroups 1 and 2) =====================
    // Warpgroup g owns rows [g * MT * 64, (g + 1) * MT * 64) of the work item: MT accumulators of 64 rows x N columns.
    // A (tap, K-chunk) step is one commit group of NK16 * MT wgmmas; a group's operand stages are released once the NEXT
    // group is issued and this one has completed (wait_group 1), so two groups are in flight.
    regs_inc<232>();
    constexpr uint32_t ROWB = CW * 2;
    constexpr int NK16 = CW / 16;
    constexpr uint32_t MT_STEP = (64u * ROWB) >> 4;
    const int g = warp / 4 - 1;
    const int tid = threadIdx.x & 127;
    const bool leader = tid == 0;
    const uint64_t desc_hi = make_desc(0, 8u * ROWB, CW == 64 ? 1u : 2u, 0);  // everything but the address
    float* stage = stage_s + g * 64 * kStageLd;
    int a_stage = 0, a_phase = 0, w_stage = 0, w_phase = 0;
    uint32_t resident_seen = 0;  // resident weight images whose arrival has already been observed
    bool w2_seen = false;        // PAIR: c2's weights have arrived
    float acc[MT][N / 2];
    const int C4 = p.Cout >> 2;
    const int ocw = f16_cw(p.Cout);  // output plane: channels per row chunk
    for (int work = blockIdx.x; work < p.n_work; work += gridDim.x) {
      const WorkItem wi = decode_work(p, work);
      const int delta = (kPadRows + wi.m0 + p.omin) & 7;  // rows the window start was rounded down by
      const int nt = p.ntaps[wi.r];
      int pend_a = -1, pend_w = -1;  // stages of the group in flight that is not yet released
      bool first = true;
      wgmma_fence();
      for (int c = 0; c < p.n_cchunks; ++c) {
        mbar_wait(&a_full[a_stage], a_phase);
        const uint32_t a_addr = smem_u32(a_base + (size_t)a_stage * p.a_stage_bytes);
        for (int t = 0; t < nt; ++t) {
          uint32_t w_addr;
          if (p.resident) {
            const int sid = p.slab[wi.r][t] * p.n_cchunks + c;
            if (!(resident_seen & (1u << sid))) {
              mbar_wait(&w_full[sid], 0);
              resident_seen |= 1u << sid;
            }
            w_addr = smem_u32(w_base + (size_t)sid * p.slab_bytes);
          } else {
            mbar_wait(&w_full[w_stage], w_phase);
            w_addr = smem_u32(w_base + (size_t)w_stage * p.slab_bytes);
          }
          uint32_t a_row = a_addr + (uint32_t)(delta + p.off[wi.r][t] - p.omin) * ROWB;
          const uint64_t a0 = desc_hi + (uint64_t)((a_row + (uint32_t)(g * MT) * 64u * ROWB) >> 4) +
                              (p.baseoff_mode ? ((uint64_t)((a_row >> 7) & 7) << 49) : 0);
          const uint64_t b0 = desc_hi + (uint64_t)(w_addr >> 4);
#pragma unroll
          for (int mt = 0; mt < MT; ++mt) fence_acc(acc[mt]);
          wgmma_fence();
#pragma unroll
          for (int s = 0; s < NK16; ++s)
#pragma unroll
            for (int mt = 0; mt < MT; ++mt)
              wgmma_f16<N>(acc[mt], a0 + (uint64_t)(2 * s + mt * MT_STEP), b0 + (uint64_t)(2 * s), (first && s == 0) ? 0u : 1u);
          wgmma_commit();
          first = false;
          wgmma_wait<1>();
#pragma unroll
          for (int mt = 0; mt < MT; ++mt) fence_acc(acc[mt]);
          if (leader) {
            if (pend_w >= 0) mbar_arrive(&w_empty[pend_w]);
            if (pend_a >= 0) mbar_arrive(&a_empty[pend_a]);
          }
          pend_w = p.resident ? -1 : w_stage;
          pend_a = (t == nt - 1) ? a_stage : -1;
          if (!p.resident) {
            if (++w_stage == p.wstages) { w_stage = 0; w_phase ^= 1; }
          }
        }
        if (++a_stage == kAStages) { a_stage = 0; a_phase ^= 1; }
      }
      wgmma_wait<0>();
#pragma unroll
      for (int mt = 0; mt < MT; ++mt) fence_acc(acc[mt]);
      if (leader) {
        if (pend_w >= 0) mbar_arrive(&w_empty[pend_w]);
        if (pend_a >= 0) mbar_arrive(&a_empty[pend_a]);
      }
      if constexpr (PAIR) {
        // ---- c1 epilogue -> mid (fp16, swizzled like the operand planes); rows outside [0, valid) are c2's zero padding
        uint8_t* mid = smem + p.mid_off;
        const int valid_mid = p.lengths ? min(p.Lin, p.lengths[wi.b] * p.len_mul_mid) : p.Lin;
        group_sync(3, 128 * kMmaGroups);  // both warpgroups are done reading the previous item's mid
        const int w = tid >> 5, l = tid & 31;
#pragma unroll
        for (int mt = 0; mt < MT; ++mt) {
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int r = (g * MT + mt) * 64 + 16 * w + (l >> 2) + 8 * h;
            const int sq = wi.m0 - p.h2 + r;
            const bool live = sq >= 0 && sq < valid_mid;
            const int sw = f16_swz(CW, r);
#pragma unroll
            for (int jj = 0; jj < N / 8; ++jj) {
              const int col = 8 * jj + 2 * (l & 3);
              float a0 = 0.f, a1 = 0.f;
              if (live) {
                a0 = lrelu(acc[mt][4 * jj + 2 * h + 0] + p.bias1[col], p.slope_mid);
                a1 = lrelu(acc[mt][4 * jj + 2 * h + 1] + p.bias1[col + 1], p.slope_mid);
              }
              *reinterpret_cast<__half2*>(mid + (size_t)r * ROWB + ((jj ^ sw) << 4) + (col & 7) * 2) = __floats2half2_rn(a0, a1);
            }
          }
        }
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // generic-proxy stores -> wgmma operand reads
        group_sync(3, 128 * kMmaGroups);
        if (!w2_seen) {
          mbar_wait(w2_full, 0);
          w2_seen = true;
        }
        // ---- c2: output row i reads mid rows i + h2 + off2[t]
        const uint32_t mid_addr = smem_u32(mid) + (uint32_t)(g * MT) * 64u * ROWB;
        for (int t = 0; t < p.k2; ++t) {
          const uint64_t a0 = desc_hi + (uint64_t)((mid_addr + (uint32_t)(p.h2 + p.off2[t]) * ROWB) >> 4);
          const uint64_t b0 = desc_hi + (uint64_t)(smem_u32(smem + p.w2_off + (size_t)t * p.slab2_bytes) >> 4);
#pragma unroll
          for (int mt = 0; mt < MT; ++mt) fence_acc(acc[mt]);
          wgmma_fence();
#pragma unroll
          for (int s = 0; s < NK16; ++s)
#pragma unroll
            for (int mt = 0; mt < MT; ++mt)
              wgmma_f16<N>(acc[mt], a0 + (uint64_t)(2 * s + mt * MT_STEP), b0 + (uint64_t)(2 * s), (t == 0 && s == 0) ? 0u : 1u);
          wgmma_commit();
        }
        wgmma_wait<0>();
#pragma unroll
        for (int mt = 0; mt < MT; ++mt) fence_acc(acc[mt]);
      }
      // ---- epilogue: per (row tile, 32-column unit) the slice goes through shared memory so that a thread owns one row and
      // 16 consecutive columns (the fp16 plane stores 8 channels and the F32B plane 4 channels per 16-byte access)
      const int valid_out = p.lengths ? min(p.Lout, p.lengths[wi.b] * p.len_mul_out) : p.Lout;
      const int row_in_tile = tid & 63;
#pragma unroll
      for (int mt = 0; mt < MT; ++mt) {
#pragma unroll
        for (int u = 0; u < N / 32; ++u) {
          const int col0 = u * 32 + (tid >> 6) * UC;
          const int q = wi.m0 + (g * MT + mt) * 64 + row_in_tile;
          const int lo = q * p.stride + wi.r;
          const bool inb = q < p.Lin && (g * MT + mt) * 64 + row_in_tile < p.rows_item;
          const bool live = inb && lo < valid_out;
          const size_t i32 = ((size_t)wi.b * C4 + (col0 >> 2)) * p.Lout + lo;  // + g * Lout per 4 channels
          float4 rv[UC / 4], ov[UC / 4];
          uint4 rh[UC / 8];
          if (inb && p.res32) {
#pragma unroll
            for (int j = 0; j < UC / 4; ++j) rv[j] = reinterpret_cast<const float4*>(p.res32)[i32 + (size_t)j * p.Lout];
          }
          if (inb && p.res16) {  // (the lo halves of a hi/lo residual share rv's registers: res32 and res16 are exclusive)
            const int rr = kPadRows + lo;
            if (!p.res_hilo) {
              const size_t rbase = (((size_t)wi.b * (p.Cout / ocw) + col0 / ocw) * p.res_Lp + rr) * (size_t)(ocw >> 3);
              const int c0 = (col0 & (ocw - 1)) >> 3, sw = f16_swz(ocw, rr);
#pragma unroll
              for (int j = 0; j < UC / 8; ++j) rh[j] = reinterpret_cast<const uint4*>(p.res16)[rbase + (size_t)((c0 + j) ^ sw)];
            } else {
              // hi/lo plane: rows of 64 channels; hi block = channels [0, Cout), lo block = [Cout, 2 Cout)
              const int nch = (2 * p.Cout) >> 6, sw = f16_swz(64, rr);
#pragma unroll
              for (int j = 0; j < UC / 8; ++j) {
                const int ch = col0 + 8 * j, cl = ch + p.Cout;
                rh[j] = reinterpret_cast<const uint4*>(p.res16)[(((size_t)wi.b * nch + (ch >> 6)) * p.res_Lp + rr) * 8 + (size_t)(((ch & 63) >> 3) ^ sw)];
                rv[j] = reinterpret_cast<const float4*>(p.res16)[(((size_t)wi.b * nch + (cl >> 6)) * p.res_Lp + rr) * 8 + (size_t)(((cl & 63) >> 3) ^ sw)];
              }
            }
          }
          if (inb && p.mode != EPI_STORE && !p.red_add) {
#pragma unroll
            for (int j = 0; j < UC / 4; ++j) ov[j] = reinterpret_cast<const float4*>(p.y32)[i32 + (size_t)j * p.Lout];
          }
          group_sync(1 + g, 128);  // the previous unit's rows have been read
          stage_acc32(stage, &acc[mt][u * 16], tid);
          group_sync(1 + g, 128);
          if (!inb) continue;
          float v[UC];
          const float* srow = stage + row_in_tile * kStageLd + (tid >> 6) * UC;
#pragma unroll
          for (int i = 0; i < UC; ++i) v[i] = srow[i] * p.acc_scale + bias_s[col0 + i];
          if (p.res32) {
#pragma unroll
            for (int j = 0; j < UC / 4; ++j) {
              v[4 * j + 0] += rv[j].x; v[4 * j + 1] += rv[j].y; v[4 * j + 2] += rv[j].z; v[4 * j + 3] += rv[j].w;
            }
          }
          if (p.res16) {
#pragma unroll
            for (int j = 0; j < UC / 8; ++j) {
              if (p.res_hilo) add_res16_hilo(&v[8 * j], rh[j], *reinterpret_cast<const uint4*>(&rv[j]), p.res_inv);
              else add_res16(&v[8 * j], rh[j], p.res_inv);
            }
          }
          if (p.mode != EPI_STORE && !p.red_add) {
#pragma unroll
            for (int j = 0; j < UC / 4; ++j) {
              v[4 * j + 0] += ov[j].x; v[4 * j + 1] += ov[j].y; v[4 * j + 2] += ov[j].z; v[4 * j + 3] += ov[j].w;
            }
            if (p.mode == EPI_ADD_DIV) {
#pragma unroll
              for (int i = 0; i < UC; ++i) v[i] /= p.div;
            }
          }
          if (!live) {
#pragma unroll
            for (int i = 0; i < UC; ++i) v[i] = 0.f;
          }
          if (p.red_add) {  // MRF sum of a middle resblock: S += v by vector reductions in L2 (rows past the length add nothing)
            if (live) {
#pragma unroll
              for (int j = 0; j < UC / 4; ++j)
                red_add_f32x4(p.y32 + (i32 + (size_t)j * p.Lout) * 4, v[4 * j + 0], v[4 * j + 1], v[4 * j + 2], v[4 * j + 3]);
            }
          } else if (p.y32) {
#pragma unroll
            for (int j = 0; j < UC / 4; ++j)
              reinterpret_cast<float4*>(p.y32)[i32 + (size_t)j * p.Lout] =
                  make_float4(v[4 * j + 0], v[4 * j + 1], v[4 * j + 2], v[4 * j + 3]);
          }
          if (p.y16) {
            const int rr = kPadRows + lo;
            const int ysw = f16_swz(p.y_cw, rr);
            const int ycw8 = p.y_cw >> 3;
#pragma unroll
            for (int j = 0; j < UC / 8; ++j) {
              float a[8];
#pragma unroll
              for (int e = 0; e < 8; ++e) a[e] = lrelu(v[8 * j + e], p.out_slope);
              __half2 h[4];
#pragma unroll
              for (int e = 0; e < 4; ++e) h[e] = __floats2half2_rn(a[2 * e], a[2 * e + 1]);
              uint4 pk;
              pk.x = *reinterpret_cast<uint32_t*>(&h[0]);
              pk.y = *reinterpret_cast<uint32_t*>(&h[1]);
              pk.z = *reinterpret_cast<uint32_t*>(&h[2]);
              pk.w = *reinterpret_cast<uint32_t*>(&h[3]);
              const int ct = p.y_c0 + col0 + 8 * j;  // channel of the (hi) block
              const int chunk = ct / p.y_cw, cc = ct - chunk * p.y_cw;
              const size_t i16 = (((size_t)wi.b * p.y_nchunks + chunk) * p.y_Lp + rr) * (size_t)ycw8 + (size_t)((cc >> 3) ^ ysw);
              reinterpret_cast<uint4*>(p.y16)[i16] = pk;
              if (p.y_lo_c >= 0) {
                __half2 l2[4];
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                  const float2 hf = __half22float2(h[e]);
                  l2[e] = __floats2half2_rn(a[2 * e] - hf.x, a[2 * e + 1] - hf.y);
                }
                uint4 pl;
                pl.x = *reinterpret_cast<uint32_t*>(&l2[0]);
                pl.y = *reinterpret_cast<uint32_t*>(&l2[1]);
                pl.z = *reinterpret_cast<uint32_t*>(&l2[2]);
                pl.w = *reinterpret_cast<uint32_t*>(&l2[3]);
                const int ctl = ct + p.y_lo_c;
                const int chl = ctl / p.y_cw, ccl = ctl - chl * p.y_cw;
                const size_t j16 = (((size_t)wi.b * p.y_nchunks + chl) * p.y_Lp + rr) * (size_t)ycw8 + (size_t)((ccl >> 3) ^ ysw);
                reinterpret_cast<uint4*>(p.y16)[j16] = pl;
              }
            }
          }
        }
      }
    }
  }
}

// fp32 slabs [K][Cin][Cout] -> fp16 images [K][n_cchunks][Cout][cw], rows swizzled like the operand planes
__global__ void pack_w16_kernel(const float* __restrict__ w32, __half* __restrict__ dst, int K, int Cin, int Cout,
                                int cw) {
  const size_t n = (size_t)K * Cin * Cout;
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  // source-linear index -> (k, ci, co)
  const int co = (int)(i % Cout);
  const int ci = (int)((i / Cout) % Cin);
  const int k = (int)(i / ((size_t)Cout * Cin));
  const int nch = Cin / cw;
  const int c = ci / cw, cc = ci - c * cw;
  const size_t img = ((size_t)k * nch + c) * (size_t)Cout * cw;
  const size_t off = (size_t)co * cw + (size_t)((((cc >> 3) ^ f16_swz(cw, co)) << 3) + (cc & 7));
  dst[img + off] = __float2half_rn(w32[i]);
}

// 3-term-split layer over an internal hi/lo plane: K-chunks [hi | lo | hi] x images [hi(w) | hi(w) | lo(w)] (Cin >= 64), or for
// Cin == 32 the single 64-channel plane chunk [hi32 | lo32] twice: images [hi(w) | hi(w)] and [lo(w) | 0].  w is pre-scaled by
// kX3WScale (power of two; the epilogue multiplies the accumulator by its inverse) so that lo(w) is a normal fp16.
__global__ void pack_w16_x3_kernel(const float* __restrict__ w32, __half* __restrict__ dst, int K, int Cin, int Cout, float wscale) {
  const int nK = Cin >= 64 ? 3 * (Cin / 64) : 2;
  const size_t n = (size_t)K * nK * Cout * 64;
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int cc = (int)(i & 63);
  const int co = (int)((i >> 6) % Cout);
  const int j = (int)((i / ((size_t)64 * Cout)) % nK);
  const int k = (int)(i / ((size_t)64 * Cout * nK));
  int ci, part;  // part 0: hi(w), 1: lo(w), 2: zero
  if (Cin >= 64) {
    const int nc = Cin / 64;
    part = j < 2 * nc ? 0 : 1;
    ci = (j % nc) * 64 + cc;
  } else {
    ci = cc & 31;
    part = j == 0 ? 0 : (cc < 32 ? 1 : 2);
  }
  __half v = __float2half_rn(0.f);
  if (part < 2) {
    const float w = w32[((size_t)k * Cin + ci) * Cout + co] * wscale;
    const __half hi = __float2half_rn(w);
    v = part == 0 ? hi : __float2half_rn(w - __half2float(hi));
  }
  const size_t img = ((size_t)k * nK + j) * (size_t)Cout * 64;
  const size_t off = (size_t)co * 64 + (size_t)((((cc >> 3) ^ f16_swz(64, co)) << 3) + (cc & 7));
  dst[img + off] = v;
}

// ---- 3-term split of an fp32 layer (conv_pre) --------------------------------------------------------
// input plane channels: [hi(x) (Cin) | lo(x) (Cin) | hi(x) (Cin) | 0 ...] (256 channels, no activation),
// weight images:        [hi(w)       | hi(w)       | lo(w)       | 0 ...]  -> sum = x*w up to ~2^-22 relative.
__device__ __forceinline__ __half split_hi(float v) { return __float2half_rn(v); }
__device__ __forceinline__ __half split_lo(float v) { return __float2half_rn(v - __half2float(__float2half_rn(v))); }

__global__ void split3_input_kernel(const float* __restrict__ x /* NCL [B][Cin][L] */, __half* __restrict__ dst, int B,
                                    int Cin, int L, const int32_t* __restrict__ lengths) {
  // one thread per (b, 16-byte chunk of the 256-channel row, l); l fastest -> coalesced reads of x
  const size_t n = (size_t)B * 32 * L;
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int l = (int)(i % L);
  const int ch8 = (int)((i / L) % 32);
  const int b = (int)(i / ((size_t)L * 32));
  __align__(16) __half h[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    const int c = ch8 * 8 + e;
    const int part = c / Cin, ci = c - part * Cin;
    float v = 0.f;
    if (part < 3 && (!lengths || l < lengths[b])) v = x[((size_t)b * Cin + ci) * L + l];  // frames past the length read as zero padding
    h[e] = part == 1 ? split_lo(v) : (part < 3 ? split_hi(v) : __float2half_rn(0.f));
  }
  const int Lp = f16_lp(L);
  const int r = kPadRows + l;
  const int chunk = ch8 >> 3, cc8 = ch8 & 7;
  const size_t o = (((size_t)b * 4 + chunk) * Lp + r) * 8 + (size_t)(cc8 ^ f16_swz(64, r));
  reinterpret_cast<uint4*>(dst)[o] = *reinterpret_cast<const uint4*>(h);
}

// fp32 slabs [K][Cin][Cout] -> per 256-output half: images [K][4 chunks][256][64] (swizzled rows)
__global__ void pack_w16_split3_kernel(const float* __restrict__ w32, __half* __restrict__ dst, int K, int Cin, int Cout) {
  const size_t n = (size_t)K * 256 * Cout;
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int co = (int)(i % Cout);
  const int c = (int)((i / Cout) % 256);
  const int k = (int)(i / ((size_t)Cout * 256));
  const int part = c / Cin, ci = c - part * Cin;
  __half v = __float2half_rn(0.f);
  if (part < 3) {
    const float w = w32[((size_t)k * Cin + ci) * Cout + co];
    v = part == 2 ? split_lo(w) : split_hi(w);
  }
  const int half_idx = co >> 8, col = co & 255;
  const int chunk = c >> 6, cc = c & 63;
  const size_t img = (((size_t)half_idx * K + k) * 4 + chunk) * (size_t)(256 * 64);
  const size_t off = (size_t)col * 64 + (size_t)((((cc >> 3) ^ f16_swz(64, col)) << 3) + (cc & 7));
  dst[img + off] = v;
}

bool tc_split3_enabled();
bool split3_capable(const TapConv& t) {
  return tc_split3_enabled() && t.stride == 1 && !t.act_tanh && t.Cin * 3 <= 256 && t.Cout % 256 == 0 && t.Cout >= 256 &&
         t.mode == EPI_STORE;
}

int pick_kc(int Cin) {
  if (Cin % 64 == 0) return 64;
  if (Cin == 32) return 32;
  return 0;
}

// shapes the 3-term-split variant of tc_conv_kernel covers (operand rows are always 64 channels wide)
bool x3_capable(const TapConv& t) {
  if (t.Cout != 32 && t.Cout != 64 && t.Cout != 128 && t.Cout != 256) return false;
  if (t.Cin != 32 && t.Cin % 64 != 0) return false;
  return !t.act_tanh;
}

bool tc_capable(const TapConv& t) {
  if (t.Cout != 32 && t.Cout != 64 && t.Cout != 128 && t.Cout != 256) return false;  // kernel instances
  if (t.Cout != 32 && pick_kc(t.Cin) != 64) return false;
  if (pick_kc(t.Cin) == 0) return false;
  if (t.act_tanh) return false;
  return true;
}

// row tiles per work item: MT x Cout <= 256 accumulator columns (128 registers per MMA thread), and as shared memory allows
int pick_mt_max(int Cout) { return Cout >= 256 ? 1 : (Cout >= 128 ? 2 : (Cout >= 64 ? 4 : 8)); }

struct SmemPlan {
  uint32_t a_stage_bytes, a_off, w_off, bias_off, bar_off, stage_off, ex_off, total;
  int wstages, resident, W, omin;
};

// `extra`: bytes of a 1024-aligned region after everything else (fused pair: c2's weights and the intermediate rows)
bool plan_smem(const TapConv& t, const TcLayer& tc, int total_slabs, SmemPlan* sp, uint32_t extra = 0) {
  int omin = 0x7fffffff, omax = -0x7fffffff;
  for (int r = 0; r < t.stride; ++r)
    for (int i = 0; i < t.ntaps[r]; ++i) {
      omin = std::min(omin, t.off[r][i]);
      omax = std::max(omax, t.off[r][i]);
    }
  if (-omin > kPadRows || omax > kPadRows) return false;
  const int row_bytes = tc.kc * 2;
  sp->omin = omin;
  sp->W = (tc.mt * 128 + (omax - omin) + 7 + 7) & ~7;  // + up to 7 rows of start rounding, multiple of 8
  sp->a_stage_bytes = (uint32_t)align_up((size_t)sp->W * row_bytes, 1024);
  sp->a_off = 0;
  sp->w_off = sp->a_off + kAStages * sp->a_stage_bytes;
  const uint32_t tail = (uint32_t)align_up((size_t)t.Cout * 4, 128) + 1024 + kStageBytes + (extra ? 1024 + extra : 0);
  const uint32_t usable = kSmemMax - 1024;  // the kernel aligns its base to 1024 B
  if (sp->w_off + tail + 2 * tc.slab_bytes > usable) return false;
  int ws = (int)((usable - sp->w_off - tail) / tc.slab_bytes);
  ws = std::min(ws, kMaxWStages);
  sp->resident = (total_slabs <= ws) ? 1 : 0;
  sp->wstages = sp->resident ? total_slabs : ws;
  sp->bias_off = sp->w_off + (uint32_t)sp->wstages * (uint32_t)tc.slab_bytes;
  sp->bar_off = sp->bias_off + (uint32_t)align_up((size_t)t.Cout * 4, 128);
  sp->stage_off = sp->bar_off + 1024;
  sp->ex_off = (uint32_t)align_up((size_t)sp->stage_off + kStageBytes, 1024);
  sp->total = extra ? sp->ex_off + extra : sp->stage_off + kStageBytes;
  return sp->total <= usable;
}

int kernel_count(const TapConv& t) {
  int k = 0;
  for (int r = 0; r < t.stride; ++r)
    for (int i = 0; i < t.ntaps[r]; ++i) k = std::max(k, t.slab[r][i] + 1);
  return k;
}

// MB_TC_FUSE=0: resblock pairs as two tc_conv launches instead of one fused launch
bool tc_fuse_enabled() {
  static int on = -1;
  if (on < 0) {
    const char* e = getenv("MB_TC_FUSE");
    on = e ? atoi(e) : 1;
  }
  return on != 0;
}

// fused resblock pair: c1's taps shifted by -h2 rows (the launch computes c1 on rows m0 - h2 ...), the row tiles per item and
// the shared-memory plan with c2's weights and the intermediate rows in the extra region
struct PairPlan {
  TapConv t1;
  int mt, h2;
  SmemPlan sp;
  uint32_t w2_off, mid_off;
};
bool pair_plan(const TcOp& c1, const TcOp& c2, PairPlan* pl) {
  const int C = c1.taps.Cout;
  if (!(C == 32 || C == 64) || c1.tc.n_cchunks != 1 || c2.tc.n_cchunks != 1) return false;
  const int k2 = c2.taps.ntaps[0];
  pl->h2 = (k2 - 1) / 2;
  pl->t1 = c1.taps;
  for (int i = 0; i < pl->t1.ntaps[0]; ++i) pl->t1.off[0][i] -= pl->h2;
  const int rowb = c1.tc.kc * 2;
  const int mts[2] = {C == 64 ? 2 : 8, C == 64 ? 1 : 4};  // kernel instances
  for (int mt : mts) {
    TcLayer tc = c1.tc;
    tc.mt = mt;
    const uint32_t w2_bytes = (uint32_t)align_up((size_t)k2 * c2.tc.slab_bytes, 1024);
    const uint32_t mid_bytes = (uint32_t)align_up((size_t)((mt * 128 + 2 * pl->h2 + 7) & ~7) * rowb, 1024);
    if (mt * 128 <= 2 * pl->h2) continue;
    if (plan_smem(pl->t1, tc, kernel_count(c1.taps), &pl->sp, w2_bytes + mid_bytes)) {
      pl->mt = mt;
      pl->w2_off = pl->sp.ex_off;
      pl->mid_off = pl->sp.ex_off + w2_bytes;
      return true;
    }
  }
  return false;
}

// MB_TC_RES16=0 keeps an fp32 residual plane in every stage (default: only in the full-rate stage; the
// other stages carry the residual stream as ONE activated fp16 plane that is both the next conv's operand
// and - through the exact inverse of the leaky-relu - the residual; error budget in DESIGN.md 3.4)
bool tc_res16_enabled() {
  static int on = -1;
  if (on < 0) {
    const char* e = getenv("MB_TC_RES16");
    on = e ? atoi(e) : 1;
  }
  return on != 0;
}

// MB_TC_X3_RES16=0: 3-term-split layers keep an fp32 residual plane (default: residual = inv_lrelu(hi + lo) of the hi/lo plane)
bool tc_x3_res16_enabled() {
  static int on = -1;
  if (on < 0) {
    const char* e = getenv("MB_TC_X3_RES16");
    on = e ? atoi(e) : 1;
  }
  return on != 0;
}

// MB_TC_SPLIT3=0 keeps conv_pre on the FP32 FFMA kernel
bool tc_split3_enabled() {
  static int on = -1;
  if (on < 0) {
    const char* e = getenv("MB_TC_SPLIT3");
    on = e ? atoi(e) : 1;
  }
  return on != 0;
}

// how the A descriptor encodes a start address that is not 1024-byte aligned (row-shifted taps).
// The operand fetch applies the swizzle XOR on absolute shared-memory address bits, so the matrix-base-offset field stays 0
// (mode 0, default; tests/test_gan_tc_layers.py checks every layer shape against torch); mode 1 (field = address bits 7..9)
// is kept for A/B checks of that assumption.
int tc_baseoff_mode() {
  static int mode = -1;
  if (mode < 0) {
    const char* e = getenv("MB_TC_BASEOFF");
    mode = e ? atoi(e) : 0;
  }
  return mode;
}

// every compiled tc_conv_kernel instance <N, MT, CW, PAIR>; launch_tc and the plan query pick from this list.  tc_plan_layers
// never picks <32, 2, 64>, <32, 4, 32> or <64, 1, 64> for a layer launched alone (a C = 32 fp16 layer's weights are resident at
// MT = 8, a C = 64 layer always fits MT >= 2), so those are not compiled.
struct TcInstance {
  int n, mt, cw;
  bool pair;
  void (*kern)(const TcParams);
};
const TcInstance kTcInstances[] = {
    {256, 1, 64, false, tc_conv_kernel<256, 1, 64>},
    {128, 2, 64, false, tc_conv_kernel<128, 2, 64>},
    {128, 1, 64, false, tc_conv_kernel<128, 1, 64>},
    {64, 4, 64, false, tc_conv_kernel<64, 4, 64>},
    {64, 2, 64, false, tc_conv_kernel<64, 2, 64>},
    {32, 8, 32, false, tc_conv_kernel<32, 8, 32>},
    {32, 4, 64, false, tc_conv_kernel<32, 4, 64>},
    {64, 2, 64, true, tc_conv_kernel<64, 2, 64, true>},
    {64, 1, 64, true, tc_conv_kernel<64, 1, 64, true>},
    {32, 8, 32, true, tc_conv_kernel<32, 8, 32, true>},
    {32, 4, 32, true, tc_conv_kernel<32, 4, 32, true>},
};
const TcInstance* find_instance(int n, int mt, int cw, bool pair) {
  for (const TcInstance& k : kTcInstances)
    if (k.n == n && k.mt == mt && k.cw == cw && k.pair == pair) return &k;
  return nullptr;
}

size_t f16_plane_bytes(size_t B, size_t T, size_t cr) {
  // rows are padded to Lp = ceil8(L + 2*kPadRows) <= L + 2*kPadRows + 7 for at most 512 channels
  return align_up(2 * B * T * cr + 2 * B * 1024 * (2 * kPadRows + 7) + kPlaneSlack, 1024);  // pad rows of <= 1024 channels (hi/lo of 512)
}
size_t f32_plane_bytes(size_t B, size_t T, size_t cr) { return align_up(4 * B * T * cr + 256, 1024); }

// red_add: an EPI_ADD launch without fp16 output may accumulate by red.global.add (else read-add-store).
// info (optional): what was launched.
int launch_tc(const TcOp& op, const char* tc_arena, const TRef& x16, const TRef& res32, const TRef& res16, float res_slope,
              const TRef& y32, const TRef& y16, float out_slope, const int32_t* lengths, int B, int Lin, cudaStream_t st,
              bool red_add, int y_c0 = 0, const float* bias_override = nullptr, const TcOp* c2 = nullptr,
              TcLaunchInfo* info = nullptr) {
  PairPlan pl;
  if (c2 && !pair_plan(op, *c2, &pl)) return fail(MB_ERR_INVALID, "tc_pair(%s): no shared-memory plan", op.name);
  const TapConv& t = c2 ? pl.t1 : op.taps;
  TcParams p;
  memset(&p, 0, sizeof(p));
  p.B = B;
  p.Lin = Lin;
  p.Lout = Lin * t.stride;
  p.Cin = t.Cin;
  p.Cout = t.Cout;
  p.stride = t.stride;
  memcpy(p.ntaps, t.ntaps, sizeof(p.ntaps));
  memcpy(p.off, t.off, sizeof(p.off));
  memcpy(p.slab, t.slab, sizeof(p.slab));
  SmemPlan sp;
  const int total_slabs = kernel_count(t) * op.tc.n_cchunks;
  if (c2) sp = pl.sp;
  else if (!plan_smem(t, op.tc, total_slabs, &sp)) return fail(MB_ERR_INVALID, "tc_conv(%s): shared memory plan failed", op.name);
  p.omin = sp.omin;
  p.W = sp.W;
  p.MT = c2 ? pl.mt : op.tc.mt;
  p.cw = op.tc.kc;
  p.row_bytes = op.tc.kc * 2;
  p.baseoff_mode = tc_baseoff_mode();
  p.nk16 = op.tc.kc / 16;
  p.n_cchunks = op.tc.n_cchunks;
  p.slab_bytes = (int)op.tc.slab_bytes;
  p.wstages = sp.wstages;
  p.resident = sp.resident;
  p.rows_item = p.MT * 128 - (c2 ? 2 * pl.h2 : 0);
  p.tiles_per_utt = (Lin + p.rows_item - 1) / p.rows_item;
  p.n_work = B * p.tiles_per_utt * p.stride;
  p.a_stage_bytes = sp.a_stage_bytes;
  p.a_off = sp.a_off;
  p.w_off = sp.w_off;
  p.bias_off = sp.bias_off;
  p.bar_off = sp.bar_off;
  p.stage_off = sp.stage_off;
  p.x16 = reinterpret_cast<const __half*>(x16.p);
  p.x_Lp = f16_lp(x16.L);
  p.x_pchunks = op.tc.x3 ? op.tc.x_pchunks : op.tc.n_cchunks;
  p.acc_scale = op.tc.x3 ? 1.f / kX3WScale : 1.f;
  if (op.tc.x3 && (!x16.hilo || x16.C != 64 * op.tc.x_pchunks))
    return fail(MB_ERR_INVALID, "tc_conv(%s): 3-term-split layer needs a hi/lo input plane", op.name);
  if (!op.tc.x3 && !op.tc.split3 && x16.hilo) return fail(MB_ERR_INVALID, "tc_conv(%s): plain layer fed a hi/lo plane", op.name);
  p.w16 = reinterpret_cast<const __half*>(tc_arena + op.tc.w16_off);
  p.bias = bias_override ? bias_override : op.b32;
  p.res32 = reinterpret_cast<const float*>(res32.p);
  p.res16 = reinterpret_cast<const __half*>(res16.p);
  p.res_Lp = f16_lp(res16.L);
  p.res_hilo = res16.p ? res16.hilo : 0;
  p.res_inv = 1.f / res_slope;
  p.y32 = reinterpret_cast<float*>(y32.p);
  p.y16 = reinterpret_cast<__half*>(y16.p);
  p.y_Lp = f16_lp(y16.L);
  p.y_cw = f16_cw(y16.p ? y16.C : t.Cout);
  p.y_nchunks = (y16.p ? y16.C : t.Cout) / p.y_cw;
  p.y_c0 = y_c0;
  p.y_lo_c = (y16.p && y16.hilo) ? (y16.C >> 1) : -1;
  p.out_slope = out_slope;
  p.mode = t.mode;
  p.red_add = (p.mode == EPI_ADD && !y16.p && y32.p && red_add) ? 1 : 0;
  p.div = t.div;
  p.lengths = lengths;
  p.len_mul_out = t.len_mul_out;
  if (c2) {  // c2 owns bias, accumulate mode and outputs; c1's bias and slope go to the intermediate
    const TapConv& u = c2->taps;
    p.k2 = u.ntaps[0];
    p.h2 = pl.h2;
    for (int i = 0; i < p.k2; ++i) p.off2[i] = u.off[0][i];
    p.w2 = reinterpret_cast<const __half*>(tc_arena + c2->tc.w16_off);
    p.slab2_bytes = (uint32_t)c2->tc.slab_bytes;
    p.w2_off = pl.w2_off;
    p.mid_off = pl.mid_off;
    p.bias1 = op.b32;
    p.bias = c2->b32;
    p.slope_mid = u.in_slope;
    p.len_mul_mid = op.taps.len_mul_out;
    p.mode = u.mode;
    p.div = u.div;
    p.len_mul_out = u.len_mul_out;
    p.red_add = (p.mode == EPI_ADD && !y16.p && y32.p && red_add) ? 1 : 0;
  }
  if (res16.p && !res16.hilo && res16.C != t.Cout) return fail(MB_ERR_INVALID, "tc_conv(%s): fp16 residual plane geometry", op.name);
  if (res16.p && res16.hilo && res16.C != (t.Cout >= 64 ? 2 * t.Cout : 64)) return fail(MB_ERR_INVALID, "tc_conv(%s): hi/lo residual plane geometry", op.name);
  if (y_c0 != 0 && (p.y32 || p.res32 || p.res16)) return fail(MB_ERR_INVALID, "tc_conv(%s): channel-offset launch supports the fp16 plane only", op.name);
  if (p.mode != EPI_STORE && !p.y32) return fail(MB_ERR_INVALID, "tc_conv(%s): accumulate mode without fp32 plane", op.name);
  const TcInstance* inst = find_instance(p.Cout, p.MT, p.cw, c2 != nullptr);
  if (!inst)
    return fail(MB_ERR_INVALID, "%s(%s): no kernel instance for Cout=%d MT=%d cw=%d", c2 ? "tc_pair" : "tc_conv", op.name, p.Cout,
                p.MT, p.cw);
  void (*kern)(const TcParams) = inst->kern;
  MB_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmemMax));
  int dev = 0, sms = 0;
  MB_CUDA_CHECK(cudaGetDevice(&dev));
  MB_CUDA_CHECK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  const int grid = std::min(p.n_work, sms);
  if (info) {
    *info = TcLaunchInfo{};
    info->n = inst->n;
    info->mt = inst->mt;
    info->cw = inst->cw;
    info->pair = inst->pair ? 1 : 0;
    info->rows_item = p.rows_item;
    info->resident = p.resident;
    info->wstages = p.wstages;
    info->n_work = p.n_work;
    info->grid = grid;
    info->red_add = p.red_add;
  }
  if (grid <= 0) return MB_OK;
  // always claim the whole shared memory: one persistent CTA per SM
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = dim3(grid);
  cfg.blockDim = dim3(kTcThreads);
  cfg.dynamicSmemBytes = kSmemMax;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  MB_CUDA_CHECK(cudaLaunchKernelEx(&cfg, kern, p));
  MB_LAUNCH_CHECK("tc_conv_kernel");
  return MB_OK;
}

TRef make_ref(void* p, int layout, int C, int L) {
  TRef t;
  t.p = p;
  t.layout = p ? layout : LAYOUT_NONE;
  t.C = C;
  t.L = L;
  return t;
}

}  // namespace

// MB_TC_RED_ADD=0: accumulate-mode epilogues read, add and store the running sum themselves (round 2)
bool tc_red_add_enabled() {
  static int on = -1;
  if (on < 0) {
    const char* e = getenv("MB_TC_RED_ADD");
    on = e ? atoi(e) : 1;
  }
  return on != 0;
}


int tc_plan_layers(std::vector<TcLayerDesc>& layers, size_t* tc_arena_bytes) {
  size_t off = 0;
  for (TcLayerDesc& d : layers) {
    if (!d.is_conv) continue;
    TcLayer& tc = *d.tc;
    const TapConv& t = *d.taps;
    tc = TcLayer{};
    if (!d.force_f32 && !tc_capable(t) && split3_capable(t)) {
      // conv_pre: runs as Cout/256 launches of the <256,1,64> instance over a 256-channel split plane
      tc.split3 = 1;
      tc.kc = 64;
      tc.n_cchunks = 4;
      tc.mt = 1;
      tc.slab_bytes = (size_t)64 * 256 * 2;
      tc.w16_off = off;
      off += align_up((size_t)(t.Cout / 256) * d.k * 4 * tc.slab_bytes, 256);
      continue;  // use_tc stays 0: every generic decision treats the layer as an FP32-input layer
    }
    const bool x3 = d.want_x3 && !d.force_f32 && x3_capable(t);
    if (d.force_f32 || (!x3 && !tc_capable(t))) continue;
    if (x3) {
      tc.x3 = 1;
      tc.kc = 64;
      tc.n_cchunks = t.Cin >= 64 ? 3 * (t.Cin / 64) : 2;
      tc.x_pchunks = t.Cin >= 64 ? 2 * (t.Cin / 64) : 1;
    } else {
      tc.kc = pick_kc(t.Cin);
      tc.n_cchunks = t.Cin / tc.kc;
      tc.x_pchunks = tc.n_cchunks;
    }
    tc.slab_bytes = (size_t)tc.kc * t.Cout * 2;
    SmemPlan sp;
    bool ok = false;
    for (tc.mt = pick_mt_max(t.Cout); tc.mt >= 1; tc.mt >>= 1) {
      // keep the weights resident if a smaller tile count allows it; otherwise take the largest that fits
      if (plan_smem(t, tc, d.k * tc.n_cchunks, &sp)) {
        ok = true;
        TcLayer half = tc;
        half.mt = tc.mt >> 1;
        SmemPlan sp2;
        if (!sp.resident && half.mt >= 1 && plan_smem(t, half, d.k * tc.n_cchunks, &sp2) && sp2.resident) tc.mt = half.mt;
        break;
      }
    }
    if (!ok) continue;  // falls back to the FP32 kernel
    if (t.Cout == 32 && tc.kc == 64 && tc.mt > 4) tc.mt = 4;  // instance list below
    plan_smem(t, tc, d.k * tc.n_cchunks, &sp);
    if (sp.resident && d.k * tc.n_cchunks > 32) continue;
    tc.use_tc = 1;
    tc.w16_off = off;
    off += align_up((size_t)d.k * tc.n_cchunks * tc.slab_bytes, 256);
  }
  *tc_arena_bytes = off;
  return MB_OK;
}

int tc_pack_weights(const TcLayer& tc, const TapConv& taps, const float* w32_slabs, char* tc_arena,
                    cudaStream_t stream) {
  if (tc.split3) {
    const int K = kernel_count(taps);
    const size_t n = (size_t)K * 256 * taps.Cout;
    pack_w16_split3_kernel<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(
        w32_slabs, reinterpret_cast<__half*>(tc_arena + tc.w16_off), K, taps.Cin, taps.Cout);
    MB_LAUNCH_CHECK("pack_w16_split3_kernel");
    return MB_OK;
  }
  if (!tc.use_tc) return MB_OK;
  if (tc.x3) {
    const int K = kernel_count(taps);
    const size_t n = (size_t)K * tc.n_cchunks * taps.Cout * 64;
    pack_w16_x3_kernel<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(w32_slabs, reinterpret_cast<__half*>(tc_arena + tc.w16_off), K,
                                                                      taps.Cin, taps.Cout, kX3WScale);
    MB_LAUNCH_CHECK("pack_w16_x3_kernel");
    return MB_OK;
  }
  const int K = kernel_count(taps);
  const size_t n = (size_t)K * taps.Cin * taps.Cout;
  pack_w16_kernel<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(
      w32_slabs, reinterpret_cast<__half*>(tc_arena + tc.w16_off), K, taps.Cin, taps.Cout, tc.kc);
  MB_LAUNCH_CHECK("pack_w16_kernel");
  return MB_OK;
}

size_t tc_workspace_bytes(const std::vector<TcBufReq>& bufs, int B, int T, int num_mels, int hop) {
  (void)num_mels;
  (void)hop;
  size_t total = 2048;
  for (const TcBufReq& b : bufs) total += f16_plane_bytes(B, T, 2 * b.cr) + f32_plane_bytes(B, T, b.cr);  // 2x: hi/lo planes
  return total;
}

std::vector<char> tc_fusion_plan(const std::vector<TcOp>& ops, int nb) {
  const int n = (int)ops.size();
  std::vector<char> fuse_next(n, 0);
  for (int i = 0; i + 1 < n; ++i) {
    const TcOp& op = ops[i];
    const TcOp& c2 = ops[i + 1];
    if (!tc_fuse_enabled() || !op.is_conv || !op.tc.use_tc || !c2.is_conv || !c2.tc.use_tc) continue;
    if (op.tc.x3 || c2.tc.x3 || op.tc.split3 || c2.tc.split3) continue;  // 3-term-split layers run unfused
    const TapConv& t1 = op.taps;
    const TapConv& t2 = c2.taps;
    const int k = t1.ntaps[0];
    const int d1 = k > 1 ? t1.off[0][1] - t1.off[0][0] : 1;
    bool ok = op.cin == op.cout && c2.cin == c2.cout && op.cin == c2.cin && t1.stride == 1 && t2.stride == 1 &&
              t2.ntaps[0] == k && (k & 1) && op.res < 0 && op.dst2 < 0 && c2.dst2 < 0 && t1.mode == EPI_STORE &&
              op.dst == c2.src && op.dst >= 0 && op.dst < nb && op.src >= 0 && op.src < nb && c2.res != op.dst &&
              op.rate_in == c2.rate_in;
    for (int t = 0; ok && t < k; ++t)
      ok = (t1.off[0][t] == t * d1 - d1 * (k - 1) / 2) && (t2.off[0][t] == t - (k - 1) / 2) && t1.slab[0][t] == t &&
           t2.slab[0][t] == t;
    // the intermediate buffer must not be read by anything but c2 before it is overwritten
    for (int j = i + 2; ok && j < n; ++j) {
      const TcOp& c = ops[j];
      if (c.src == op.dst || (c.is_conv && (c.res == op.dst || c.dst2 == op.dst))) ok = false;
      if (c.is_conv && c.dst == op.dst && c.taps.mode == EPI_STORE) break;
    }
    PairPlan pl;
    if (ok && pair_plan(op, c2, &pl)) {
      fuse_next[i] = 1;
      ++i;  // c2 belongs to this pair
    }
  }
  return fuse_next;
}

int tc_op_plan(const std::vector<TcOp>& ops, const std::vector<char>& fuse_next, int i, TcOpPlan* out) {
  *out = TcOpPlan{};
  const TcOp& op = ops[i];
  if (!op.is_conv) return MB_OK;
  out->use_tc = op.tc.use_tc;
  out->x3 = op.tc.x3;
  out->split3 = op.tc.split3;
  out->fuse_next = fuse_next[i];
  out->fused_prev = i > 0 && fuse_next[i - 1];
  if (!op.tc.use_tc && !op.tc.split3) return MB_OK;
  // the geometry launch_tc runs: conv_pre's split as 256-channel halves, everything else as planned
  TcOp o = op;
  if (op.tc.split3) {
    o.taps.Cin = 256;
    o.taps.Cout = 256;
  }
  const TapConv& t = o.taps;
  out->kc = o.tc.kc;
  out->n_cchunks = o.tc.n_cchunks;
  out->mt = o.tc.mt;
  SmemPlan sp;
  if (!plan_smem(t, o.tc, kernel_count(t) * o.tc.n_cchunks, &sp))
    return fail(MB_ERR_INVALID, "tc_plan(%s): shared memory plan failed", op.name);
  out->resident = sp.resident;
  out->wstages = sp.wstages;
  out->omin = sp.omin;
  out->omax = -0x7fffffff;
  for (int r = 0; r < t.stride; ++r)
    for (int k = 0; k < t.ntaps[r]; ++k) out->omax = std::max(out->omax, t.off[r][k]);
  out->rows_item = o.tc.mt * 128;
  const TcInstance* inst = find_instance(t.Cout, o.tc.mt, o.tc.kc, false);
  if (out->fuse_next) {
    PairPlan pl;
    if (!pair_plan(op, ops[i + 1], &pl)) return fail(MB_ERR_INVALID, "tc_plan(%s): fused pair without a plan", op.name);
    out->pair_mt = pl.mt;
    out->pair_rows_item = pl.mt * 128 - 2 * pl.h2;
    out->pair_resident = pl.sp.resident;
    out->pair_wstages = pl.sp.wstages;
    out->pair_omin = pl.sp.omin;
    inst = find_instance(t.Cout, pl.mt, o.tc.kc, true);
  }
  if (out->fused_prev) return MB_OK;  // launched by the previous op
  if (!inst) return fail(MB_ERR_INVALID, "tc_plan(%s): no kernel instance", op.name);
  out->kn = inst->n;
  out->kmt = inst->mt;
  out->kcw = inst->cw;
  out->kpair = inst->pair ? 1 : 0;
  return MB_OK;
}

int tc_forward(const std::vector<TcOp>& ops, const std::vector<TcBufReq>& bufs, const char* tc_arena,
               const float* mel, const int32_t* lengths, int B, int T, int num_mels, int hop, float* wav,
               void* workspace, cudaStream_t st, cudaEvent_t* events) {
  (void)hop;
  constexpr int BUF_IN = 100, BUF_OUT = 101;
  const int nb = (int)bufs.size();
  // carve planes
  std::vector<char*> p16(nb), p32(nb);
  std::vector<TRef> cur16(nb), cur32(nb);  // geometry each plane currently holds
  char* ws = (char*)(((uintptr_t)workspace + 1023) & ~(uintptr_t)1023);
  for (int i = 0; i < nb; ++i) {
    p16[i] = ws;
    ws += f16_plane_bytes(B, T, 2 * bufs[i].cr);
    p32[i] = ws;
    ws += f32_plane_bytes(B, T, bufs[i].cr);
  }
  // buffer -> fp16 / fp32 plane storage (identity: every layer writes its own buffer's planes)
  std::vector<int> map16(nb);
  for (int i = 0; i < nb; ++i) map16[i] = i;
  std::vector<int> map32(nb);
  for (int i = 0; i < nb; ++i) map32[i] = i;
  std::vector<float> plane_slope(nb, 1.f);  // leaky-relu slope each fp16 storage was written with
  const int n = (int)ops.size();
  int full_rate = 1;
  for (const TcOp& o : ops) full_rate = std::max(full_rate, o.rate_out);
  // residual taken from the activated fp16 plane (no fp32 residual plane) in every stage but the full-rate one
  auto res16_ok = [&](const TcOp& c) {
    // 3-term-split layers take the residual from the hi/lo plane their pair's first conv reads anyway (hi + lo carries 22 bits:
    // FP32-equivalent), in every stage; plain fp16 layers from the activated fp16 plane in every stage but the full-rate one
    if (!(tc_res16_enabled() && c.is_conv && c.tc.use_tc && c.res >= 0 && c.res < nb && c.taps.stride == 1)) return false;
    return c.tc.x3 ? tc_x3_res16_enabled() : c.rate_out < full_rate;
  };
  // does a 3-term-split layer consume buffer `buf` (scanning forward from op `from` until the buffer is overwritten)?
  auto wants_hilo = [&](int buf, int from) {
    for (int j = from; j < n; ++j) {
      const TcOp& c = ops[j];
      if (c.is_conv && c.src == buf && c.tc.use_tc && c.tc.x3) return true;
      if (c.is_conv && c.dst == buf) break;  // the next writer (store or accumulate) produces the plane its own consumers need
    }
    return false;
  };
  const std::vector<char> fuse_next = tc_fusion_plan(ops, nb);
  for (int i = 0; i < n; ++i) {
    const TcOp& op = ops[i];
    if (events) MB_CUDA_CHECK(cudaEventRecord(events[i], st));
    const int Lin = T * op.rate_in, Lout = T * op.rate_out;
    if (!op.is_conv) {
      // dst32 += src32 ; refresh dst16 if a tensor-core consumer follows
      if (op.dst < 0 || op.dst >= nb || op.src < 0 || op.src >= nb) return fail(MB_ERR_INVALID, "tc_forward: bad add op");
      bool need16 = false;
      float slope16 = 1.f;
      for (int j = i + 1; j < n; ++j) {
        if (ops[j].is_conv && ops[j].src == op.dst && ops[j].tc.use_tc) { need16 = true; slope16 = ops[j].taps.in_slope; }
        if (ops[j].is_conv && ops[j].dst == op.dst) break;
      }
      TRef d32 = make_ref(p32[map32[op.dst]], LAYOUT_F32B, op.cout, Lout);
      TRef s32 = make_ref(p32[map32[op.src]], LAYOUT_F32B, op.cout, Lout);
      const bool add_hilo = need16 && wants_hilo(op.dst, i + 1);
      TRef d16 = need16 ? make_ref(p16[map16[op.dst]], LAYOUT_F16B, op.cout * (add_hilo ? 2 : 1), Lout) : TRef{};
      d16.hilo = add_hilo ? 1 : 0;
      if (need16) {
        plane_slope[map16[op.dst]] = slope16;
        if (cur16[map16[op.dst]].C != d16.C || cur16[map16[op.dst]].L != Lout || cur16[map16[op.dst]].hilo != d16.hilo) {
          cudaError_t ez = launch_zero_pads_f16(d16, B, st);
          if (ez != cudaSuccess) return fail(MB_ERR_CUDA, "zero_pads: %s", cudaGetErrorString(ez));
          count_launch();
          cur16[map16[op.dst]] = d16;
        }
      }
      cudaError_t e = launch_add_inplace_f32(d32, s32, d16, slope16, B, st);
      if (e != cudaSuccess) return fail(MB_ERR_CUDA, "add kernel: %s", cudaGetErrorString(e));
      count_launch();
      continue;
    }
    const bool fuse = fuse_next[i] != 0;
    const TcOp& oop = fuse ? ops[i + 1] : op;  // the op whose outputs this launch produces
    const int x16_idx = (op.src >= 0 && op.src < nb) ? map16[op.src] : -1;  // storage of the input plane (before any swap)
    const bool use_res16 = res16_ok(oop);
    TRef res16 = use_res16 ? make_ref(p16[map16[oop.res]], LAYOUT_F16B, oop.cout, Lout) : TRef{};
    if (use_res16 && cur16[map16[oop.res]].hilo) {  // the residual buffer currently holds a hi/lo plane (3-term-split consumers)
      res16.C = cur16[map16[oop.res]].C;
      res16.hilo = 1;
    }
    const float res_slope = use_res16 ? plane_slope[map16[oop.res]] : 1.f;
    const TRef res32 = (oop.res >= 0 && !use_res16) ? make_ref(p32[map32[oop.res]], LAYOUT_F32B, oop.cout, Lout) : TRef{};
    // a fused pair must not write the fp16 plane other CTAs still read halos from: an in-place pair (c2 writes c1's input buffer)
    // writes the storage of the (dead) intermediate buffer instead
    if (fuse && oop.dst == op.src) std::swap(map16[oop.dst], map16[op.dst]);
    const int scan_from = fuse ? i + 2 : i + 1;
    // ---- which planes must this op produce? (scan the consumers of dst until it is overwritten)
    bool need16 = false, need32 = false;
    float slope16 = 1.f;
    bool have_slope = false;
    auto scan = [&](int buf, bool& n16, bool& n32, float& s16, bool& hs) -> int {
      for (int j = scan_from; j < n; ++j) {
        const TcOp& c = ops[j];
        if (c.is_conv) {
          if (c.src == buf) {
            if (c.tc.use_tc) {
              if (hs && s16 != c.taps.in_slope) return fail(MB_ERR_INVALID, "tc_forward: consumers of one buffer disagree on slope");
              n16 = true;
              s16 = c.taps.in_slope;
              hs = true;
            } else {
              n32 = true;
            }
          }
          if (c.res == buf) {
            if (res16_ok(c)) n16 = true;
            else n32 = true;
          }
          if (c.dst2 == buf) n32 = true;
          if (c.dst == buf) {
            if (c.taps.mode != EPI_STORE) n32 = true;
            break;
          }
        } else {
          if (c.src == buf || c.dst == buf) n32 = true;
        }
      }
      return MB_OK;
    };
    TRef y32, y16, y2_32, y2_16;
    float y2_slope = 1.f;
    if (oop.dst == BUF_OUT) {
      y32 = make_ref(wav, LAYOUT_NCL, oop.cout, Lout);
    } else {
      if (oop.dst < 0 || oop.dst >= nb) return fail(MB_ERR_INVALID, "tc_forward: bad dst");
      int rc = scan(oop.dst, need16, need32, slope16, have_slope);
      if (rc != MB_OK) return rc;
      if (oop.taps.mode != EPI_STORE) need32 = true;
      if (need32) y32 = make_ref(p32[map32[oop.dst]], LAYOUT_F32B, oop.cout, Lout);
      if (need16) {
        const bool hl = wants_hilo(oop.dst, scan_from);
        y16 = make_ref(p16[map16[oop.dst]], LAYOUT_F16B, oop.cout * (hl ? 2 : 1), Lout);
        y16.hilo = hl ? 1 : 0;
        if (cur16[map16[oop.dst]].C != y16.C || cur16[map16[oop.dst]].L != Lout || cur16[map16[oop.dst]].hilo != y16.hilo) {
          cudaError_t e = launch_zero_pads_f16(y16, B, st);
          if (e != cudaSuccess) return fail(MB_ERR_CUDA, "zero_pads: %s", cudaGetErrorString(e));
          count_launch();
          cur16[map16[oop.dst]] = y16;
        }
        plane_slope[map16[oop.dst]] = slope16;
      }
    }
    if (oop.dst2 >= 0) {
      if (oop.dst2 >= nb) return fail(MB_ERR_INVALID, "tc_forward: bad dst2");
      bool n16 = false, n32 = true, hs = false;
      int rc = scan(oop.dst2, n16, n32, y2_slope, hs);
      if (rc != MB_OK) return rc;
      y2_32 = make_ref(p32[map32[oop.dst2]], LAYOUT_F32B, oop.cout, Lout);
      if (n16) {
        const bool hl = wants_hilo(oop.dst2, scan_from);
        y2_16 = make_ref(p16[map16[oop.dst2]], LAYOUT_F16B, oop.cout * (hl ? 2 : 1), Lout);
        y2_16.hilo = hl ? 1 : 0;
        plane_slope[map16[oop.dst2]] = y2_slope;
      }
    }
    if (op.tc.split3 && op.src == BUF_IN && y16.p && !y32.p && op.res < 0 && op.dst2 < 0) {
      // conv_pre on the tensor cores, fp32-accurate: split the fp32 input into fp16 hi/lo planes (scratch = any
      // other buffer's fp16 storage; all planes are dead at this point of the forward)
      int sidx = -1;
      const size_t need = (size_t)B * 256 * f16_lp(Lin) * 2;
      for (int j = 0; j < nb && sidx < 0; ++j)
        if (j != map16[op.dst] && f16_plane_bytes(B, T, 2 * bufs[j].cr) >= need + kPlaneSlack) sidx = j;
      if (sidx < 0) return fail(MB_ERR_WORKSPACE, "tc_forward: no scratch plane for %s", op.name);
      TRef xs = make_ref(p16[sidx], LAYOUT_F16B, 256, Lin);
      if (cur16[sidx].C != 256 || cur16[sidx].L != Lin) {
        cudaError_t e = launch_zero_pads_f16(xs, B, st);
        if (e != cudaSuccess) return fail(MB_ERR_CUDA, "zero_pads: %s", cudaGetErrorString(e));
        count_launch();
        cur16[sidx] = xs;
      }
      {
        const size_t nthr = (size_t)B * 32 * Lin;
        split3_input_kernel<<<(unsigned)((nthr + 255) / 256), 256, 0, st>>>(mel, reinterpret_cast<__half*>(p16[sidx]), B, op.cin, Lin, lengths);
        MB_LAUNCH_CHECK("split3_input_kernel");
      }
      for (int hf = 0; hf < op.cout / 256; ++hf) {
        TcOp half = op;
        half.taps.Cin = 256;
        half.taps.Cout = 256;
        half.tc.w16_off = op.tc.w16_off + (size_t)hf * kernel_count(op.taps) * 4 * op.tc.slab_bytes;
        int rc = launch_tc(half, tc_arena, xs, TRef{}, TRef{}, 1.f, TRef{}, y16, slope16, lengths, B, Lin, st,
                           tc_red_add_enabled(), hf * 256, op.b32 ? op.b32 + hf * 256 : nullptr);
        if (rc != MB_OK) return rc;
      }
    } else if (op.tc.use_tc) {
      if (op.src < 0 || op.src >= nb) return fail(MB_ERR_INVALID, "tc_forward: tensor-core layer %s reads an external buffer", op.name);
      TRef x16 = make_ref(p16[x16_idx], LAYOUT_F16B, op.tc.x3 ? 64 * op.tc.x_pchunks : op.cin, Lin);
      x16.hilo = op.tc.x3;
      if (cur16[x16_idx].hilo != x16.hilo)
        return fail(MB_ERR_INVALID, "tc_forward: %s expects a %s input plane", op.name, x16.hilo ? "hi/lo" : "plain");
      int rc = launch_tc(op, tc_arena, x16, res32, res16, res_slope, y32, y16, slope16, lengths, B, Lin, st,
                         tc_red_add_enabled(), 0, nullptr, fuse ? &ops[i + 1] : nullptr);
      if (rc != MB_OK) return rc;
      if (fuse) {
        if (events) MB_CUDA_CHECK(cudaEventRecord(events[i + 1], st));
        ++i;  // c2 is done as well
      }
    } else {
      TapConv p = op.taps;
      p.B = B;
      p.Lin = Lin;
      p.Lout = Lout;
      p.lengths = lengths;
      TapConvIO io;
      if (op.src == BUF_IN) io.x = make_ref(const_cast<float*>(mel), LAYOUT_NCL, num_mels, Lin);
      else if (op.src >= 0 && op.src < nb) io.x = make_ref(p32[map32[op.src]], LAYOUT_F32B, op.cin, Lin);
      else return fail(MB_ERR_INVALID, "tc_forward: bad src");
      io.res = res32;
      io.y32 = y32;
      io.y16 = y16;
      io.out16_slope = slope16;
      io.y2_32 = y2_32;
      io.y2_16 = y2_16;
      io.y2_16_slope = y2_slope;
      cudaError_t e = (op.cout == 1 && p.stride == 1) ? launch_tapconv_cout1_f32(p, io, op.w32, op.b32, st)
                                                      : launch_tapconv_f32(p, io, op.w32, op.b32, st);
      if (e != cudaSuccess) return fail(MB_ERR_CUDA, "tapconv_f32 (%s): %s", op.name, cudaGetErrorString(e));
      count_launch();
    }
  }
  if (events) MB_CUDA_CHECK(cudaEventRecord(events[n], st));
  return MB_OK;
}

int tc_debug_layer(const TcOp& op, const char* tc_arena, const float* x, const float* residual, int B, int Lin,
                   float* y, void* workspace, size_t workspace_bytes, cudaStream_t st) {
  const TapConv& t = op.taps;
  const int Lout = Lin * t.stride;
  TRef xn = make_ref(const_cast<float*>(x), LAYOUT_NCL, t.Cin, Lin);
  TRef yn = make_ref(y, LAYOUT_NCL, t.Cout, Lout);
  if (!op.tc.use_tc) {
    TapConv p = t;
    p.B = B;
    p.Lin = Lin;
    p.Lout = Lout;
    p.lengths = nullptr;
    TapConvIO io;
    io.x = xn;
    io.res = make_ref(const_cast<float*>(residual), LAYOUT_NCL, t.Cout, Lout);
    io.y32 = yn;
    cudaError_t e = (t.Cout == 1 && p.stride == 1) ? launch_tapconv_cout1_f32(p, io, op.w32, op.b32, st)
                                                   : launch_tapconv_f32(p, io, op.w32, op.b32, st);
    if (e != cudaSuccess) return fail(MB_ERR_CUDA, "tapconv_f32: %s", cudaGetErrorString(e));
    count_launch();
    return MB_OK;
  }
  // planes: x16 (activated), res32, y32
  const int xC = op.tc.x3 ? 64 * op.tc.x_pchunks : t.Cin;  // hi/lo plane: twice the channels
  const size_t b_x16 = align_up((size_t)B * xC * f16_lp(Lin) * 2 + kPlaneSlack, 1024);
  const size_t b_r32 = align_up((size_t)B * t.Cout * Lout * 4, 1024);
  if (workspace_bytes < b_x16 + 2 * b_r32 + 2048) return fail(MB_ERR_WORKSPACE, "tc_debug_layer: workspace too small");
  char* ws = (char*)(((uintptr_t)workspace + 1023) & ~(uintptr_t)1023);
  TRef x16 = make_ref(ws, LAYOUT_F16B, xC, Lin);
  x16.hilo = op.tc.x3;
  TRef r32 = residual ? make_ref(ws + b_x16, LAYOUT_F32B, t.Cout, Lout) : TRef{};
  TRef y32 = make_ref(ws + b_x16 + b_r32, LAYOUT_F32B, t.Cout, Lout);
  MB_CUDA_CHECK(cudaMemsetAsync(ws, 0, b_x16, st));
  cudaError_t e = launch_convert_layout(xn, x16, B, t.in_slope, st);
  if (e != cudaSuccess) return fail(MB_ERR_CUDA, "convert: %s", cudaGetErrorString(e));
  if (residual) {
    e = launch_convert_layout(make_ref(const_cast<float*>(residual), LAYOUT_NCL, t.Cout, Lout), r32, B, 1.f, st);
    if (e != cudaSuccess) return fail(MB_ERR_CUDA, "convert: %s", cudaGetErrorString(e));
  }
  int rc = launch_tc(op, tc_arena, x16, r32, TRef{}, 1.f, y32, TRef{}, 1.f, nullptr, B, Lin, st, tc_red_add_enabled());
  if (rc != MB_OK) return rc;
  e = launch_convert_layout(y32, yn, B, 1.f, st);
  if (e != cudaSuccess) return fail(MB_ERR_CUDA, "convert: %s", cudaGetErrorString(e));
  count_launch(3);
  return MB_OK;
}

int tc_debug_launch(const TcOp& op, const TcOp* c2, const TcDebugSpec& s, const char* tc_arena, void* workspace,
                    size_t workspace_bytes, cudaStream_t st, TcLaunchInfo* info, int* n_launches) {
  *n_launches = 0;
  const TcOp& last = c2 ? *c2 : op;  // the op whose outputs the launch produces
  if (!op.tc.use_tc || !last.tc.use_tc) return fail(MB_ERR_INVALID, "tc_debug_launch(%s): not a tensor-core layer", op.name);
  const int B = s.B, Lin = s.Lin, Lout = Lin * op.taps.stride;
  const int Cout = last.taps.Cout;
  const int xC = op.tc.x3 ? 64 * op.tc.x_pchunks : op.taps.Cin;
  const int hlC = Cout >= 64 ? 2 * Cout : 64;  // hi/lo plane of Cout channels
  const int y16C = s.out16 == 2 ? hlC : Cout;
  auto f16b = [&](int C, int L) { return align_up((size_t)B * C * f16_lp(L) * 2 + kPlaneSlack, 1024); };
  const size_t b_x16 = f16b(xC, Lin), b_mid = c2 ? f16b(Cout, Lin) : 0, b_res = f16b(hlC, Lout),
               b_r32 = align_up((size_t)B * Cout * Lout * 4, 1024), b_y16 = f16b(y16C, Lout);
  const size_t need = b_x16 + b_mid + b_res + 2 * b_r32 + b_y16 + 1024;
  if (workspace_bytes < need) return fail(MB_ERR_WORKSPACE, "tc_debug_launch: workspace %zu < %zu bytes", workspace_bytes, need);
  char* ws = (char*)(((uintptr_t)workspace + 1023) & ~(uintptr_t)1023);
  MB_CUDA_CHECK(cudaMemsetAsync(ws, 0, need - 1024, st));  // zero pad rows of every fp16 plane
  char* p_mid = ws + b_x16;
  char* p_res = p_mid + b_mid;
  char* p_r32 = p_res + b_res;
  char* p_y32 = p_r32 + b_r32;
  char* p_y16 = p_y32 + b_r32;
  TRef x16 = make_ref(ws, LAYOUT_F16B, xC, Lin);
  x16.hilo = op.tc.x3;
  cudaError_t e = launch_convert_layout(make_ref(const_cast<float*>(s.x), LAYOUT_NCL, op.taps.Cin, Lin), x16, B, op.taps.in_slope, st);
  if (e != cudaSuccess) return fail(MB_ERR_CUDA, "convert: %s", cudaGetErrorString(e));
  TRef res32, res16;
  const TRef res_ncl = make_ref(const_cast<float*>(s.res), LAYOUT_NCL, Cout, Lout);
  if (s.res_kind != 0 && !s.res) return fail(MB_ERR_INVALID, "tc_debug_launch: residual kind %d without residual", s.res_kind);
  if (s.res_kind == 1) {
    res32 = make_ref(p_r32, LAYOUT_F32B, Cout, Lout);
    e = launch_convert_layout(res_ncl, res32, B, 1.f, st);
  } else if (s.res_kind == 2 || s.res_kind == 3) {
    res16 = make_ref(p_res, LAYOUT_F16B, s.res_kind == 3 ? hlC : Cout, Lout);
    res16.hilo = s.res_kind == 3;
    e = launch_convert_layout(res_ncl, res16, B, s.res_slope, st);
  } else if (s.res_kind != 0) {
    return fail(MB_ERR_INVALID, "tc_debug_launch: residual kind %d", s.res_kind);
  }
  if (e != cudaSuccess) return fail(MB_ERR_CUDA, "convert: %s", cudaGetErrorString(e));
  const TRef y_ncl = make_ref(s.y, LAYOUT_NCL, Cout, Lout);
  const TRef y32 = s.y ? make_ref(p_y32, LAYOUT_F32B, Cout, Lout) : TRef{};
  if (s.y) {  // the running sum of the accumulate modes
    e = launch_convert_layout(y_ncl, y32, B, 1.f, st);
    if (e != cudaSuccess) return fail(MB_ERR_CUDA, "convert: %s", cudaGetErrorString(e));
  }
  TRef y16;
  if (s.out16 == 1 || s.out16 == 2) {
    if (!s.y16) return fail(MB_ERR_INVALID, "tc_debug_launch: fp16 output plane without destination");
    y16 = make_ref(p_y16, LAYOUT_F16B, y16C, Lout);
    y16.hilo = s.out16 == 2;
  } else if (s.out16 != 0) {
    return fail(MB_ERR_INVALID, "tc_debug_launch: fp16 output kind %d", s.out16);
  }
  int rc;
  if (c2 && s.two_launches) {
    // c1 -> activated fp16 intermediate plane (what tc_forward does for an unfused pair), then c2 reads it
    const TRef mid = make_ref(p_mid, LAYOUT_F16B, Cout, Lin);
    rc = launch_tc(op, tc_arena, x16, TRef{}, TRef{}, 1.f, TRef{}, mid, c2->taps.in_slope, s.lengths, B, Lin, st, s.red_add, 0,
                   nullptr, nullptr, &info[0]);
    if (rc != MB_OK) return rc;
    rc = launch_tc(*c2, tc_arena, mid, res32, res16, s.res_slope, y32, y16, s.out_slope, s.lengths, B, Lin, st, s.red_add, 0,
                   nullptr, nullptr, &info[1]);
    *n_launches = 2;
  } else {
    rc = launch_tc(op, tc_arena, x16, res32, res16, s.res_slope, y32, y16, s.out_slope, s.lengths, B, Lin, st, s.red_add, 0,
                   nullptr, c2, &info[0]);
    *n_launches = 1;
  }
  if (rc != MB_OK) return rc;
  if (s.y) {
    e = launch_convert_layout(y32, y_ncl, B, 1.f, st);
    if (e != cudaSuccess) return fail(MB_ERR_CUDA, "convert: %s", cudaGetErrorString(e));
  }
  if (y16.p) {
    e = launch_convert_layout(y16, make_ref(s.y16, LAYOUT_NCL, y16C, Lout), B, 1.f, st);
    if (e != cudaSuccess) return fail(MB_ERR_CUDA, "convert: %s", cudaGetErrorString(e));
  }
  return MB_OK;
}

}  // namespace mb
