// Tensor-core GEMMs of the Tacotron decoder step (sm_90a: wgmma / bulk-TMA / mbarrier), FP32-accurate.
//
// The decoder's LSTM cells (tacotron.py:118-127: two LSTMCell(1024) with residuals) are 84 % of the
// per-step MACs with only batch-many (<= 128) rows: Y[M][4H] = [x | h] . [W_ih | W_hh]^T.  FP32 FFMA
// kernels are compute-bound there at ~7 TFLOP/s; the tensor cores need fp16 operands, which alone would
// break the 1e-3 parity bar after 200 recurrent steps.  So every product is computed as a 3-term split
//     a*w ~= hi(a)*hi(w) + lo(a)*hi(w) + hi(a)*lo(w),   hi(v) = fp16(v), lo(v) = fp16(v - hi(v))
// with FP32 accumulation in registers: ~2^-21 relative per product, i.e. FP32-equivalent (weights are
// pre-scaled by a power of two so that their lo parts stay out of the fp16 subnormal range).
//
//   grid      : one CTA per 32 output columns (LSTM: the 4 gates of 8 hidden units, interleaved at pack
//               time, so the cell update c' = f*c + i*g, h' = o*tanh(c') runs in the epilogue)
//   operands  : K-major SWIZZLE_128B tiles of 64 k: activations [K/64][rows_pad][64] (hi and lo, written
//               by act_split_kernel), weights [tile][K/64][hi|lo][32][64]; each tile is one bulk copy
//   pipeline  : warp 0 producer (4-stage ring), warpgroups 1-2 MMA (12 wgmmas M64 x N32 x K16 per stage, 64 batch rows
//               each; the second only for more than 64 rows) and epilogue (one batch row per thread)
#include <cuda_fp16.h>

#include <cstdlib>
#include <cstring>

#include "gan_tc_dev.cuh"
#include "tacotron_kernels.cuh"

namespace mb {
namespace taco {

namespace {

using namespace tcdev;

constexpr int kStages = 4;          // ring depth of the 32-column kernels (5 stages measured no faster: 37.8 vs 36.0 ms on cfg 4)
constexpr int kBigStages = 3;       // ring depth of the 128-column kernel (64 KB per stage)
constexpr int kThreads = 384;    // copy-producer warpgroup + two MMA / epilogue warpgroups (64 rows each)
constexpr size_t kEpiStageBytes = 2 * 64 * kStageLd * 4;
constexpr uint32_t kATile = 16384;  // 128 rows x 128 B (rows >= rows_pad stay zero)
constexpr uint32_t kWTile = 4096;   // 32 rows x 128 B
constexpr uint32_t kStageBytes = 2 * kATile + 2 * kWTile;
template <int NT>
__host__ __device__ constexpr uint32_t w_tile_bytes() { return (uint32_t)NT * 128u; }
template <int NT>
__host__ __device__ constexpr uint32_t stage_bytes() { return 2 * kATile + 2 * w_tile_bytes<NT>(); }

__device__ __forceinline__ float sigm(float x) { return 1.f / (1.f + expf(-x)); }

// ---- thread-block-cluster helpers (activation-tile multicast of the skinny GEMMs) ----
__device__ __forceinline__ uint32_t cluster_nctaid_x() {
  uint32_t v;
  asm volatile("mov.u32 %0, %%cluster_nctaid.x;" : "=r"(v));
  return v;
}
__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t v;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(v));
  return v;
}
__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// bulk copy global -> the same shared-memory offset of every CTA in `mask`, complete_tx on the mbarrier at the same offset in each
__device__ __forceinline__ void bulk_g2s_mc(uint32_t dst_smem, const void* src, uint32_t bytes, uint64_t* bar, uint16_t mask) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster [%0], [%1], %2, [%3], %4;" ::"r"(dst_smem),
      "l"(src), "r"(bytes), "r"(smem_u32(bar)), "h"(mask)
      : "memory");
}
// Shared main loop: operands for output tile `tile` stream through the ring; `epi(m, v)` is called by the
// epilogue warps with the 32 accumulator columns (already scaled, bias added) of row m.
template <int NT, int STAGES, typename Epi>
__device__ __forceinline__ void skinny_body_t(const __half* a_hi_g, const __half* a_lo_g, const __half* w_g, const float* bias,
                                              int n_valid, int KB, int M, int rows_pad, float inv_scale, int tile, Epi epi,
                                              size_t a_kb_stride = 0, int kb0 = 0, int KBw = 0, bool compact = false) {
  constexpr uint32_t kWTile = w_tile_bytes<NT>();
  // `compact` (32-column kernels with <= 64 rows, MB_TACO_RING8): an activation slot is 8 KB (64 rows) instead of 16, so a stage
  // shrinks from 40 to 24 KB and the ring holds 8 k-blocks instead of 4: half as many dependent L2 round trips per launch.
  const int kStages = compact ? 2 * STAGES : STAGES;
  const uint32_t kASlot = compact ? kATile / 2 : kATile;
  const uint32_t kStageBytes = 2 * kASlot + 2 * kWTile;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + (size_t)kStages * kStageBytes);
  uint64_t* full = bars;
  uint64_t* empty = bars + kStages;
  float* bias_s = reinterpret_cast<float*>(bars + 2 * kStages);

  float* stage_s = reinterpret_cast<float*>(smem + (size_t)kStages * kStageBytes + 1024);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t a_bytes = (uint32_t)rows_pad * 128u;
  if (a_kb_stride == 0) a_kb_stride = a_bytes;  // bytes between the k-blocks of the activation tiles
  // Optionally launched as clusters of `csize` CTAs (launch_tc_skinny, MB_TACO_MC; off by default, see there): the activation tiles are
  // the same for every output tile, so each CTA fetches 1 / csize of a tile and multicasts it to the whole cluster.
  // A stage is refilled only when ALL CTAs of the cluster have consumed it: every consumer arrives on every CTA's `empty` barrier.
  const uint32_t csize = cluster_nctaid_x();
  const uint32_t crank = cluster_ctarank();
  const bool mc = csize > 1;
  const uint16_t cmask = (uint16_t)((1u << csize) - 1u);
  // warpgroup g (1, 2) multiplies rows [64 (g - 1), 64 g); the second one only when there are more than 64 rows
  const uint32_t n_mma_groups = M > 64 ? 2u : 1u;

  if (threadIdx.x == 0) {
    for (int i = 0; i < kStages; ++i) {
      mbar_init(&full[i], 1);
      mbar_init(&empty[i], n_mma_groups * (mc ? csize : 1u));
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  if (threadIdx.x < NT) bias_s[threadIdx.x] = (bias && tile * NT + (int)threadIdx.x < n_valid) ? bias[tile * NT + threadIdx.x] : 0.f;
  __syncthreads();
  if (mc) cluster_sync_all();  // every CTA's barriers are initialised before a peer's multicast / arrive can reach them
  // Programmatic dependent launch: everything above (barriers, bias) touched no tensor another kernel writes and may overlap
  // the tail of the previous launch (recurrences are chains of these kernels); its outputs are only read below.  A plain
  // launch makes both instructions no-ops.
  asm volatile("griddepcontrol.wait;" ::: "memory");
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");

  if (warp < 4) {
    regs_dec<40>();
    if (warp == 0 && lane == 0) {
      const uint8_t* wt = reinterpret_cast<const uint8_t*>(w_g) + (size_t)tile * (KBw > 0 ? KBw : KB) * (2 * kWTile);
      for (int kb = 0; kb < KB; ++kb) {
        const int s = kb % kStages, ph = (kb / kStages) & 1;
        const size_t kg = (size_t)(kb0 + kb);  // k-block inside the activation tiles / the weight image
        mbar_wait(&empty[s], ph ^ 1);
        uint8_t* st = smem + (size_t)s * kStageBytes;
        mbar_expect_tx(&full[s], 2 * a_bytes + 2 * kWTile);
        if (mc) {
          const uint32_t slice = a_bytes / csize, off = crank * slice;  // my byte range of both tiles, sent to every CTA of the cluster
          bulk_g2s_mc(smem_u32(st + off), reinterpret_cast<const uint8_t*>(a_hi_g) + kg * a_kb_stride + off, slice, &full[s], cmask);
          bulk_g2s_mc(smem_u32(st + kASlot + off), reinterpret_cast<const uint8_t*>(a_lo_g) + kg * a_kb_stride + off, slice, &full[s],
                      cmask);
        } else {
          bulk_g2s(smem_u32(st), reinterpret_cast<const uint8_t*>(a_hi_g) + kg * a_kb_stride, a_bytes, &full[s]);
          bulk_g2s(smem_u32(st + kASlot), reinterpret_cast<const uint8_t*>(a_lo_g) + kg * a_kb_stride, a_bytes, &full[s]);
        }
        bulk_g2s(smem_u32(st + 2 * kASlot), wt + kg * (2 * kWTile), 2 * kWTile, &full[s]);
      }
    }
  } else {
    regs_inc<232>();
    const int g = warp / 4 - 1;
    const int tid = threadIdx.x & 127;
    if ((uint32_t)g < n_mma_groups) {
      // one commit group per stage (12 wgmmas: 4 k-steps x 3 split terms); a stage is released once the next one is issued
      // and it has completed (wait_group 1)
      const uint64_t desc_hi = make_desc(0, 1024u, 1u, 0);
      const uint32_t row_off = (uint32_t)g * 64u * 128u;
      float acc[NT / 2];
      auto release = [&](int s) {
        if (tid != 0) return;
        if (mc) {
          for (uint32_t c = 0; c < csize; ++c) mbar_arrive_cluster(&empty[s], c);
        } else {
          mbar_arrive(&empty[s]);
        }
      };
      wgmma_fence();
      for (int kb = 0; kb < KB; ++kb) {
        const int s = kb % kStages, ph = (kb / kStages) & 1;
        mbar_wait(&full[s], ph);
        const uint32_t base = smem_u32(smem + (size_t)s * kStageBytes);
        const uint64_t ah = desc_hi + (uint64_t)((base + row_off) >> 4);
        const uint64_t al = desc_hi + (uint64_t)((base + kASlot + row_off) >> 4);
        const uint64_t wh = desc_hi + (uint64_t)((base + 2 * kASlot) >> 4);
        const uint64_t wl = desc_hi + (uint64_t)((base + 2 * kASlot + kWTile) >> 4);
        fence_acc(acc);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          wgmma_f16<NT>(acc, ah + (uint64_t)(2 * k), wh + (uint64_t)(2 * k), (kb | k) ? 1u : 0u);
          wgmma_f16<NT>(acc, al + (uint64_t)(2 * k), wh + (uint64_t)(2 * k), 1u);
          wgmma_f16<NT>(acc, ah + (uint64_t)(2 * k), wl + (uint64_t)(2 * k), 1u);
        }
        wgmma_commit();
        wgmma_wait<1>();
        fence_acc(acc);
        if (kb > 0) release((kb - 1) % kStages);
      }
      wgmma_wait<0>();
      fence_acc(acc);
      release((KB - 1) % kStages);
      // epilogue: 32-column slices through shared memory, one row per thread of the first two warps
      float* stage = stage_s + g * 64 * kStageLd;
      const int m = g * 64 + tid;
#pragma unroll
      for (int c0 = 0; c0 < NT; c0 += 32) {
        group_sync(1 + g, 128);
        stage_acc32(stage, &acc[c0 / 2], tid);
        group_sync(1 + g, 128);
        if (tid < 64 && m < M) {
          float v[32];
#pragma unroll
          for (int i = 0; i < 32; ++i) v[i] = stage[tid * kStageLd + i] * inv_scale + bias_s[c0 + i];
          epi(m, v, c0);
        }
      }
    }
  }
  if (mc) cluster_sync_all();  // no CTA leaves while a peer's arrive may still reach its barriers
}

// the 32-column instance used by the recurrent kernels (bias already in tile order, all 32 columns valid)
template <typename Epi>
__device__ __forceinline__ void skinny_body(const __half* a_hi_g, const __half* a_lo_g, const __half* w_g, const float* bias,
                                            int KB, int M, int rows_pad, float inv_scale, int tile, Epi epi,
                                            size_t a_kb_stride = 0, int kb0 = 0, int KBw = 0, bool compact = false) {
  skinny_body_t<32, kStages>(a_hi_g, a_lo_g, w_g, bias, 0x7fffffff, KB, M, rows_pad, inv_scale, tile,
                             [&](int m, float* v, int) { epi(m, v); }, a_kb_stride, kb0, KBw, compact);
}

// 8 fp32 values of row m, hidden units [u0, u0 + 8) -> the 16-byte chunk of the hi / lo operand tiles of the NEXT GEMM
__device__ __forceinline__ void store_split_chunk(const float* x, int m, int rows_pad, int k0, __half* t_hi, __half* t_lo) {
  __align__(16) __half hi[8], lo[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    hi[e] = __float2half_rn(x[e]);
    lo[e] = __float2half_rn(x[e] - __half2float(hi[e]));
  }
  const int kb = k0 >> 6, c8 = (k0 & 63) >> 3;
  const size_t o = ((size_t)kb * rows_pad + m) * 8 + (size_t)(c8 ^ (m & 7));
  reinterpret_cast<uint4*>(t_hi)[o] = *reinterpret_cast<const uint4*>(hi);
  reinterpret_cast<uint4*>(t_lo)[o] = *reinterpret_cast<const uint4*>(lo);
}

__global__ void __launch_bounds__(kThreads, 1) tc_skinny_kernel(const __grid_constant__ TcSkinnyArgs p) {
  const int tile = blockIdx.x;
  skinny_body(p.a_hi, p.a_lo, p.w, p.bias, p.KB, p.M, p.rows_pad, p.inv_scale, tile, [&](int m, float* v) {
    if (p.pre) {  // partial product over the other k-blocks, computed earlier by a TCS_PLAIN launch (tile column order)
      const float4* pp = reinterpret_cast<const float4*>(p.pre + (size_t)m * p.ldpre + (size_t)tile * 32);
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const float4 q = pp[i];
        v[4 * i + 0] += q.x; v[4 * i + 1] += q.y; v[4 * i + 2] += q.z; v[4 * i + 3] += q.w;
      }
    }
    if (p.mode == TCS_LSTM) {
      const size_t o = (size_t)m * p.H + (size_t)tile * 8;
      float cn[8], hn[8], xn[8];
      const float4 c0 = *reinterpret_cast<const float4*>(p.c + o), c1 = *reinterpret_cast<const float4*>(p.c + o + 4);
      const float co[8] = {c0.x, c0.y, c0.z, c0.w, c1.x, c1.y, c1.z, c1.w};
      const float4 x0 = *reinterpret_cast<const float4*>(p.x + o), x1 = *reinterpret_cast<const float4*>(p.x + o + 4);
      const float xo[8] = {x0.x, x0.y, x0.z, x0.w, x1.x, x1.y, x1.z, x1.w};
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const float ig = sigm(v[e]), fg = sigm(v[8 + e]), cg = tanhf(v[16 + e]), og = sigm(v[24 + e]);
        cn[e] = fg * co[e] + ig * cg;
        hn[e] = og * tanhf(cn[e]);
        xn[e] = xo[e] + hn[e];
      }
      *reinterpret_cast<float4*>(p.c + o) = make_float4(cn[0], cn[1], cn[2], cn[3]);
      *reinterpret_cast<float4*>(p.c + o + 4) = make_float4(cn[4], cn[5], cn[6], cn[7]);
      *reinterpret_cast<float4*>(p.h + o) = make_float4(hn[0], hn[1], hn[2], hn[3]);
      *reinterpret_cast<float4*>(p.h + o + 4) = make_float4(hn[4], hn[5], hn[6], hn[7]);
      *reinterpret_cast<float4*>(p.x + o) = make_float4(xn[0], xn[1], xn[2], xn[3]);
      *reinterpret_cast<float4*>(p.x + o + 4) = make_float4(xn[4], xn[5], xn[6], xn[7]);
      if (p.s_hi[0]) store_split_chunk(xn, m, p.rows_pad, p.s_k0[0] + tile * 8, p.s_hi[0], p.s_lo[0]);
      if (p.s_hi[1]) store_split_chunk(hn, m, p.rows_pad, p.s_k0[1] + tile * 8, p.s_hi[1], p.s_lo[1]);
    } else {
      float* y = p.y + (long long)step_index(p.step_ptr, p.step_j) * p.y_step + (size_t)m * p.ldy + (size_t)tile * 32;
#pragma unroll
      for (int i = 0; i < 32; i += 4) {
        if (tile * 32 + i < p.N) *reinterpret_cast<float4*>(y + i) = make_float4(v[i], v[i + 1], v[i + 2], v[i + 3]);
      }
      if (p.s_hi[0]) {
#pragma unroll
        for (int i = 0; i < 32; i += 8)
          if (tile * 32 + i + 8 <= p.N) store_split_chunk(v + i, m, p.rows_pad, p.s_k0[0] + tile * 32 + i, p.s_hi[0], p.s_lo[0]);
      }
    }
  }, 0, p.kb0, p.KBw, p.compact != 0);
}

// One recurrent step of a (bi)directional GRU: blockIdx.y = direction, blockIdx.x = 8 hidden units.
//   gh = W_hh h + b_hh (this GEMM, gates r|z|n interleaved per tile);  r = sig(gi_r + gh_r), z = sig(gi_z + gh_z),
//   n = tanh(gi_n + r * gh_n), h' = (h - n) z + n   (ATen gru_cell; gi = W_ih x_t + b_ih precomputed for all t)
// h' goes to the state, to the output sequence and - as hi/lo operand chunks - into the NEXT step's A tiles.
__global__ void __launch_bounds__(kThreads, 1) tc_gru_kernel(const __grid_constant__ TcGruArgs p) {
  const int tile = blockIdx.x, dir = blockIdx.y;
  const int H = p.H;
  skinny_body(p.a_hi[dir], p.a_lo[dir], p.w[dir], p.bias[dir], p.KB, p.M, p.rows_pad, p.inv_scale[dir], tile,
              [&](int m, float* v) {
                const float* gi = p.gi[dir] + (size_t)m * p.ldgi + (size_t)tile * 8;
                float* hp = p.h[dir] + (size_t)m * H + (size_t)tile * 8;
                float hn[8];
#pragma unroll
                for (int e = 0; e < 8; ++e) {
                  const float r = sigm(v[e] + gi[e]);
                  const float z = sigm(v[8 + e] + gi[H + e]);
                  const float n = tanhf(gi[2 * H + e] + v[16 + e] * r);
                  hn[e] = (hp[e] - n) * z + n;
                }
                *reinterpret_cast<float4*>(hp) = make_float4(hn[0], hn[1], hn[2], hn[3]);
                *reinterpret_cast<float4*>(hp + 4) = make_float4(hn[4], hn[5], hn[6], hn[7]);
                float* op = p.out[dir] + (size_t)m * p.ldout + (size_t)tile * 8;
                *reinterpret_cast<float4*>(op) = make_float4(hn[0], hn[1], hn[2], hn[3]);
                *reinterpret_cast<float4*>(op + 4) = make_float4(hn[4], hn[5], hn[6], hn[7]);
                store_split_chunk(hn, m, p.rows_pad, tile * 8, p.nxt_hi[dir], p.nxt_lo[dir]);
                if (dir == 0 && p.s_hi) store_split_chunk(hn, m, p.rows_pad, p.s_k0 + tile * 8, p.s_hi, p.s_lo);
              });
}

// One time step of one LSTM layer over many rows (speaker encoder: rows = partial windows): blockIdx.x = 8 hidden
// units, blockIdx.y = block of 128 rows.  gates = W_hh h_{t-1} (this GEMM) + gi (W_ih x_t + b_ih + b_hh, precomputed
// for all t); c' = f c + i g, h' = o tanh(c') (ATen lstm_cell, gate order i|f|g|o).  h' goes to the layer's
// output sequence and - as hi/lo operand chunks - into the next step's A tiles (ping-pong).
__global__ void __launch_bounds__(kThreads, 1) tc_lstm_seq_kernel(const __grid_constant__ TcLstmSeqArgs p) {
  const int tile = blockIdx.x, mb = blockIdx.y;
  const int H = p.H;
  const int rows_here = min(128, p.M - mb * 128);
  const size_t blk = (size_t)mb * 128 * 128;  // byte offset of this row block inside a k-block slab
  skinny_body(reinterpret_cast<const __half*>(reinterpret_cast<const char*>(p.a_hi) + blk),
              reinterpret_cast<const __half*>(reinterpret_cast<const char*>(p.a_lo) + blk), p.w, nullptr, p.KB, rows_here, 128,
              p.inv_scale, tile,
              [&](int ml, float* v) {
                const int m = mb * 128 + ml;
                const float* gi = p.gi + (size_t)m * p.ldgi + (size_t)tile * 8;
                float* cp = p.c + (size_t)m * H + (size_t)tile * 8;
                float hn[8], cn[8];
#pragma unroll
                for (int e = 0; e < 8; ++e) {
                  const float ig = sigm(v[e] + gi[e]), fg = sigm(v[8 + e] + gi[H + e]);
                  const float cg = tanhf(v[16 + e] + gi[2 * H + e]), og = sigm(v[24 + e] + gi[3 * H + e]);
                  cn[e] = fg * cp[e] + ig * cg;
                  hn[e] = og * tanhf(cn[e]);
                }
                *reinterpret_cast<float4*>(cp) = make_float4(cn[0], cn[1], cn[2], cn[3]);
                *reinterpret_cast<float4*>(cp + 4) = make_float4(cn[4], cn[5], cn[6], cn[7]);
                float* op = p.out + (size_t)m * p.ldout + (size_t)tile * 8;
                *reinterpret_cast<float4*>(op) = make_float4(hn[0], hn[1], hn[2], hn[3]);
                *reinterpret_cast<float4*>(op + 4) = make_float4(hn[4], hn[5], hn[6], hn[7]);
                store_split_chunk(hn, m, p.rows_total, tile * 8, p.nxt_hi, p.nxt_lo);
              },
              (size_t)p.rows_total * 128);
}

// Large-M GEMM / Conv1d-over-time of the CBHG stacks (encoder, postnet), same 3-term split: blockIdx.x = 128 output
// columns, blockIdx.y = 128 rows.  The operand tiles hold the im2col of the layer input (one K segment per conv
// tap, im2col_split_kernel); epilogue = bias, ReLU, eval-BatchNorm affine (after the ReLU, batch_norm_conv.py:11-14),
// residual -> fp32 channels-last.
__global__ void __launch_bounds__(kThreads, 1) tc_big_kernel(const __grid_constant__ TcBigArgs p) {
  const int tile = blockIdx.x, mb = blockIdx.y;
  const int rows_here = min(128, p.M - mb * 128);
  const size_t blk = (size_t)mb * 128 * 128;
  skinny_body_t<128, kBigStages>(
      reinterpret_cast<const __half*>(reinterpret_cast<const char*>(p.a_hi) + blk),
      reinterpret_cast<const __half*>(reinterpret_cast<const char*>(p.a_lo) + blk), p.w, p.bias, p.N, p.KB, rows_here, 128,
      p.inv_scale, tile,
      [&](int ml, float* v, int c0) {
        const int m = mb * 128 + ml;
        const int n0 = tile * 128 + c0;
        if (n0 >= p.N) return;
        float* y = p.y + (size_t)m * p.ldy + n0;
        const float* res = p.res ? p.res + (size_t)m * p.ldres + n0 : nullptr;
#pragma unroll
        for (int i = 0; i < 32; i += 4) {
          if (n0 + i >= p.N) break;
          float o[4];
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            float t = v[i + e];
            if (p.act == ACT_RELU) t = fmaxf(t, 0.f);
            if (p.bn_scale) t = fmaf(t, p.bn_scale[n0 + i + e], p.bn_shift[n0 + i + e]);
            if (res) t += res[i + e];
            o[e] = t;
          }
          *reinterpret_cast<float4*>(y + i) = make_float4(o[0], o[1], o[2], o[3]);
        }
      },
      (size_t)p.rows_total * 128);
}

// im2col of a channels-last fp32 tensor into hi / lo operand tiles [nseg * KBs][rows_total][64]: segment s holds
// x[row + shift_s][0 .. K) (zero outside the row's own length-T sequence, zero for k >= K and rows >= M)
__global__ void im2col_split_kernel(const TcIm2col q, __half* __restrict__ a_hi, __half* __restrict__ a_lo) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;  // one thread per 16-byte chunk
  const size_t total = (size_t)q.nseg * q.KBs * q.rows_total * 8;
  if (i >= total) return;
  const int c8 = (int)(i & 7);
  const int m = (int)((i >> 3) % q.rows_total);
  const int kb = (int)(i / ((size_t)8 * q.rows_total));
  const int sg = kb / q.KBs, kbs = kb - sg * q.KBs;
  __align__(16) __half hi[8], lo[8];
  bool ok = m < q.M;
  int row = m;
  if (ok && q.shift[sg] != 0) {
    const int t = m % q.T + q.shift[sg];
    ok = (t >= 0 && t < q.T);
    row = m + q.shift[sg];
  }
  const float* src = q.x[sg] + (size_t)row * q.ld[sg];
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    const int k = kbs * 64 + c8 * 8 + e;
    const float v = (ok && k < q.K) ? src[k] : 0.f;
    hi[e] = __float2half_rn(v);
    lo[e] = __float2half_rn(v - __half2float(hi[e]));
  }
  const size_t o = ((size_t)kb * q.rows_total + m) * 8 + (size_t)(c8 ^ (m & 7));
  reinterpret_cast<uint4*>(a_hi)[o] = *reinterpret_cast<const uint4*>(hi);
  reinterpret_cast<uint4*>(a_lo)[o] = *reinterpret_cast<const uint4*>(lo);
}

// weights described like GemmArgs segments (W[n * ldw + w_off_s + k * w_stride_s]) * scale -> tiles
// [n_tile(128)][nseg * KBs][hi|lo][128][64]
__global__ void pack_big_w_kernel(const TcBigPack q, __half* __restrict__ dst) {
  const size_t n_tiles = (size_t)(q.N + 127) / 128;
  const size_t KB = (size_t)q.nseg * q.KBs;
  const size_t total = n_tiles * KB * 128 * 8;
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int c8 = (int)(i & 7);
  const int n = (int)((i >> 3) & 127);
  const int kb = (int)((i >> 10) % KB);
  const int j = (int)(i / ((size_t)1024 * KB));
  const int sg = kb / q.KBs, kbs = kb - sg * q.KBs;
  const int row = 128 * j + n;
  __align__(16) __half hi[8], lo[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    const int k = kbs * 64 + c8 * 8 + e;
    float v = 0.f;
    if (row < q.N && k < q.K) v = q.W[(size_t)row * q.ldw + q.w_off[sg] + (size_t)k * q.w_stride[sg]] * q.scale;
    hi[e] = __float2half_rn(v);
    lo[e] = __float2half_rn(v - __half2float(hi[e]));
  }
  const size_t t = ((size_t)j * KB + kb) * 2;
  const size_t o = (size_t)n * 8 + (size_t)(c8 ^ (n & 7));
  reinterpret_cast<uint4*>(dst)[(t + 0) * 1024 + o] = *reinterpret_cast<const uint4*>(hi);
  reinterpret_cast<uint4*>(dst)[(t + 1) * 1024 + o] = *reinterpret_cast<const uint4*>(lo);
}

__device__ __forceinline__ __half split_hi(float v) { return __float2half_rn(v); }
__device__ __forceinline__ __half split_lo(float v) { return __float2half_rn(v - __half2float(__float2half_rn(v))); }

// activations [M][K0 | K1] fp32 -> hi / lo operand tiles [KB][rows_pad][64] (16-byte chunks XOR (row & 7))
__global__ void act_split_kernel(const float* __restrict__ s0, int K0, int ld0, const float* __restrict__ s1, int K1, int ld1,
                                 int M, int rows_pad, int KB, __half* __restrict__ a_hi, __half* __restrict__ a_lo) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;  // one thread per 8 consecutive k of one row
  const int n = KB * rows_pad * 8;
  if (i >= n) return;
  const int c8 = i & 7;
  const int m = (i >> 3) % rows_pad;
  const int kb = i / (8 * rows_pad);
  __align__(16) __half hi[8], lo[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    const int k = kb * 64 + c8 * 8 + e;
    float v = 0.f;
    if (m < M) {
      if (k < K0) v = s0[(size_t)m * ld0 + k];
      else if (k < K0 + K1) v = s1[(size_t)m * ld1 + (k - K0)];
    }
    hi[e] = split_hi(v);
    lo[e] = split_lo(v);
  }
  const size_t o = ((size_t)kb * rows_pad + m) * 8 + (size_t)(c8 ^ (m & 7));
  reinterpret_cast<uint4*>(a_hi)[o] = *reinterpret_cast<const uint4*>(hi);
  reinterpret_cast<uint4*>(a_lo)[o] = *reinterpret_cast<const uint4*>(lo);
}

// weights -> tiles [tile][KB][hi|lo][32][64].  Row n of tile j is source row
//   lstm_H > 0 : (n / 8) * lstm_H + 8 j + (n % 8)   (gate-interleaved: i,f,g,o of 8 units)
//   else       : 32 j + n  (rows >= N are zero)
// and its K axis is [w0 (K0 columns) | w1 (K1 columns)], zero padded to 64 KB.
__global__ void pack_split_w_kernel(const float* __restrict__ w0, int K0, const float* __restrict__ w1, int K1, int N,
                                    int lstm_H, int KB, float scale, __half* __restrict__ dst) {
  const size_t n_tiles = lstm_H > 0 ? (size_t)lstm_H / 8 : (size_t)(N + 31) / 32;
  const size_t total = n_tiles * KB * 32 * 8;
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int c8 = (int)(i & 7);
  const int n = (int)((i >> 3) & 31);
  const int kb = (int)((i >> 8) % KB);
  const int j = (int)(i / ((size_t)256 * KB));
  const int row = lstm_H > 0 ? (n / 8) * lstm_H + 8 * j + (n % 8) : 32 * j + n;  // gate-interleaved: N / H gates of 8 units
  __align__(16) __half hi[8], lo[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    const int k = kb * 64 + c8 * 8 + e;
    float v = 0.f;
    if (row < N) {
      if (k < K0) v = w0[(size_t)row * K0 + k];
      else if (k < K0 + K1) v = w1[(size_t)row * K1 + (k - K0)];
    }
    v *= scale;
    hi[e] = split_hi(v);
    lo[e] = split_lo(v);
  }
  const size_t t = ((size_t)j * KB + kb) * 2;
  const size_t o = (size_t)n * 8 + (size_t)(c8 ^ (n & 7));
  reinterpret_cast<uint4*>(dst)[(t + 0) * 256 + o] = *reinterpret_cast<const uint4*>(hi);
  reinterpret_cast<uint4*>(dst)[(t + 1) * 256 + o] = *reinterpret_cast<const uint4*>(lo);
}

// bias in tile order (LSTM: gate-interleaved b_ih + b_hh)
__global__ void pack_split_bias_kernel(const float* __restrict__ b0, const float* __restrict__ b1, int N, int lstm_H,
                                       float* __restrict__ dst) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const int n_pad = lstm_H > 0 ? lstm_H * 4 : (N + 31) / 32 * 32;
  if (i >= n_pad) return;
  const int j = i / 32, n = i % 32;
  const int row = lstm_H > 0 ? (n / 8) * lstm_H + 8 * j + (n % 8) : i;
  float v = 0.f;
  if (row < N) v = (b0 ? b0[row] : 0.f) + (b1 ? b1[row] : 0.f);
  dst[i] = v;
}

__global__ void absmax_kernel(const float* __restrict__ w, size_t n, unsigned int* __restrict__ out) {
  float m = 0.f;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) m = fmaxf(m, fabsf(w[i]));
  for (int o = 16; o; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0) atomicMax(out, __float_as_uint(m));  // non-negative floats order like their bit patterns
}

}  // namespace

// launch with the programmatic-stream-serialization attribute (MB_TACO_PDL=0: plain launches)
template <typename Args>
cudaError_t launch_pdl(void (*kern)(const Args), dim3 grid, size_t smem, cudaStream_t st, const Args& args, int cluster_x = 1) {
  static const bool pdl = [] {
    const char* e = getenv("MB_TACO_PDL");
    return e ? atoi(e) != 0 : true;
  }();
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = grid;
  cfg.blockDim = dim3(kThreads);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[2];
  int na = 0;
  if (pdl) {
    attr[na].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[na].val.programmaticStreamSerializationAllowed = 1;
    ++na;
  }
  if (cluster_x > 1) {
    attr[na].id = cudaLaunchAttributeClusterDimension;
    attr[na].val.clusterDim.x = (unsigned)cluster_x;
    attr[na].val.clusterDim.y = 1;
    attr[na].val.clusterDim.z = 1;
    ++na;
  }
  cfg.attrs = attr;
  cfg.numAttrs = na;
  return cudaLaunchKernelEx(&cfg, kern, args);
}

size_t tc_skinny_weight_bytes(int N, int K) {
  const size_t n_tiles = (size_t)(N + 31) / 32, KB = (size_t)(K + 63) / 64;
  return n_tiles * KB * 2 * kWTile;
}

size_t tc_gated_weight_bytes(int H, int K) {  // gate-interleaved images: H / 8 tiles whatever the gate count (<= 4)
  return (size_t)(H / 8) * ((size_t)(K + 63) / 64) * 2 * kWTile;
}

size_t tc_skinny_act_bytes(int M, int K) {
  const size_t KB = (size_t)(K + 63) / 64;
  return KB * (size_t)(M <= 64 ? 64 : 128) * 128;
}

cudaError_t tc_skinny_absmax(const float* w, size_t n, unsigned int* dev_out, cudaStream_t st) {
  absmax_kernel<<<132, 256, 0, st>>>(w, n, dev_out);
  return cudaGetLastError();
}

cudaError_t tc_skinny_pack(const float* w0, int K0, const float* w1, int K1, const float* b0, const float* b1, int N,
                           int lstm_H, float scale, __half* w_dst, float* bias_dst, cudaStream_t st) {
  const int KB = (K0 + K1 + 63) / 64;
  const size_t total = (size_t)(lstm_H > 0 ? lstm_H / 8 : (N + 31) / 32) * KB * 256;
  pack_split_w_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(w0, K0, w1, K1, N, lstm_H, KB, scale, w_dst);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return e;
  const int n_pad = lstm_H > 0 ? lstm_H * 4 : (N + 31) / 32 * 32;
  pack_split_bias_kernel<<<(n_pad + 255) / 256, 256, 0, st>>>(b0, b1, N, lstm_H, bias_dst);
  return cudaGetLastError();
}

cudaError_t launch_act_split(const float* s0, int K0, int ld0, const float* s1, int K1, int ld1, int M, __half* a_hi,
                             __half* a_lo, cudaStream_t st) {
  const int KB = (K0 + K1 + 63) / 64;
  const int rows_pad = M <= 64 ? 64 : 128;
  const int n = KB * rows_pad * 8;
  act_split_kernel<<<(n + 255) / 256, 256, 0, st>>>(s0, K0, ld0, s1, K1, ld1, M, rows_pad, KB, a_hi, a_lo);
  return cudaGetLastError();
}

size_t tc_big_weight_bytes(int N, int nseg, int K) {
  return (size_t)((N + 127) / 128) * nseg * ((K + 63) / 64) * 2 * w_tile_bytes<128>();
}
size_t tc_big_act_bytes(int M, int nseg, int K) {  // one plane (hi or lo)
  return (size_t)nseg * ((K + 63) / 64) * ((size_t)(M + 127) / 128 * 128) * 128;
}

cudaError_t launch_im2col_split(const TcIm2col& q, __half* a_hi, __half* a_lo, cudaStream_t st) {
  const size_t total = (size_t)q.nseg * q.KBs * q.rows_total * 8;
  im2col_split_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(q, a_hi, a_lo);
  return cudaGetLastError();
}

cudaError_t launch_pack_big_w(const TcBigPack& q, __half* dst, cudaStream_t st) {
  const size_t total = (size_t)((q.N + 127) / 128) * q.nseg * q.KBs * 1024;
  pack_big_w_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(q, dst);
  return cudaGetLastError();
}

cudaError_t launch_tc_big(const TcBigArgs& a, cudaStream_t st) {
  if (a.M <= 0 || a.N <= 0 || a.N % 4 || a.KB <= 0 || a.rows_total % 128 || a.rows_total < a.M) return cudaErrorInvalidValue;
  constexpr size_t smem = kBigStages * stage_bytes<128>() + 1024 + 1024 + kEpiStageBytes;
  static bool attr = false;
  if (!attr) {
    cudaError_t e = cudaFuncSetAttribute(tc_big_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    attr = true;
  }
  return launch_pdl(tc_big_kernel, dim3((a.N + 127) / 128, (a.M + 127) / 128), smem, st, a);
}

cudaError_t launch_tc_lstm_seq(const TcLstmSeqArgs& a, cudaStream_t st) {
  if (a.M <= 0 || a.H <= 0 || a.H % 8 || a.KB <= 0 || a.rows_total % 128 || a.rows_total < a.M) return cudaErrorInvalidValue;
  constexpr size_t smem = kStages * kStageBytes + 1024 + 1024 + kEpiStageBytes;
  static bool attr = false;
  if (!attr) {
    cudaError_t e = cudaFuncSetAttribute(tc_lstm_seq_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    attr = true;
  }
  return launch_pdl(tc_lstm_seq_kernel, dim3(a.H / 8, (a.M + 127) / 128), smem, st, a);
}

cudaError_t launch_tc_gru(const TcGruArgs& a, cudaStream_t st) {
  if (a.M <= 0 || a.M > 128 || a.H <= 0 || a.H % 8 || a.KB <= 0 || a.ndir < 1 || a.ndir > 2) return cudaErrorInvalidValue;
  TcGruArgs p = a;
  p.rows_pad = a.M <= 64 ? 64 : 128;
  constexpr size_t smem = kStages * kStageBytes + 1024 + 1024 + kEpiStageBytes;
  static bool attr = false;
  if (!attr) {
    cudaError_t e = cudaFuncSetAttribute(tc_gru_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    attr = true;
  }
  return launch_pdl(tc_gru_kernel, dim3(a.H / 8, a.ndir), smem, st, p);
}

cudaError_t launch_tc_skinny(const TcSkinnyArgs& a, cudaStream_t st) {
  if (a.M <= 0 || a.M > 128 || a.N <= 0 || a.KB <= 0) return cudaErrorInvalidValue;
  TcSkinnyArgs p = a;
  p.rows_pad = a.M <= 64 ? 64 : 128;
  static const bool ring8 = [] {
    const char* e = getenv("MB_TACO_RING8");  // A/B switch: 0 = 4 stages of 40 KB for every batch size (round 2)
    return e ? atoi(e) != 0 : true;
  }();
  p.compact = (ring8 && p.rows_pad == 64) ? 1 : 0;
  constexpr size_t smem = (kStages * kStageBytes > 2 * kStages * (kATile + 2 * kWTile) ? kStages * kStageBytes : 2 * kStages * (kATile + 2 * kWTile)) + 1024 + 1024 + kEpiStageBytes;
  static bool attr = false;
  if (!attr) {
    cudaError_t e = cudaFuncSetAttribute(tc_skinny_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    attr = true;
  }
  // MB_TACO_MC = 2 / 4 / 8: cluster size of the activation-tile multicast (launches whose tile count it divides).  Default 1 (no
  // clusters): MEASURED SLOWER - cfg 4 takes 42.1 ms with clusters of 8 and 36.3 ms with 4 against 35.6 ms without (same box, ABAB).
  // The launches are not bound by L2 traffic; co-scheduling 8 SMs of a GPC per cluster and refilling a stage only when the slowest
  // of 8 CTAs has consumed it cost more than the 2.4 x smaller operand traffic saves.
  static const int mc_env = [] {
    const char* e = getenv("MB_TACO_MC");
    const int v = e ? atoi(e) : 1;
    return (v == 2 || v == 4 || v == 8) ? v : 1;
  }();
  const int tiles = (a.N + 31) / 32;
  const int cl = (mc_env > 1 && tiles % mc_env == 0 && (p.rows_pad * 128) % (16 * mc_env) == 0) ? mc_env : 1;
  return launch_pdl(tc_skinny_kernel, dim3(tiles), smem, st, p, cl);
}

}  // namespace taco
}  // namespace mb
