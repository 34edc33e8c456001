// Tacotron inference on H100 (mb_tacotron_*): encoder (embedding, PreNet, CBHG), global style token,
// attention decoder loop and postnet CBHG, lowered onto the FP32 kernels of tacotron_kernels.cu plus
// the location-sensitive-attention step kernel below.
//
// reference: models/synthesizer/models/tacotron.py:199-298 (forward/generate), :71-138 (Decoder.forward),
//            sublayer/cbhg.py:42-79, sublayer/lsa.py:21-42, sublayer/pre_net.py:11-27,
//            sublayer/global_style_token.py:9-145
// Activations are channels-last [rows][features]; Conv1d over time = shifted-row GEMM segments.
#include "tacotron_kernels.cuh"

#include <cstdlib>
#include <cstring>
#include <algorithm>
#include <map>
#include <memory>
#include <set>
#include <string>
#include <vector>

#include "../../include/mb_wavernn_math.h"
#include "mb_common.h"

namespace mb {
namespace taco {

namespace {

// ---- location sensitive attention step: one CTA per batch row ---------------------------------------
//   pq[d]   = W q + b                       (precomputed, [B][128])
//   loc[f]  = conv1d(cumulative, k=31)[t]   (32 filters)
//   u[t]    = v . tanh(pq + proj[b,t] + L loc) * (chars[b,t] != 0)
//   scores  = softmax_t(u); cumulative += scores; ctx = scores @ seq[b]
// Ragged rows (lens != nullptr): row b has lens[b] characters.  Positions >= lens[b] get the energy -inf, so their exp is
// exactly 0: every max, sum and score of the row is bitwise what it would be with the loops cut at lens[b], i.e. what the row
// computes alone, and their cumulative attention stays at its initial 0, which is what the location conv reads past the row's
// end.  (Cutting the loops instead keeps the length live in a register and makes ptxas spill.)
constexpr int ATT_D = 128, ATT_F = 32, ATT_K = 31;

// launch with the programmatic-stream-serialization attribute (MB_TACO_PDL2=0: plain launch): the kernel may start while the
// previous one drains; it must not touch anything another kernel writes before its griddepcontrol.wait
template <typename... KArgs, typename... Args>
cudaError_t launch_pdl2(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args... args) {
  static const bool pdl = [] {
    const char* e = getenv("MB_TACO_PDL2");
    return e ? atoi(e) != 0 : true;
  }();
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(args)...);
}

__global__ void __launch_bounds__(512) lsa_step_kernel(const float* __restrict__ pq, const float* __restrict__ proj,
                                                       const float* __restrict__ seq, int seq_dim,
                                                       const int32_t* __restrict__ chars, float* cum,
                                                       const float* __restrict__ conv_w, const float* __restrict__ conv_b,
                                                       const float* __restrict__ Lw, const float* __restrict__ vw,
                                                       float* __restrict__ scores_out, int scores_ld, float* ctx, int Tc,
                                                       const int* step_ptr, int step_j, const float* __restrict__ q_in,
                                                       const float* __restrict__ Wq, const float* __restrict__ bq,
                                                       const int* __restrict__ lens, const int* __restrict__ row_start, int ring) {
  extern __shared__ float sm[];
  // this decoder step's row of the alignment matrix (the row's own step in a ring with a per-row step origin)
  scores_out += (size_t)ring_slot(row_step(step_index(step_ptr, step_j), row_start, blockIdx.x), row_start, ring) * Tc;
  float* s_cw = sm;                         // [32][31]
  float* s_Lt = s_cw + ATT_F * ATT_K;       // [32][128]  (L transposed: conflict-free for d-major threads)
  float* s_v = s_Lt + ATT_D * ATT_F;        // [128]
  float* s_pq = s_v + ATT_D;                // [128]
  float* s_cb = s_pq + ATT_D;               // [32]
  float* s_cum = s_cb + ATT_F;              // [Tc + 30] zero padded
  float* s_u = s_cum + Tc + 2 * 15;         // [Tc]
  float* s_red = s_u + Tc;                  // [32]
  float* s_loc = s_red + 32;                // [Tc][32]
  float* s_part = s_loc + (size_t)Tc * ATT_F;  // [Tc][4]
  const int b = blockIdx.x, tid = threadIdx.x;
  for (int i = tid; i < ATT_F * ATT_K; i += blockDim.x) s_cw[i] = conv_w[i];
  for (int i = tid; i < ATT_D * ATT_F; i += blockDim.x) {
    const int d = i / ATT_F, f = i - d * ATT_F;
    s_Lt[f * ATT_D + d] = Lw[i];
  }
  for (int i = tid; i < ATT_D; i += blockDim.x) s_v[i] = vw[i];
  for (int i = tid; i < ATT_F; i += blockDim.x) s_cb[i] = conv_b[i];
  // programmatic dependent launch: the weights above are never written by a kernel and were staged while the previous launch drained
  asm volatile("griddepcontrol.wait;" ::: "memory");
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  for (int i = tid; i < ATT_D; i += blockDim.x) {
    if (!q_in) s_pq[i] = pq[(size_t)b * ATT_D + i];
  }
  if (q_in) {
    // processed query pq = W q + b (lsa.py:29) computed here instead of by a GEMM launch of its own: one warp per output,
    // lanes over k (coalesced rows of W), 128 x 128 MACs per batch row
    const int warp = tid >> 5, lane = tid & 31, nw = (int)(blockDim.x >> 5);
    float qv[ATT_D / 32];
#pragma unroll
    for (int j = 0; j < ATT_D / 32; ++j) qv[j] = q_in[(size_t)b * ATT_D + lane + 32 * j];
    for (int o = warp; o < ATT_D; o += nw) {
      float a = 0.f;
#pragma unroll
      for (int j = 0; j < ATT_D / 32; ++j) a = fmaf(Wq[(size_t)o * ATT_D + lane + 32 * j], qv[j], a);
      for (int sh = 16; sh; sh >>= 1) a += __shfl_xor_sync(0xffffffffu, a, sh);
      if (lane == 0) s_pq[o] = a + bq[o];
    }
  }
  for (int i = tid; i < Tc + 30; i += blockDim.x) {
    const int t = i - 15;
    s_cum[i] = (t >= 0 && t < Tc) ? cum[(size_t)b * Tc + t] : 0.f;
  }
  __syncthreads();
  // location features loc[t][f] = conv1d(cumulative, k = 31)[t] + bias: one (t, f) per thread and pass
  for (int i = tid; i < Tc * ATT_F; i += blockDim.x) {
    const int t = i >> 5, f = i & 31;
    float a = 0.f;
#pragma unroll
    for (int j = 0; j < ATT_K; ++j) a = fmaf(s_cw[f * ATT_K + j], s_cum[t + j], a);
    s_loc[i] = a + s_cb[f];
  }
  __syncthreads();
  // energies: thread = (d, t parity); u[t] = sum_d v[d] * tanh(pq[d] + proj[t][d] + sum_f L[d][f] loc[t][f])
  {
    const int d = tid & (ATT_D - 1), tg = tid >> 7, wq = (tid >> 5) & 3;
    const int ntg = (int)(blockDim.x >> 7);  // time-step groups of 128 threads (2 at 256 threads, 4 at 512)
    float lreg[ATT_F];
#pragma unroll
    for (int f = 0; f < ATT_F; ++f) lreg[f] = s_Lt[f * ATT_D + d];
    const float vd = s_v[d], pqd = s_pq[d];
    const float* pb = proj + (size_t)b * Tc * ATT_D + d;
    // blocks of 8 time steps: the 8 (independent) loads of the processed memory are issued before any is used -
    // a plain loop is bound by one L2 round trip per step
    for (int t0 = tg; t0 < Tc; t0 += 8 * ntg) {
      float pr[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int t = t0 + ntg * j;
        pr[j] = t < Tc ? pb[(size_t)t * ATT_D] : 0.f;
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int t = t0 + ntg * j;
        if (t >= Tc) break;  // warp-uniform
        float pl = 0.f;
        const float* lc = s_loc + (size_t)t * ATT_F;
#pragma unroll
        for (int f = 0; f < ATT_F; ++f) pl = fmaf(lreg[f], lc[f], pl);
        float e = vd * tanhf(pqd + pr[j] + pl);
        for (int o = 16; o; o >>= 1) e += __shfl_xor_sync(0xffffffffu, e, o);
        if ((tid & 31) == 0) s_part[t * 4 + wq] = e;
      }
    }
  }
  __syncthreads();
  const int len = lens ? lens[b] : Tc;
  for (int t = tid; t < Tc; t += blockDim.x) {
    const float u = (s_part[t * 4 + 0] + s_part[t * 4 + 1]) + (s_part[t * 4 + 2] + s_part[t * 4 + 3]);
    // u * (chars != 0): padded positions of the row score exp(0); positions past a ragged row's end are out of it
    s_u[t] = t >= len ? -INFINITY : chars[(size_t)b * Tc + t] != 0 ? u : 0.f;
  }
  __syncthreads();
  // softmax over t
  float mx = -3.0e38f;
  for (int t = tid; t < Tc; t += blockDim.x) mx = fmaxf(mx, s_u[t]);
  for (int o = 16; o; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  if ((tid & 31) == 0) s_red[tid >> 5] = mx;
  __syncthreads();
  mx = s_red[0];
  for (int w = 1; w < (int)(blockDim.x >> 5); ++w) mx = fmaxf(mx, s_red[w]);
  __syncthreads();
  float sum = 0.f;
  for (int t = tid; t < Tc; t += blockDim.x) {
    const float e = expf(s_u[t] - mx);
    s_u[t] = e;
    sum += e;
  }
  for (int o = 16; o; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  if ((tid & 31) == 0) s_red[tid >> 5] = sum;
  __syncthreads();
  sum = 0.f;
  for (int w = 0; w < (int)(blockDim.x >> 5); ++w) sum += s_red[w];
  for (int t = tid; t < Tc; t += blockDim.x) {
    const float sc = s_u[t] / sum;
    s_u[t] = sc;
    scores_out[(size_t)b * scores_ld + t] = sc;
    cum[(size_t)b * Tc + t] = s_cum[t + 15] + sc;
  }
  if (ctx == nullptr) return;  // context vector computed by lsa_ctx_kernel (more CTAs, vector loads)
  __syncthreads();
  // t < len: a ragged row never reads the encoder sequence past its end (0 * seq[t] would be NaN there were seq[t] not finite)
  for (int f = tid; f < seq_dim; f += blockDim.x) {
    float a = 0.f;
    const float* sp = seq + (size_t)b * Tc * seq_dim + f;
    for (int t = 0; t < len; ++t) a = fmaf(s_u[t], sp[(size_t)t * seq_dim], a);
    ctx[(size_t)b * seq_dim + f] = a;
  }
}

// dynamic shared memory of lsa_step_kernel (the layout at its top): 4 * (5438 + 38 Tc) bytes
size_t lsa_step_smem_bytes(int Tc) {
  return sizeof(float) * (ATT_F * ATT_K + ATT_D * ATT_F + 2 * ATT_D + ATT_F + (Tc + 30) + Tc + 32 + (size_t)Tc * ATT_F + (size_t)Tc * 4);
}

// the longest input (characters per utterance) lsa_step_kernel can take on the current device: its shared memory must fit the
// per-block opt-in limit (1386 at the H100's 227 KB); 0 when there is no device to ask
int lsa_max_chars() {
  int dev = 0, optin = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev) != cudaSuccess) {
    cudaGetLastError();
    return 0;
  }
  const size_t fixed = lsa_step_smem_bytes(0), per_char = lsa_step_smem_bytes(1) - fixed;
  return (size_t)optin > fixed ? (int)(((size_t)optin - fixed) / per_char) : 0;
}

// raises the kernel's dynamic shared memory limit where the input needs more than the default 48 KB
cudaError_t lsa_step_prepare(int Tc) {
  const size_t smem = lsa_step_smem_bytes(Tc);
  return smem > 48 * 1024 ? cudaFuncSetAttribute(lsa_step_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) : cudaSuccess;
}

// context = scores @ encoder_seq (tacotron.py:104 via lsa.py:40): ctx[b][f] = sum_t scores[b][t] seq[b][t][f].
// grid (seq_dim / 256, B): 64 float4 feature lanes x 4 interleaved t-groups per CTA, partials reduced in smem.
// The whole encoder sequence (B x Tc x 1024 fp32) is re-read every decoder step from L2: the kernel needs many
// 16-byte loads in flight, which one CTA per batch row cannot provide.  Ragged rows (lens): only t < lens[b] is read.
__global__ void __launch_bounds__(256) lsa_ctx_kernel(const float* __restrict__ scores, int scores_ld, const float* __restrict__ seq,
                                                      int seq_dim, int Tc, float* __restrict__ ctx, const int* step_ptr,
                                                      int step_j, __half* sa_hi, __half* sa_lo, __half* sb_hi, __half* sb_lo,
                                                      int s_rows_pad, const int* __restrict__ lens, const int* __restrict__ row_start,
                                                      int ring) {
  __shared__ float4 part[4][64];
  extern __shared__ float s_sc[];
  asm volatile("griddepcontrol.wait;" ::: "memory");
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  const int b = blockIdx.y, f4 = blockIdx.x * 64 + (threadIdx.x & 63), tg = threadIdx.x >> 6;
  const int sb = ring_slot(row_step(step_index(step_ptr, step_j), row_start, b), row_start, ring);
  const float* sc = scores + (size_t)sb * Tc + (size_t)b * scores_ld;
  const int Tb = lens ? lens[b] : Tc;
  for (int t = threadIdx.x; t < Tb; t += 256) s_sc[t] = sc[t];
  __syncthreads();
  float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
  const float4* sp = reinterpret_cast<const float4*>(seq + (size_t)b * Tc * seq_dim) + f4;
  const int q4 = seq_dim >> 2;
#pragma unroll 6
  for (int t = tg; t < Tb; t += 4) {
    const float4 v = sp[(size_t)t * q4];
    const float w = s_sc[t];
    a.x = fmaf(w, v.x, a.x);
    a.y = fmaf(w, v.y, a.y);
    a.z = fmaf(w, v.z, a.z);
    a.w = fmaf(w, v.w, a.w);
  }
  part[tg][threadIdx.x & 63] = a;
  __syncthreads();
  if (tg == 0) {
    const float4 p0 = part[0][threadIdx.x], p1 = part[1][threadIdx.x], p2 = part[2][threadIdx.x], p3 = part[3][threadIdx.x];
    float4 r;
    r.x = (p0.x + p1.x) + (p2.x + p3.x);
    r.y = (p0.y + p1.y) + (p2.y + p3.y);
    r.z = (p0.z + p1.z) + (p2.z + p3.z);
    r.w = (p0.w + p1.w) + (p2.w + p3.w);
    reinterpret_cast<float4*>(ctx + (size_t)b * seq_dim)[f4] = r;
    // the context is the leading K segment of two tensor-core GEMMs (attention GRU input of the NEXT step, rnn_input of this one):
    // write their hi / lo operand chunks here instead of launching act_split twice
    if (sa_hi) taco::store_split_quad(r, b, s_rows_pad, f4 * 4, sa_hi, sa_lo);
    if (sb_hi) taco::store_split_quad(r, b, s_rows_pad, f4 * 4, sb_hi, sb_lo);
  }
}

// global style token attention for one batch row: q [512] -> 8 heads over `ntok` tokens (K,V [ntok][512])
__global__ void gst_attention_kernel(const float* __restrict__ q, const float* __restrict__ Kt, const float* __restrict__ Vt,
                                     int ntok, float* __restrict__ out, int E, int heads, float inv_sqrt_dk) {
  __shared__ float sc[8][16];
  const int b = blockIdx.x, tid = threadIdx.x;
  const int hd = E / heads;
  if (tid < heads * ntok) {
    const int h = tid / ntok, k = tid - h * ntok;
    float a = 0.f;
    for (int d = 0; d < hd; ++d) a = fmaf(q[(size_t)b * E + h * hd + d], Kt[(size_t)k * E + h * hd + d], a);
    sc[h][k] = a * inv_sqrt_dk;
  }
  __syncthreads();
  if (tid < heads) {
    float mx = -3.0e38f;
    for (int k = 0; k < ntok; ++k) mx = fmaxf(mx, sc[tid][k]);
    float s = 0.f;
    for (int k = 0; k < ntok; ++k) {
      sc[tid][k] = expf(sc[tid][k] - mx);
      s += sc[tid][k];
    }
    for (int k = 0; k < ntok; ++k) sc[tid][k] /= s;
  }
  __syncthreads();
  for (int e = tid; e < E; e += blockDim.x) {
    const int h = e / hd;
    float a = 0.f;
    for (int k = 0; k < ntok; ++k) a = fmaf(sc[h][k], Vt[(size_t)k * E + e], a);
    out[(size_t)b * E + e] = a;
  }
}

__global__ void bn_fold_kernel(const float* g, const float* b, const float* mean, const float* var, float* scale,
                               float* shift, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float s = g[i] * (1.0f / sqrtf(var[i] + 1e-5f));
  scale[i] = s;
  shift[i] = b[i] - mean[i] * s;
}

__global__ void tanh_kernel(const float* x, float* y, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) y[i] = tanhf(x[i]);
}

// compact mel projection rows: dst[(j*80 + m)][:] = W[(m*max_r + j)][:]
__global__ void pack_melproj_kernel(const float* __restrict__ W, float* __restrict__ dst, int n_mels, int max_r, int r,
                                    int K) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)r * n_mels * K) return;
  const int k = (int)(i % K);
  const int row = (int)(i / K);
  const int j = row / n_mels, m = row - j * n_mels;
  dst[i] = W[((size_t)m * max_r + j) * K + k];
}

__global__ void fill_masks_kernel(uint8_t* m, size_t n, uint64_t seed, uint32_t stream_id, const int* step_ptr = nullptr) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  if (step_ptr) stream_id += (uint32_t)*step_ptr;  // decoder step = *step_ptr + offset (graph replay)
  uint32_t o[4];
  mb_philox4x32((uint32_t)(i >> 2), (uint32_t)(i >> 34), stream_id, 0x7461636fu, (uint32_t)seed, (uint32_t)(seed >> 32), o);
  m[i] = (uint8_t)((o[i & 3] >> 16) & 1u);  // Bernoulli(0.5) keep flag
}

// the PreNet dropout masks of ALL decoder steps in one launch (same bits as fill_masks_kernel called with stream_id = step)
__global__ void fill_masks_steps_kernel(uint8_t* m, size_t n_per_step, int n_steps, uint64_t seed) {
  const size_t g = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= n_per_step * (size_t)n_steps) return;
  const uint32_t step = (uint32_t)(g / n_per_step);
  const size_t i = g - (size_t)step * n_per_step;
  uint32_t o[4];
  mb_philox4x32((uint32_t)(i >> 2), (uint32_t)(i >> 34), step, 0x7461636fu, (uint32_t)seed, (uint32_t)(seed >> 32), o);
  m[g] = (uint8_t)((o[i & 3] >> 16) & 1u);
}

// PreNet dropout keep flags of ragged rows, keyed by each utterance's own seed: the Philox counter is (unit / 4, position, layer),
// position = character (encoder) or decoder step, so an utterance draws the same flags whatever its row, batch or neighbours.
//   encoder (dec == 0): m [2 layers][B][npos][units];  decoder (dec == 1): m [npos steps][2 layers][B][units]
__global__ void fill_masks_seeded_kernel(uint8_t* m, int B, int npos, int units, const uint64_t* __restrict__ seeds, int dec) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)2 * B * npos * units) return;
  const int u = (int)(i % units);
  size_t q = i / units;
  int b, l, pos;
  if (dec) {
    b = (int)(q % B);
    q /= B;
    l = (int)(q & 1);
    pos = (int)(q >> 1);
  } else {
    pos = (int)(q % npos);
    q /= npos;
    b = (int)(q % B);
    l = (int)(q / B);
  }
  const uint64_t seed = seeds[b];
  uint32_t o[4];
  mb_philox4x32((uint32_t)u >> 2, (uint32_t)pos, (uint32_t)(2 * dec + l), 0x72616767u, (uint32_t)seed, (uint32_t)(seed >> 32), o);
  m[i] = (uint8_t)((o[u & 3] >> 16) & 1u);
}

// stop rule of tacotron.py:275 at decoder step si (frame t = si * r) over the B stop values stopv[b * ld].  Padded batch
// (row_done == nullptr): flags[si] = every row passes and t > 10.  Ragged rows: row b ends at the first step where it passes with
// t > 10 or reaches its cap of row_caps[b] steps (row_done[b] = that step, -1 before); flags[si] = every row has ended.  With a
// per-row step origin (row_start) each row applies the rule at its own step and flags is null: the global step is unbounded, so
// nothing is indexed by it, and the host polls row_done instead.
__device__ void apply_stop_rule(const float* stopv, int ld, int B, float min_stop_token, int r, int si, int* flags, int* row_done,
                                const int* row_caps, const int* row_start) {
  bool all = true;
  for (int b = 0; b < B; ++b) {
    const bool pass = __ldcg(stopv + (size_t)b * ld) * 10.f > min_stop_token;
    if (row_done) {
      const int s = row_step(si, row_start, b);
      if (row_done[b] < 0 && ((pass && s * r > 10) || s + 1 >= row_caps[b])) row_done[b] = s;
      all = all && row_done[b] >= 0;
    } else {
      all = all && pass;
    }
  }
  if (flags) flags[si] = row_done ? (all ? 1 : 0) : ((all && si * r > 10) ? 1 : 0);
}

// decoder step si = (step_ptr ? *step_ptr : 0) + step_j; frame t = si * r; flags[si] = stop rule of tacotron.py:275
__global__ void stop_flag_kernel(const float* stopv, int B, float min_stop_token, int r, int* flags, const int* step_ptr,
                                 int step_j, int* row_done = nullptr, const int* row_caps = nullptr, const int* row_start = nullptr) {
  if (threadIdx.x == 0 && blockIdx.x == 0)
    apply_stop_rule(stopv, 1, B, min_stop_token, r, step_index(step_ptr, step_j), flags, row_done, row_caps, row_start);
}

// stop projection (sigmoid(w . [x | ctx] + b), tacotron.py:131-133) of one batch row per CTA, then - in the CTA that takes the
// last ticket - the stop rule over all rows.  Same summation order as rowdot_kernel.
__global__ void __launch_bounds__(256) stop_step_kernel(const GemmArgs a, int B, float min_stop_token, int r, int* flags,
                                                        const int* step_ptr, int step_j, unsigned int* ticket,
                                                        int* row_done = nullptr, const int* row_caps = nullptr,
                                                        const int* row_start = nullptr) {
  __shared__ float red[8];
  __shared__ bool last;
  const int m = blockIdx.x, tid = threadIdx.x;
  float s = 0.f;
  for (int sgi = 0; sgi < a.nseg; ++sgi) {
    const Seg sg = a.seg[sgi];
    for (int k = tid; k < sg.K; k += 256) s = fmaf(sg.x[(size_t)m * sg.ld + k], a.W[sg.w_off + (size_t)k * sg.w_stride], s);
  }
  for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if ((tid & 31) == 0) red[tid >> 5] = s;
  __syncthreads();
  if (tid == 0) {
    float v = 0.f;
    for (int w = 0; w < 8; ++w) v += red[w];
    if (a.bias) v += a.bias[0];
    a.Y[(size_t)m * a.ldy] = 1.f / (1.f + expf(-v));
    __threadfence();
    last = atomicAdd(ticket, 1u) == (unsigned int)(B - 1);
  }
  __syncthreads();
  if (last && tid == 0) {
    *ticket = 0u;
    __threadfence();
    apply_stop_rule(a.Y, a.ldy, B, min_stop_token, r, step_index(step_ptr, step_j), flags, row_done, row_caps, row_start);
  }
}

__global__ void step_advance_kernel(int* step_ptr, int n) {
  if (threadIdx.x == 0 && blockIdx.x == 0) *step_ptr += n;
}

// [B][T][C] (first `frames` of `steps` rows) -> [B][C][frames]
__global__ void to_ncl_kernel(const float* __restrict__ x, int steps, float* __restrict__ y, int B, int C, int frames) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)B * C * frames) return;
  const int t = (int)(i % frames);
  const int c = (int)((i / frames) % C);
  const int b = (int)(i / ((size_t)frames * C));
  y[i] = x[((size_t)b * steps + t) * C + c];
}


// a few host bytes carried into device memory as a kernel argument (upload() in the stream entry points)
constexpr int kUploadBytes = 8192;
struct UploadBlob {
  unsigned char b[kUploadBytes];
};
__global__ void upload_kernel(const __grid_constant__ UploadBlob src, unsigned char* dst, int n) {
  for (int i = threadIdx.x; i < n; i += blockDim.x) dst[i] = src.b[i];
}

// ---- streamed decoding (mb_tacotron_stream_*): row admission -----------------------------------------------------------------
// One launch puts n texts into their slots between graph replays: every recurrent state, ctx, cum, the side stream's half-sums and
// both parities of the fused-split operand tiles of the slot go to the zeros a fresh row starts from; the text's encoder rows
// (seq, encoder_proj keys) and characters are copied from the staging pool; its decoder dropout masks are copied (injected) or drawn
// (Philox keyed by its seed, as fill_masks_seeded_kernel) for its steps 0 .. cap - 1; its length, cap, done step (-1) and start
// step are set.  blockIdx.y = admitted row.
struct AdmitRow {
  int slot, src, len, cap;  // slot, staging-pool row, characters, decoder-step cap
  uint64_t seed;
  const uint8_t* dmask;     // injected masks [>= cap][2][units], or null: drawn from seed
};
struct RowZero {            // row `slot` of a region: nchunks chunks of chunk_bytes at p + c * chunk_stride + slot * row_stride
  char* p;
  long long row_stride, chunk_stride;
  int nchunks, chunk_bytes;
};
constexpr int kMaxZero = 32;
struct AdmitArgs {
  const AdmitRow* rows;
  int start;                // global step the rows start at
  RowZero zero[kMaxZero];
  int nzero;
  const float* src_seq;     // staging pool [2 * slots][Tc][seq_row / Tc]
  float* seq;
  long long seq_row;
  const float* src_proj;
  float* proj;
  long long proj_row;
  const int32_t* src_chars;
  int32_t* chars;
  int Tc;
  int* lens;
  int* caps;
  int* done;
  int* starts;
  uint8_t* dmask;           // [ring][2][S][units]
  int S, units;
};

__global__ void admit_rows_kernel(const __grid_constant__ AdmitArgs a) {
  const AdmitRow row = a.rows[blockIdx.y];
  const long long tid = (long long)blockIdx.x * blockDim.x + threadIdx.x, nth = (long long)gridDim.x * blockDim.x;
  for (int z = 0; z < a.nzero; ++z) {
    const RowZero& r = a.zero[z];
    const int words = r.chunk_bytes / 4;
    for (long long i = tid; i < (long long)r.nchunks * words; i += nth) {
      const long long c = i / words, w = i - c * words;
      reinterpret_cast<uint32_t*>(r.p + c * r.chunk_stride + (long long)row.slot * r.row_stride)[w] = 0u;
    }
  }
  for (long long i = tid; i < a.seq_row; i += nth) a.seq[row.slot * a.seq_row + i] = a.src_seq[row.src * a.seq_row + i];
  for (long long i = tid; i < a.proj_row; i += nth) a.proj[row.slot * a.proj_row + i] = a.src_proj[row.src * a.proj_row + i];
  for (long long i = tid; i < a.Tc; i += nth) a.chars[(long long)row.slot * a.Tc + i] = a.src_chars[(long long)row.src * a.Tc + i];
  for (long long i = tid; i < (long long)row.cap * 2 * a.units; i += nth) {
    const int u = (int)(i % a.units), l = (int)((i / a.units) & 1), pos = (int)(i / (2 * a.units));
    uint8_t v;
    if (row.dmask) {
      v = row.dmask[i];
    } else {
      uint32_t o[4];
      mb_philox4x32((uint32_t)u >> 2, (uint32_t)pos, (uint32_t)(2 + l), 0x72616767u, (uint32_t)row.seed, (uint32_t)(row.seed >> 32), o);
      v = (uint8_t)((o[u & 3] >> 16) & 1u);
    }
    a.dmask[(((size_t)pos * 2 + l) * a.S + row.slot) * a.units + u] = v;
  }
  if (tid == 0) {
    a.lens[row.slot] = row.len;
    a.caps[row.slot] = row.cap;
    a.done[row.slot] = -1;
    a.starts[row.slot] = a.start;
  }
}

}  // namespace
}  // namespace taco
}  // namespace mb

// =================================================================================================
using namespace mb;
using namespace mb::taco;

struct mb_tacotron {
  mb_tacotron_config cfg{};
  WeightTable w;
  bool finalized = false;
  int packed_r = 0;
  std::map<std::string, float> tc_inv_scale;  // tensor-core weight images: 1 / pack scale per tensor
  // generate() runs on an internal non-blocking stream ordered after / before the caller's stream by events: the
  // decoder loop is replayed from a CUDA graph, and stream capture is not allowed on the legacy default stream
  std::set<std::string> big_packed;  // CBHG GEMMs whose tensor-core images ("<key>.bigw") are packed
  cudaStream_t own_stream = nullptr;
  cudaEvent_t ev_in = nullptr, ev_out = nullptr;
  // side stream of the decoder loop (the parts of a step's GEMMs whose inputs are known a step early, the stop rule) + its events
  cudaStream_t side_stream = nullptr;
  cudaEvent_t ev_side[8] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
};

namespace {

float* P(const mb_tacotron* h, const std::string& name) { return h->w.ptr(name); }

void cbhg_slots(WeightTable& w, const std::string& p, int K, int cin, int ch, int p0, int p1, int nh) {
  auto bnconv = [&](const std::string& n, int ci, int co, int k) {
    w.add(n + ".conv.weight", {co, ci, k});
    for (const char* leaf : {".bnorm.weight", ".bnorm.bias", ".bnorm.running_mean", ".bnorm.running_var"}) w.add(n + leaf, {co});
    w.add_derived(n + ".bn_scale", co);  // at finalize
    w.add_derived(n + ".bn_shift", co);
  };
  for (int i = 0; i < K; ++i) bnconv(p + ".conv1d_bank." + std::to_string(i), cin, ch, i + 1);
  bnconv(p + ".conv_project1", K * ch, p0, 3);
  bnconv(p + ".conv_project2", p0, p1, 3);
  if (p1 != ch) w.add(p + ".pre_highway.weight", {ch, p1});
  // derived: tensor-core images of the large-M GEMMs (cbhg_gemm), packed on first use
  for (int i = 0; i < K; ++i) w.add_derived(p + ".conv1d_bank." + std::to_string(i) + ".bigw", tc_big_weight_bytes(ch, i + 1, cin) / 4);
  w.add_derived(p + ".conv_project1.bigw", tc_big_weight_bytes(p0, 3, K * ch) / 4);
  w.add_derived(p + ".conv_project2.bigw", tc_big_weight_bytes(p1, 3, p0) / 4);
  if (p1 != ch) w.add_derived(p + ".pre_highway.bigw", tc_big_weight_bytes(ch, 1, p1) / 4);
  for (int i = 0; i < nh; ++i) w.add_derived(p + ".highways." + std::to_string(i) + ".bigw", tc_big_weight_bytes(2 * ch, 1, ch) / 4);
  for (const char* sfx : {"", "_reverse"}) w.add_derived(p + ".rnn.ih" + sfx + ".bigw", tc_big_weight_bytes(3 * (ch / 2), 1, ch) / 4);
  for (int i = 0; i < nh; ++i) {
    const std::string q = p + ".highways." + std::to_string(i);
    w.add(q + ".W1.weight", {ch, ch});
    w.add(q + ".W1.bias", {ch});
    w.add(q + ".W2.weight", {ch, ch});
    w.add(q + ".W2.bias", {ch});
    w.add_derived(q + ".W12", (size_t)2 * ch * ch);  // [W1; W2] stacked
    w.add_derived(q + ".b12", (size_t)2 * ch);
  }
  const int H = ch / 2;
  for (const char* sfx : {"", "_reverse"}) {
    w.add(p + ".rnn.weight_ih_l0" + sfx, {3 * H, ch});
    w.add(p + ".rnn.weight_hh_l0" + sfx, {3 * H, H});
    w.add(p + ".rnn.bias_ih_l0" + sfx, {3 * H});
    w.add(p + ".rnn.bias_hh_l0" + sfx, {3 * H});
    // derived: tensor-core images of W_hh (gates r|z|n interleaved per 8 units) + tile-order b_hh
    w.add_derived(p + ".rnn.hh" + sfx + ".tcw", tc_gated_weight_bytes(H, H) / 4);
    w.add_derived(p + ".rnn.hh" + sfx + ".tcb", (size_t)4 * H);
  }
}

// byte offsets (inside Ws::fsp) of the hi planes of the operand tiles the decoder kernels write for each other; lo = hi + bytes
struct FusedSplit {
  size_t p1, p2, p3[2], p4[2], p5, b1, b2, b3, b5, total;
};
FusedSplit fused_split_layout(int Bc, int proj_dims, int D, int LD) {
  FusedSplit f{};
  f.b1 = tc_skinny_act_bytes(Bc, proj_dims + 2 * D);
  f.b2 = tc_skinny_act_bytes(Bc, proj_dims + D);
  f.b3 = tc_skinny_act_bytes(Bc, 2 * LD);
  f.b5 = tc_skinny_act_bytes(Bc, LD);
  size_t o = 0;
  f.p1 = o; o += 2 * f.b1;
  f.p2 = o; o += 2 * f.b2;
  for (int q = 0; q < 2; ++q) { f.p3[q] = o; o += 2 * f.b3; }
  for (int q = 0; q < 2; ++q) { f.p4[q] = o; o += 2 * f.b3; }
  f.p5 = o; o += 2 * f.b5;
  f.total = o;
  return f;
}

struct Ws {
  // encoder
  size_t ids, emb, m_enc, p1, x0, bank, pool, pj1, y, hw12, gi_f, gi_b, gh, hst, seq, proj, style_q, style;
  // decoder
  size_t attn_h, h1, c1, h2, c2, ctx, cum, dp1, dp2, dgi, dgh, pq, x, gates, a_hi, a_lo, ah_hi, ah_lo, fsp, pre1, pre2, gic, stopv, step, flags, dmask;
  size_t big_hi, big_lo, big_bytes;
  // outputs / postnet
  size_t mel_all, scores_all, pbank, ppool, ppj1, ppj2, py, phw12, pgi_f, pgi_b, pgh, phst, pout, lin;
  // ragged batches only: int32 characters, caps (decoder steps), done step, frames [B] each, seeds [B] u64
  size_t rows;
  size_t total;  // bytes; every other field is an offset in floats
};

// What a workspace holds: the encoder's scratch, the decoder loop (its state, the encoder rows it reads, its per-step buffers), the
// postnet's scratch.  generate uses all three in one workspace; a stream (mb_tacotron_stream_*) gives each its own, because the
// encoder and the postnet run on their own streams while the decoder loop runs.  Fields of a part left out take no space.
enum WsPart : int { WS_ENC = 1, WS_DEC = 2, WS_POST = 4, WS_ALL = 7 };

Ws ws_layout(const mb_tacotron_config& c, int B, int Tc, int steps, int r, bool ragged = false, int parts = WS_ALL) {
  Ws L{};
  WsLayout W;
  auto in = [&](int part, size_t n) { return (parts & part) ? n : (size_t)0; };
  const size_t Me = (size_t)B * Tc, Mp = (size_t)B * steps;
  const int E = c.encoder_dims, PD = c.postnet_dims, proj_dims = E + c.speaker_embedding_size + c.gst_E;
  L.ids = W.take<float>(in(WS_DEC, Me));  // int32 characters of the rows (streams; generate reads the caller's)
  L.emb = W.take<float>(in(WS_ENC, Me * c.embed_dims));
  L.m_enc = W.take<float>(in(WS_ENC, (2 * Me * E + 3) / 4 + 64));  // uint8 masks
  L.p1 = W.take<float>(in(WS_ENC, Me * E));
  L.x0 = W.take<float>(in(WS_ENC, Me * E));
  L.bank = W.take<float>(in(WS_ENC, Me * c.encoder_K * E));
  L.pool = W.take<float>(in(WS_ENC, Me * c.encoder_K * E));
  L.pj1 = W.take<float>(in(WS_ENC, Me * E));
  L.y = W.take<float>(in(WS_ENC, Me * E));
  L.hw12 = W.take<float>(in(WS_ENC, Me * 2 * E));
  L.gi_f = W.take<float>(in(WS_ENC, Me * 3 * (E / 2)));
  L.gi_b = W.take<float>(in(WS_ENC, Me * 3 * (E / 2)));
  L.gh = W.take<float>(in(WS_ENC | WS_POST, (size_t)2 * B * 3 * (PD / 2)));
  L.hst = W.take<float>(in(WS_ENC | WS_POST, (size_t)2 * B * (PD / 2)));
  L.seq = W.take<float>(in(WS_DEC, Me * proj_dims));
  L.proj = W.take<float>(in(WS_DEC, Me * c.decoder_dims));
  L.style_q = W.take<float>(in(WS_ENC, (size_t)B * c.gst_E));
  L.style = W.take<float>(in(WS_ENC, (size_t)B * c.gst_E));
  L.attn_h = W.take<float>(in(WS_DEC, (size_t)B * c.decoder_dims));
  L.h1 = W.take<float>(in(WS_DEC, (size_t)B * c.lstm_dims));
  L.c1 = W.take<float>(in(WS_DEC, (size_t)B * c.lstm_dims));
  L.h2 = W.take<float>(in(WS_DEC, (size_t)B * c.lstm_dims));
  L.c2 = W.take<float>(in(WS_DEC, (size_t)B * c.lstm_dims));
  L.ctx = W.take<float>(in(WS_DEC, (size_t)B * proj_dims));
  L.cum = W.take<float>(in(WS_DEC, Me));
  L.dp1 = W.take<float>(in(WS_DEC, (size_t)B * 2 * c.decoder_dims));
  L.dp2 = W.take<float>(in(WS_DEC, (size_t)B * 2 * c.decoder_dims));
  L.dgi = W.take<float>(in(WS_DEC, (size_t)B * 3 * c.decoder_dims));
  L.dgh = W.take<float>(in(WS_DEC, (size_t)B * 3 * c.decoder_dims));
  L.pq = W.take<float>(in(WS_DEC, (size_t)B * c.decoder_dims));
  L.x = W.take<float>(in(WS_DEC, (size_t)B * c.lstm_dims));
  L.gates = W.take<float>(in(WS_DEC, (size_t)B * 4 * c.lstm_dims));
  L.a_hi = W.take<float>(tc_skinny_act_bytes(B > 128 ? 128 : B, 2 * c.lstm_dims) / 4);
  L.a_lo = W.take<float>(tc_skinny_act_bytes(B > 128 ? 128 : B, 2 * c.lstm_dims) / 4);
  L.ah_hi = W.take<float>(in(WS_DEC, 2 * tc_skinny_act_bytes(B > 128 ? 128 : B, c.decoder_dims) / 4));  // attention-GRU state tiles, 2 parities
  L.ah_lo = W.take<float>(in(WS_DEC, 2 * tc_skinny_act_bytes(B > 128 ? 128 : B, c.decoder_dims) / 4));
  {
    // operand tiles written by the producing kernels (fused act_split): P1 [ctx | prenet], P2 [ctx | attn_h], P3 / P4 [x | h] of the
    // two LSTMs (two step parities each), P5 [x]; hi and lo of each; zeroed with the attention-GRU tiles at the start of generate()
    const int Bc = B > 128 ? 128 : B;
    const FusedSplit f = fused_split_layout(Bc, proj_dims, c.decoder_dims, c.lstm_dims);
    L.fsp = W.take<float>(in(WS_DEC, f.total / 4));
  }
  // partial GEMM results computed a step early on the side stream: W_hh h of the two LSTMs, W_ih[:, ctx] ctx of the attention GRU
  L.pre1 = W.take<float>(in(WS_DEC, (size_t)B * 4 * c.lstm_dims));
  L.pre2 = W.take<float>(in(WS_DEC, (size_t)B * 4 * c.lstm_dims));
  L.gic = W.take<float>(in(WS_DEC, (size_t)B * 3 * c.decoder_dims));
  L.stopv = W.take<float>(in(WS_DEC, B));
  L.step = W.take<float>(in(WS_DEC, 64));
  const int nst = (steps + r - 1) / r;
  L.flags = W.take<float>(in(WS_DEC, nst));
  L.dmask = W.take<float>(in(WS_DEC, ((size_t)nst * 2 * B * 2 * c.decoder_dims + 3) / 4 + 64));  // PreNet dropout masks of every decoder step
  L.mel_all = W.take<float>(in(WS_DEC, Mp * c.n_mels + (size_t)r * c.n_mels));
  L.scores_all = W.take<float>(in(WS_DEC, (size_t)B * nst * Tc));
  L.pbank = W.take<float>(in(WS_POST, Mp * c.postnet_K * PD));
  L.ppool = W.take<float>(in(WS_POST, Mp * c.postnet_K * PD));
  L.ppj1 = W.take<float>(in(WS_POST, Mp * PD));
  L.ppj2 = W.take<float>(in(WS_POST, Mp * c.n_mels));
  L.py = W.take<float>(in(WS_POST, Mp * PD));
  L.phw12 = W.take<float>(in(WS_POST, Mp * 2 * PD));
  L.pgi_f = W.take<float>(in(WS_POST, Mp * 3 * (PD / 2)));
  L.pgi_b = W.take<float>(in(WS_POST, Mp * 3 * (PD / 2)));
  L.pgh = W.take<float>(in(WS_POST, (size_t)2 * B * 3 * (PD / 2)));
  L.phst = W.take<float>(in(WS_POST, (size_t)2 * B * (PD / 2)));
  L.pout = W.take<float>(in(WS_POST, Mp * PD));
  L.lin = W.take<float>(in(WS_POST, Mp * c.n_mels));
  {  // im2col operand planes of the large-M tensor-core GEMMs: the widest layer is conv_project1 (3 taps x K * ch)
    const size_t enc = in(WS_ENC, tc_big_act_bytes((int)Me, 3, c.encoder_K * E)), post = in(WS_POST, tc_big_act_bytes((int)Mp, 3, c.postnet_K * PD));
    L.big_bytes = enc > post ? enc : post;
    L.big_hi = W.take<float>(L.big_bytes / 4);
    L.big_lo = W.take<float>(L.big_bytes / 4);
  }
  if (ragged) L.rows = W.take<float>(in(WS_DEC, (size_t)6 * B));
  L.total = W.total();
  return L;
}

#define TK(expr)                                                                                          \
  do {                                                                                                    \
    cudaError_t _e = (expr);                                                                              \
    if (_e != cudaSuccess) return fail(MB_ERR_CUDA, "%s: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
    count_launch();                                                                                       \
  } while (0)

GemmArgs gemm1(const float* x, int K, int ld, const float* W, int ldw, const float* bias, int M, int N, float* Y, int ldy,
               int act = ACT_NONE) {
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

struct BigWs {
  float* hi = nullptr;
  float* lo = nullptr;
  size_t bytes = 0;
};

// A large-M GEMM / conv of the CBHG stacks: tensor cores (tc_big_kernel, 3-term fp16 split) when the layer qualifies,
// else the FP32 FFMA kernels.  MB_TACO_CONV_TC=0 disables the tensor-core route.  Ragged batches (lens = valid length of each
// length-T sequence) always take the tensor-core route, whatever M, so a row's arithmetic does not depend on the batch.
int cbhg_gemm(mb_tacotron* h, const std::string& key, const GemmArgs& a, cudaStream_t st, const BigWs& bw, const int* lens = nullptr) {
  static const bool env = [] {
    const char* e = getenv("MB_TACO_CONV_TC");
    return e ? atoi(e) != 0 : true;
  }();
  bool ok = (env || lens) && bw.hi && (a.M >= 512 || lens) && a.N % 4 == 0 && a.nseg >= 1 && a.nseg <= kMaxSeg && !a.mask && !a.step_mode &&
            a.act != ACT_SIGMOID && a.act != ACT_TANH && h->w.has(key + ".bigw") && (a.ldy % 4) == 0 &&
            (!a.res || (a.ldres % 4) == 0);
  const int K = a.seg[0].K;
  for (int s = 1; ok && s < a.nseg; ++s) ok = a.seg[s].K == K;
  if (ok) ok = tc_big_act_bytes(a.M, a.nseg, K) <= bw.bytes && tc_big_weight_bytes(a.N, a.nseg, K) / 4 <= h->w.size(key + ".bigw");
  if (!ok && lens) return fail(MB_ERR_STATE, "%s: no tensor-core route for this layer of a ragged batch", key.c_str());
  if (!ok) {
    TK(launch_gemm(a, st));
    return MB_OK;
  }
  const int KBs = (K + 63) / 64;
  __half* wimg = reinterpret_cast<__half*>(P(h, key + ".bigw"));
  if (!h->big_packed.count(key)) {
    unsigned int* dmax = reinterpret_cast<unsigned int*>(P(h, "scratch.absmax.tcb"));
    MB_CUDA_CHECK(cudaMemsetAsync(dmax, 0, sizeof(unsigned int), st));
    TK(tc_skinny_absmax(a.W, (size_t)a.N * a.ldw, dmax, st));
    unsigned int hmax = 0;
    MB_CUDA_CHECK(cudaMemcpyAsync(&hmax, dmax, sizeof(hmax), cudaMemcpyDeviceToHost, st));
    MB_CUDA_CHECK(cudaStreamSynchronize(st));
    TcBigPack q;
    memset(&q, 0, sizeof(q));
    q.W = a.W;
    q.ldw = a.ldw;
    q.N = a.N;
    q.nseg = a.nseg;
    q.K = K;
    q.KBs = KBs;
    for (int s = 0; s < a.nseg; ++s) {
      q.w_off[s] = a.seg[s].w_off;
      q.w_stride[s] = a.seg[s].w_stride;
    }
    q.scale = tc_weight_scale(hmax);
    h->tc_inv_scale[key + ".bigw"] = 1.f / q.scale;
    TK(launch_pack_big_w(q, wimg, st));
    h->big_packed.insert(key);
  }
  TcIm2col q;
  memset(&q, 0, sizeof(q));
  for (int s = 0; s < a.nseg; ++s) {
    q.x[s] = a.seg[s].x;
    q.ld[s] = a.seg[s].ld;
    q.shift[s] = a.seg[s].shift;
  }
  q.nseg = a.nseg;
  q.K = K;
  q.KBs = KBs;
  q.M = a.M;
  q.T = a.T > 0 ? a.T : 1;
  q.rows_total = (a.M + 127) / 128 * 128;
  q.len = lens;
  TK(launch_im2col_split(q, reinterpret_cast<__half*>(bw.hi), reinterpret_cast<__half*>(bw.lo), st));
  TcBigArgs t;
  memset(&t, 0, sizeof(t));
  t.a_hi = reinterpret_cast<const __half*>(bw.hi);
  t.a_lo = reinterpret_cast<const __half*>(bw.lo);
  t.w = wimg;
  t.bias = a.bias;
  t.KB = a.nseg * KBs;
  t.M = a.M;
  t.N = a.N;
  t.rows_total = q.rows_total;
  t.act = a.act;
  t.inv_scale = h->tc_inv_scale[key + ".bigw"];
  t.bn_scale = a.bn_scale;
  t.bn_shift = a.bn_shift;
  t.res = a.res;
  t.ldres = a.ldres;
  t.y = a.Y;
  t.ldy = a.ldy;
  TK(launch_tc_big(t, st));
  return MB_OK;
}

// CBHG (sublayer/cbhg.py:42-79) on x [B*T][cin] channels-last -> out [B*T][ch] written at out (ld ldout).  Ragged batches
// (lens: sequence b is its first lens[b] of T rows) run every layer on the tensor cores; the convolutions read zeros past a
// sequence's end and the backward GRU starts at its last row from h = 0, so rows past the end never reach rows before it.
int run_cbhg(mb_tacotron* h, const std::string& p, int K, int cin, int ch, int p0, int p1, int nh, const float* x, int B,
             int T, float* bank, float* pool, float* pj1, float* y, float* hw12, float* gi_f, float* gi_b, float* gh,
             float* hst, float* out, int ldout, cudaStream_t st, float* tc_hi = nullptr, float* tc_lo = nullptr,
             size_t tc_bytes = 0, const BigWs& bw = BigWs(), const int* lens = nullptr) {
  const int M = B * T;
#define CG(key, args)                                    \
  do {                                                   \
    int _rc = cbhg_gemm(h, (key), (args), st, bw, lens); \
    if (_rc != MB_OK) return _rc;                        \
  } while (0)
  // convolution bank: k = 1..K, "same" padding k//2 cropped to T, ReLU then BatchNorm
  for (int i = 0; i < K; ++i) {
    const int k = i + 1;
    const std::string n = p + ".conv1d_bank." + std::to_string(i);
    GemmArgs a;
    memset(&a, 0, sizeof(a));
    a.nseg = k;
    for (int tap = 0; tap < k; ++tap) a.seg[tap] = {x, cin, cin, tap - k / 2, tap, k};
    a.W = P(h, n + ".conv.weight");
    a.ldw = cin * k;
    a.M = M;
    a.N = ch;
    a.T = T;
    a.act = ACT_RELU;
    a.bn_scale = P(h, n + ".bn_scale");
    a.bn_shift = P(h, n + ".bn_shift");
    a.Y = bank + (size_t)i * ch;
    a.ldy = K * ch;
    CG(n, a);
  }
  TK(launch_maxpool2(bank, pool, B, T, K * ch, st));
  {
    GemmArgs a;
    memset(&a, 0, sizeof(a));
    a.nseg = 3;
    for (int tap = 0; tap < 3; ++tap) a.seg[tap] = {pool, K * ch, K * ch, tap - 1, tap, 3};
    a.W = P(h, p + ".conv_project1.conv.weight");
    a.ldw = K * ch * 3;
    a.M = M;
    a.N = p0;
    a.T = T;
    a.act = ACT_RELU;
    a.bn_scale = P(h, p + ".conv_project1.bn_scale");
    a.bn_shift = P(h, p + ".conv_project1.bn_shift");
    a.Y = pj1;
    a.ldy = p0;
    CG(p + ".conv_project1", a);
  }
  float* cur = y;  // [M][ch] highway stream
  {
    // conv_project2 (no ReLU) + BN + residual x
    GemmArgs a;
    memset(&a, 0, sizeof(a));
    a.nseg = 3;
    for (int tap = 0; tap < 3; ++tap) a.seg[tap] = {pj1, p0, p0, tap - 1, tap, 3};
    a.W = P(h, p + ".conv_project2.conv.weight");
    a.ldw = p0 * 3;
    a.M = M;
    a.N = p1;
    a.T = T;
    a.act = ACT_NONE;
    a.bn_scale = P(h, p + ".conv_project2.bn_scale");
    a.bn_shift = P(h, p + ".conv_project2.bn_shift");
    a.res = x;
    a.ldres = cin;
    if (p1 != ch) {
      a.Y = hw12;  // scratch: [M][p1] before the pre_highway projection
      a.ldy = p1;
      CG(p + ".conv_project2", a);
      GemmArgs b = gemm1(hw12, p1, p1, P(h, p + ".pre_highway.weight"), p1, nullptr, M, ch, cur, ch);
      CG(p + ".pre_highway", b);
    } else {
      a.Y = cur;
      a.ldy = ch;
      CG(p + ".conv_project2", a);
    }
  }
  for (int i = 0; i < nh; ++i) {
    const std::string q = p + ".highways." + std::to_string(i);
    GemmArgs a = gemm1(cur, ch, ch, P(h, q + ".W12"), ch, P(h, q + ".b12"), M, 2 * ch, hw12, 2 * ch);
    CG(q, a);
    TK(launch_highway(hw12, cur, M, ch, st));
  }
  // bidirectional GRU: input projections for all t, then the two recurrences
  const int H = ch / 2;
  {
    GemmArgs a = gemm1(cur, ch, ch, P(h, p + ".rnn.weight_ih_l0"), ch, P(h, p + ".rnn.bias_ih_l0"), M, 3 * H, gi_f, 3 * H);
    CG(p + ".rnn.ih", a);
    GemmArgs b = gemm1(cur, ch, ch, P(h, p + ".rnn.weight_ih_l0_reverse"), ch, P(h, p + ".rnn.bias_ih_l0_reverse"), M, 3 * H,
                       gi_b, 3 * H);
    CG(p + ".rnn.ih_reverse", b);
  }
  const size_t tile_bytes = tc_skinny_act_bytes(B, H);
  if (tc_hi && tc_lo && B <= 128 && H % 64 == 0 && 4 * tile_bytes <= tc_bytes) {
    // recurrences on the tensor cores: one launch per time step covers both directions; the epilogue applies
    // the GRU cell and writes h_t straight into the next step's operand tiles (ping-pong)
    MB_CUDA_CHECK(cudaMemsetAsync(hst, 0, sizeof(float) * 2 * B * H, st));
    MB_CUDA_CHECK(cudaMemsetAsync(tc_hi, 0, 4 * tile_bytes, st));
    MB_CUDA_CHECK(cudaMemsetAsync(tc_lo, 0, 4 * tile_bytes, st));
    auto tile = [&](float* base, int dir, int par) {
      return reinterpret_cast<__half*>(reinterpret_cast<char*>(base) + (size_t)(dir * 2 + par) * tile_bytes);
    };
    TcGruArgs g;
    memset(&g, 0, sizeof(g));
    g.ldgi = T * 3 * H;
    g.ldout = T * ldout;
    g.KB = H / 64;
    g.M = B;
    g.H = H;
    g.ndir = 2;
    g.len1 = lens;
    const char* sfx[2] = {"", "_reverse"};
    for (int d = 0; d < 2; ++d) {
      g.w[d] = reinterpret_cast<const __half*>(P(h, p + ".rnn.hh" + sfx[d] + ".tcw"));
      g.bias[d] = P(h, p + ".rnn.hh" + sfx[d] + ".tcb");
      g.inv_scale[d] = h->tc_inv_scale[p + ".rnn.hh" + sfx[d]];
      g.h[d] = hst + (size_t)d * B * H;
    }
    for (int s = 0; s < T; ++s) {
      const int par = s & 1, t_b = T - 1 - s;
      for (int d = 0; d < 2; ++d) {
        g.a_hi[d] = tile(tc_hi, d, par);
        g.a_lo[d] = tile(tc_lo, d, par);
        g.nxt_hi[d] = tile(tc_hi, d, par ^ 1);
        g.nxt_lo[d] = tile(tc_lo, d, par ^ 1);
      }
      g.gi[0] = gi_f + (size_t)s * 3 * H;
      g.gi[1] = gi_b + (size_t)t_b * 3 * H;
      g.out[0] = out + (size_t)s * ldout;
      g.out[1] = out + (size_t)t_b * ldout + H;
      g.t1 = t_b;
      TK(launch_tc_gru(g, st));
    }
    return MB_OK;
  }
  if (lens) return fail(MB_ERR_STATE, "%s: no tensor-core GRU route for a ragged batch", p.c_str());
  MB_CUDA_CHECK(cudaMemsetAsync(hst, 0, sizeof(float) * 2 * B * H, st));
  float* hf = hst;
  float* hb = hst + (size_t)B * H;
  float* ghf = gh;
  float* ghb = gh + (size_t)B * 3 * H;
  for (int s = 0; s < T; ++s) {
    {  // forward direction, time s
      GemmArgs a = gemm1(hf, H, H, P(h, p + ".rnn.weight_hh_l0"), H, P(h, p + ".rnn.bias_hh_l0"), B, 3 * H, ghf, 3 * H);
      TK(launch_gemm(a, st));
      TK(launch_gru_cell(gi_f + (size_t)s * 3 * H, T * 3 * H, ghf, hf, H, out + (size_t)s * ldout, T * ldout, B, H, st));
    }
    {  // reverse direction, time T-1-s
      const int t = T - 1 - s;
      GemmArgs a = gemm1(hb, H, H, P(h, p + ".rnn.weight_hh_l0_reverse"), H, P(h, p + ".rnn.bias_hh_l0_reverse"), B, 3 * H,
                         ghb, 3 * H);
      TK(launch_gemm(a, st));
      TK(launch_gru_cell(gi_b + (size_t)t * 3 * H, T * 3 * H, ghb, hb, H, out + (size_t)t * ldout + H, T * ldout, B, H, st));
    }
  }
  return MB_OK;
}

// absmax -> power-of-two scale (tc_weight_scale) -> hi/lo tile images "<name>.tcw" + tile-order bias "<name>.tcb".  Synchronises the stream.
int tc_prepare(mb_tacotron* h, const std::string& name, const float* w0, int K0, const float* w1, int K1, const float* b0,
               const float* b1, int N, int lstm_H, cudaStream_t st) {
  unsigned int* dmax = reinterpret_cast<unsigned int*>(P(h, "scratch.absmax.tcb"));
  MB_CUDA_CHECK(cudaMemsetAsync(dmax, 0, sizeof(unsigned int), st));
  TK(tc_skinny_absmax(w0, (size_t)N * K0, dmax, st));
  if (w1) TK(tc_skinny_absmax(w1, (size_t)N * K1, dmax, st));
  unsigned int hmax = 0;
  MB_CUDA_CHECK(cudaMemcpyAsync(&hmax, dmax, sizeof(hmax), cudaMemcpyDeviceToHost, st));
  MB_CUDA_CHECK(cudaStreamSynchronize(st));
  const float scale = tc_weight_scale(hmax);
  h->tc_inv_scale[name] = 1.f / scale;
  TK(tc_skinny_pack(w0, K0, w1, K1, b0, b1, N, lstm_H, scale, reinterpret_cast<__half*>(P(h, name + ".tcw")),
                    P(h, name + ".tcb"), st));
  return MB_OK;
}

}  // namespace

extern "C" {

int mb_tacotron_create(const mb_tacotron_config* cfg, mb_tacotron** out) {
  if (!cfg || !out) return fail(MB_ERR_INVALID, "mb_tacotron_create: null argument");
  const mb_tacotron_config& c = *cfg;
  if (c.decoder_dims != ATT_D || c.encoder_dims % 2 || c.postnet_dims % 2 || c.gst_heads > 8 || c.gst_tokens > 16 ||
      c.encoder_K > kMaxSeg || c.postnet_K > kMaxSeg)
    return fail(MB_ERR_INVALID, "mb_tacotron_create: unsupported hyper-parameters");
  mb_tacotron* h = new mb_tacotron();
  h->cfg = c;
  const int E = c.encoder_dims, D = c.decoder_dims, proj_dims = E + c.speaker_embedding_size + c.gst_E;
  const int dk = c.gst_E / c.gst_heads, L = c.lstm_dims;
  WeightTable& w = h->w;
  w.add_derived("scratch.absmax.tcb", 64);  // device scratch of the weight-image packers (no cudaMalloc after create)
  w.add("encoder.embedding.weight", {c.num_chars, c.embed_dims});
  w.add("encoder.pre_net.fc1.weight", {E, c.embed_dims});
  w.add("encoder.pre_net.fc1.bias", {E});
  w.add("encoder.pre_net.fc2.weight", {E, E});
  w.add("encoder.pre_net.fc2.bias", {E});
  cbhg_slots(w, "encoder.cbhg", c.encoder_K, E, E, E, E, c.num_highways);
  w.add("encoder_proj.weight", {D, proj_dims});
  w.add("gst.const_enc", {c.gst_E / 2});  // ReferenceEncoder(zeros): input independent, folded by the host
  w.add("gst.stl.embed", {c.gst_tokens, dk});
  w.add("gst.stl.attention.W_query.weight", {c.gst_E, c.gst_E / 2 + c.speaker_embedding_size});
  w.add("gst.stl.attention.W_key.weight", {c.gst_E, dk});
  w.add("gst.stl.attention.W_value.weight", {c.gst_E, dk});
  w.add_derived("gst.tanh_embed", (size_t)c.gst_tokens * dk);
  w.add_derived("gst.keys", (size_t)c.gst_tokens * c.gst_E);
  w.add_derived("gst.values", (size_t)c.gst_tokens * c.gst_E);
  w.add("decoder.prenet.fc1.weight", {2 * D, c.n_mels});
  w.add("decoder.prenet.fc1.bias", {2 * D});
  w.add("decoder.prenet.fc2.weight", {2 * D, 2 * D});
  w.add("decoder.prenet.fc2.bias", {2 * D});
  w.add("decoder.attn_net.conv.weight", {ATT_F, 1, ATT_K});
  w.add("decoder.attn_net.conv.bias", {ATT_F});
  w.add("decoder.attn_net.L.weight", {ATT_D, ATT_F});
  w.add("decoder.attn_net.W.weight", {ATT_D, ATT_D});
  w.add("decoder.attn_net.W.bias", {ATT_D});
  w.add("decoder.attn_net.v.weight", {1, ATT_D});
  w.add("decoder.attn_rnn.weight_ih", {3 * D, proj_dims + 2 * D});
  w.add("decoder.attn_rnn.weight_hh", {3 * D, D});
  w.add("decoder.attn_rnn.bias_ih", {3 * D});
  w.add("decoder.attn_rnn.bias_hh", {3 * D});
  w.add_derived("decoder.attn_rnn.ih.tcw", tc_skinny_weight_bytes(3 * D, proj_dims + 2 * D) / 4);  // tensor-core images
  w.add_derived("decoder.attn_rnn.ih.tcb", 3 * D);
  w.add_derived("decoder.attn_rnn.hh.tcw", tc_gated_weight_bytes(D, D) / 4);
  w.add_derived("decoder.attn_rnn.hh.tcb", 4 * D);
  w.add("decoder.rnn_input.weight", {L, proj_dims + D});
  w.add("decoder.rnn_input.bias", {L});
  for (const char* n : {"decoder.res_rnn1", "decoder.res_rnn2"}) {
    w.add(std::string(n) + ".weight_ih", {4 * L, L});
    w.add(std::string(n) + ".weight_hh", {4 * L, L});
    w.add(std::string(n) + ".bias_ih", {4 * L});
    w.add(std::string(n) + ".bias_hh", {4 * L});
    w.add_derived(std::string(n) + ".bias_sum", 4 * L);                                   // b_hh + b_ih
    w.add_derived(std::string(n) + ".tcw", tc_skinny_weight_bytes(4 * L, 2 * L) / 4);  // hi/lo tiles
    w.add_derived(std::string(n) + ".tcb", 4 * L);                                        // tile-order bias
  }
  w.add("decoder.mel_proj.weight", {c.n_mels * c.max_r, L});
  w.add_derived("decoder.mel_proj.packed", (size_t)c.n_mels * c.max_r * L);                     // for the current r
  w.add_derived("decoder.mel_proj.tcw", tc_skinny_weight_bytes(c.n_mels * c.max_r, L) / 4);  // (current r)
  w.add_derived("decoder.mel_proj.tcb", (size_t)c.n_mels * c.max_r + 32);
  w.add_derived("decoder.rnn_input.tcw", tc_skinny_weight_bytes(L, proj_dims + D) / 4);
  w.add_derived("decoder.rnn_input.tcb", L);
  w.add("decoder.stop_proj.weight", {1, proj_dims + L});
  w.add("decoder.stop_proj.bias", {1});
  cbhg_slots(w, "postnet", c.postnet_K, c.n_mels, c.postnet_dims, c.postnet_dims, c.n_mels, c.num_highways);
  w.add("post_proj.weight", {c.n_mels, c.postnet_dims});
  w.add_derived("post_proj.bigw", tc_big_weight_bytes(c.n_mels, 1, c.postnet_dims) / 4);
  *out = h;
  return MB_OK;
}

void mb_tacotron_destroy(mb_tacotron* h) {
  if (!h) return;
  if (h->ev_in) cudaEventDestroy(h->ev_in);
  if (h->ev_out) cudaEventDestroy(h->ev_out);
  if (h->own_stream) cudaStreamDestroy(h->own_stream);
  for (cudaEvent_t e : h->ev_side)
    if (e) cudaEventDestroy(e);
  if (h->side_stream) cudaStreamDestroy(h->side_stream);
  delete h;
}

size_t mb_tacotron_arena_bytes(const mb_tacotron* h) { return h ? h->w.floats() * sizeof(float) : 0; }

int mb_tacotron_set_arena(mb_tacotron* h, void* arena, size_t bytes) {
  if (int rc = check_arena("mb_tacotron_set_arena", h, arena, bytes, mb_tacotron_arena_bytes(h), 256)) return rc;
  h->w.attach((float*)arena);
  h->finalized = false;
  // a new arena holds none of the derived images: forget every lazily packed tensor-core image and its scale
  h->big_packed.clear();
  h->tc_inv_scale.clear();
  h->packed_r = 0;
  return MB_OK;
}

int mb_tacotron_set_weight(mb_tacotron* h, const char* name, const float* w, const int64_t* dims, int32_t ndim,
                           void* stream) {
  if (!h) return fail(MB_ERR_INVALID, "mb_tacotron_set_weight: null argument");
  if (int rc = h->w.set("mb_tacotron_set_weight", name, w, dims, ndim, stream)) return rc;
  h->finalized = false;
  h->big_packed.clear();  // images packed from the previous weights are stale
  h->packed_r = 0;
  return MB_OK;
}

int mb_tacotron_finalize(mb_tacotron* h, void* stream) {
  if (!h) return fail(MB_ERR_INVALID, "mb_tacotron_finalize: null handle");
  cudaStream_t st = (cudaStream_t)stream;
  h->big_packed.clear();  // re-packed from the current weights at first use
  const mb_tacotron_config& c = h->cfg;
  if (int rc = h->w.check_all_set("mb_tacotron_finalize")) return rc;
  // the BatchNorm'd convolutions and the highways of both CBHG stacks
  std::vector<std::string> bnconvs, highways;
  for (const auto& cb : {std::make_pair(std::string("encoder.cbhg"), c.encoder_K), std::make_pair(std::string("postnet"), c.postnet_K)}) {
    for (int i = 0; i < cb.second; ++i) bnconvs.push_back(cb.first + ".conv1d_bank." + std::to_string(i));
    bnconvs.push_back(cb.first + ".conv_project1");
    bnconvs.push_back(cb.first + ".conv_project2");
    for (int i = 0; i < c.num_highways; ++i) highways.push_back(cb.first + ".highways." + std::to_string(i));
  }
  // fold eval BatchNorm into scale/shift
  for (const std::string& base : bnconvs) {
    const int co = (int)h->w.size(base + ".bnorm.weight");
    bn_fold_kernel<<<(co + 255) / 256, 256, 0, st>>>(P(h, base + ".bnorm.weight"), P(h, base + ".bnorm.bias"),
                                                     P(h, base + ".bnorm.running_mean"), P(h, base + ".bnorm.running_var"),
                                                     P(h, base + ".bn_scale"), P(h, base + ".bn_shift"), co);
    MB_LAUNCH_CHECK("bn_fold_kernel");
  }
  // stacked highway weights [W1; W2]
  for (const std::string& base : highways) {
    const size_t nn = h->w.size(base + ".W1.weight"), ch = h->w.size(base + ".W1.bias");
    MB_CUDA_CHECK(cudaMemcpyAsync(P(h, base + ".W12"), P(h, base + ".W1.weight"), nn * 4, cudaMemcpyDeviceToDevice, st));
    MB_CUDA_CHECK(cudaMemcpyAsync(P(h, base + ".W12") + nn, P(h, base + ".W2.weight"), nn * 4, cudaMemcpyDeviceToDevice, st));
    MB_CUDA_CHECK(cudaMemcpyAsync(P(h, base + ".b12"), P(h, base + ".W1.bias"), ch * 4, cudaMemcpyDeviceToDevice, st));
    MB_CUDA_CHECK(cudaMemcpyAsync(P(h, base + ".b12") + ch, P(h, base + ".W2.bias"), ch * 4, cudaMemcpyDeviceToDevice, st));
  }
  // GST constants: keys/values of the tanh'd tokens
  {
    const int dk = c.gst_E / c.gst_heads, nt = c.gst_tokens;
    tanh_kernel<<<(nt * dk + 255) / 256, 256, 0, st>>>(P(h, "gst.stl.embed"), P(h, "gst.tanh_embed"), nt * dk);
    MB_LAUNCH_CHECK("tanh_kernel");
    GemmArgs a = gemm1(P(h, "gst.tanh_embed"), dk, dk, P(h, "gst.stl.attention.W_key.weight"), dk, nullptr, nt, c.gst_E,
                       P(h, "gst.keys"), c.gst_E);
    TK(launch_gemm(a, st));
    GemmArgs b = gemm1(P(h, "gst.tanh_embed"), dk, dk, P(h, "gst.stl.attention.W_value.weight"), dk, nullptr, nt, c.gst_E,
                       P(h, "gst.values"), c.gst_E);
    TK(launch_gemm(b, st));
  }
  // tensor-core images: the two residual LSTMs ([W_ih | W_hh], gate-interleaved) and rnn_input
  {
    const char* names[2] = {"decoder.res_rnn1", "decoder.res_rnn2"};
    for (int l = 0; l < 2; ++l) {
      const std::string n = names[l];
      int rc = tc_prepare(h, n, P(h, n + ".weight_ih"), c.lstm_dims, P(h, n + ".weight_hh"), c.lstm_dims, P(h, n + ".bias_ih"),
                          P(h, n + ".bias_hh"), 4 * c.lstm_dims, c.lstm_dims, st);
      if (rc != MB_OK) return rc;
    }
    for (const std::string p : {std::string("encoder.cbhg"), std::string("postnet")}) {
      const int H = (p == "postnet" ? c.postnet_dims : c.encoder_dims) / 2;
      for (const char* sfx : {"", "_reverse"}) {
        int rc = tc_prepare(h, p + ".rnn.hh" + sfx, P(h, p + ".rnn.weight_hh_l0" + sfx), H, nullptr, 0,
                            P(h, p + ".rnn.bias_hh_l0" + sfx), nullptr, 3 * H, H, st);
        if (rc != MB_OK) return rc;
      }
    }
    const int pd = c.encoder_dims + c.speaker_embedding_size + c.gst_E;
    {
      const int Dd = c.decoder_dims;
      int rc = tc_prepare(h, "decoder.attn_rnn.ih", P(h, "decoder.attn_rnn.weight_ih"), pd + 2 * Dd, nullptr, 0,
                          P(h, "decoder.attn_rnn.bias_ih"), nullptr, 3 * Dd, 0, st);
      if (rc != MB_OK) return rc;
      rc = tc_prepare(h, "decoder.attn_rnn.hh", P(h, "decoder.attn_rnn.weight_hh"), Dd, nullptr, 0,
                      P(h, "decoder.attn_rnn.bias_hh"), nullptr, 3 * Dd, Dd, st);
      if (rc != MB_OK) return rc;
    }
    int rc = tc_prepare(h, "decoder.rnn_input", P(h, "decoder.rnn_input.weight"), pd + c.decoder_dims, nullptr, 0,
                        P(h, "decoder.rnn_input.bias"), nullptr, c.lstm_dims, 0, st);
    if (rc != MB_OK) return rc;
  }
  h->packed_r = 0;
  h->finalized = true;
  return MB_OK;
}

size_t mb_tacotron_workspace_bytes(const mb_tacotron* h, int32_t B, int32_t Tc, int32_t steps, int32_t r) {
  if (!h || B <= 0 || Tc <= 0 || steps <= 0 || r <= 0) return 0;
  const int max_chars = lsa_max_chars();  // 0: no device to ask; mb_tacotron_generate still refuses
  if (max_chars > 0 && Tc > max_chars) return 0;
  const int nst = (steps + r - 1) / r;
  return ws_layout(h->cfg, B, Tc, nst * r, r).total;
}

}  // extern "C"

namespace {

// per-row description of a ragged batch (mb_tacotron_generate_ragged), host arrays of B entries
struct RaggedRows {
  const int32_t* chars;   // characters of each row (<= Tc)
  const int32_t* steps;   // frame cap of each row: ceil(steps / r) decoder steps
  const uint64_t* seeds;  // dropout seed of each utterance
  int32_t* frames;        // out: frames of each row
};

// the handle's internal streams and events (created at the first decoder loop)
int ensure_streams(mb_tacotron* h) {
  if (!h->own_stream) {
    MB_CUDA_CHECK(cudaStreamCreateWithFlags(&h->own_stream, cudaStreamNonBlocking));
    MB_CUDA_CHECK(cudaEventCreateWithFlags(&h->ev_in, cudaEventDisableTiming));
    MB_CUDA_CHECK(cudaEventCreateWithFlags(&h->ev_out, cudaEventDisableTiming));
    MB_CUDA_CHECK(cudaStreamCreateWithFlags(&h->side_stream, cudaStreamNonBlocking));
    for (cudaEvent_t& e : h->ev_side) MB_CUDA_CHECK(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
  }
  return MB_OK;
}

// the mel projection's packed rows and tensor-core image for reduction factor r (re-packed when r changes)
int prepare_mel_proj(mb_tacotron* h, int r, cudaStream_t st) {
  const mb_tacotron_config& c = h->cfg;
  const int NM = c.n_mels, LD = c.lstm_dims;
  if (h->packed_r == r) return MB_OK;
  const size_t n = (size_t)r * NM * LD;
  pack_melproj_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(P(h, "decoder.mel_proj.weight"), P(h, "decoder.mel_proj.packed"),
                                                                   NM, c.max_r, r, LD);
  MB_LAUNCH_CHECK("pack_melproj_kernel");
  int rc = tc_prepare(h, "decoder.mel_proj", P(h, "decoder.mel_proj.packed"), LD, nullptr, 0, nullptr, nullptr, r * NM, 0, st);
  if (rc != MB_OK) return rc;
  h->packed_r = r;
  return MB_OK;
}

// the encoder (embedding, PreNet, CBHG), speaker and style columns and encoder_proj of B rows of Tc characters: seq [B][Tc][proj_dims]
// and proj [B][Tc][decoder_dims].  Ragged rows (d_lens) take the routes whose arithmetic per row does not depend on the batch.
int run_encoder(mb_tacotron* h, const Ws& L, float* ws, const int32_t* chars, const float* spk, int B, int Tc, int style_idx,
                const uint8_t* enc_masks, uint64_t seed, bool ragged, const int* d_lens, const uint64_t* d_seeds, bool use_tc,
                float* seq, float* proj, cudaStream_t st) {
  const mb_tacotron_config& c = h->cfg;
  const int E = c.encoder_dims, D = c.decoder_dims, LD = c.lstm_dims, SE = c.speaker_embedding_size, proj_dims = E + SE + c.gst_E;
  const int Me = B * Tc;
  BigWs bw;
  bw.hi = ws + L.big_hi;
  bw.lo = ws + L.big_lo;
  bw.bytes = L.big_bytes;
  TK(launch_embedding(chars, P(h, "encoder.embedding.weight"), ws + L.emb, Me, c.embed_dims, st));
  uint8_t* em = reinterpret_cast<uint8_t*>(ws + L.m_enc);
  const size_t enc_mask_n = (size_t)Me * E;
  if (enc_masks) {
    MB_CUDA_CHECK(cudaMemcpyAsync(em, enc_masks, 2 * enc_mask_n, cudaMemcpyDeviceToDevice, st));
  } else if (ragged) {
    fill_masks_seeded_kernel<<<(unsigned)((2 * enc_mask_n + 255) / 256), 256, 0, st>>>(em, B, Tc, E, d_seeds, 0);
    MB_LAUNCH_CHECK("fill_masks_seeded_kernel");
  } else {
    fill_masks_kernel<<<(unsigned)((2 * enc_mask_n + 255) / 256), 256, 0, st>>>(em, 2 * enc_mask_n, seed, 0xffffffffu);
    MB_LAUNCH_CHECK("fill_masks_kernel");
  }
  {
    GemmArgs a = gemm1(ws + L.emb, c.embed_dims, c.embed_dims, P(h, "encoder.pre_net.fc1.weight"), c.embed_dims,
                       P(h, "encoder.pre_net.fc1.bias"), Me, E, ws + L.p1, E, ACT_RELU);
    a.mask = em;
    a.fma_chain = ragged;
    TK(launch_gemm(a, st));
    GemmArgs b = gemm1(ws + L.p1, E, E, P(h, "encoder.pre_net.fc2.weight"), E, P(h, "encoder.pre_net.fc2.bias"), Me, E,
                       ws + L.x0, E, ACT_RELU);
    b.mask = em + enc_mask_n;
    b.fma_chain = ragged;
    TK(launch_gemm(b, st));
  }
  int rc = run_cbhg(h, "encoder.cbhg", c.encoder_K, E, E, E, E, c.num_highways, ws + L.x0, B, Tc, ws + L.bank, ws + L.pool,
                    ws + L.pj1, ws + L.y, ws + L.hw12, ws + L.gi_f, ws + L.gi_b, ws + L.gh, ws + L.hst, seq, proj_dims, st,
                    use_tc ? ws + L.a_hi : nullptr, use_tc ? ws + L.a_lo : nullptr, tc_skinny_act_bytes(B > 128 ? 128 : B, 2 * LD), bw,
                    d_lens);
  if (rc != MB_OK) return rc;
  // speaker embedding per char (tacotron.py:236), style embedding (tacotron.py:238-253)
  TK(launch_copy_cols(spk, SE, Tc, seq, proj_dims, E, Me, SE, st));
  if (style_idx >= 0 && style_idx < c.gst_tokens) {
    // zero query over a single token: softmax over one key == 1  ->  style = W_value tanh(embed[idx])
    TK(launch_copy_cols(P(h, "gst.values") + (size_t)style_idx * c.gst_E, c.gst_E, Me, seq, proj_dims, E + SE, Me, c.gst_E, st));
  } else {
    GemmArgs a;
    memset(&a, 0, sizeof(a));
    a.nseg = 2;
    a.seg[0] = {P(h, "gst.const_enc"), c.gst_E / 2, 0, 0, 0, 1};  // ld 0: the same row for every batch element
    a.seg[1] = {spk, SE, SE, 0, c.gst_E / 2, 1};
    a.W = P(h, "gst.stl.attention.W_query.weight");
    a.ldw = c.gst_E / 2 + SE;
    a.M = B;
    a.N = c.gst_E;
    a.T = 1;
    a.Y = ws + L.style_q;
    a.ldy = c.gst_E;
    a.fma_chain = ragged;
    TK(launch_gemm(a, st));
    const int dk = c.gst_E / c.gst_heads;
    gst_attention_kernel<<<B, 256, 0, st>>>(ws + L.style_q, P(h, "gst.keys"), P(h, "gst.values"), c.gst_tokens,
                                            ws + L.style, c.gst_E, c.gst_heads, 1.0f / sqrtf((float)dk));
    MB_LAUNCH_CHECK("gst_attention_kernel");
    TK(launch_copy_cols(ws + L.style, c.gst_E, Tc, seq, proj_dims, E + SE, Me, c.gst_E, st));
  }
  {
    GemmArgs a = gemm1(seq, proj_dims, proj_dims, P(h, "encoder_proj.weight"), proj_dims, nullptr, Me, D, proj, D);
    a.fma_chain = ragged;
    TK(launch_gemm(a, st));
  }

  return MB_OK;
}

// the postnet CBHG and post_proj over B rows of `frames` mel frames (melc [B][frames][n_mels]; ragged rows: d_flen) -> ws + L.lin
int run_postnet(mb_tacotron* h, const Ws& L, float* ws, const float* melc, int B, int frames, const int* d_flen, bool use_tc,
                cudaStream_t st) {
  const mb_tacotron_config& c = h->cfg;
  const int PD = c.postnet_dims, NM = c.n_mels, LD = c.lstm_dims;
  BigWs bw;
  bw.hi = ws + L.big_hi;
  bw.lo = ws + L.big_lo;
  bw.bytes = L.big_bytes;
  int rc = run_cbhg(h, "postnet", c.postnet_K, NM, PD, PD, NM, c.num_highways, melc, B, frames, ws + L.pbank, ws + L.ppool,
                ws + L.ppj1, ws + L.py, ws + L.phw12, ws + L.pgi_f, ws + L.pgi_b, ws + L.pgh, ws + L.phst, ws + L.pout, PD, st,
                use_tc ? ws + L.a_hi : nullptr, use_tc ? ws + L.a_lo : nullptr, tc_skinny_act_bytes(B > 128 ? 128 : B, 2 * LD), bw,
                d_flen);
  if (rc != MB_OK) return rc;
  {
    GemmArgs a = gemm1(ws + L.pout, PD, PD, P(h, "post_proj.weight"), PD, nullptr, B * frames, NM, ws + L.lin, NM);
    int rc2 = cbhg_gemm(h, "post_proj", a, st, bw, d_flen);
    if (rc2 != MB_OK) return rc2;
  }
  return MB_OK;
}

// One decoder step of B rows (tacotron.py:71-138), launched on st (+ the side stream sd of the step DAG).  The step index is
// (sp ? *sp : 0) + sj, resolved ON THE DEVICE by the few kernels that need it (PreNet input frame and dropout masks, alignment row,
// mel output frames, stop rule), so the same launch sequence can be captured once into a CUDA graph and replayed for every group
// of steps.  With a per-row step origin (d_start) each row reads and writes its per-step buffers (nst steps: alignment rows, mel
// frames, masks) at its own step modulo nst.
// Fused operand split (MB_TACO_SPLIT_FUSED, default 1): the five act_split launches of a step disappear - every kernel that
// produces an input of a tensor-core GEMM (PreNet, context, attention GRU, rnn_input, the two LSTM cells) writes the fp16 hi / lo
// operand chunks itself, into per-consumer tiles (the LSTM tiles ping-pong on the step parity: a cell writes h' for the next step
// while other CTAs of the same launch still read this step's tiles).
// Step DAG (MB_TACO_DAG, default 1, needs the fused split): a step's critical path is a chain of ~10 latency-bound kernels.  Three
// of its GEMMs have a K segment that is known a whole step early - W_hh h_{t-1} of both LSTM cells and the context half of the
// attention GRU's input projection - so those halves run on a side stream (TCS_PLAIN over a k-block range, result added to the
// accumulator of the short main-path GEMM), and so does the stop projection / stop rule, which nothing in the next step needs.
// The side stream forks from / joins the main one with events, inside the captured graph as well.
struct DecoderLoop {
  mb_tacotron* h;
  Ws L;
  float* ws;
  int B, Tc, r, nst, steps_alloc;  // nst: steps the per-step buffers hold (steps_alloc = nst * r frames per row)
  const int32_t* chars;
  float* seq;
  float* mel_all;
  const uint8_t* dec_masks;  // injected masks [nst][2][B][2D], else dm (drawn before the loop / written at admission)
  uint8_t* dm;
  float min_stop_token;
  int* flags;                // [nst] stop flags of the padded / ragged loop, or null (per-row step origin)
  const int* d_lens;         // ragged rows: characters, caps, done steps; or null
  const int* d_caps;
  int* d_done;
  const int* d_start;        // per-row step origin, or null
  bool use_tc;
  // derived by init()
  int NM, D, LD, proj_dims, f_rows_pad;
  size_t dmask_n, lsa_smem;
  bool prenet_fused_env, fsplit, dag;
  FusedSplit fs;
  char* fbase;
  cudaStream_t st, sd;
  bool have_gic = false, have_p1 = false, have_p2 = false, have_stop = false, side_open = false;

  void init(cudaStream_t main_stream) {
    const mb_tacotron_config& c = h->cfg;
    NM = c.n_mels;
    D = c.decoder_dims;
    LD = c.lstm_dims;
    proj_dims = c.encoder_dims + c.speaker_embedding_size + c.gst_E;
    dmask_n = (size_t)B * 2 * D;
    lsa_smem = lsa_step_smem_bytes(Tc);
    static const bool split_fused_env = [] {
      const char* e = getenv("MB_TACO_SPLIT_FUSED");
      return e ? atoi(e) != 0 : true;
    }();
    static const bool prenet_env = [] {
      const char* e = getenv("MB_TACO_PRENET_FUSED");
      return e ? atoi(e) != 0 : true;
    }();
    prenet_fused_env = prenet_env;
    fsplit = split_fused_env && prenet_fused_env && use_tc && D % 64 == 0 && proj_dims % 256 == 0 && LD % 64 == 0 &&
             (r * NM) % 4 == 0 && NM <= 128 && 2 * D <= 256 && B <= 128;
    fs = fused_split_layout(B > 128 ? 128 : B, proj_dims, D, LD);
    fbase = reinterpret_cast<char*>(ws + L.fsp);
    f_rows_pad = B <= 64 ? 64 : 128;
    static const bool dag_env = [] {
      const char* e = getenv("MB_TACO_DAG");
      return e ? atoi(e) != 0 : true;
    }();
    dag = dag_env && fsplit && proj_dims % 64 == 0;
    st = main_stream;
    sd = h->side_stream;
  }
  __half* fhi(size_t off) const { return reinterpret_cast<__half*>(fbase + off); }
  // fork: side stream waits for everything enqueued on the main stream so far
  int side_after_main(cudaEvent_t ev) {
    MB_CUDA_CHECK(cudaEventRecord(ev, st));
    MB_CUDA_CHECK(cudaStreamWaitEvent(sd, ev, 0));
    side_open = true;
    return MB_OK;
  }
  int main_after_side(cudaEvent_t ev) {
    MB_CUDA_CHECK(cudaEventRecord(ev, sd));
    MB_CUDA_CHECK(cudaStreamWaitEvent(st, ev, 0));
    return MB_OK;
  }
  // join everything outstanding on the side stream (end of a captured group / of a directly launched step)
  int join_side() {
    if (side_open) {
      int rcj = main_after_side(h->ev_side[7]);
      if (rcj != MB_OK) return rcj;
    }
    side_open = have_gic = have_p1 = have_p2 = have_stop = false;
    return MB_OK;
  }
  int emit_step(const int* sp, int sj);
};

int DecoderLoop::emit_step(const int* sp, int sj) {
  // PreNet on the last frame of the previous step (go frame = zeros)
  const uint8_t* m1;
  const uint8_t* m2;
  long long mstep = 0;
  if (dec_masks) {
    m1 = dec_masks;
    m2 = m1 + dmask_n;
    mstep = (long long)(2 * dmask_n);
  } else {  // generated for all steps before the loop (fill_masks_steps_kernel)
    m1 = dm;
    m2 = dm + dmask_n;
    mstep = (long long)(2 * dmask_n);
  }
  const bool prenet_fused = prenet_fused_env;  // A/B switch MB_TACO_PRENET_FUSED: 0 = two skinny GEMM launches (round 1)
  const int par = sj & 1;  // graph groups start at even steps, so the parity of (base + sj) is that of sj
  if (prenet_fused && NM <= 128 && 2 * D <= 256) {
    // both PreNet layers in one launch; frame (step * r - 1) of every utterance, step 0 = the all-zero go frame
    PrenetArgs pa;
    memset(&pa, 0, sizeof(pa));
    pa.x = mel_all - NM;
    pa.x_ld = (long long)steps_alloc * NM;
    pa.x_step = (long long)r * NM;
    pa.x_first = mel_all + (size_t)B * steps_alloc * NM;
    pa.W1 = P(h, "decoder.prenet.fc1.weight");
    pa.b1 = P(h, "decoder.prenet.fc1.bias");
    pa.W2 = P(h, "decoder.prenet.fc2.weight");
    pa.b2 = P(h, "decoder.prenet.fc2.bias");
    pa.m1 = m1;
    pa.m2 = m2;
    pa.mask_step = mstep;
    pa.step_ptr = sp;
    pa.step_j = sj;
    pa.row_start = d_start;
    pa.ring = nst;
    pa.B = B;
    pa.K = NM;
    pa.H = 2 * D;
    pa.y = ws + L.dp2;
    pa.ldy = 2 * D;
    if (fsplit) {  // [ctx | prenet] tiles of the attention GRU's input GEMM
      pa.s_hi = fhi(fs.p1);
      pa.s_lo = fhi(fs.p1 + fs.b1);
      pa.s_k0 = proj_dims;
      pa.s_rows_pad = f_rows_pad;
    }
    TK(launch_prenet_fused(pa, st));
  } else {
    // frame (step * r - 1) of every utterance; step 0 reads the zero block behind mel_all with row stride 0
    GemmArgs a = gemm1(mel_all - NM, NM, steps_alloc * NM, P(h, "decoder.prenet.fc1.weight"), NM,
                       P(h, "decoder.prenet.fc1.bias"), B, 2 * D, ws + L.dp1, 2 * D, ACT_RELU);
    a.mask = m1;
    a.step_mode = 1;
    a.step_ptr = sp;
    a.step_j = sj;
    a.x_step = (long long)r * NM;
    a.x_first = mel_all + (size_t)B * steps_alloc * NM;
    a.mask_step = mstep;
    TK(launch_gemm(a, st));
    GemmArgs b = gemm1(ws + L.dp1, 2 * D, 2 * D, P(h, "decoder.prenet.fc2.weight"), 2 * D, P(h, "decoder.prenet.fc2.bias"),
                       B, 2 * D, ws + L.dp2, 2 * D, ACT_RELU);
    b.mask = m2;
    b.step_mode = 1;
    b.step_ptr = sp;
    b.step_j = sj;
    b.mask_step = mstep;
    TK(launch_gemm(b, st));
  }
  if (use_tc && D % 64 == 0) {  // attention GRU on [context, prenet]: input projection + recurrent step on tensor cores
    __half* a_hi = reinterpret_cast<__half*>(ws + L.a_hi);
    __half* a_lo = reinterpret_cast<__half*>(ws + L.a_lo);
    if (fsplit) {
      a_hi = fhi(fs.p1);
      a_lo = fhi(fs.p1 + fs.b1);
    } else {
      TK(launch_act_split(ws + L.ctx, proj_dims, proj_dims, ws + L.dp2, 2 * D, 2 * D, B, a_hi, a_lo, st));
    }
    TcSkinnyArgs ta;
    memset(&ta, 0, sizeof(ta));
    ta.a_hi = a_hi;
    ta.a_lo = a_lo;
    ta.w = reinterpret_cast<const __half*>(P(h, "decoder.attn_rnn.ih.tcw"));
    ta.bias = P(h, "decoder.attn_rnn.ih.tcb");
    ta.KB = (proj_dims + 2 * D + 63) / 64;
    if (dag) {  // the context half was multiplied on the side stream after the previous step's attention (zero at step 0)
      if (have_gic) {
        MB_CUDA_CHECK(cudaStreamWaitEvent(st, h->ev_side[1], 0));
        have_gic = false;
      }
      ta.KBw = ta.KB;
      ta.kb0 = proj_dims / 64;
      ta.KB = ta.KBw - ta.kb0;
      ta.pre = ws + L.gic;
      ta.ldpre = 3 * D;
    }
    ta.M = B;
    ta.N = 3 * D;
    ta.mode = TCS_PLAIN;
    ta.inv_scale = h->tc_inv_scale["decoder.attn_rnn.ih"];
    ta.y = ws + L.dgi;
    ta.ldy = 3 * D;
    TK(launch_tc_skinny(ta, st));
    const size_t tb = tc_skinny_act_bytes(B, D);
    TcGruArgs g;
    memset(&g, 0, sizeof(g));
    if (fsplit) {  // attn_h is the trailing K segment of rnn_input's [ctx | attn_h] tiles
      g.s_hi = fhi(fs.p2);
      g.s_lo = fhi(fs.p2 + fs.b2);
      g.s_k0 = proj_dims;
    }
    g.a_hi[0] = reinterpret_cast<const __half*>(reinterpret_cast<const char*>(ws + L.ah_hi) + par * tb);
    g.a_lo[0] = reinterpret_cast<const __half*>(reinterpret_cast<const char*>(ws + L.ah_lo) + par * tb);
    g.nxt_hi[0] = reinterpret_cast<__half*>(reinterpret_cast<char*>(ws + L.ah_hi) + (par ^ 1) * tb);
    g.nxt_lo[0] = reinterpret_cast<__half*>(reinterpret_cast<char*>(ws + L.ah_lo) + (par ^ 1) * tb);
    g.w[0] = reinterpret_cast<const __half*>(P(h, "decoder.attn_rnn.hh.tcw"));
    g.bias[0] = P(h, "decoder.attn_rnn.hh.tcb");
    g.gi[0] = ws + L.dgi;
    g.h[0] = ws + L.attn_h;
    g.out[0] = ws + L.attn_h;
    g.inv_scale[0] = h->tc_inv_scale["decoder.attn_rnn.hh"];
    g.ldgi = 3 * D;
    g.ldout = D;
    g.KB = D / 64;
    g.M = B;
    g.H = D;
    g.ndir = 1;
    TK(launch_tc_gru(g, st));
  } else {  // attention GRU on [context, prenet]
    GemmArgs a;
    memset(&a, 0, sizeof(a));
    a.nseg = 2;
    a.seg[0] = {ws + L.ctx, proj_dims, proj_dims, 0, 0, 1};
    a.seg[1] = {ws + L.dp2, 2 * D, 2 * D, 0, proj_dims, 1};
    a.W = P(h, "decoder.attn_rnn.weight_ih");
    a.ldw = proj_dims + 2 * D;
    a.bias = P(h, "decoder.attn_rnn.bias_ih");
    a.M = B;
    a.N = 3 * D;
    a.T = 1;
    a.Y = ws + L.dgi;
    a.ldy = 3 * D;
    TK(launch_gemm(a, st));
    GemmArgs b = gemm1(ws + L.attn_h, D, D, P(h, "decoder.attn_rnn.weight_hh"), D, P(h, "decoder.attn_rnn.bias_hh"), B, 3 * D,
                       ws + L.dgh, 3 * D);
    TK(launch_gemm(b, st));
    TK(launch_gru_cell(ws + L.dgi, 3 * D, ws + L.dgh, ws + L.attn_h, D, nullptr, 0, B, D, st));
  }
  {  // location sensitive attention + context
    // MB_TACO_LSA_FUSED (default 1): 512 threads per batch row (4 time-step groups in the energy phase) and the query
    // projection W q + b inside the kernel; 0 = round-2 shape (256 threads, separate GEMM launch)
    static const bool lsa_fused = [] {
      const char* e = getenv("MB_TACO_LSA_FUSED");
      return e ? atoi(e) != 0 : true;
    }();
    const bool qf = lsa_fused && D == ATT_D;
    if (!qf) {
      GemmArgs a = gemm1(ws + L.attn_h, D, D, P(h, "decoder.attn_net.W.weight"), D, P(h, "decoder.attn_net.W.bias"), B, D,
                         ws + L.pq, D);
      TK(launch_gemm(a, st));
    }
    MB_CUDA_CHECK(launch_pdl2(lsa_step_kernel, dim3(B), dim3(lsa_fused ? 512 : 256), lsa_smem, st, ws + L.pq, ws + L.proj, seq,
                              proj_dims, chars, ws + L.cum, P(h, "decoder.attn_net.conv.weight"),
                              P(h, "decoder.attn_net.conv.bias"), P(h, "decoder.attn_net.L.weight"),
                              P(h, "decoder.attn_net.v.weight"), ws + L.scores_all, nst * Tc,
                              (proj_dims % 256 == 0) ? nullptr : ws + L.ctx, Tc, sp, sj, qf ? ws + L.attn_h : nullptr,
                              P(h, "decoder.attn_net.W.weight"), P(h, "decoder.attn_net.W.bias"), d_lens, d_start, nst));
    MB_LAUNCH_CHECK("lsa_step_kernel");
    if (proj_dims % 256 == 0) {
      if (have_stop) {  // the previous step's stop projection (side stream) still reads ctx and x, which are rewritten from here on
        MB_CUDA_CHECK(cudaStreamWaitEvent(st, h->ev_side[6], 0));
        have_stop = false;
      }
      MB_CUDA_CHECK(launch_pdl2(lsa_ctx_kernel, dim3(proj_dims / 256, B), dim3(256), sizeof(float) * Tc, st, ws + L.scores_all,
                                nst * Tc, seq, proj_dims, Tc, ws + L.ctx, sp, sj, fsplit ? fhi(fs.p1) : nullptr,
                                fsplit ? fhi(fs.p1 + fs.b1) : nullptr, fsplit ? fhi(fs.p2) : nullptr,
                                fsplit ? fhi(fs.p2 + fs.b2) : nullptr, f_rows_pad, d_lens, d_start, nst));
      MB_LAUNCH_CHECK("lsa_ctx_kernel");
    }
    if (dag) {  // side stream: context half of the NEXT step's attention-GRU input projection
      int rcs = side_after_main(h->ev_side[0]);
      if (rcs != MB_OK) return rcs;
      TcSkinnyArgs tp;
      memset(&tp, 0, sizeof(tp));
      tp.a_hi = fhi(fs.p1);
      tp.a_lo = fhi(fs.p1 + fs.b1);
      tp.w = reinterpret_cast<const __half*>(P(h, "decoder.attn_rnn.ih.tcw"));
      tp.KBw = (proj_dims + 2 * D + 63) / 64;
      tp.kb0 = 0;
      tp.KB = proj_dims / 64;
      tp.M = B;
      tp.N = 3 * D;
      tp.mode = TCS_PLAIN;
      tp.inv_scale = h->tc_inv_scale["decoder.attn_rnn.ih"];
      tp.y = ws + L.gic;
      tp.ldy = 3 * D;
      TK(launch_tc_skinny(tp, sd));
      MB_CUDA_CHECK(cudaEventRecord(h->ev_side[1], sd));
      have_gic = true;
    }
  }
  if (use_tc) {  // rnn_input on [context, attn_hidden] (tensor cores)
    __half* a_hi = reinterpret_cast<__half*>(ws + L.a_hi);
    __half* a_lo = reinterpret_cast<__half*>(ws + L.a_lo);
    if (fsplit) {
      a_hi = fhi(fs.p2);
      a_lo = fhi(fs.p2 + fs.b2);
    } else {
      TK(launch_act_split(ws + L.ctx, proj_dims, proj_dims, ws + L.attn_h, D, D, B, a_hi, a_lo, st));
    }
    TcSkinnyArgs ta;
    memset(&ta, 0, sizeof(ta));
    ta.a_hi = a_hi;
    ta.a_lo = a_lo;
    if (fsplit) {  // x is the leading K segment of the first LSTM's [x | h1] tiles of this step
      ta.s_hi[0] = fhi(fs.p3[par]);
      ta.s_lo[0] = fhi(fs.p3[par] + fs.b3);
      ta.s_k0[0] = 0;
    }
    ta.w = reinterpret_cast<const __half*>(P(h, "decoder.rnn_input.tcw"));
    ta.bias = P(h, "decoder.rnn_input.tcb");
    ta.KB = (proj_dims + D + 63) / 64;
    ta.M = B;
    ta.N = LD;
    ta.mode = TCS_PLAIN;
    ta.inv_scale = h->tc_inv_scale["decoder.rnn_input"];
    ta.y = ws + L.x;
    ta.ldy = LD;
    TK(launch_tc_skinny(ta, st));
  } else {  // rnn_input on [context, attn_hidden]
    GemmArgs a;
    memset(&a, 0, sizeof(a));
    a.nseg = 2;
    a.seg[0] = {ws + L.ctx, proj_dims, proj_dims, 0, 0, 1};
    a.seg[1] = {ws + L.attn_h, D, D, 0, proj_dims, 1};
    a.W = P(h, "decoder.rnn_input.weight");
    a.ldw = proj_dims + D;
    a.bias = P(h, "decoder.rnn_input.bias");
    a.M = B;
    a.N = LD;
    a.T = 1;
    a.Y = ws + L.x;
    a.ldy = LD;
    TK(launch_gemm(a, st));
  }
  for (int l = 0; l < 2; ++l) {  // residual LSTMs
    const std::string n = l == 0 ? "decoder.res_rnn1" : "decoder.res_rnn2";
    float* hh = ws + (l == 0 ? L.h1 : L.h2);
    float* cc = ws + (l == 0 ? L.c1 : L.c2);
    if (use_tc) {
      // gates GEMM on the tensor cores (3-term fp16 split, FP32 accumulate) with the cell update fused
      __half* a_hi = reinterpret_cast<__half*>(ws + L.a_hi);
      __half* a_lo = reinterpret_cast<__half*>(ws + L.a_lo);
      TcSkinnyArgs ta;
      memset(&ta, 0, sizeof(ta));
      if (fsplit) {
        // this step's [x | h] tiles; x' (residual stream) goes to the next consumer's tiles, h' to this cell's tiles of the
        // NEXT step (other parity)
        const size_t* mine = l == 0 ? fs.p3 : fs.p4;
        a_hi = fhi(mine[par]);
        a_lo = fhi(mine[par] + fs.b3);
        ta.s_hi[1] = fhi(mine[par ^ 1]);
        ta.s_lo[1] = fhi(mine[par ^ 1] + fs.b3);
        ta.s_k0[1] = LD;
        ta.s_hi[0] = l == 0 ? fhi(fs.p4[par]) : fhi(fs.p5);
        ta.s_lo[0] = l == 0 ? fhi(fs.p4[par] + fs.b3) : fhi(fs.p5 + fs.b5);
        ta.s_k0[0] = 0;
      } else {
        TK(launch_act_split(ws + L.x, LD, LD, hh, LD, LD, B, a_hi, a_lo, st));
      }
      ta.a_hi = a_hi;
      ta.a_lo = a_lo;
      ta.w = reinterpret_cast<const __half*>(P(h, n + ".tcw"));
      ta.bias = P(h, n + ".tcb");
      ta.KB = 2 * LD / 64;
      if (dag) {  // W_hh h_{t-1} was multiplied on the side stream right after the previous step's cell (zero at step 0)
        bool& have = l == 0 ? have_p1 : have_p2;
        if (have) {
          MB_CUDA_CHECK(cudaStreamWaitEvent(st, h->ev_side[l == 0 ? 3 : 5], 0));
          have = false;
        }
        ta.KBw = ta.KB;
        ta.kb0 = 0;
        ta.KB = LD / 64;
        ta.pre = ws + (l == 0 ? L.pre1 : L.pre2);
        ta.ldpre = 4 * LD;
      }
      ta.M = B;
      ta.N = 4 * LD;
      ta.mode = TCS_LSTM;
      ta.inv_scale = h->tc_inv_scale[n];
      ta.c = cc;
      ta.h = hh;
      ta.x = ws + L.x;
      ta.H = LD;
      TK(launch_tc_skinny(ta, st));
      if (dag) {  // side stream: W_hh h_t for the next step, from the h tiles this launch just wrote (other parity)
        int rcs = side_after_main(h->ev_side[l == 0 ? 2 : 4]);
        if (rcs != MB_OK) return rcs;
        const size_t* mine = l == 0 ? fs.p3 : fs.p4;
        TcSkinnyArgs tp;
        memset(&tp, 0, sizeof(tp));
        tp.a_hi = fhi(mine[par ^ 1]);
        tp.a_lo = fhi(mine[par ^ 1] + fs.b3);
        tp.w = reinterpret_cast<const __half*>(P(h, n + ".tcw"));
        tp.KBw = 2 * LD / 64;
        tp.kb0 = LD / 64;
        tp.KB = LD / 64;
        tp.M = B;
        tp.N = 4 * LD;
        tp.mode = TCS_PLAIN;
        tp.inv_scale = h->tc_inv_scale[n];
        tp.y = ws + (l == 0 ? L.pre1 : L.pre2);
        tp.ldy = 4 * LD;
        TK(launch_tc_skinny(tp, sd));
        MB_CUDA_CHECK(cudaEventRecord(h->ev_side[l == 0 ? 3 : 5], sd));
        (l == 0 ? have_p1 : have_p2) = true;
      }
      continue;
    }
    GemmArgs a;
    memset(&a, 0, sizeof(a));
    // gates = linear_hh(h) + linear_ih(x): two GEMMs chained through the residual input of the second
    GemmArgs g1 = gemm1(hh, LD, LD, P(h, n + ".weight_hh"), LD, P(h, n + ".bias_hh"), B, 4 * LD, ws + L.gates, 4 * LD);
    TK(launch_gemm(g1, st));
    GemmArgs g2 = gemm1(ws + L.x, LD, LD, P(h, n + ".weight_ih"), LD, P(h, n + ".bias_ih"), B, 4 * LD, ws + L.gates, 4 * LD);
    g2.res = ws + L.gates;
    g2.ldres = 4 * LD;
    TK(launch_gemm(g2, st));
    TK(launch_lstm_cell(ws + L.gates, cc, hh, ws + L.x, B, LD, st));
  }
  {  // mel frames of this step, written straight into mel_all[b][t..t+r)[:]
    if (use_tc && (r * NM) % 4 == 0) {
      __half* a_hi = reinterpret_cast<__half*>(ws + L.a_hi);
      __half* a_lo = reinterpret_cast<__half*>(ws + L.a_lo);
      if (fsplit) {
        a_hi = fhi(fs.p5);
        a_lo = fhi(fs.p5 + fs.b5);
      } else {
        TK(launch_act_split(ws + L.x, LD, LD, nullptr, 0, 0, B, a_hi, a_lo, st));
      }
      TcSkinnyArgs ta;
      memset(&ta, 0, sizeof(ta));
      ta.a_hi = a_hi;
      ta.a_lo = a_lo;
      ta.w = reinterpret_cast<const __half*>(P(h, "decoder.mel_proj.tcw"));
      ta.bias = nullptr;
      ta.KB = LD / 64;
      ta.M = B;
      ta.N = r * NM;
      ta.mode = TCS_PLAIN;
      ta.inv_scale = h->tc_inv_scale["decoder.mel_proj"];
      ta.y = mel_all;
      ta.ldy = steps_alloc * NM;
      ta.step_ptr = sp;
      ta.step_j = sj;
      ta.y_step = (long long)r * NM;
      ta.row_start = d_start;
      ta.ring = nst;
      TK(launch_tc_skinny(ta, st));
    } else {
      if (sp) return fail(MB_ERR_STATE, "mb_tacotron_generate: graph replay needs the tensor-core mel projection");
      GemmArgs a = gemm1(ws + L.x, LD, LD, P(h, "decoder.mel_proj.packed"), LD, nullptr, B, r * NM,
                         mel_all + (size_t)sj * r * NM, steps_alloc * NM);
      TK(launch_gemm(a, st));
    }
    GemmArgs s;
    memset(&s, 0, sizeof(s));
    s.nseg = 2;
    s.seg[0] = {ws + L.x, LD, LD, 0, 0, 1};
    s.seg[1] = {ws + L.ctx, proj_dims, proj_dims, 0, LD, 1};
    s.W = P(h, "decoder.stop_proj.weight");
    s.ldw = LD + proj_dims;
    s.bias = P(h, "decoder.stop_proj.bias");
    s.M = B;
    s.N = 1;
    s.T = 1;
    s.act = ACT_SIGMOID;
    s.Y = ws + L.stopv;
    s.ldy = 1;
    static const bool stop_fused = [] {
      const char* e = getenv("MB_TACO_STOP_FUSED");  // 0 = stop projection and stop rule as two launches (round 2)
      return e ? atoi(e) != 0 : true;
    }();
    if (stop_fused) {
      // the CTA that finishes last applies the stop rule (ticket counter behind the step counter, reset by that CTA).
      // With the step DAG it runs on the side stream (after the second LSTM's fork): the next step does not need it.
      stop_step_kernel<<<B, 256, 0, dag ? sd : st>>>(s, B, min_stop_token, r, flags, sp, sj,
                                                     reinterpret_cast<unsigned int*>(ws + L.step) + 16, d_done, d_caps,
                                                     d_start);
      MB_LAUNCH_CHECK("stop_step_kernel");
      if (dag) {
        MB_CUDA_CHECK(cudaEventRecord(h->ev_side[6], sd));
        have_stop = true;
      }
    } else {
      TK(launch_gemm(s, st));
      stop_flag_kernel<<<1, 32, 0, st>>>(ws + L.stopv, B, min_stop_token, r, flags, sp, sj, d_done, d_caps, d_start);
      MB_LAUNCH_CHECK("stop_flag_kernel");
    }
  }
  return MB_OK;
}

// Groups of kGraphSteps decoder steps are captured once and replayed (the loop is launch-bound: ~20 kernels of a few
// microseconds per step); MB_TACO_GRAPH=0 or a capture failure falls back to direct launches.  The group ends by advancing the
// device step counter.  false (error cleared): no graph.
constexpr int kGraphSteps = 8;
bool capture_group(DecoderLoop& dl, int* step_dev, cudaGraph_t* graph, cudaGraphExec_t* exec, int* per_graph) {
  cudaStream_t st = dl.st;
  const uint64_t launches_before = mb_launch_count();
  bool ok = cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal) == cudaSuccess;
  int rc_cap = MB_OK;
  if (ok) {
    for (int j = 0; j < kGraphSteps && rc_cap == MB_OK; ++j) rc_cap = dl.emit_step(step_dev, j);
    if (rc_cap == MB_OK) rc_cap = dl.join_side();
    if (rc_cap == MB_OK) step_advance_kernel<<<1, 32, 0, st>>>(step_dev, kGraphSteps);
    ok = cudaStreamEndCapture(st, graph) == cudaSuccess && rc_cap == MB_OK && *graph != nullptr;
  }
  if (ok) ok = cudaGraphInstantiate(exec, *graph, 0) == cudaSuccess;
  *per_graph = (int)(mb_launch_count() - launches_before);
  count_launch(-*per_graph);  // captured, not launched; every replay counts them
  if (!ok) cudaGetLastError();
  return ok;
}

// Tacotron.generate of one padded batch (rg == nullptr) or of B ragged rows, each computed as that utterance alone (rg)
int generate_impl(mb_tacotron* h, const int32_t* chars, const float* spk, int32_t B, int32_t Tc, int32_t steps,
                  int32_t r, int32_t style_idx, float min_stop_token, const uint8_t* enc_masks,
                  const uint8_t* dec_masks, uint64_t seed, float* mel_out, float* linear_out, float* attn_out,
                  int32_t* frames_out_host, void* workspace, size_t workspace_bytes, void* stream, const RaggedRows* rg) {
  if (!h || !chars || !spk || !mel_out || !linear_out || !frames_out_host)
    return fail(MB_ERR_INVALID, "mb_tacotron_generate: null argument");
  if (!h->finalized) return fail(MB_ERR_STATE, "mb_tacotron_generate: weights not finalized");
  const mb_tacotron_config& c = h->cfg;
  if (B <= 0 || Tc <= 0 || steps <= 0 || r <= 0 || r > c.max_r) return fail(MB_ERR_INVALID, "mb_tacotron_generate: bad shape");
  const int max_chars = lsa_max_chars();
  if (Tc > max_chars)
    return fail(MB_ERR_INVALID, "mb_tacotron_generate: %d characters exceed the limit of %d (the attention step's shared memory)",
                Tc, max_chars);
  const int nst = (steps + r - 1) / r;
  const int steps_alloc = nst * r;  // the reference emits r frames per decoder step (tacotron.py:264-272)
  const Ws L = ws_layout(c, B, Tc, steps_alloc, r, rg != nullptr);
  float* ws;
  if (int rc = bind("mb_tacotron_generate", workspace, workspace_bytes, L.total, &ws)) return rc;
  cudaStream_t caller = (cudaStream_t)stream;
  if (int rc = ensure_streams(h)) return rc;
  cudaStream_t st = h->own_stream;
  MB_CUDA_CHECK(cudaEventRecord(h->ev_in, caller));
  MB_CUDA_CHECK(cudaStreamWaitEvent(st, h->ev_in, 0));
  const int E = c.encoder_dims, D = c.decoder_dims, LD = c.lstm_dims, PD = c.postnet_dims, NM = c.n_mels;
  // MB_TACO_TC=0 keeps the decoder LSTMs on the FP32 FFMA kernels (A/B measurements); batches > 128 rows always do
  static const bool tc_env = [] {
    const char* e = getenv("MB_TACO_TC");
    return e ? atoi(e) != 0 : true;
  }();
  // a ragged batch always takes the tensor-core routes: their arithmetic per row does not depend on the row count
  const bool use_tc = (tc_env || rg) && B <= 128 && LD % 64 == 0;
  if (rg && !use_tc) return fail(MB_ERR_INVALID, "mb_tacotron_generate_ragged: more than 128 rows or lstm_dims %% 64 != 0");
  BigWs bw;
  bw.hi = ws + L.big_hi;
  bw.lo = ws + L.big_lo;
  bw.bytes = L.big_bytes;
  const int SE = c.speaker_embedding_size, proj_dims = E + SE + c.gst_E;
  const int Me = B * Tc;
  int* d_lens = nullptr;   // ragged rows: characters, caps, done steps, frames, seeds (device copies)
  int* d_caps = nullptr;
  int* d_done = nullptr;
  int* d_flen = nullptr;
  const uint64_t* d_seeds = nullptr;
  if (rg) {
    int32_t* base = reinterpret_cast<int32_t*>(ws + L.rows);
    std::vector<int32_t> hv((size_t)6 * B, 0);
    for (int b = 0; b < B; ++b) {
      hv[b] = rg->chars[b];
      hv[B + b] = (rg->steps[b] + r - 1) / r;
      hv[2 * B + b] = -1;
    }
    memcpy(hv.data() + 4 * B, rg->seeds, sizeof(uint64_t) * B);
    MB_CUDA_CHECK(cudaMemcpyAsync(base, hv.data(), sizeof(int32_t) * hv.size(), cudaMemcpyHostToDevice, st));
    d_lens = base;
    d_caps = base + B;
    d_done = base + 2 * B;
    d_flen = base + 3 * B;
    d_seeds = reinterpret_cast<const uint64_t*>(base + 4 * B);
  }

  if (int rc = prepare_mel_proj(h, r, st)) return rc;

  float* seq = ws + L.seq;
  int rc = run_encoder(h, L, ws, chars, spk, B, Tc, style_idx, enc_masks, seed, rg != nullptr, d_lens, d_seeds, use_tc, seq, ws + L.proj, st);
  if (rc != MB_OK) return rc;

  // ------------------------------------------------------------------ decoder loop (tacotron.py:264-275)
  MB_CUDA_CHECK(cudaMemsetAsync(ws + L.attn_h, 0, sizeof(float) * (L.dp1 - L.attn_h), st));  // states, ctx, cum
  MB_CUDA_CHECK(cudaMemsetAsync(ws + L.ah_hi, 0, sizeof(float) * (L.stopv - L.ah_hi), st));  // h0 = 0 operand tiles
  MB_CUDA_CHECK(cudaMemsetAsync(ws + L.step, 0, sizeof(float) * 64, st));  // step counter, stop-rule ticket
  float* mel_all = ws + L.mel_all;
  MB_CUDA_CHECK(cudaMemsetAsync(mel_all, 0, sizeof(float) * ((size_t)B * steps_alloc * NM + (size_t)r * NM), st));
  int* flags = reinterpret_cast<int*>(ws + L.flags);
  MB_CUDA_CHECK(cudaMemsetAsync(flags, 0, sizeof(int) * nst, st));
  uint8_t* dm = reinterpret_cast<uint8_t*>(ws + L.dmask);
  const size_t dmask_n = (size_t)B * 2 * D;
  MB_CUDA_CHECK(lsa_step_prepare(Tc));
  if (!dec_masks && rg) {
    fill_masks_seeded_kernel<<<(unsigned)((2 * dmask_n * (size_t)nst + 255) / 256), 256, 0, st>>>(dm, B, nst, 2 * D, d_seeds, 1);
    MB_LAUNCH_CHECK("fill_masks_seeded_kernel");
  } else if (!dec_masks) {
    const size_t total = 2 * dmask_n * (size_t)nst;
    fill_masks_steps_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(dm, 2 * dmask_n, nst, seed);
    MB_LAUNCH_CHECK("fill_masks_steps_kernel");
  }
  int done_step = -1;
  std::vector<int> hflags(nst, 0);
  int checked = 0;
  DecoderLoop dl;
  dl.h = h;
  dl.L = L;
  dl.ws = ws;
  dl.B = B;
  dl.Tc = Tc;
  dl.r = r;
  dl.nst = nst;
  dl.steps_alloc = steps_alloc;
  dl.chars = chars;
  dl.seq = seq;
  dl.mel_all = mel_all;
  dl.dec_masks = dec_masks;
  dl.dm = dm;
  dl.min_stop_token = min_stop_token;
  dl.flags = flags;
  dl.d_lens = d_lens;
  dl.d_caps = d_caps;
  dl.d_done = d_done;
  dl.d_start = nullptr;
  dl.use_tc = use_tc;
  dl.init(st);
  auto emit_step = [&](const int* sp, int sj) { return dl.emit_step(sp, sj); };
  auto join_side = [&]() { return dl.join_side(); };

  // poll the early-stop rule (tacotron.py:275) after every group of 16 decoder steps
  auto poll = [&](int upto) -> int {
    MB_CUDA_CHECK(cudaMemcpyAsync(hflags.data() + checked, flags + checked, sizeof(int) * (upto + 1 - checked),
                                  cudaMemcpyDeviceToHost, st));
    MB_CUDA_CHECK(cudaStreamSynchronize(st));
    for (int j = checked; j <= upto && done_step < 0; ++j)
      if (hflags[j]) done_step = j;
    checked = upto + 1;
    return MB_OK;
  };
  static const bool graph_env = [] {
    const char* e = getenv("MB_TACO_GRAPH");
    return e ? atoi(e) != 0 : true;
  }();
  int si = 0;
  if (graph_env && use_tc && (r * NM) % 4 == 0 && nst >= 2 * kGraphSteps) {
    int* step_dev = reinterpret_cast<int*>(ws + L.step);
    MB_CUDA_CHECK(cudaMemsetAsync(step_dev, 0, sizeof(int), st));
    cudaGraph_t graph = nullptr;
    cudaGraphExec_t exec = nullptr;
    int per_graph = 0;
    const bool ok = capture_group(dl, step_dev, &graph, &exec, &per_graph);
    if (ok) {
      while (si + kGraphSteps <= nst && done_step < 0) {
        if (cudaGraphLaunch(exec, st) != cudaSuccess) {
          cudaGraphExecDestroy(exec);
          cudaGraphDestroy(graph);
          return fail(MB_ERR_CUDA, "mb_tacotron_generate: cudaGraphLaunch failed");
        }
        count_launch(per_graph + 1);
        si += kGraphSteps;
        if ((si % 16) == 0 || si + kGraphSteps > nst) {
          int rc2 = poll(si - 1);
          if (rc2 != MB_OK) return rc2;
        }
      }
    }
    if (exec) cudaGraphExecDestroy(exec);
    if (graph) cudaGraphDestroy(graph);
  }
  for (; si < nst && done_step < 0; ++si) {  // tail (or everything, without the graph): direct launches
    int rc2 = emit_step(nullptr, si);
    if (rc2 == MB_OK) rc2 = join_side();
    if (rc2 != MB_OK) return rc2;
    if ((si % 16) == 15 || si == nst - 1) {
      rc2 = poll(si);
      if (rc2 != MB_OK) return rc2;
    }
  }
  int frames = 0;
  if (rg) {  // a ragged row ends at its own done step; the postnet runs over the longest row, each row over its own frames
    std::vector<int32_t> hdone(B), hflen(B);
    MB_CUDA_CHECK(cudaMemcpyAsync(hdone.data(), d_done, sizeof(int32_t) * B, cudaMemcpyDeviceToHost, st));
    MB_CUDA_CHECK(cudaStreamSynchronize(st));
    for (int b = 0; b < B; ++b) {
      hflen[b] = ((hdone[b] >= 0 ? hdone[b] : nst - 1) + 1) * r;
      rg->frames[b] = hflen[b];
      if (hflen[b] > frames) frames = hflen[b];
    }
    MB_CUDA_CHECK(cudaMemcpyAsync(d_flen, hflen.data(), sizeof(int32_t) * B, cudaMemcpyHostToDevice, st));
  } else {
    frames = ((done_step >= 0 ? done_step : nst - 1) + 1) * r;
  }
  const int nsteps_done = frames / r;
  *frames_out_host = frames;

  // ------------------------------------------------------------------ postnet (tacotron.py:281-283)
  // the postnet sees exactly `frames` frames per utterance: compact mel_all to [B][frames][80] first
  float* melc = ws + L.lin;  // reuse the output buffer as the compact input, then overwrite
  if (frames != steps_alloc) {
    for (int b = 0; b < B; ++b)
      MB_CUDA_CHECK(cudaMemcpyAsync(ws + L.ppj2 + (size_t)b * frames * NM, mel_all + (size_t)b * steps_alloc * NM,
                                    sizeof(float) * frames * NM, cudaMemcpyDeviceToDevice, st));
    melc = ws + L.ppj2;
    // ppj2 is also run_cbhg's conv_project2 scratch only when p1 != ch (it uses hw12), so it is free here
  } else {
    melc = mel_all;
  }
  rc = run_postnet(h, L, ws, melc, B, frames, d_flen, use_tc, st);
  if (rc != MB_OK) return rc;
  // outputs in the reference's layouts: mel [B][80][frames], linear [B][80][frames], attn [B][nsteps][Tc]
  {
    const size_t n = (size_t)B * NM * frames;
    to_ncl_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(mel_all, steps_alloc, mel_out, B, NM, frames);
    MB_LAUNCH_CHECK("to_ncl_kernel");
    to_ncl_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(ws + L.lin, frames, linear_out, B, NM, frames);
    MB_LAUNCH_CHECK("to_ncl_kernel");
    if (attn_out)
      for (int b = 0; b < B; ++b)
        MB_CUDA_CHECK(cudaMemcpyAsync(attn_out + (size_t)b * nsteps_done * Tc, ws + L.scores_all + (size_t)b * nst * Tc,
                                      sizeof(float) * nsteps_done * Tc, cudaMemcpyDeviceToDevice, st));
  }
  MB_CUDA_CHECK(cudaEventRecord(h->ev_out, st));
  MB_CUDA_CHECK(cudaStreamWaitEvent(caller, h->ev_out, 0));
  return MB_OK;
}

}  // namespace

extern "C" {

int mb_tacotron_generate(mb_tacotron* h, const int32_t* chars, const float* spk, int32_t B, int32_t Tc, int32_t steps,
                         int32_t r, int32_t style_idx, float min_stop_token, const uint8_t* enc_masks,
                         const uint8_t* dec_masks, uint64_t seed, float* mel_out, float* linear_out, float* attn_out,
                         int32_t* frames_out_host, void* workspace, size_t workspace_bytes, void* stream) {
  return generate_impl(h, chars, spk, B, Tc, steps, r, style_idx, min_stop_token, enc_masks, dec_masks, seed, mel_out, linear_out,
                       attn_out, frames_out_host, workspace, workspace_bytes, stream, nullptr);
}

size_t mb_tacotron_ragged_workspace_bytes(const mb_tacotron* h, int32_t B, int32_t Tc, int32_t steps, int32_t r) {
  if (B > 128 || !mb_tacotron_workspace_bytes(h, B, Tc, steps, r)) return 0;
  return ws_layout(h->cfg, B, Tc, (steps + r - 1) / r * r, r, true).total;
}

int mb_tacotron_generate_ragged(mb_tacotron* h, const int32_t* chars, const float* spk, int32_t B, int32_t Tc,
                                const int32_t* row_chars, const int32_t* row_steps, const uint64_t* row_seeds, int32_t r,
                                int32_t style_idx, float min_stop_token, const uint8_t* enc_masks, const uint8_t* dec_masks,
                                float* mel_out, float* linear_out, float* attn_out, int32_t* frames_out_host,
                                int32_t* row_frames_host, void* workspace, size_t workspace_bytes, void* stream) {
  const char* me = "mb_tacotron_generate_ragged";
  if (!h || !row_chars || !row_steps || !row_seeds || !row_frames_host) return fail(MB_ERR_INVALID, "%s: null argument", me);
  if (B <= 0 || B > 128 || Tc <= 0) return fail(MB_ERR_INVALID, "%s: %d rows of %d characters (1 to 128 rows)", me, B, Tc);
  int steps = 0;
  for (int b = 0; b < B; ++b) {
    if (row_chars[b] < 1 || row_chars[b] > Tc)
      return fail(MB_ERR_INVALID, "%s: row %d has %d characters, outside [1, %d]", me, b, row_chars[b], Tc);
    if (row_steps[b] < 1) return fail(MB_ERR_INVALID, "%s: row %d has a frame cap of %d", me, b, row_steps[b]);
    if (row_steps[b] > steps) steps = row_steps[b];
  }
  RaggedRows rg{row_chars, row_steps, row_seeds, row_frames_host};
  return generate_impl(h, chars, spk, B, Tc, steps, r, style_idx, min_stop_token, enc_masks, dec_masks, 0, mel_out, linear_out,
                       attn_out, frames_out_host, workspace, workspace_bytes, stream, &rg);
}

int32_t mb_tacotron_max_chars(void) { return lsa_max_chars(); }

}  // extern "C"

namespace {

// ---- streamed decoding (mb_tacotron_stream_*) ----------------------------------------------------------------------------------
// A decoder loop over a fixed set of slots.  A text enters a free slot between graph replays (admission) and leaves when its row
// stops; its frames and alignment rows are then copied to a pool the postnet reads from its own stream.  Each row's step is the
// global step minus its start step (DecoderLoop::d_start), and its per-step buffers are rings of kStreamRing steps beyond its cap,
// so a row finished at its last step still has its frames when the next poll (at most 15 steps later) finds it.
constexpr int kStreamPoll = 16;

struct StreamLayout {
  Ws enc, dec, post;
  // byte offsets
  size_t enc_at, dec_at, post_at, pool_seq, pool_proj, pool_chars, pool_tab, post_mel, post_attn, post_flen, admit_tab, start, total;
};

StreamLayout stream_layout(const mb_tacotron_config& c, int S, int Tc, int nst, int r) {
  StreamLayout L{};
  const int ring = nst + kStreamPoll, proj_dims = c.encoder_dims + c.speaker_embedding_size + c.gst_E;
  L.enc = ws_layout(c, S, Tc, r, r, true, WS_ENC);
  L.dec = ws_layout(c, S, Tc, ring * r, r, true, WS_DEC);
  L.post = ws_layout(c, S, Tc, nst * r, r, true, WS_POST);
  WsLayout W;
  L.enc_at = W.take(L.enc.total);
  L.dec_at = W.take(L.dec.total);
  L.post_at = W.take(L.post.total);
  L.pool_seq = W.take(sizeof(float) * (size_t)2 * S * Tc * proj_dims);
  L.pool_proj = W.take(sizeof(float) * (size_t)2 * S * Tc * c.decoder_dims);
  L.pool_chars = W.take(sizeof(int32_t) * (size_t)2 * S * Tc);
  L.pool_tab = W.take(sizeof(int32_t) * (size_t)2 * S * 3);  // characters [2S] | seeds (u64) [2S] of each staging-pool row
  L.post_mel = W.take(sizeof(float) * (size_t)2 * S * nst * r * c.n_mels);
  L.post_attn = W.take(sizeof(float) * (size_t)2 * S * nst * Tc);
  L.post_flen = W.take(sizeof(int32_t) * S);
  L.admit_tab = W.take(sizeof(AdmitRow) * S);
  L.start = W.take(sizeof(int32_t) * S);
  L.total = W.total();
  return L;
}

}  // namespace

struct mb_taco_stream {
  mb_tacotron* h = nullptr;
  int S = 0, Tc = 0, nst = 0, ring = 0, r = 0, style_idx = 0;
  StreamLayout L;
  char* base = nullptr;
  float *we = nullptr, *wd = nullptr, *wp = nullptr;
  int* d_done = nullptr;
  DecoderLoop dl;
  cudaGraph_t graph = nullptr;
  cudaGraphExec_t exec = nullptr;
  int per_graph = 0;
  cudaStream_t enc_st = nullptr;
  cudaEvent_t ev_enc[2] = {nullptr, nullptr}, ev_admit = nullptr, ev_copied = nullptr, ev_post = nullptr, ev_in = nullptr;
  int global = 0;                     // decoder steps run so far (the device step counter)
  long long steps_run = 0;
  std::vector<int64_t> occupant;      // text in each slot, -1: free
  std::vector<int> pool;              // postnet pool rows: 0 free, 1 finished and waiting, 2 read by a postnet in flight
  std::vector<int64_t> pool_id;
  std::vector<int> pool_frames;
  std::vector<int> pending;           // pool rows in the order their rows finished
  std::vector<int32_t> hdone;
  // releases the stream's graph, events and encoder stream (mb_tacotron_stream_close first waits for their work)
  ~mb_taco_stream() {
    if (exec) cudaGraphExecDestroy(exec);
    if (graph) cudaGraphDestroy(graph);
    for (cudaEvent_t e : {ev_enc[0], ev_enc[1], ev_admit, ev_copied, ev_post, ev_in})
      if (e) cudaEventDestroy(e);
    if (enc_st) cudaStreamDestroy(enc_st);
  }
};

namespace {

int stream_check(const char* fn, mb_taco_stream* s) {
  if (!s || !s->h) return fail(MB_ERR_INVALID, "%s: null stream", fn);
  return MB_OK;
}

int caller_to(mb_taco_stream* s, cudaStream_t caller, cudaStream_t to) {
  MB_CUDA_CHECK(cudaEventRecord(s->ev_in, caller));
  MB_CUDA_CHECK(cudaStreamWaitEvent(to, s->ev_in, 0));
  return MB_OK;
}

// A few host bytes into device memory in stream order, carried as a kernel argument.  A copy from pageable host memory would
// first wait for the stream, which would block the host behind an encode or a postnet that is still running.
int upload(void* dst, const void* src, size_t n, cudaStream_t st) {
  if (n > (size_t)kUploadBytes) return fail(MB_ERR_INVALID, "upload of %zu bytes (at most %d)", n, kUploadBytes);
  UploadBlob b;
  memcpy(b.b, src, n);
  upload_kernel<<<1, 256, 0, st>>>(b, reinterpret_cast<unsigned char*>(dst), (int)n);
  MB_LAUNCH_CHECK("upload_kernel");
  return MB_OK;
}

// The per-slot regions of a stream's decoder loop and its staging pool.  Admission zeroes the rows of the `reset` regions (the
// state a fresh row starts from, as generate zeroes it) and fills the rest of a slot's rows; mb_tacotron_stream_regions hands the
// same list to tests.
void stream_regions(const mb_taco_stream* s, std::vector<mb_taco_stream_region>& out) {
  const mb_tacotron_config& c = s->h->cfg;
  const Ws& D = s->L.dec;
  float* wd = s->wd;
  const int S = s->S, Dd = c.decoder_dims, LD = c.lstm_dims, proj_dims = c.encoder_dims + c.speaker_embedding_size + c.gst_E;
  const int rows_pad = S <= 64 ? 64 : 128;
  auto add = [&](const char* name, void* p, int kind, int rows, int width, int depth, int reset) {
    mb_taco_stream_region r;
    memset(&r, 0, sizeof(r));
    snprintf(r.name, sizeof(r.name), "%s", name);
    r.ptr = p;
    r.kind = kind;
    r.rows = rows;
    r.width = width;
    r.depth = depth;
    r.reset = reset;
    out.push_back(r);
  };
  add("attn_h", wd + D.attn_h, MB_TACO_REGION_F32, S, Dd, 1, 1);
  add("h1", wd + D.h1, MB_TACO_REGION_F32, S, LD, 1, 1);
  add("c1", wd + D.c1, MB_TACO_REGION_F32, S, LD, 1, 1);
  add("h2", wd + D.h2, MB_TACO_REGION_F32, S, LD, 1, 1);
  add("c2", wd + D.c2, MB_TACO_REGION_F32, S, LD, 1, 1);
  add("ctx", wd + D.ctx, MB_TACO_REGION_F32, S, proj_dims, 1, 1);
  add("cum", wd + D.cum, MB_TACO_REGION_F32, S, s->Tc, 1, 1);
  add("pre1", wd + D.pre1, MB_TACO_REGION_F32, S, 4 * LD, 1, 1);
  add("pre2", wd + D.pre2, MB_TACO_REGION_F32, S, 4 * LD, 1, 1);
  add("gic", wd + D.gic, MB_TACO_REGION_F32, S, 3 * Dd, 1, 1);
  const size_t tb = tc_skinny_act_bytes(S, Dd);
  for (int par = 0; par < 2; ++par) {
    add(par ? "ah_hi.1" : "ah_hi.0", reinterpret_cast<char*>(wd + D.ah_hi) + par * tb, MB_TACO_REGION_TILE, rows_pad, Dd, 1, 1);
    add(par ? "ah_lo.1" : "ah_lo.0", reinterpret_cast<char*>(wd + D.ah_lo) + par * tb, MB_TACO_REGION_TILE, rows_pad, Dd, 1, 1);
  }
  const FusedSplit& fs = s->dl.fs;
  char* fb = s->dl.fbase;
  auto pair = [&](const char* hi, const char* lo, size_t off, size_t bytes, int K) {
    add(hi, fb + off, MB_TACO_REGION_TILE, rows_pad, K, 1, 1);
    add(lo, fb + off + bytes, MB_TACO_REGION_TILE, rows_pad, K, 1, 1);
  };
  pair("p1_hi", "p1_lo", fs.p1, fs.b1, proj_dims + 2 * Dd);
  pair("p2_hi", "p2_lo", fs.p2, fs.b2, proj_dims + Dd);
  pair("p3_hi.0", "p3_lo.0", fs.p3[0], fs.b3, 2 * LD);
  pair("p3_hi.1", "p3_lo.1", fs.p3[1], fs.b3, 2 * LD);
  pair("p4_hi.0", "p4_lo.0", fs.p4[0], fs.b3, 2 * LD);
  pair("p4_hi.1", "p4_lo.1", fs.p4[1], fs.b3, 2 * LD);
  pair("p5_hi", "p5_lo", fs.p5, fs.b5, LD);
  add("seq", wd + D.seq, MB_TACO_REGION_F32, S, s->Tc * proj_dims, 1, 0);
  add("proj", wd + D.proj, MB_TACO_REGION_F32, S, s->Tc * Dd, 1, 0);
  add("chars", wd + D.ids, MB_TACO_REGION_I32, S, s->Tc, 1, 0);
  int32_t* drows = reinterpret_cast<int32_t*>(wd + D.rows);
  add("lens", drows, MB_TACO_REGION_I32, S, 1, 1, 0);
  add("caps", drows + S, MB_TACO_REGION_I32, S, 1, 1, 0);
  add("done", drows + 2 * S, MB_TACO_REGION_I32, S, 1, 1, 0);
  add("start", s->base + s->L.start, MB_TACO_REGION_I32, S, 1, 1, 0);
  add("dmask", wd + D.dmask, MB_TACO_REGION_U8, S, 2 * Dd, s->ring, 0);
  add("pool_seq", s->base + s->L.pool_seq, MB_TACO_REGION_F32, 2 * S, s->Tc * proj_dims, 1, 0);
  add("pool_proj", s->base + s->L.pool_proj, MB_TACO_REGION_F32, 2 * S, s->Tc * Dd, 1, 0);
  add("pool_chars", s->base + s->L.pool_chars, MB_TACO_REGION_I32, 2 * S, s->Tc, 1, 0);
}

}  // namespace

extern "C" {

size_t mb_tacotron_stream_workspace_bytes(const mb_tacotron* h, int32_t slots, int32_t n_chars, int32_t max_steps, int32_t r) {
  if (!h || slots < 1 || slots > 128 || !mb_tacotron_workspace_bytes(h, slots, n_chars, max_steps, r)) return 0;
  return stream_layout(h->cfg, slots, n_chars, (max_steps + r - 1) / r, r).total;
}

int mb_tacotron_stream_open(mb_tacotron* h, int32_t slots, int32_t n_chars, int32_t max_steps, int32_t r, int32_t style_idx,
                            float min_stop_token, void* workspace, size_t workspace_bytes, void* stream, mb_taco_stream** out) {
  const char* me = "mb_tacotron_stream_open";
  if (!h || !out) return fail(MB_ERR_INVALID, "%s: null argument", me);
  if (!h->finalized) return fail(MB_ERR_STATE, "%s: weights not finalized", me);
  const mb_tacotron_config& c = h->cfg;
  if (slots < 1 || slots > 128 || n_chars < 1 || max_steps < 1 || r < 1 || r > c.max_r)
    return fail(MB_ERR_INVALID, "%s: %d slots (1 to 128), %d characters, %d frames, r = %d", me, slots, n_chars, max_steps, r);
  if (n_chars > lsa_max_chars())
    return fail(MB_ERR_INVALID, "%s: %d characters exceed the limit of %d (the attention step's shared memory)", me, n_chars,
                lsa_max_chars());
  const size_t need = mb_tacotron_stream_workspace_bytes(h, slots, n_chars, max_steps, r);
  char* base;
  if (int rc = bind(me, workspace, workspace_bytes, need, &base)) return rc;
  if (int rc = ensure_streams(h)) return rc;
  cudaStream_t st = h->own_stream;
  std::unique_ptr<mb_taco_stream> s(new mb_taco_stream());
  s->h = h;
  s->S = slots;
  s->Tc = n_chars;
  s->r = r;
  s->nst = (max_steps + r - 1) / r;
  s->ring = s->nst + kStreamPoll;
  s->style_idx = style_idx;
  s->L = stream_layout(c, slots, n_chars, s->nst, r);
  s->base = base;
  s->we = reinterpret_cast<float*>(base + s->L.enc_at);
  s->wd = reinterpret_cast<float*>(base + s->L.dec_at);
  s->wp = reinterpret_cast<float*>(base + s->L.post_at);
  s->occupant.assign(slots, -1);
  s->pool.assign(2 * slots, 0);
  s->pool_id.assign(2 * slots, -1);
  s->pool_frames.assign(2 * slots, 0);
  s->hdone.assign(slots, 0);
  MB_CUDA_CHECK(cudaStreamCreateWithFlags(&s->enc_st, cudaStreamNonBlocking));
  for (cudaEvent_t* e : {&s->ev_enc[0], &s->ev_enc[1], &s->ev_admit, &s->ev_copied, &s->ev_post, &s->ev_in})
    MB_CUDA_CHECK(cudaEventCreateWithFlags(e, cudaEventDisableTiming));
  if (int rc = caller_to(s.get(), (cudaStream_t)stream, st)) return rc;
  if (int rc = prepare_mel_proj(h, r, st)) return rc;
  MB_CUDA_CHECK(lsa_step_prepare(n_chars));
  const Ws& D = s->L.dec;
  float* wd = s->wd;
  // every slot starts empty: zero state, one character, done at step 0 (a finished row that is never reported)
  MB_CUDA_CHECK(cudaMemsetAsync(wd, 0, D.total, st));
  int32_t* rows = reinterpret_cast<int32_t*>(wd + D.rows);
  std::vector<int32_t> init((size_t)3 * slots, 0);
  for (int b = 0; b < slots; ++b) init[b] = init[slots + b] = 1;
  MB_CUDA_CHECK(cudaMemcpyAsync(rows, init.data(), sizeof(int32_t) * init.size(), cudaMemcpyHostToDevice, st));
  MB_CUDA_CHECK(cudaMemsetAsync(base + s->L.start, 0, sizeof(int32_t) * slots, st));
  s->d_done = rows + 2 * slots;
  DecoderLoop& dl = s->dl;
  dl.h = h;
  dl.L = D;
  dl.ws = wd;
  dl.B = slots;
  dl.Tc = n_chars;
  dl.r = r;
  dl.nst = s->ring;
  dl.steps_alloc = s->ring * r;
  dl.chars = reinterpret_cast<const int32_t*>(wd + D.ids);
  dl.seq = wd + D.seq;
  dl.mel_all = wd + D.mel_all;
  dl.dec_masks = nullptr;
  dl.dm = reinterpret_cast<uint8_t*>(wd + D.dmask);
  dl.min_stop_token = min_stop_token;
  dl.flags = nullptr;
  dl.d_lens = rows;
  dl.d_caps = rows + slots;
  dl.d_done = s->d_done;
  dl.d_start = reinterpret_cast<const int*>(base + s->L.start);
  dl.use_tc = true;
  dl.init(st);
  if (!dl.fsplit || (r * c.n_mels) % 4)
    return fail(MB_ERR_STATE, "%s: streaming needs the fused decoder step (MB_TACO_SPLIT_FUSED, MB_TACO_PRENET_FUSED)", me);
  if (!capture_group(dl, reinterpret_cast<int*>(wd + D.step), &s->graph, &s->exec, &s->per_graph))
    return fail(MB_ERR_CUDA, "%s: capturing the decoder step graph failed", me);
  MB_CUDA_CHECK(cudaEventRecord(s->ev_admit, st));
  MB_CUDA_CHECK(cudaEventRecord(s->ev_enc[0], st));
  MB_CUDA_CHECK(cudaEventRecord(s->ev_enc[1], st));
  MB_CUDA_CHECK(cudaEventRecord(s->ev_post, st));
  MB_CUDA_CHECK(cudaEventRecord(h->ev_out, st));
  MB_CUDA_CHECK(cudaStreamWaitEvent((cudaStream_t)stream, h->ev_out, 0));
  *out = s.release();
  return MB_OK;
}

int mb_tacotron_stream_encode(mb_taco_stream* s, int32_t pool_row, int32_t n, const int32_t* chars, const float* spk,
                              const int32_t* row_chars, const uint64_t* row_seeds, const uint8_t* enc_masks, void* stream) {
  const char* me = "mb_tacotron_stream_encode";
  if (int rc = stream_check(me, s)) return rc;
  if (!chars || !spk || !row_chars || !row_seeds) return fail(MB_ERR_INVALID, "%s: null argument", me);
  if (n < 1 || pool_row < 0 || pool_row / s->S != (pool_row + n - 1) / s->S || pool_row + n > 2 * s->S)
    return fail(MB_ERR_INVALID, "%s: rows [%d, %d) are not inside one half of the staging pool (2 x %d rows)", me, pool_row,
                pool_row + n, s->S);
  for (int i = 0; i < n; ++i)
    if (row_chars[i] < 1 || row_chars[i] > s->Tc)
      return fail(MB_ERR_INVALID, "%s: row %d has %d characters, outside [1, %d]", me, i, row_chars[i], s->Tc);
  mb_tacotron* h = s->h;
  const mb_tacotron_config& c = h->cfg;
  const int proj_dims = c.encoder_dims + c.speaker_embedding_size + c.gst_E, Tc = s->Tc, S2 = 2 * s->S;
  cudaStream_t st = s->enc_st;
  if (int rc = caller_to(s, (cudaStream_t)stream, st)) return rc;
  MB_CUDA_CHECK(cudaStreamWaitEvent(st, s->ev_admit, 0));  // the rows it overwrites have been admitted
  int32_t* tab = reinterpret_cast<int32_t*>(s->base + s->L.pool_tab);
  uint64_t* seeds = reinterpret_cast<uint64_t*>(tab + S2);
  if (int rc = upload(tab + pool_row, row_chars, sizeof(int32_t) * n, st)) return rc;
  if (int rc = upload(seeds + pool_row, row_seeds, sizeof(uint64_t) * n, st)) return rc;
  MB_CUDA_CHECK(cudaMemcpyAsync(reinterpret_cast<int32_t*>(s->base + s->L.pool_chars) + (size_t)pool_row * Tc, chars,
                                sizeof(int32_t) * n * Tc, cudaMemcpyDeviceToDevice, st));
  float* seq = reinterpret_cast<float*>(s->base + s->L.pool_seq) + (size_t)pool_row * Tc * proj_dims;
  float* proj = reinterpret_cast<float*>(s->base + s->L.pool_proj) + (size_t)pool_row * Tc * c.decoder_dims;
  if (int rc = run_encoder(h, s->L.enc, s->we, chars, spk, n, Tc, s->style_idx, enc_masks, 0, true, tab + pool_row, seeds + pool_row,
                           true, seq, proj, st))
    return rc;
  // only the admissions that copy these rows wait for them (mb_tacotron_stream_admit): the caller's stream does not, so the
  // decoder keeps running while the encoder works; the inputs must stay allocated until the stream is closed
  MB_CUDA_CHECK(cudaEventRecord(s->ev_enc[pool_row / s->S], st));
  return MB_OK;
}

int mb_tacotron_stream_admit(mb_taco_stream* s, int32_t n, const int32_t* slot, const int32_t* pool_row, const int64_t* text_id,
                             const int32_t* row_chars, const int32_t* row_steps, const uint64_t* row_seeds,
                             const uint8_t* const* dec_masks, void* stream) {
  const char* me = "mb_tacotron_stream_admit";
  if (int rc = stream_check(me, s)) return rc;
  if (!slot || !pool_row || !text_id || !row_chars || !row_steps || !row_seeds) return fail(MB_ERR_INVALID, "%s: null argument", me);
  if (n < 1 || n > s->S) return fail(MB_ERR_INVALID, "%s: %d rows (1 to %d)", me, n, s->S);
  std::vector<AdmitRow> rows(n);
  std::vector<int> seen(s->S, 0);
  for (int i = 0; i < n; ++i) {
    if (slot[i] < 0 || slot[i] >= s->S || s->occupant[slot[i]] >= 0 || seen[slot[i]]++)
      return fail(MB_ERR_INVALID, "%s: slot %d is not free", me, slot[i]);
    if (pool_row[i] < 0 || pool_row[i] >= 2 * s->S) return fail(MB_ERR_INVALID, "%s: pool row %d", me, pool_row[i]);
    if (row_chars[i] < 1 || row_chars[i] > s->Tc)
      return fail(MB_ERR_INVALID, "%s: row %d has %d characters, outside [1, %d]", me, i, row_chars[i], s->Tc);
    if (row_steps[i] < 1 || row_steps[i] > s->nst * s->r)
      return fail(MB_ERR_INVALID, "%s: frame cap %d outside [1, %d]", me, row_steps[i], s->nst * s->r);
  }
  mb_tacotron* h = s->h;
  const mb_tacotron_config& c = h->cfg;
  cudaStream_t st = h->own_stream;
  if (int rc = caller_to(s, (cudaStream_t)stream, st)) return rc;
  bool half[2] = {false, false};
  for (int i = 0; i < n; ++i) half[pool_row[i] / s->S] = true;
  for (int q = 0; q < 2; ++q)  // the encoder rows this admission copies
    if (half[q]) MB_CUDA_CHECK(cudaStreamWaitEvent(st, s->ev_enc[q], 0));
  for (int i = 0; i < n; ++i) {
    rows[i] = AdmitRow{slot[i], pool_row[i], row_chars[i], (row_steps[i] + s->r - 1) / s->r, row_seeds[i],
                       dec_masks ? dec_masks[i] : nullptr};
    s->occupant[slot[i]] = text_id[i];
  }
  AdmitRow* d_rows = reinterpret_cast<AdmitRow*>(s->base + s->L.admit_tab);
  if (int rc = upload(d_rows, rows.data(), sizeof(AdmitRow) * n, st)) return rc;
  const Ws& D = s->L.dec;
  float* wd = s->wd;
  const int Dd = c.decoder_dims, proj_dims = c.encoder_dims + c.speaker_embedding_size + c.gst_E, S = s->S;
  AdmitArgs a;
  memset(&a, 0, sizeof(a));
  a.rows = d_rows;
  a.start = s->global;
  std::vector<mb_taco_stream_region> regs;
  stream_regions(s, regs);
  for (const mb_taco_stream_region& g : regs) {
    if (!g.reset) continue;
    if (a.nzero == kMaxZero) return fail(MB_ERR_STATE, "%s: more than %d regions to reset", me, kMaxZero);
    char* p = reinterpret_cast<char*>(g.ptr);
    if (g.kind == MB_TACO_REGION_TILE)  // the slot's 128 bytes in every k-block of a plane [K/64][rows_pad][64] halves
      a.zero[a.nzero++] = RowZero{p, 128, (long long)g.rows * 128, (g.width + 63) / 64, 128};
    else
      a.zero[a.nzero++] = RowZero{p, (long long)g.width * 4, 0, 1, g.width * 4};
  }
  a.src_seq = reinterpret_cast<const float*>(s->base + s->L.pool_seq);
  a.seq = wd + D.seq;
  a.seq_row = (long long)s->Tc * proj_dims;
  a.src_proj = reinterpret_cast<const float*>(s->base + s->L.pool_proj);
  a.proj = wd + D.proj;
  a.proj_row = (long long)s->Tc * Dd;
  a.src_chars = reinterpret_cast<const int32_t*>(s->base + s->L.pool_chars);
  a.chars = reinterpret_cast<int32_t*>(wd + D.ids);
  a.Tc = s->Tc;
  int32_t* drows = reinterpret_cast<int32_t*>(wd + D.rows);
  a.lens = drows;
  a.caps = drows + S;
  a.done = drows + 2 * S;
  a.starts = reinterpret_cast<int*>(s->base + s->L.start);
  a.dmask = reinterpret_cast<uint8_t*>(wd + D.dmask);
  a.S = S;
  a.units = 2 * Dd;
  admit_rows_kernel<<<dim3(16, n), 256, 0, st>>>(a);
  MB_LAUNCH_CHECK("admit_rows_kernel");
  MB_CUDA_CHECK(cudaEventRecord(s->ev_admit, st));
  MB_CUDA_CHECK(cudaStreamWaitEvent((cudaStream_t)stream, s->ev_admit, 0));
  return MB_OK;
}

int mb_tacotron_stream_run(mb_taco_stream* s, int32_t* n_done, int64_t* done_ids, int32_t* done_frames, int64_t* steps_run) {
  const char* me = "mb_tacotron_stream_run";
  if (int rc = stream_check(me, s)) return rc;
  if (!n_done || !done_ids || !done_frames) return fail(MB_ERR_INVALID, "%s: null argument", me);
  *n_done = 0;
  const int S = s->S;
  int busy = 0;
  for (int b = 0; b < S; ++b) busy += s->occupant[b] >= 0;
  cudaStream_t st = s->h->own_stream;
  std::vector<int> fin;
  while (busy && fin.empty()) {
    for (int g = 0; g < kStreamPoll / kGraphSteps; ++g) {
      if (cudaGraphLaunch(s->exec, st) != cudaSuccess) return fail(MB_ERR_CUDA, "%s: cudaGraphLaunch failed", me);
      count_launch(s->per_graph + 1);
    }
    s->global += kStreamPoll;
    s->steps_run += kStreamPoll;
    MB_CUDA_CHECK(cudaMemcpyAsync(s->hdone.data(), s->d_done, sizeof(int32_t) * S, cudaMemcpyDeviceToHost, st));
    MB_CUDA_CHECK(cudaStreamSynchronize(st));
    for (int b = 0; b < S; ++b)
      if (s->occupant[b] >= 0 && s->hdone[b] >= 0) fin.push_back(b);
  }
  int nfree = 0;
  for (int v : s->pool) nfree += v == 0;
  if (nfree < (int)fin.size()) {  // rows a postnet still reads come back once it has finished
    MB_CUDA_CHECK(cudaStreamWaitEvent(st, s->ev_post, 0));
    for (int& v : s->pool)
      if (v == 2) v = 0, ++nfree;
  }
  if (nfree < (int)fin.size())
    return fail(MB_ERR_STATE, "%s: %zu finished rows wait for the postnet: harvest them first", me, s->pending.size());
  const mb_tacotron_config& c = s->h->cfg;
  const int NM = c.n_mels, r = s->r;
  const Ws& D = s->L.dec;
  float* pmel = reinterpret_cast<float*>(s->base + s->L.post_mel);
  float* pattn = reinterpret_cast<float*>(s->base + s->L.post_attn);
  int p = 0;
  for (int b : fin) {
    while (s->pool[p]) ++p;
    const int steps = s->hdone[b] + 1;
    MB_CUDA_CHECK(cudaMemcpyAsync(pmel + (size_t)p * s->nst * r * NM, s->wd + D.mel_all + (size_t)b * s->ring * r * NM,
                                  sizeof(float) * steps * r * NM, cudaMemcpyDeviceToDevice, st));
    MB_CUDA_CHECK(cudaMemcpyAsync(pattn + (size_t)p * s->nst * s->Tc, s->wd + D.scores_all + (size_t)b * s->ring * s->Tc,
                                  sizeof(float) * steps * s->Tc, cudaMemcpyDeviceToDevice, st));
    s->pool[p] = 1;
    s->pool_id[p] = s->occupant[b];
    s->pool_frames[p] = steps * r;
    s->pending.push_back(p);
    done_ids[*n_done] = s->occupant[b];
    done_frames[*n_done] = steps * r;
    ++*n_done;
    s->occupant[b] = -1;
  }
  MB_CUDA_CHECK(cudaEventRecord(s->ev_copied, st));
  if (steps_run) *steps_run = s->steps_run;
  return MB_OK;
}

int mb_tacotron_stream_harvest(mb_taco_stream* s, int32_t n, int32_t frames, float* mel, float* linear, float* attn, void* stream) {
  const char* me = "mb_tacotron_stream_harvest";
  if (int rc = stream_check(me, s)) return rc;
  if (!mel || !linear || !attn) return fail(MB_ERR_INVALID, "%s: null argument", me);
  if (n < 1 || n > s->S || n > (int)s->pending.size())
    return fail(MB_ERR_INVALID, "%s: %d rows (1 to %d, %zu finished)", me, n, s->S, s->pending.size());
  std::vector<int32_t> flen(n);
  int fmax = 0;
  for (int i = 0; i < n; ++i) fmax = std::max(fmax, flen[i] = s->pool_frames[s->pending[i]]);
  if (frames != fmax) return fail(MB_ERR_INVALID, "%s: frames %d, the longest of these rows has %d", me, frames, fmax);
  mb_tacotron* h = s->h;
  const mb_tacotron_config& c = h->cfg;
  const int NM = c.n_mels, r = s->r, Tc = s->Tc;
  cudaStream_t st = (cudaStream_t)stream;
  MB_CUDA_CHECK(cudaStreamWaitEvent(st, s->ev_copied, 0));
  const Ws& Lp = s->L.post;
  float* wp = s->wp;
  float* melc = wp + Lp.ppj2;
  const float* pmel = reinterpret_cast<const float*>(s->base + s->L.post_mel);
  const float* pattn = reinterpret_cast<const float*>(s->base + s->L.post_attn);
  for (int i = 0; i < n; ++i) {
    const int p = s->pending[i];
    MB_CUDA_CHECK(cudaMemcpyAsync(melc + (size_t)i * frames * NM, pmel + (size_t)p * s->nst * r * NM, sizeof(float) * frames * NM,
                                  cudaMemcpyDeviceToDevice, st));
    MB_CUDA_CHECK(cudaMemcpyAsync(attn + (size_t)i * (frames / r) * Tc, pattn + (size_t)p * s->nst * Tc,
                                  sizeof(float) * (frames / r) * Tc, cudaMemcpyDeviceToDevice, st));
  }
  int32_t* d_flen = reinterpret_cast<int32_t*>(s->base + s->L.post_flen);
  if (int rc = upload(d_flen, flen.data(), sizeof(int32_t) * n, st)) return rc;
  if (int rc = run_postnet(h, Lp, wp, melc, n, frames, d_flen, true, st)) return rc;
  const size_t cnt = (size_t)n * NM * frames;
  to_ncl_kernel<<<(unsigned)((cnt + 255) / 256), 256, 0, st>>>(melc, frames, mel, n, NM, frames);
  MB_LAUNCH_CHECK("to_ncl_kernel");
  to_ncl_kernel<<<(unsigned)((cnt + 255) / 256), 256, 0, st>>>(wp + Lp.lin, frames, linear, n, NM, frames);
  MB_LAUNCH_CHECK("to_ncl_kernel");
  MB_CUDA_CHECK(cudaEventRecord(s->ev_post, st));
  for (int i = 0; i < n; ++i) s->pool[s->pending[i]] = 2;
  s->pending.erase(s->pending.begin(), s->pending.begin() + n);
  return MB_OK;
}

int32_t mb_tacotron_stream_regions(const mb_taco_stream* s, mb_taco_stream_region* out, int32_t max) {
  if (!s || !s->h) return fail(MB_ERR_INVALID, "mb_tacotron_stream_regions: null stream");
  std::vector<mb_taco_stream_region> regs;
  stream_regions(s, regs);
  for (int i = 0; out && i < max && i < (int)regs.size(); ++i) out[i] = regs[i];
  return (int32_t)regs.size();
}

void mb_tacotron_stream_close(mb_taco_stream* s) {
  if (!s) return;
  if (s->h && s->h->own_stream) cudaStreamSynchronize(s->h->own_stream);
  if (s->enc_st) cudaStreamSynchronize(s->enc_st);
  if (s->ev_post) cudaEventSynchronize(s->ev_post);
  delete s;
}

}  // extern "C"

// ---- mb_taco_debug: one FP32 kernel of this path per call, launched as the forward launches it ----------------------------
namespace {

GemmArgs debug_gemm_args(const mb_taco_debug_spec& s) {
  GemmArgs a;
  memset(&a, 0, sizeof(a));
  a.nseg = s.nseg;
  for (int j = 0; j < s.nseg && j < kMaxSeg; ++j) a.seg[j] = {s.x[j], s.K[j], s.ld[j], s.shift[j], s.w_off[j], s.w_stride[j]};
  a.W = s.W;
  a.ldw = s.ldw;
  a.bias = s.bias;
  a.M = s.M;
  a.N = s.N;
  a.T = s.T;
  a.act = s.act;
  a.bn_scale = s.bn_scale;
  a.bn_shift = s.bn_shift;
  a.mask = s.mask;
  a.res = s.res;
  a.ldres = s.ldres;
  a.Y = s.y;
  a.ldy = s.ldy;
  a.step_mode = s.step_mode;
  a.step_ptr = s.step_ptr;
  a.step_j = s.step_j;
  a.x_step = s.x_step;
  a.x_first = s.x_first;
  a.mask_step = s.mask_step;
  a.fma_chain = s.fma_chain;
  return a;
}

int debug_check(const mb_taco_debug_spec& s) {
  const char* me = "mb_taco_debug";
  if (s.kind < MB_TACO_DBG_GEMM || s.kind > MB_TACO_DBG_FILL_MASKS_SEEDED) return fail(MB_ERR_INVALID, "%s: bad kind %d", me, s.kind);
  if ((s.row_done == nullptr) != (s.row_caps == nullptr)) return fail(MB_ERR_INVALID, "%s: row_done and row_caps go together", me);
  if (s.row_start && s.ring < 1) return fail(MB_ERR_INVALID, "%s: row_start needs a ring of at least one step", me);
  if (s.row_start && (s.kind == MB_TACO_DBG_STOP_STEP || s.kind == MB_TACO_DBG_STOP_FLAG) && (!s.row_done || s.out[0]))
    return fail(MB_ERR_INVALID, "%s: with row_start the stop rule is per row (row_done, row_caps) and writes no flags", me);
  if (s.kind == MB_TACO_DBG_GEMM || s.kind == MB_TACO_DBG_STOP_STEP) {
    if (s.nseg < 1 || s.nseg > kMaxSeg || !s.W || !s.y || s.M <= 0 || s.N <= 0)
      return fail(MB_ERR_INVALID, "%s: GEMM nseg %d, M %d, N %d or a null operand", me, s.nseg, s.M, s.N);
    for (int j = 0; j < s.nseg; ++j)
      if (!s.x[j] || s.K[j] <= 0) return fail(MB_ERR_INVALID, "%s: segment %d empty", me, j);
    if (s.kind == MB_TACO_DBG_STOP_STEP && (s.N != 1 || (!s.out[0] && !s.row_start) || !s.out[1] || s.n[0] != s.M))
      return fail(MB_ERR_INVALID, "%s: STOP_STEP needs N = 1, flags (unless row_start), ticket and B = M", me);
    return MB_OK;
  }
  for (int i = 0; i < 10; ++i)
    if (s.n[i] < 0) return fail(MB_ERR_INVALID, "%s: n[%d] = %lld", me, i, (long long)s.n[i]);
  if (s.kind == MB_TACO_DBG_LSA_STEP) {
    if (s.n[4] != 256 && s.n[4] != 512) return fail(MB_ERR_INVALID, "%s: LSA_STEP threads %lld", me, (long long)s.n[4]);
    if (s.n[1] < 1 || s.n[1] > lsa_max_chars()) return fail(MB_ERR_INVALID, "%s: Tc = %lld outside [1, %d]", me, (long long)s.n[1], lsa_max_chars());
  }
  if (s.kind == MB_TACO_DBG_LSA_CTX && (s.n[2] <= 0 || s.n[2] % 256 || s.n[1] < 1))
    return fail(MB_ERR_INVALID, "%s: LSA_CTX seq_dim %lld must be a positive multiple of 256", me, (long long)s.n[2]);
  if (s.kind == MB_TACO_DBG_FILL_MASKS_SEEDED && (!s.row_seeds || !s.out[0] || s.n[3] > 1))
    return fail(MB_ERR_INVALID, "%s: FILL_MASKS_SEEDED needs row_seeds, m and dec 0 or 1", me);
  if (s.kind == MB_TACO_DBG_GST_ATTENTION && (s.n[1] < 1 || s.n[1] > 16 || s.n[3] < 1 || s.n[3] > 8 || s.n[2] % s.n[3]))
    return fail(MB_ERR_INVALID, "%s: GST ntok %lld (<= 16), heads %lld (<= 8, dividing E)", me, (long long)s.n[1], (long long)s.n[3]);
  return MB_OK;
}

}  // namespace

extern "C" {

size_t mb_taco_debug_workspace_bytes(const mb_taco_debug_spec* spec) {
  return spec && debug_check(*spec) == MB_OK ? 256 : 0;
}

int mb_taco_debug(const mb_taco_debug_spec* spec, void* workspace, size_t workspace_bytes, void* stream, char* report,
                  size_t report_len) {
  if (!spec) return fail(MB_ERR_INVALID, "mb_taco_debug: null spec");
  const mb_taco_debug_spec& s = *spec;
  int rc = debug_check(s);
  if (rc != MB_OK) return rc;
  if ((rc = bind("mb_taco_debug", workspace, workspace_bytes, mb_taco_debug_workspace_bytes(spec)))) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  const int64_t* n = s.n;
  auto fin = [&](int i) { return reinterpret_cast<const float*>(s.in[i]); };
  auto fout = [&](int i) { return reinterpret_cast<float*>(s.out[i]); };
  auto hout = [&](int i) { return reinterpret_cast<__half*>(s.out[i]); };
  auto blocks = [](int64_t count) { return (unsigned)((count + 255) / 256); };
  GemmLaunchInfo info{"", 0, 1, 256, 0};
  switch (s.kind) {
    case MB_TACO_DBG_GEMM:
      TK(launch_gemm(debug_gemm_args(s), st, &info));
      break;
    case MB_TACO_DBG_PRENET: {
      PrenetArgs pa;
      memset(&pa, 0, sizeof(pa));
      pa.x = fin(0);
      pa.x_first = fin(1);
      pa.W1 = fin(2);
      pa.b1 = fin(3);
      pa.W2 = fin(4);
      pa.b2 = fin(5);
      pa.m1 = reinterpret_cast<const uint8_t*>(s.in[6]);
      pa.m2 = reinterpret_cast<const uint8_t*>(s.in[7]);
      pa.y = fout(0);
      pa.s_hi = hout(1);
      pa.s_lo = hout(2);
      pa.B = (int)n[0];
      pa.K = (int)n[1];
      pa.H = (int)n[2];
      pa.ldy = (int)n[3];
      pa.x_ld = n[4];
      pa.x_step = n[5];
      pa.mask_step = n[6];
      pa.s_k0 = (int)n[7];
      pa.s_rows_pad = (int)n[8];
      pa.step_ptr = s.step_ptr;
      pa.step_j = s.step_j;
      pa.row_start = s.row_start;
      pa.ring = s.ring;
      TK(launch_prenet_fused(pa, st));
      info = {"prenet_fused", (pa.B + 3) / 4, 1, 512, 0};
      break;
    }
    case MB_TACO_DBG_GRU_CELL:
      TK(launch_gru_cell(fin(0), (int)n[2], fin(1), fout(0), (int)n[3], fout(1), (int)n[4], (int)n[0], (int)n[1], st));
      info = {"gru_cell", (int)blocks(n[0] * n[1]), 1, 256, 0};
      break;
    case MB_TACO_DBG_LSTM_CELL:
      TK(launch_lstm_cell(fin(0), fout(0), fout(1), fout(2), (int)n[0], (int)n[1], st));
      info = {"lstm_cell", (int)blocks(n[0] * n[1]), 1, 256, 0};
      break;
    case MB_TACO_DBG_HIGHWAY:
      TK(launch_highway(fin(0), fout(0), (int)n[0], (int)n[1], st));
      info = {"highway", (int)blocks(n[0] * n[1]), 1, 256, 0};
      break;
    case MB_TACO_DBG_MAXPOOL2:
      TK(launch_maxpool2(fin(0), fout(0), (int)n[0], (int)n[1], (int)n[2], st));
      info = {"maxpool2", (int)blocks(n[0] * n[1] * n[2]), 1, 256, 0};
      break;
    case MB_TACO_DBG_EMBEDDING:
      TK(launch_embedding(reinterpret_cast<const int32_t*>(s.in[0]), fin(1), fout(0), (int)n[0], (int)n[1], st));
      info = {"embedding", (int)blocks(n[0] * n[1]), 1, 256, 0};
      break;
    case MB_TACO_DBG_COPY_COLS:
      TK(launch_copy_cols(fin(0), (int)n[2], (int)n[3], fout(0), (int)n[4], (int)n[5], (int)n[0], (int)n[1], st));
      info = {"copy_cols", (int)blocks(n[0] * n[1]), 1, 256, 0};
      break;
    case MB_TACO_DBG_LSA_STEP: {
      const int B = (int)n[0], Tc = (int)n[1], threads = (int)n[4];
      const size_t smem = lsa_step_smem_bytes(Tc);
      MB_CUDA_CHECK(lsa_step_prepare(Tc));
      MB_CUDA_CHECK(launch_pdl2(lsa_step_kernel, dim3(B), dim3(threads), smem, st, fin(0), fin(1), fin(2), (int)n[2],
                                reinterpret_cast<const int32_t*>(s.in[3]), fout(0), fin(4), fin(5), fin(6), fin(7), fout(1),
                                (int)n[3], fout(2), Tc, s.step_ptr, s.step_j, fin(8), fin(9), fin(10), s.row_len, s.row_start,
                                s.ring));
      MB_LAUNCH_CHECK("lsa_step_kernel");
      info = {"lsa_step", B, 1, threads, smem};
      break;
    }
    case MB_TACO_DBG_LSA_CTX: {
      const int B = (int)n[0], Tc = (int)n[1], seq_dim = (int)n[2];
      const size_t smem = sizeof(float) * Tc;
      MB_CUDA_CHECK(launch_pdl2(lsa_ctx_kernel, dim3(seq_dim / 256, B), dim3(256), smem, st, fin(0), (int)n[3], fin(1), seq_dim, Tc,
                                fout(0), s.step_ptr, s.step_j, hout(1), hout(2), hout(3), hout(4), (int)n[4], s.row_len, s.row_start,
                                s.ring));
      MB_LAUNCH_CHECK("lsa_ctx_kernel");
      info = {"lsa_ctx", seq_dim / 256, B, 256, smem};
      break;
    }
    case MB_TACO_DBG_GST_ATTENTION: {
      const int B = (int)n[0], E = (int)n[2], heads = (int)n[3];
      gst_attention_kernel<<<B, 256, 0, st>>>(fin(0), fin(1), fin(2), (int)n[1], fout(0), E, heads, 1.0f / sqrtf((float)(E / heads)));
      MB_LAUNCH_CHECK("gst_attention_kernel");
      info = {"gst_attention", B, 1, 256, 0};
      break;
    }
    case MB_TACO_DBG_STOP_STEP: {
      const int B = (int)n[0];
      stop_step_kernel<<<B, 256, 0, st>>>(debug_gemm_args(s), B, s.fval, (int)n[1], reinterpret_cast<int*>(s.out[0]), s.step_ptr,
                                          s.step_j, reinterpret_cast<unsigned int*>(s.out[1]), s.row_done, s.row_caps, s.row_start);
      MB_LAUNCH_CHECK("stop_step_kernel");
      info = {"stop_step", B, 1, 256, 0};
      break;
    }
    case MB_TACO_DBG_STOP_FLAG:
      stop_flag_kernel<<<1, 32, 0, st>>>(fin(0), (int)n[0], s.fval, (int)n[1], reinterpret_cast<int*>(s.out[0]), s.step_ptr, s.step_j,
                                         s.row_done, s.row_caps, s.row_start);
      MB_LAUNCH_CHECK("stop_flag_kernel");
      info = {"stop_flag", 1, 1, 32, 0};
      break;
    case MB_TACO_DBG_FILL_MASKS:
      fill_masks_kernel<<<blocks(n[0]), 256, 0, st>>>(reinterpret_cast<uint8_t*>(s.out[0]), (size_t)n[0], s.seed, (uint32_t)n[1],
                                                       s.step_ptr);
      MB_LAUNCH_CHECK("fill_masks_kernel");
      info = {"fill_masks", (int)blocks(n[0]), 1, 256, 0};
      break;
    case MB_TACO_DBG_FILL_MASKS_STEPS:
      fill_masks_steps_kernel<<<blocks(n[0] * n[1]), 256, 0, st>>>(reinterpret_cast<uint8_t*>(s.out[0]), (size_t)n[0], (int)n[1],
                                                                    s.seed);
      MB_LAUNCH_CHECK("fill_masks_steps_kernel");
      info = {"fill_masks_steps", (int)blocks(n[0] * n[1]), 1, 256, 0};
      break;
    case MB_TACO_DBG_PACK_MELPROJ:
      pack_melproj_kernel<<<blocks(n[2] * n[0] * n[3]), 256, 0, st>>>(fin(0), fout(0), (int)n[0], (int)n[1], (int)n[2], (int)n[3]);
      MB_LAUNCH_CHECK("pack_melproj_kernel");
      info = {"pack_melproj", (int)blocks(n[2] * n[0] * n[3]), 1, 256, 0};
      break;
    case MB_TACO_DBG_TO_NCL:
      to_ncl_kernel<<<blocks(n[1] * n[2] * n[3]), 256, 0, st>>>(fin(0), (int)n[0], fout(0), (int)n[1], (int)n[2], (int)n[3]);
      MB_LAUNCH_CHECK("to_ncl_kernel");
      info = {"to_ncl", (int)blocks(n[1] * n[2] * n[3]), 1, 256, 0};
      break;
    case MB_TACO_DBG_BN_FOLD:
      bn_fold_kernel<<<blocks(n[0]), 256, 0, st>>>(fin(0), fin(1), fin(2), fin(3), fout(0), fout(1), (int)n[0]);
      MB_LAUNCH_CHECK("bn_fold_kernel");
      info = {"bn_fold", (int)blocks(n[0]), 1, 256, 0};
      break;
    case MB_TACO_DBG_FILL_MASKS_SEEDED: {
      const int64_t count = 2 * n[0] * n[1] * n[2];
      fill_masks_seeded_kernel<<<blocks(count), 256, 0, st>>>(reinterpret_cast<uint8_t*>(s.out[0]), (int)n[0], (int)n[1], (int)n[2],
                                                              s.row_seeds, (int)n[3]);
      MB_LAUNCH_CHECK("fill_masks_seeded_kernel");
      info = {"fill_masks_seeded", (int)blocks(count), 1, 256, 0};
      break;
    }
  }
  if (report && report_len)
    snprintf(report, report_len, "kernel=%s grid=%d,%d block=%d smem=%zu\n", info.kernel, info.grid_x, info.grid_y, info.block,
             info.smem);
  return MB_OK;
}

}  // extern "C"
