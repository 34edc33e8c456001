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
#include <map>
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
                                                       const float* __restrict__ Wq, const float* __restrict__ bq) {
  extern __shared__ float sm[];
  scores_out += (size_t)step_index(step_ptr, step_j) * Tc;  // this decoder step's row of the alignment matrix
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
  for (int t = tid; t < Tc; t += blockDim.x) {
    const float u = (s_part[t * 4 + 0] + s_part[t * 4 + 1]) + (s_part[t * 4 + 2] + s_part[t * 4 + 3]);
    s_u[t] = chars[(size_t)b * Tc + t] != 0 ? u : 0.f;  // u * (chars != 0): padded positions score exp(0)
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
  for (int f = tid; f < seq_dim; f += blockDim.x) {
    float a = 0.f;
    const float* sp = seq + (size_t)b * Tc * seq_dim + f;
    for (int t = 0; t < Tc; ++t) a = fmaf(s_u[t], sp[(size_t)t * seq_dim], a);
    ctx[(size_t)b * seq_dim + f] = a;
  }
}

// context = scores @ encoder_seq (tacotron.py:104 via lsa.py:40): ctx[b][f] = sum_t scores[b][t] seq[b][t][f].
// grid (seq_dim / 256, B): 64 float4 feature lanes x 4 interleaved t-groups per CTA, partials reduced in smem.
// The whole encoder sequence (B x Tc x 1024 fp32) is re-read every decoder step from L2: the kernel needs many
// 16-byte loads in flight, which one CTA per batch row cannot provide.
__global__ void __launch_bounds__(256) lsa_ctx_kernel(const float* __restrict__ scores, int scores_ld, const float* __restrict__ seq,
                                                      int seq_dim, int Tc, float* __restrict__ ctx, const int* step_ptr,
                                                      int step_j, __half* sa_hi, __half* sa_lo, __half* sb_hi, __half* sb_lo,
                                                      int s_rows_pad) {
  __shared__ float4 part[4][64];
  extern __shared__ float s_sc[];
  asm volatile("griddepcontrol.wait;" ::: "memory");
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  const int b = blockIdx.y, f4 = blockIdx.x * 64 + (threadIdx.x & 63), tg = threadIdx.x >> 6;
  const float* sc = scores + (size_t)step_index(step_ptr, step_j) * Tc + (size_t)b * scores_ld;
  for (int t = threadIdx.x; t < Tc; t += 256) s_sc[t] = sc[t];
  __syncthreads();
  float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
  const float4* sp = reinterpret_cast<const float4*>(seq + (size_t)b * Tc * seq_dim) + f4;
  const int q4 = seq_dim >> 2;
#pragma unroll 6
  for (int t = tg; t < Tc; t += 4) {
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

// decoder step si = (step_ptr ? *step_ptr : 0) + step_j; frame t = si * r; flags[si] = stop rule of tacotron.py:275
__global__ void stop_flag_kernel(const float* stopv, int B, float min_stop_token, int r, int* flags, const int* step_ptr,
                                 int step_j) {
  if (threadIdx.x == 0 && blockIdx.x == 0) {
    const int si = step_index(step_ptr, step_j);
    bool all = true;
    for (int b = 0; b < B; ++b) all = all && (stopv[b] * 10.f > min_stop_token);
    flags[si] = (all && si * r > 10) ? 1 : 0;
  }
}

// stop projection (sigmoid(w . [x | ctx] + b), tacotron.py:131-133) of one batch row per CTA, then - in the CTA that takes the
// last ticket - the stop rule over all rows.  Same summation order as rowdot_kernel.
__global__ void __launch_bounds__(256) stop_step_kernel(const GemmArgs a, int B, float min_stop_token, int r, int* flags,
                                                        const int* step_ptr, int step_j, unsigned int* ticket) {
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
    const int si = step_index(step_ptr, step_j);
    bool all = true;
    for (int b = 0; b < B; ++b) all = all && (__ldcg(a.Y + (size_t)b * a.ldy) * 10.f > min_stop_token);
    flags[si] = (all && si * r > 10) ? 1 : 0;
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

}  // namespace
}  // namespace taco
}  // namespace mb

// =================================================================================================
using namespace mb;
using namespace mb::taco;

struct mb_tacotron {
  mb_tacotron_config cfg{};
  struct Slot {
    size_t off;
    size_t n;
    bool set;
  };
  std::map<std::string, Slot> slots;
  size_t total = 0;
  float* arena = nullptr;
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

void slot(mb_tacotron* h, const std::string& name, size_t n) {
  h->slots[name] = {h->total, n, false};
  h->total += align_up(n, 64);
}

float* P(const mb_tacotron* h, const std::string& name) {
  auto it = h->slots.find(name);
  return it == h->slots.end() ? nullptr : h->arena + it->second.off;
}

void cbhg_slots(mb_tacotron* h, const std::string& p, int K, int cin, int ch, int p0, int p1, int nh) {
  auto bnconv = [&](const std::string& n, int ci, int co, int k) {
    slot(h, n + ".conv.weight", (size_t)co * ci * k);
    for (const char* leaf : {".bnorm.weight", ".bnorm.bias", ".bnorm.running_mean", ".bnorm.running_var"}) slot(h, n + leaf, co);
    slot(h, n + ".bn_scale", co);  // derived at finalize
    slot(h, n + ".bn_shift", co);
  };
  for (int i = 0; i < K; ++i) bnconv(p + ".conv1d_bank." + std::to_string(i), cin, ch, i + 1);
  bnconv(p + ".conv_project1", K * ch, p0, 3);
  bnconv(p + ".conv_project2", p0, p1, 3);
  if (p1 != ch) slot(h, p + ".pre_highway.weight", (size_t)ch * p1);
  // derived: tensor-core images of the large-M GEMMs (cbhg_gemm), packed on first use
  for (int i = 0; i < K; ++i) slot(h, p + ".conv1d_bank." + std::to_string(i) + ".bigw", tc_big_weight_bytes(ch, i + 1, cin) / 4);
  slot(h, p + ".conv_project1.bigw", tc_big_weight_bytes(p0, 3, K * ch) / 4);
  slot(h, p + ".conv_project2.bigw", tc_big_weight_bytes(p1, 3, p0) / 4);
  if (p1 != ch) slot(h, p + ".pre_highway.bigw", tc_big_weight_bytes(ch, 1, p1) / 4);
  for (int i = 0; i < nh; ++i) slot(h, p + ".highways." + std::to_string(i) + ".bigw", tc_big_weight_bytes(2 * ch, 1, ch) / 4);
  for (const char* sfx : {"", "_reverse"}) slot(h, p + ".rnn.ih" + sfx + ".bigw", tc_big_weight_bytes(3 * (ch / 2), 1, ch) / 4);
  for (int i = 0; i < nh; ++i) {
    const std::string q = p + ".highways." + std::to_string(i);
    slot(h, q + ".W1.weight", (size_t)ch * ch);
    slot(h, q + ".W1.bias", ch);
    slot(h, q + ".W2.weight", (size_t)ch * ch);
    slot(h, q + ".W2.bias", ch);
    slot(h, q + ".W12", (size_t)2 * ch * ch);  // derived: [W1; W2] stacked
    slot(h, q + ".b12", (size_t)2 * ch);
  }
  for (const char* sfx : {"", "_reverse"}) {
    slot(h, p + ".rnn.weight_ih_l0" + sfx, (size_t)3 * (ch / 2) * ch);
    slot(h, p + ".rnn.weight_hh_l0" + sfx, (size_t)3 * (ch / 2) * (ch / 2));
    slot(h, p + ".rnn.bias_ih_l0" + sfx, (size_t)3 * (ch / 2));
    slot(h, p + ".rnn.bias_hh_l0" + sfx, (size_t)3 * (ch / 2));
    // derived: tensor-core images of W_hh (gates r|z|n interleaved per 8 units) + tile-order b_hh
    slot(h, p + ".rnn.hh" + sfx + ".tcw", tc_gated_weight_bytes(ch / 2, ch / 2) / 4);
    slot(h, p + ".rnn.hh" + sfx + ".tcb", (size_t)4 * (ch / 2));
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
  size_t total;
};

Ws ws_layout(const mb_tacotron_config& c, int B, int Tc, int steps, int r) {
  Ws L{};
  size_t o = 0;
  auto take = [&](size_t n) {
    size_t q = o;
    o += align_up(n, 64);
    return q;
  };
  const size_t Me = (size_t)B * Tc, Mp = (size_t)B * steps;
  const int E = c.encoder_dims, PD = c.postnet_dims, proj_dims = E + c.speaker_embedding_size + c.gst_E;
  L.ids = take(Me);
  L.emb = take(Me * c.embed_dims);
  L.m_enc = take((2 * Me * E + 3) / 4 + 64);  // uint8 masks
  L.p1 = take(Me * E);
  L.x0 = take(Me * E);
  L.bank = take(Me * c.encoder_K * E);
  L.pool = take(Me * c.encoder_K * E);
  L.pj1 = take(Me * E);
  L.y = take(Me * E);
  L.hw12 = take(Me * 2 * E);
  L.gi_f = take(Me * 3 * (E / 2));
  L.gi_b = take(Me * 3 * (E / 2));
  L.gh = take((size_t)2 * B * 3 * (PD / 2));
  L.hst = take((size_t)2 * B * (PD / 2));
  L.seq = take(Me * proj_dims);
  L.proj = take(Me * c.decoder_dims);
  L.style_q = take((size_t)B * c.gst_E);
  L.style = take((size_t)B * c.gst_E);
  L.attn_h = take((size_t)B * c.decoder_dims);
  L.h1 = take((size_t)B * c.lstm_dims);
  L.c1 = take((size_t)B * c.lstm_dims);
  L.h2 = take((size_t)B * c.lstm_dims);
  L.c2 = take((size_t)B * c.lstm_dims);
  L.ctx = take((size_t)B * proj_dims);
  L.cum = take(Me);
  L.dp1 = take((size_t)B * 2 * c.decoder_dims);
  L.dp2 = take((size_t)B * 2 * c.decoder_dims);
  L.dgi = take((size_t)B * 3 * c.decoder_dims);
  L.dgh = take((size_t)B * 3 * c.decoder_dims);
  L.pq = take((size_t)B * c.decoder_dims);
  L.x = take((size_t)B * c.lstm_dims);
  L.gates = take((size_t)B * 4 * c.lstm_dims);
  L.a_hi = take(tc_skinny_act_bytes(B > 128 ? 128 : B, 2 * c.lstm_dims) / 4);
  L.a_lo = take(tc_skinny_act_bytes(B > 128 ? 128 : B, 2 * c.lstm_dims) / 4);
  L.ah_hi = take(2 * tc_skinny_act_bytes(B > 128 ? 128 : B, c.decoder_dims) / 4);  // attention-GRU state tiles, 2 parities
  L.ah_lo = take(2 * tc_skinny_act_bytes(B > 128 ? 128 : B, c.decoder_dims) / 4);
  {
    // operand tiles written by the producing kernels (fused act_split): P1 [ctx | prenet], P2 [ctx | attn_h], P3 / P4 [x | h] of the
    // two LSTMs (two step parities each), P5 [x]; hi and lo of each; zeroed with the attention-GRU tiles at the start of generate()
    const int Bc = B > 128 ? 128 : B;
    const FusedSplit f = fused_split_layout(Bc, proj_dims, c.decoder_dims, c.lstm_dims);
    L.fsp = take(f.total / 4);
  }
  // partial GEMM results computed a step early on the side stream: W_hh h of the two LSTMs, W_ih[:, ctx] ctx of the attention GRU
  L.pre1 = take((size_t)B * 4 * c.lstm_dims);
  L.pre2 = take((size_t)B * 4 * c.lstm_dims);
  L.gic = take((size_t)B * 3 * c.decoder_dims);
  L.stopv = take(B);
  L.step = take(64);
  const int nst = (steps + r - 1) / r;
  L.flags = take(nst);
  L.dmask = take(((size_t)nst * 2 * B * 2 * c.decoder_dims + 3) / 4 + 64);  // PreNet dropout masks of every decoder step
  L.mel_all = take(Mp * c.n_mels + (size_t)r * c.n_mels);
  L.scores_all = take((size_t)B * nst * Tc);
  L.pbank = take(Mp * c.postnet_K * PD);
  L.ppool = take(Mp * c.postnet_K * PD);
  L.ppj1 = take(Mp * PD);
  L.ppj2 = take(Mp * c.n_mels);
  L.py = take(Mp * PD);
  L.phw12 = take(Mp * 2 * PD);
  L.pgi_f = take(Mp * 3 * (PD / 2));
  L.pgi_b = take(Mp * 3 * (PD / 2));
  L.pgh = take((size_t)2 * B * 3 * (PD / 2));
  L.phst = take((size_t)2 * B * (PD / 2));
  L.pout = take(Mp * PD);
  L.lin = take(Mp * c.n_mels);
  {  // im2col operand planes of the large-M tensor-core GEMMs: the widest layer is conv_project1 (3 taps x K * ch)
    const size_t enc = tc_big_act_bytes((int)Me, 3, c.encoder_K * E), post = tc_big_act_bytes((int)Mp, 3, c.postnet_K * PD);
    L.big_bytes = enc > post ? enc : post;
    L.big_hi = take(L.big_bytes / 4);
    L.big_lo = take(L.big_bytes / 4);
  }
  L.total = o;
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
// else the FP32 FFMA kernels.  MB_TACO_CONV_TC=0 disables the tensor-core route.
int cbhg_gemm(mb_tacotron* h, const std::string& key, const GemmArgs& a, cudaStream_t st, const BigWs& bw) {
  static const bool env = [] {
    const char* e = getenv("MB_TACO_CONV_TC");
    return e ? atoi(e) != 0 : true;
  }();
  bool ok = env && bw.hi && a.M >= 512 && a.N % 4 == 0 && a.nseg >= 1 && a.nseg <= kMaxSeg && !a.mask && !a.step_mode &&
            a.act != ACT_SIGMOID && a.act != ACT_TANH && h->slots.count(key + ".bigw") && (a.ldy % 4) == 0 &&
            (!a.res || (a.ldres % 4) == 0);
  const int K = a.seg[0].K;
  for (int s = 1; ok && s < a.nseg; ++s) ok = a.seg[s].K == K;
  if (ok) ok = tc_big_act_bytes(a.M, a.nseg, K) <= bw.bytes && tc_big_weight_bytes(a.N, a.nseg, K) / 4 <= h->slots[key + ".bigw"].n;
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
    float mx;
    memcpy(&mx, &hmax, sizeof(float));
    int e = 0;
    if (mx > 0.f && mx < 3.0e38f) frexpf(mx, &e);
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
    q.scale = ldexpf(1.f, 12 - e);
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

// CBHG (sublayer/cbhg.py:42-79) on x [B*T][cin] channels-last -> out [B*T][ch] written at out (ld ldout)
int run_cbhg(mb_tacotron* h, const std::string& p, int K, int cin, int ch, int p0, int p1, int nh, const float* x, int B,
             int T, float* bank, float* pool, float* pj1, float* y, float* hw12, float* gi_f, float* gi_b, float* gh,
             float* hst, float* out, int ldout, cudaStream_t st, float* tc_hi = nullptr, float* tc_lo = nullptr,
             size_t tc_bytes = 0, const BigWs& bw = BigWs()) {
  const int M = B * T;
#define CG(key, args)                                 \
  do {                                                \
    int _rc = cbhg_gemm(h, (key), (args), st, bw);    \
    if (_rc != MB_OK) return _rc;                     \
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
      TK(launch_tc_gru(g, st));
    }
    return MB_OK;
  }
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

// absmax -> power-of-two scale (max |w| lands in [2^11, 2^12): the lo parts of the fp16 split stay clear of the
// subnormal range) -> hi/lo tile images "<name>.tcw" + tile-order bias "<name>.tcb".  Synchronises the stream.
int tc_prepare(mb_tacotron* h, const std::string& name, const float* w0, int K0, const float* w1, int K1, const float* b0,
               const float* b1, int N, int lstm_H, cudaStream_t st) {
  unsigned int* dmax = reinterpret_cast<unsigned int*>(P(h, "scratch.absmax.tcb"));
  MB_CUDA_CHECK(cudaMemsetAsync(dmax, 0, sizeof(unsigned int), st));
  TK(tc_skinny_absmax(w0, (size_t)N * K0, dmax, st));
  if (w1) TK(tc_skinny_absmax(w1, (size_t)N * K1, dmax, st));
  unsigned int hmax = 0;
  MB_CUDA_CHECK(cudaMemcpyAsync(&hmax, dmax, sizeof(hmax), cudaMemcpyDeviceToHost, st));
  MB_CUDA_CHECK(cudaStreamSynchronize(st));
  float mx;
  memcpy(&mx, &hmax, sizeof(float));
  int e = 0;
  if (mx > 0.f && mx < 3.0e38f) frexpf(mx, &e);  // mx = f * 2^e, f in [0.5, 1)
  const float scale = ldexpf(1.f, 12 - e);
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
  slot(h, "scratch.absmax.tcb", 64);  // device scratch of the weight-image packers (derived slot: no cudaMalloc after create)
  slot(h, "encoder.embedding.weight", (size_t)c.num_chars * c.embed_dims);
  slot(h, "encoder.pre_net.fc1.weight", (size_t)E * c.embed_dims);
  slot(h, "encoder.pre_net.fc1.bias", E);
  slot(h, "encoder.pre_net.fc2.weight", (size_t)E * E);
  slot(h, "encoder.pre_net.fc2.bias", E);
  cbhg_slots(h, "encoder.cbhg", c.encoder_K, E, E, E, E, c.num_highways);
  slot(h, "encoder_proj.weight", (size_t)D * proj_dims);
  slot(h, "gst.const_enc", c.gst_E / 2);  // ReferenceEncoder(zeros): input independent, folded by the host
  slot(h, "gst.stl.embed", (size_t)c.gst_tokens * (c.gst_E / c.gst_heads));
  slot(h, "gst.stl.attention.W_query.weight", (size_t)c.gst_E * (c.gst_E / 2 + c.speaker_embedding_size));
  slot(h, "gst.stl.attention.W_key.weight", (size_t)c.gst_E * (c.gst_E / c.gst_heads));
  slot(h, "gst.stl.attention.W_value.weight", (size_t)c.gst_E * (c.gst_E / c.gst_heads));
  slot(h, "gst.tanh_embed", (size_t)c.gst_tokens * (c.gst_E / c.gst_heads));  // derived
  slot(h, "gst.keys", (size_t)c.gst_tokens * c.gst_E);
  slot(h, "gst.values", (size_t)c.gst_tokens * c.gst_E);
  slot(h, "decoder.prenet.fc1.weight", (size_t)2 * D * c.n_mels);
  slot(h, "decoder.prenet.fc1.bias", 2 * D);
  slot(h, "decoder.prenet.fc2.weight", (size_t)2 * D * 2 * D);
  slot(h, "decoder.prenet.fc2.bias", 2 * D);
  slot(h, "decoder.attn_net.conv.weight", ATT_F * ATT_K);
  slot(h, "decoder.attn_net.conv.bias", ATT_F);
  slot(h, "decoder.attn_net.L.weight", ATT_D * ATT_F);
  slot(h, "decoder.attn_net.W.weight", ATT_D * ATT_D);
  slot(h, "decoder.attn_net.W.bias", ATT_D);
  slot(h, "decoder.attn_net.v.weight", ATT_D);
  slot(h, "decoder.attn_rnn.weight_ih", (size_t)3 * D * (proj_dims + 2 * D));
  slot(h, "decoder.attn_rnn.weight_hh", (size_t)3 * D * D);
  slot(h, "decoder.attn_rnn.bias_ih", 3 * D);
  slot(h, "decoder.attn_rnn.bias_hh", 3 * D);
  slot(h, "decoder.attn_rnn.ih.tcw", tc_skinny_weight_bytes(3 * D, proj_dims + 2 * D) / 4);  // derived tensor-core images
  slot(h, "decoder.attn_rnn.ih.tcb", 3 * D);
  slot(h, "decoder.attn_rnn.hh.tcw", tc_gated_weight_bytes(D, D) / 4);
  slot(h, "decoder.attn_rnn.hh.tcb", 4 * D);
  slot(h, "decoder.rnn_input.weight", (size_t)c.lstm_dims * (proj_dims + D));
  slot(h, "decoder.rnn_input.bias", c.lstm_dims);
  for (const char* n : {"decoder.res_rnn1", "decoder.res_rnn2"}) {
    slot(h, std::string(n) + ".weight_ih", (size_t)4 * c.lstm_dims * c.lstm_dims);
    slot(h, std::string(n) + ".weight_hh", (size_t)4 * c.lstm_dims * c.lstm_dims);
    slot(h, std::string(n) + ".bias_ih", 4 * c.lstm_dims);
    slot(h, std::string(n) + ".bias_hh", 4 * c.lstm_dims);
    slot(h, std::string(n) + ".bias_sum", 4 * c.lstm_dims);  // derived: b_hh + b_ih
    slot(h, std::string(n) + ".tcw", tc_skinny_weight_bytes(4 * c.lstm_dims, 2 * c.lstm_dims) / 4);  // derived: hi/lo tiles
    slot(h, std::string(n) + ".tcb", 4 * c.lstm_dims);                                                // derived: tile-order bias
  }
  slot(h, "decoder.mel_proj.weight", (size_t)c.n_mels * c.max_r * c.lstm_dims);
  slot(h, "decoder.mel_proj.packed", (size_t)c.n_mels * c.max_r * c.lstm_dims);  // derived for the current r
  slot(h, "decoder.mel_proj.tcw", tc_skinny_weight_bytes(c.n_mels * c.max_r, c.lstm_dims) / 4);  // derived (current r)
  slot(h, "decoder.mel_proj.tcb", (size_t)c.n_mels * c.max_r + 32);
  slot(h, "decoder.rnn_input.tcw", tc_skinny_weight_bytes(c.lstm_dims, proj_dims + D) / 4);     // derived
  slot(h, "decoder.rnn_input.tcb", c.lstm_dims);
  slot(h, "decoder.stop_proj.weight", (size_t)(proj_dims + c.lstm_dims));
  slot(h, "decoder.stop_proj.bias", 1);
  cbhg_slots(h, "postnet", c.postnet_K, c.n_mels, c.postnet_dims, c.postnet_dims, c.n_mels, c.num_highways);
  slot(h, "post_proj.weight", (size_t)c.n_mels * c.postnet_dims);
  slot(h, "post_proj.bigw", tc_big_weight_bytes(c.n_mels, 1, c.postnet_dims) / 4);
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

size_t mb_tacotron_arena_bytes(const mb_tacotron* h) { return h ? h->total * sizeof(float) : 0; }

int mb_tacotron_set_arena(mb_tacotron* h, void* arena, size_t bytes) {
  if (!h || !arena) return fail(MB_ERR_INVALID, "mb_tacotron_set_arena: null argument");
  if (bytes < mb_tacotron_arena_bytes(h)) return fail(MB_ERR_WORKSPACE, "mb_tacotron_set_arena: arena too small");
  if (((uintptr_t)arena & 255) != 0) return fail(MB_ERR_INVALID, "mb_tacotron_set_arena: arena must be 256-byte aligned");
  h->arena = (float*)arena;
  // a new arena holds none of the derived images: forget every lazily packed tensor-core image and its scale
  h->big_packed.clear();
  h->tc_inv_scale.clear();
  h->packed_r = 0;
  h->finalized = false;
  return MB_OK;
}

int mb_tacotron_set_weight(mb_tacotron* h, const char* name, const float* w, const int64_t* dims, int32_t ndim,
                           void* stream) {
  if (!h || !name || !w) return fail(MB_ERR_INVALID, "mb_tacotron_set_weight: null argument");
  if (!h->arena) return fail(MB_ERR_STATE, "mb_tacotron_set_weight: call mb_tacotron_set_arena first");
  auto it = h->slots.find(name);
  if (it == h->slots.end()) return fail(MB_ERR_INVALID, "mb_tacotron_set_weight: unknown tensor '%s'", name);
  size_t n = 1;
  for (int i = 0; i < ndim; ++i) n *= (size_t)dims[i];
  if (n != it->second.n)
    return fail(MB_ERR_INVALID, "mb_tacotron_set_weight: %s has %zu elements, expected %zu", name, n, it->second.n);
  MB_CUDA_CHECK(cudaMemcpyAsync(h->arena + it->second.off, w, n * sizeof(float), cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
  it->second.set = true;
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
  auto derived = [](const std::string& n) {
    return n.find(".bn_scale") != std::string::npos || n.find(".bn_shift") != std::string::npos ||
           n.find(".W12") != std::string::npos || n.find(".b12") != std::string::npos || n == "gst.tanh_embed" ||
           n == "gst.keys" || n == "gst.values" || n.find(".bias_sum") != std::string::npos || n.find(".tcw") != std::string::npos ||
           n.find(".tcb") != std::string::npos || n.find(".tcw") != std::string::npos || n.find(".bigw") != std::string::npos ||
           n == "decoder.mel_proj.packed";
  };
  for (auto& kv : h->slots)
    if (!kv.second.set && !derived(kv.first))
      return fail(MB_ERR_STATE, "mb_tacotron_finalize: tensor %s was never set", kv.first.c_str());
  // fold eval BatchNorm into scale/shift
  for (auto& kv : h->slots) {
    const std::string& n = kv.first;
    const size_t pos = n.find(".bnorm.weight");
    if (pos == std::string::npos) continue;
    const std::string base = n.substr(0, pos);
    const int co = (int)kv.second.n;
    bn_fold_kernel<<<(co + 255) / 256, 256, 0, st>>>(P(h, base + ".bnorm.weight"), P(h, base + ".bnorm.bias"),
                                                     P(h, base + ".bnorm.running_mean"), P(h, base + ".bnorm.running_var"),
                                                     P(h, base + ".bn_scale"), P(h, base + ".bn_shift"), co);
    MB_LAUNCH_CHECK("bn_fold_kernel");
  }
  // stacked highway weights [W1; W2]
  for (auto& kv : h->slots) {
    const std::string& n = kv.first;
    const size_t pos = n.find(".W1.weight");
    if (pos == std::string::npos) continue;
    const std::string base = n.substr(0, pos);
    const size_t nn = kv.second.n;
    const size_t ch = h->slots[base + ".W1.bias"].n;
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
  const int nst = (steps + r - 1) / r;
  return ws_layout(h->cfg, B, Tc, nst * r, r).total * sizeof(float) + 256;
}

int mb_tacotron_generate(mb_tacotron* h, const int32_t* chars, const float* spk, int32_t B, int32_t Tc, int32_t steps,
                         int32_t r, int32_t style_idx, float min_stop_token, const uint8_t* enc_masks,
                         const uint8_t* dec_masks, uint64_t seed, float* mel_out, float* linear_out, float* attn_out,
                         int32_t* frames_out_host, void* workspace, size_t workspace_bytes, void* stream) {
  if (!h || !chars || !spk || !mel_out || !linear_out || !frames_out_host || !workspace)
    return fail(MB_ERR_INVALID, "mb_tacotron_generate: null argument");
  if (!h->finalized) return fail(MB_ERR_STATE, "mb_tacotron_generate: weights not finalized");
  const mb_tacotron_config& c = h->cfg;
  if (B <= 0 || Tc <= 0 || steps <= 0 || r <= 0 || r > c.max_r) return fail(MB_ERR_INVALID, "mb_tacotron_generate: bad shape");
  const int nst = (steps + r - 1) / r;
  const int steps_alloc = nst * r;  // the reference emits r frames per decoder step (tacotron.py:264-272)
  const Ws L = ws_layout(c, B, Tc, steps_alloc, r);
  if (workspace_bytes < L.total * sizeof(float) + 256) return fail(MB_ERR_WORKSPACE, "mb_tacotron_generate: workspace too small");
  float* ws = (float*)(((uintptr_t)workspace + 255) & ~(uintptr_t)255);
  cudaStream_t caller = (cudaStream_t)stream;
  if (!h->own_stream) {
    MB_CUDA_CHECK(cudaStreamCreateWithFlags(&h->own_stream, cudaStreamNonBlocking));
    MB_CUDA_CHECK(cudaEventCreateWithFlags(&h->ev_in, cudaEventDisableTiming));
    MB_CUDA_CHECK(cudaEventCreateWithFlags(&h->ev_out, cudaEventDisableTiming));
    MB_CUDA_CHECK(cudaStreamCreateWithFlags(&h->side_stream, cudaStreamNonBlocking));
    for (cudaEvent_t& e : h->ev_side) MB_CUDA_CHECK(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
  }
  cudaStream_t st = h->own_stream;
  MB_CUDA_CHECK(cudaEventRecord(h->ev_in, caller));
  MB_CUDA_CHECK(cudaStreamWaitEvent(st, h->ev_in, 0));
  const int E = c.encoder_dims, D = c.decoder_dims, LD = c.lstm_dims, PD = c.postnet_dims, NM = c.n_mels;
  // MB_TACO_TC=0 keeps the decoder LSTMs on the FP32 FFMA kernels (A/B measurements); batches > 128 rows always do
  static const bool tc_env = [] {
    const char* e = getenv("MB_TACO_TC");
    return e ? atoi(e) != 0 : true;
  }();
  const bool use_tc = tc_env && B <= 128 && LD % 64 == 0;
  BigWs bw;
  bw.hi = ws + L.big_hi;
  bw.lo = ws + L.big_lo;
  bw.bytes = L.big_bytes;
  const int SE = c.speaker_embedding_size, proj_dims = E + SE + c.gst_E;
  const int Me = B * Tc;

  if (h->packed_r != r) {
    const size_t n = (size_t)r * NM * LD;
    pack_melproj_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(P(h, "decoder.mel_proj.weight"),
                                                                     P(h, "decoder.mel_proj.packed"), NM, c.max_r, r, LD);
    MB_LAUNCH_CHECK("pack_melproj_kernel");
    int rc = tc_prepare(h, "decoder.mel_proj", P(h, "decoder.mel_proj.packed"), LD, nullptr, 0, nullptr, nullptr, r * NM, 0, st);
    if (rc != MB_OK) return rc;
    h->packed_r = r;
  }

  // ------------------------------------------------------------------ encoder (tacotron.py:31-44)
  TK(launch_embedding(chars, P(h, "encoder.embedding.weight"), ws + L.emb, Me, c.embed_dims, st));
  uint8_t* em = reinterpret_cast<uint8_t*>(ws + L.m_enc);
  const size_t enc_mask_n = (size_t)Me * E;
  if (enc_masks) {
    MB_CUDA_CHECK(cudaMemcpyAsync(em, enc_masks, 2 * enc_mask_n, cudaMemcpyDeviceToDevice, st));
  } else {
    fill_masks_kernel<<<(unsigned)((2 * enc_mask_n + 255) / 256), 256, 0, st>>>(em, 2 * enc_mask_n, seed, 0xffffffffu);
    MB_LAUNCH_CHECK("fill_masks_kernel");
  }
  {
    GemmArgs a = gemm1(ws + L.emb, c.embed_dims, c.embed_dims, P(h, "encoder.pre_net.fc1.weight"), c.embed_dims,
                       P(h, "encoder.pre_net.fc1.bias"), Me, E, ws + L.p1, E, ACT_RELU);
    a.mask = em;
    TK(launch_gemm(a, st));
    GemmArgs b = gemm1(ws + L.p1, E, E, P(h, "encoder.pre_net.fc2.weight"), E, P(h, "encoder.pre_net.fc2.bias"), Me, E,
                       ws + L.x0, E, ACT_RELU);
    b.mask = em + enc_mask_n;
    TK(launch_gemm(b, st));
  }
  float* seq = ws + L.seq;
  int rc = run_cbhg(h, "encoder.cbhg", c.encoder_K, E, E, E, E, c.num_highways, ws + L.x0, B, Tc, ws + L.bank, ws + L.pool,
                    ws + L.pj1, ws + L.y, ws + L.hw12, ws + L.gi_f, ws + L.gi_b, ws + L.gh, ws + L.hst, seq, proj_dims, st,
                    use_tc ? ws + L.a_hi : nullptr, use_tc ? ws + L.a_lo : nullptr, tc_skinny_act_bytes(B > 128 ? 128 : B, 2 * LD), bw);
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
    TK(launch_gemm(a, st));
    const int dk = c.gst_E / c.gst_heads;
    gst_attention_kernel<<<B, 256, 0, st>>>(ws + L.style_q, P(h, "gst.keys"), P(h, "gst.values"), c.gst_tokens,
                                            ws + L.style, c.gst_E, c.gst_heads, 1.0f / sqrtf((float)dk));
    MB_LAUNCH_CHECK("gst_attention_kernel");
    TK(launch_copy_cols(ws + L.style, c.gst_E, Tc, seq, proj_dims, E + SE, Me, c.gst_E, st));
  }
  {
    GemmArgs a = gemm1(seq, proj_dims, proj_dims, P(h, "encoder_proj.weight"), proj_dims, nullptr, Me, D, ws + L.proj, D);
    TK(launch_gemm(a, st));
  }

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
  const size_t lsa_smem = sizeof(float) * (ATT_F * ATT_K + ATT_D * ATT_F + 2 * ATT_D + ATT_F + (Tc + 30) + Tc + 32 + (size_t)Tc * ATT_F + (size_t)Tc * 4);
  if (lsa_smem > 48 * 1024) MB_CUDA_CHECK(cudaFuncSetAttribute(lsa_step_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)lsa_smem));
  if (!dec_masks) {
    const size_t total = 2 * dmask_n * (size_t)nst;
    fill_masks_steps_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(dm, 2 * dmask_n, nst, seed);
    MB_LAUNCH_CHECK("fill_masks_steps_kernel");
  }
  int done_step = -1;
  std::vector<int> hflags(nst, 0);
  int checked = 0;
  // One decoder step.  The step index is (sp ? *sp : 0) + sj, resolved ON THE DEVICE by the few kernels that
  // need it (PreNet input frame and dropout masks, alignment row, mel output frames, stop flag), so the same
  // launch sequence can be captured once into a CUDA graph and replayed for every group of steps.
  // Fused operand split (MB_TACO_SPLIT_FUSED, default 1): the five act_split launches of a step disappear - every kernel that
  // produces an input of a tensor-core GEMM (PreNet, context, attention GRU, rnn_input, the two LSTM cells) writes the fp16 hi / lo
  // operand chunks itself, into per-consumer tiles (the LSTM tiles ping-pong on the step parity: a cell writes h' for the next step
  // while other CTAs of the same launch still read this step's tiles).
  static const bool split_fused_env = [] {
    const char* e = getenv("MB_TACO_SPLIT_FUSED");
    return e ? atoi(e) != 0 : true;
  }();
  static const bool prenet_fused_env = [] {
    const char* e = getenv("MB_TACO_PRENET_FUSED");
    return e ? atoi(e) != 0 : true;
  }();
  const bool fsplit = split_fused_env && prenet_fused_env && use_tc && D % 64 == 0 && proj_dims % 256 == 0 && LD % 64 == 0 &&
                      (r * NM) % 4 == 0 && NM <= 128 && 2 * D <= 256 && B <= 128;
  const FusedSplit fs = fused_split_layout(B > 128 ? 128 : B, proj_dims, D, LD);
  char* fbase = reinterpret_cast<char*>(ws + L.fsp);
  auto fhi = [&](size_t off) { return reinterpret_cast<__half*>(fbase + off); };
  const int f_rows_pad = B <= 64 ? 64 : 128;
  // Step DAG (MB_TACO_DAG, default 1, needs the fused split): a step's critical path is a chain of ~10 latency-bound kernels.  Three
  // of its GEMMs have a K segment that is known a whole step early - W_hh h_{t-1} of both LSTM cells and the context half of the
  // attention GRU's input projection - so those halves run on a side stream (TCS_PLAIN over a k-block range, result added to the
  // accumulator of the short main-path GEMM), and so does the stop projection / stop rule, which nothing in the next step needs.
  // The side stream forks from / joins the main one with events, inside the captured graph as well.
  static const bool dag_env = [] {
    const char* e = getenv("MB_TACO_DAG");
    return e ? atoi(e) != 0 : true;
  }();
  const bool dag = dag_env && fsplit && proj_dims % 64 == 0;
  cudaStream_t sd = h->side_stream;
  bool have_gic = false, have_p1 = false, have_p2 = false, have_stop = false, side_open = false;
  // fork: side stream waits for everything enqueued on the main stream so far
  auto side_after_main = [&](cudaEvent_t ev) -> int {
    MB_CUDA_CHECK(cudaEventRecord(ev, st));
    MB_CUDA_CHECK(cudaStreamWaitEvent(sd, ev, 0));
    side_open = true;
    return MB_OK;
  };
  auto main_after_side = [&](cudaEvent_t ev) -> int {
    MB_CUDA_CHECK(cudaEventRecord(ev, sd));
    MB_CUDA_CHECK(cudaStreamWaitEvent(st, ev, 0));
    return MB_OK;
  };
  // join everything outstanding on the side stream (end of a captured group / of a directly launched step)
  auto join_side = [&]() -> int {
    if (side_open) {
      int rcj = main_after_side(h->ev_side[7]);
      if (rcj != MB_OK) return rcj;
    }
    side_open = have_gic = have_p1 = have_p2 = have_stop = false;
    return MB_OK;
  };
  auto emit_step = [&](const int* sp, int sj) -> int {
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
                                P(h, "decoder.attn_net.W.weight"), P(h, "decoder.attn_net.W.bias")));
      MB_LAUNCH_CHECK("lsa_step_kernel");
      if (proj_dims % 256 == 0) {
        if (have_stop) {  // the previous step's stop projection (side stream) still reads ctx and x, which are rewritten from here on
          MB_CUDA_CHECK(cudaStreamWaitEvent(st, h->ev_side[6], 0));
          have_stop = false;
        }
        MB_CUDA_CHECK(launch_pdl2(lsa_ctx_kernel, dim3(proj_dims / 256, B), dim3(256), sizeof(float) * Tc, st, ws + L.scores_all,
                                  nst * Tc, seq, proj_dims, Tc, ws + L.ctx, sp, sj, fsplit ? fhi(fs.p1) : nullptr,
                                  fsplit ? fhi(fs.p1 + fs.b1) : nullptr, fsplit ? fhi(fs.p2) : nullptr,
                                  fsplit ? fhi(fs.p2 + fs.b2) : nullptr, f_rows_pad));
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
                                                       reinterpret_cast<unsigned int*>(ws + L.step) + 16);
        MB_LAUNCH_CHECK("stop_step_kernel");
        if (dag) {
          MB_CUDA_CHECK(cudaEventRecord(h->ev_side[6], sd));
          have_stop = true;
        }
      } else {
        TK(launch_gemm(s, st));
        stop_flag_kernel<<<1, 32, 0, st>>>(ws + L.stopv, B, min_stop_token, r, flags, sp, sj);
        MB_LAUNCH_CHECK("stop_flag_kernel");
      }
    }
    return MB_OK;
  };

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
  // Groups of kGraphSteps steps are captured once and replayed (the loop is launch-bound: ~20 kernels of a few
  // microseconds per step); MB_TACO_GRAPH=0 or a capture failure falls back to direct launches.
  constexpr int kGraphSteps = 8;
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
    const uint64_t launches_before = mb_launch_count();
    bool ok = cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal) == cudaSuccess;
    int rc_cap = MB_OK;
    if (ok) {
      for (int j = 0; j < kGraphSteps && rc_cap == MB_OK; ++j) rc_cap = emit_step(step_dev, j);
      if (rc_cap == MB_OK) rc_cap = join_side();
      if (rc_cap == MB_OK) step_advance_kernel<<<1, 32, 0, st>>>(step_dev, kGraphSteps);
      ok = cudaStreamEndCapture(st, &graph) == cudaSuccess && rc_cap == MB_OK && graph != nullptr;
    }
    if (ok) ok = cudaGraphInstantiate(&exec, graph, 0) == cudaSuccess;
    const int per_graph = (int)(mb_launch_count() - launches_before);
    count_launch(-per_graph);  // captured, not launched; every replay below counts them
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
    } else {
      cudaGetLastError();  // clear the capture error; direct launches below
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
  const int nsteps_done = (done_step >= 0 ? done_step : nst - 1) + 1;
  int frames = nsteps_done * r;
  if (frames > steps_alloc) frames = steps_alloc;
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
  rc = run_cbhg(h, "postnet", c.postnet_K, NM, PD, PD, NM, c.num_highways, melc, B, frames, ws + L.pbank, ws + L.ppool,
                ws + L.ppj1, ws + L.py, ws + L.phw12, ws + L.pgi_f, ws + L.pgi_b, ws + L.pgh, ws + L.phst, ws + L.pout, PD, st,
                use_tc ? ws + L.a_hi : nullptr, use_tc ? ws + L.a_lo : nullptr, tc_skinny_act_bytes(B > 128 ? 128 : B, 2 * LD), bw);
  if (rc != MB_OK) return rc;
  {
    GemmArgs a = gemm1(ws + L.pout, PD, PD, P(h, "post_proj.weight"), PD, nullptr, B * frames, NM, ws + L.lin, NM);
    int rc2 = cbhg_gemm(h, "post_proj", a, st, bw);
    if (rc2 != MB_OK) return rc2;
  }
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

}  // extern "C"
