// DeepMind-style dual-softmax WaveRNN on the H100 (SURVEY.md 8f row N3; mb_deepmind_*).
//   replaces  models/vocoder/wavernn/models/deepmind_version.py:75-162 (WaveRNN.generate): one unconditioned row, per sample two
//             dependent half-steps (coarse 8 bits, then fine 8 bits given the coarse draw):
//               R h (896 -> 2688, split coarse/fine x u,r,e) ; gates u,r = sigmoid, e = tanh(r * R_e + I_e + b_e) ;
//               h' = u h + (1 - u) e ; logits = O2 relu(O1 h'_coarse) resp. O4 relu(O3 h'_fine) ; Categorical draw.
// Same skeleton as the fatchord sample loop (wavernn.cu): ONE persistent cooperative kernel, the 12 MB of fp32 weights sliced
// across 112 CTAs and kept in shared memory for the whole call (114 KB per CTA: 24 rows of R, 4+4 rows of O1/O3, 4+4 rows of
// O2/O4), activations exchanged through L2-resident global vectors, 6 grid barriers per sample.  FP32 FFMA on purpose: the
// integer coarse / fine samples must equal the reference's under a fixed seed, which rules out fp16/tf32 operand rounding.
// Sampling = argmax(p / q) with q from the caller's Exp(1) stream (the torch-identical MT19937 stream of mt_stream.cu:
// 256 coarse draws then 256 fine draws per sample) or from the built-in counter-based generator; every CTA evaluates the
// 256-way draw redundantly (one warp), which saves a barrier per half-step.
#include <cstring>
#include <string>
#include <vector>

#include "../../include/mb_wavernn_math.h"
#include "mb_common.h"

namespace mb {
namespace {

constexpr int H = 896, S = 448, Q = 256;
constexpr int NCTA = 112, UPC = H / NCTA;          // 8 hidden units per CTA; CTAs [0,56) own coarse units, [56,112) fine units
constexpr int OPC = S / NCTA;                      // 4 outputs of O1 / O3 per CTA
constexpr int QCTA = Q / OPC;                      // 64 CTAs own 4 outputs of O2 / O4 each
constexpr int kThreads = 256;
// per-CTA weight pack (floats)
constexpr int OFF_R = 0;                           // [3 gates][8 units][896]
constexpr int OFF_O1 = OFF_R + 3 * UPC * H;        // [4][448]
constexpr int OFF_O3 = OFF_O1 + OPC * S;
constexpr int OFF_O2 = OFF_O3 + OPC * S;           // [4][448] (CTAs < 64, zeros elsewhere)
constexpr int OFF_O4 = OFF_O2 + OPC * S;
constexpr int OFF_MISC = OFF_O4 + OPC * S;         // gate biases [3][8], I rows [3][8][3], O1b[4] O3b[4] O2b[4] O4b[4]
constexpr int MISC = 3 * UPC + 3 * UPC * 3 + 4 * OPC;
constexpr int WPACK = (OFF_MISC + MISC + 3) / 4 * 4;
constexpr int SMEM_FLOATS = WPACK + H + S + Q + 64;

struct DmParams {
  const float* wpack;      // [NCTA][WPACK]
  float* hidden;           // [2][896] ping-pong (coarse | fine)
  float* x1;               // [448] relu(O1 h_c) / relu(O3 h_f)
  float* logits;           // [2][256] coarse / fine
  int* prev;               // [2] previous coarse / fine class (persist between calls)
  const float* noise;      // [nsteps][2][256] or nullptr
  uint64_t seed;
  int step0, nsteps, steps_total;
  int16_t* coarse;         // [steps_total]
  int16_t* fine;
  unsigned int* barrier;
};

__device__ __forceinline__ void grid_barrier(unsigned int* counter, unsigned int& target) {
  __syncthreads();
  if (threadIdx.x == 0) {
    target += gridDim.x;
    __threadfence();
    atomicAdd(counter, 1u);
    unsigned int v;
    do {
      asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(counter) : "memory");
    } while (v < target);
    __threadfence();
  }
  __syncthreads();
}

// warp dot product of a shared-memory weight row with a shared-memory vector: per-lane sequential fma chain over
// k = lane, lane+32, ... then xor butterfly (fixed order -> deterministic)
__device__ __forceinline__ float warp_dot(const float* __restrict__ w, const float* __restrict__ x, int n, int lane) {
  float a = 0.f;
  for (int k = lane; k < n; k += 32) a = fmaf(w[k], x[k], a);
#pragma unroll
  for (int off = 16; off >= 1; off >>= 1) a = a + __shfl_xor_sync(0xffffffffu, a, off);
  return a;
}

// 256-way Categorical draw by one warp: softmax, Categorical's renormalisation, argmax(p / q) (first maximum wins)
__device__ __forceinline__ int warp_sample(const float* __restrict__ lg_s, const float* __restrict__ noise, uint64_t seed,
                                           uint32_t gstep, uint32_t which, int lane) {
  float lg[8], e[8];
  float m = -3.0e38f;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    lg[j] = lg_s[lane + 32 * j];
    m = lg[j] > m ? lg[j] : m;
  }
#pragma unroll
  for (int off = 16; off >= 1; off >>= 1) {
    const float o = __shfl_xor_sync(0xffffffffu, m, off);
    m = o > m ? o : m;
  }
  float s = 0.f;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    e[j] = mb_expf(lg[j] - m);
    s = s + e[j];
  }
#pragma unroll
  for (int off = 16; off >= 1; off >>= 1) s = s + __shfl_xor_sync(0xffffffffu, s, off);
  const float S1 = s;
  float s2 = 0.f;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    e[j] = e[j] / S1;
    s2 = s2 + e[j];
  }
#pragma unroll
  for (int off = 16; off >= 1; off >>= 1) s2 = s2 + __shfl_xor_sync(0xffffffffu, s2, off);
  float bestv = -1.f;
  int best = 0;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int cls = lane + 32 * j;
    const float q = noise ? noise[cls] : mb_exp1_noise(seed, gstep, which, (uint32_t)cls);
    const float v = (e[j] / s2) / q;
    if (v > bestv) {
      bestv = v;
      best = cls;
    }
  }
#pragma unroll
  for (int off = 16; off >= 1; off >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, bestv, off);
    const int ob = __shfl_xor_sync(0xffffffffu, best, off);
    if (ov > bestv || (ov == bestv && ob < best)) {
      bestv = ov;
      best = ob;
    }
  }
  return best;
}

__global__ void __launch_bounds__(kThreads, 1) k_deepmind_loop(const DmParams p) {
  extern __shared__ __align__(16) float sm[];
  float* wsm = sm;
  float* hs = sm + WPACK;        // [896] hidden of the previous sample
  float* vs = hs + H;            // [448] staging of h'_coarse / x1 / h'_fine / x3
  float* ls = vs + S;            // [256] logits
  float* rf = ls + Q;            // [24] R_fine u,r,e of this CTA's units (fine CTAs) + scalars
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int cta = blockIdx.x;
  const bool fine_cta = cta >= NCTA / 2;
  {
    const float4* src = reinterpret_cast<const float4*>(p.wpack + (size_t)cta * WPACK);
    float4* dst = reinterpret_cast<float4*>(wsm);
    for (int i = tid; i < WPACK / 4; i += kThreads) dst[i] = src[i];
  }
  __syncthreads();
  const float* gb = wsm + OFF_MISC;                 // gate biases [3][8]
  const float* iw = gb + 3 * UPC;                   // I rows [3][8][3] (coarse CTAs use 2 inputs, the third weight is 0)
  const float* ob = iw + 3 * UPC * 3;               // O1b[4] O3b[4] O2b[4] O4b[4]
  unsigned int bar_target = 0;
  int prev_c = p.prev[0], prev_f = p.prev[1];

  for (int i = 0; i < p.nsteps; ++i) {
    const int gstep = p.step0 + i;
    const float* h_old = p.hidden + (size_t)(gstep & 1) * H;
    float* h_new = p.hidden + (size_t)((gstep & 1) ^ 1) * H;
    const float oc = (float)prev_c / 127.5f - 1.f;
    const float of = (float)prev_f / 127.5f - 1.f;
    // ---- P1: R h for this CTA's 8 units x 3 gates; coarse CTAs finish their gates -------------------------------
    for (int k = tid; k < H; k += kThreads) hs[k] = __ldcg(h_old + k);
    __syncthreads();
#pragma unroll 1
    for (int r = warp; r < 3 * UPC; r += kThreads / 32) {
      const float d = warp_dot(wsm + OFF_R + (size_t)r * H, hs, H, lane);
      if (lane == 0) rf[r] = d;
    }
    __syncthreads();
    if (!fine_cta && tid < UPC) {
      const int j = tid, unit = cta * UPC + j;
      const float Iu = fmaf(iw[(0 * UPC + j) * 3 + 1], of, iw[(0 * UPC + j) * 3 + 0] * oc);
      const float Ir = fmaf(iw[(1 * UPC + j) * 3 + 1], of, iw[(1 * UPC + j) * 3 + 0] * oc);
      const float Ie = fmaf(iw[(2 * UPC + j) * 3 + 1], of, iw[(2 * UPC + j) * 3 + 0] * oc);
      const float u = mb_sigmoidf(rf[0 * UPC + j] + Iu + gb[0 * UPC + j]);
      const float r = mb_sigmoidf(rf[1 * UPC + j] + Ir + gb[1 * UPC + j]);
      const float e = mb_tanhf(r * rf[2 * UPC + j] + Ie + gb[2 * UPC + j]);
      h_new[unit] = u * hs[unit] + (1.f - u) * e;
    }
    grid_barrier(p.barrier, bar_target);
    // ---- P2: x1 = relu(O1 h'_coarse + b) ----------------------------------------------------------------------
    for (int k = tid; k < S; k += kThreads) vs[k] = __ldcg(h_new + k);
    __syncthreads();
    if (warp < OPC) {
      const float d = warp_dot(wsm + OFF_O1 + (size_t)warp * S, vs, S, lane) + ob[warp];
      if (lane == 0) p.x1[cta * OPC + warp] = d > 0.f ? d : 0.f;
    }
    grid_barrier(p.barrier, bar_target);
    // ---- P3: coarse logits = O2 x1 + b (64 CTAs) ---------------------------------------------------------------
    if (cta < QCTA) {
      for (int k = tid; k < S; k += kThreads) vs[k] = __ldcg(p.x1 + k);
      __syncthreads();
      if (warp < OPC) {
        const float d = warp_dot(wsm + OFF_O2 + (size_t)warp * S, vs, S, lane) + ob[2 * OPC + warp];
        if (lane == 0) p.logits[cta * OPC + warp] = d;
      }
    }
    grid_barrier(p.barrier, bar_target);
    // ---- P4: coarse draw (every CTA, redundantly); fine CTAs finish their gates -------------------------------
    for (int k = tid; k < Q; k += kThreads) ls[k] = __ldcg(p.logits + k);
    __syncthreads();
    if (warp == 0) {
      const int c = warp_sample(ls, p.noise ? p.noise + ((size_t)i * 2 + 0) * Q : nullptr, p.seed, (uint32_t)gstep, 0u, lane);
      if (lane == 0) {
        reinterpret_cast<int*>(rf)[32] = c;
        if (cta == 0) p.coarse[gstep] = (int16_t)c;
      }
    }
    __syncthreads();
    const int cur_c = reinterpret_cast<int*>(rf)[32];
    if (fine_cta && tid < UPC) {
      const int j = tid, unit = cta * UPC + j;
      const float cp = (float)cur_c / 127.5f - 1.f;
      const float* w0 = iw + (0 * UPC + j) * 3;
      const float* w1 = iw + (1 * UPC + j) * 3;
      const float* w2 = iw + (2 * UPC + j) * 3;
      const float Iu = fmaf(w0[2], cp, fmaf(w0[1], of, w0[0] * oc));
      const float Ir = fmaf(w1[2], cp, fmaf(w1[1], of, w1[0] * oc));
      const float Ie = fmaf(w2[2], cp, fmaf(w2[1], of, w2[0] * oc));
      const float u = mb_sigmoidf(rf[0 * UPC + j] + Iu + gb[0 * UPC + j]);
      const float r = mb_sigmoidf(rf[1 * UPC + j] + Ir + gb[1 * UPC + j]);
      const float e = mb_tanhf(r * rf[2 * UPC + j] + Ie + gb[2 * UPC + j]);
      h_new[unit] = u * hs[unit] + (1.f - u) * e;
    }
    grid_barrier(p.barrier, bar_target);
    // ---- P5: x3 = relu(O3 h'_fine + b) --------------------------------------------------------------------------
    for (int k = tid; k < S; k += kThreads) vs[k] = __ldcg(h_new + S + k);
    __syncthreads();
    if (warp < OPC) {
      const float d = warp_dot(wsm + OFF_O3 + (size_t)warp * S, vs, S, lane) + ob[OPC + warp];
      if (lane == 0) p.x1[cta * OPC + warp] = d > 0.f ? d : 0.f;
    }
    grid_barrier(p.barrier, bar_target);
    // ---- P6: fine logits = O4 x3 + b ---------------------------------------------------------------------------
    if (cta < QCTA) {
      for (int k = tid; k < S; k += kThreads) vs[k] = __ldcg(p.x1 + k);
      __syncthreads();
      if (warp < OPC) {
        const float d = warp_dot(wsm + OFF_O4 + (size_t)warp * S, vs, S, lane) + ob[3 * OPC + warp];
        if (lane == 0) p.logits[Q + cta * OPC + warp] = d;
      }
    }
    grid_barrier(p.barrier, bar_target);
    // ---- P7: fine draw (every CTA); the next sample's P1 follows without another barrier ------------------------
    for (int k = tid; k < Q; k += kThreads) ls[k] = __ldcg(p.logits + Q + k);
    __syncthreads();
    if (warp == 0) {
      const int f = warp_sample(ls, p.noise ? p.noise + ((size_t)i * 2 + 1) * Q : nullptr, p.seed, (uint32_t)gstep, 1u, lane);
      if (lane == 0) {
        reinterpret_cast<int*>(rf)[33] = f;
        if (cta == 0) p.fine[gstep] = (int16_t)f;
      }
    }
    __syncthreads();
    prev_c = cur_c;
    prev_f = reinterpret_cast<int*>(rf)[33];
  }
  if (cta == 0 && tid == 0) {
    p.prev[0] = prev_c;
    p.prev[1] = prev_f;
  }
}

// [3H][H] R, O1..O4 (+bias), I_coarse [3S][2], I_fine [3S][3], bias_u/r/e [H]  ->  per-CTA packs
__global__ void k_deepmind_pack(const float* __restrict__ R, const float* __restrict__ O1, const float* __restrict__ O1b,
                                const float* __restrict__ O2, const float* __restrict__ O2b, const float* __restrict__ O3,
                                const float* __restrict__ O3b, const float* __restrict__ O4, const float* __restrict__ O4b,
                                const float* __restrict__ Ic, const float* __restrict__ If, const float* __restrict__ bu,
                                const float* __restrict__ br, const float* __restrict__ be, float* __restrict__ pack) {
  const int cta = blockIdx.x;
  float* dst = pack + (size_t)cta * WPACK;
  for (int i = threadIdx.x; i < WPACK; i += blockDim.x) {
    float v = 0.f;
    if (i < OFF_O1) {
      const int g = i / (UPC * H), j = (i / H) % UPC, k = i % H;
      v = R[((size_t)g * H + cta * UPC + j) * H + k];
    } else if (i < OFF_O3) {
      const int o = (i - OFF_O1) / S, k = (i - OFF_O1) % S;
      v = O1[(size_t)(cta * OPC + o) * S + k];
    } else if (i < OFF_O2) {
      const int o = (i - OFF_O3) / S, k = (i - OFF_O3) % S;
      v = O3[(size_t)(cta * OPC + o) * S + k];
    } else if (i < OFF_O4) {
      const int o = (i - OFF_O2) / S, k = (i - OFF_O2) % S;
      v = cta < QCTA ? O2[(size_t)(cta * OPC + o) * S + k] : 0.f;
    } else if (i < OFF_MISC) {
      const int o = (i - OFF_O4) / S, k = (i - OFF_O4) % S;
      v = cta < QCTA ? O4[(size_t)(cta * OPC + o) * S + k] : 0.f;
    } else {
      const int m = i - OFF_MISC;
      if (m < 3 * UPC) {
        const int g = m / UPC, j = m % UPC;
        const float* b = g == 0 ? bu : (g == 1 ? br : be);
        v = b[cta * UPC + j];
      } else if (m < 3 * UPC + 3 * UPC * 3) {
        const int q = m - 3 * UPC;
        const int g = q / (UPC * 3), j = (q / 3) % UPC, c = q % 3;
        const int unit = cta * UPC + j;
        if (unit < S) v = c < 2 ? Ic[((size_t)g * S + unit) * 2 + c] : 0.f;          // I_coarse: gate g rows [g*S, (g+1)*S)
        else v = If[((size_t)g * S + (unit - S)) * 3 + c];
      } else if (m < MISC) {
        const int q = m - (3 * UPC + 3 * UPC * 3);
        const int which = q / OPC, o = q % OPC;  // O1b, O3b, O2b, O4b
        if (which == 0) v = O1b[cta * OPC + o];
        else if (which == 1) v = O3b[cta * OPC + o];
        else if (which == 2) v = cta < QCTA ? O2b[cta * OPC + o] : 0.f;
        else v = cta < QCTA ? O4b[cta * OPC + o] : 0.f;
      }
    }
    dst[i] = v;
  }
}

}  // namespace
}  // namespace mb

using namespace mb;

struct mb_deepmind {
  WeightTable w;
  float* arena = nullptr;
  bool finalized = false;
};

namespace {
// workspace (floats): hidden [2][896] | x1 [448] | logits [512] | prev [2 ints] | barrier
constexpr size_t WS_HIDDEN = 0, WS_X1 = 2 * H, WS_LOGITS = WS_X1 + S, WS_PREV = WS_LOGITS + 2 * Q, WS_BAR = WS_PREV + 64, WS_TOTAL = WS_BAR + 64;
WsLayout ws_layout() {
  WsLayout L;
  L.take<float>(WS_TOTAL);
  return L;
}
}  // namespace

extern "C" {

int mb_deepmind_create(int32_t hidden_size, int32_t quantisation, mb_deepmind** out) {
  if (!out) return fail(MB_ERR_INVALID, "mb_deepmind_create: null argument");
  if (hidden_size != H || quantisation != Q)
    return fail(MB_ERR_INVALID, "mb_deepmind_create: only hidden_size=%d, quantisation=%d (the reference defaults) are built", H, Q);
  mb_deepmind* h = new mb_deepmind();
  WeightTable& w = h->w;
  w.add("R.weight", {3 * H, H});
  for (const auto& o : {std::make_pair("O1", S), std::make_pair("O2", Q), std::make_pair("O3", S), std::make_pair("O4", Q)}) {
    w.add(std::string(o.first) + ".weight", {o.second, S});
    w.add(std::string(o.first) + ".bias", {o.second});
  }
  w.add("I_coarse.weight", {3 * S, 2});
  w.add("I_fine.weight", {3 * S, 3});
  for (const char* b : {"bias_u", "bias_r", "bias_e"}) w.add(b, {H});
  *out = h;
  return MB_OK;
}

void mb_deepmind_destroy(mb_deepmind* h) { delete h; }

size_t mb_deepmind_arena_bytes(const mb_deepmind* h) { return h ? (h->w.floats() + (size_t)NCTA * WPACK) * sizeof(float) : 0; }

int mb_deepmind_set_arena(mb_deepmind* h, void* arena, size_t bytes) {
  if (int rc = check_arena("mb_deepmind_set_arena", h, arena, bytes, mb_deepmind_arena_bytes(h), 256)) return rc;
  h->w.attach((float*)arena);
  h->arena = (float*)arena;
  h->finalized = false;
  return MB_OK;
}

int mb_deepmind_set_weight(mb_deepmind* h, const char* name, const float* w, const int64_t* dims, int32_t ndim, void* stream) {
  if (!h) return fail(MB_ERR_INVALID, "mb_deepmind_set_weight: null argument");
  if (int rc = h->w.set("mb_deepmind_set_weight", name, w, dims, ndim, stream)) return rc;
  h->finalized = false;
  return MB_OK;
}

int mb_deepmind_finalize(mb_deepmind* h, void* stream) {
  if (!h || !h->arena) return fail(MB_ERR_STATE, "mb_deepmind_finalize: no arena");
  if (int rc = h->w.check_all_set("mb_deepmind_finalize")) return rc;
  k_deepmind_pack<<<NCTA, 256, 0, (cudaStream_t)stream>>>(
      h->w.ptr("R.weight"), h->w.ptr("O1.weight"), h->w.ptr("O1.bias"), h->w.ptr("O2.weight"), h->w.ptr("O2.bias"),
      h->w.ptr("O3.weight"), h->w.ptr("O3.bias"), h->w.ptr("O4.weight"), h->w.ptr("O4.bias"), h->w.ptr("I_coarse.weight"),
      h->w.ptr("I_fine.weight"), h->w.ptr("bias_u"), h->w.ptr("bias_r"), h->w.ptr("bias_e"), h->arena + h->w.floats());
  MB_LAUNCH_CHECK("k_deepmind_pack");
  h->finalized = true;
  return MB_OK;
}

size_t mb_deepmind_workspace_bytes(const mb_deepmind* h) { return h ? ws_layout().total() : 0; }

/* samples [step0, step0+nsteps) of one generate(seq_len = steps) call; step0 == 0 resets hidden / previous outputs to zero
 * (deepmind_version.py:86-91).  noise: Exp(1) draws fp32 [nsteps][2][256] (coarse draw then fine draw per sample, the order
 * Categorical.sample() consumes the torch generator) or NULL for the built-in generator.  coarse / fine: int16 [steps]. */
int mb_deepmind_generate(mb_deepmind* h, int32_t steps, int32_t step0, int32_t nsteps, const float* noise, uint64_t seed,
                         int16_t* coarse, int16_t* fine, void* workspace, size_t workspace_bytes, void* stream) {
  if (!h || !coarse || !fine) return fail(MB_ERR_INVALID, "mb_deepmind_generate: null argument");
  if (!h->finalized) return fail(MB_ERR_STATE, "mb_deepmind_generate: weights not finalized");
  if (nsteps <= 0 || step0 < 0 || step0 + nsteps > steps) return fail(MB_ERR_INVALID, "mb_deepmind_generate: bad step range");
  float* ws;
  if (int rc = bind("mb_deepmind_generate", workspace, workspace_bytes, ws_layout().total(), &ws)) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  if (step0 == 0) MB_CUDA_CHECK(cudaMemsetAsync(ws, 0, WS_TOTAL * sizeof(float), st));
  MB_CUDA_CHECK(cudaMemsetAsync(ws + WS_BAR, 0, 256, st));
  DmParams p;
  memset(&p, 0, sizeof(p));
  p.wpack = h->arena + h->w.floats();
  p.hidden = ws + WS_HIDDEN;
  p.x1 = ws + WS_X1;
  p.logits = ws + WS_LOGITS;
  p.prev = reinterpret_cast<int*>(ws + WS_PREV);
  p.noise = noise;
  p.seed = seed;
  p.step0 = step0;
  p.nsteps = nsteps;
  p.steps_total = steps;
  p.coarse = coarse;
  p.fine = fine;
  p.barrier = reinterpret_cast<unsigned int*>(ws + WS_BAR);
  const size_t smem = sizeof(float) * SMEM_FLOATS;
  static bool attr = false;
  if (!attr) {
    MB_CUDA_CHECK(cudaFuncSetAttribute(k_deepmind_loop, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    attr = true;
  }
  void* args[] = {(void*)&p};
  MB_CUDA_CHECK(cudaLaunchCooperativeKernel((void*)k_deepmind_loop, dim3(NCTA), dim3(kThreads), args, smem, st));
  count_launch();
  return MB_OK;
}

}  // extern "C"
