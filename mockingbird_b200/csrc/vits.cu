// VITS synthesizer (mb_vits_*): Vits.infer (models/synthesizer/models/vits.py:498-527) as FP32 kernels for the text
// encoder, the duration predictors, the path expansion and the reverse coupling flow, and an MB_GAN_VITS generator for the
// decoder.  See include/mockingbird_b200.h for the contract and DESIGN.md section 4l for the arithmetic.
#include <cmath>
#include <string>
#include <vector>

#include "mb_common.h"

namespace mb {
namespace {

constexpr int kMaxTokens = 1024;  // attention scores row in shared memory
constexpr int kMaxHead = 256;
constexpr int kWindow = 4;        // Encoder(window_size=4) (vits_modules.py:386)
constexpr int kBins = 10;         // ConvFlow(num_bins=10, tail_bound=5) (vits_modules.py:340)
constexpr float kTail = 5.f;
constexpr int kEmo = 1024;        // TextEncoder.emo_proj = Linear(1024, hidden) (vits.py:154)
constexpr int kSdpLayers = 3;     // DDSConv(n_layers=3) in the SDP and its ConvFlows
constexpr int kWnLayers = 4;      // ResidualCouplingBlock(inter, hidden, 5, 1, 4) (vits.py:448)
constexpr int kWnK = 5;

enum { EPI_STORE_ = 0, EPI_ACC = 1, EPI_SUB = 2 };

// y[b, co, t] = epi(bias[co] + bbias[b, co] + sum_{ci, j} w[co, ci, j] * xm[b, ci, t + j*dil - pad]), xm = x masked at
// t >= len[b] when in_mask.  epi: relu, then store / y += v / y -= v, then * mask(t) when out_mask.  Each output sums its
// terms in one fixed order (ci ascending, tap ascending), whatever B and T are: a row is bitwise the same in any batch.
struct ConvArgs {
  const float* x;
  long long xbs;  // batch stride of x (floats); channel stride is T
  int Cin;
  const float* w;  // [Cout][Cin][K]
  const float* bias;
  const float* bbias;  // [B][bbs] per-utterance bias (nullable)
  int bbs;
  float* y;
  long long ybs;
  int Cout, T, K, dil, pad;
  const int32_t* len;
  int in_mask, out_mask, relu, mode;
};

constexpr int CV_CO = 32, CV_T = 64, CV_CI = 16, CV_MAXK = 7;

__global__ void __launch_bounds__(256) conv1d_kernel(ConvArgs a) {
  __shared__ float xs[CV_CI][CV_T + (CV_MAXK - 1) * 1 + 8];
  __shared__ float ws[CV_CO][CV_CI * CV_MAXK + 1];
  const int b = blockIdx.z, co0 = blockIdx.y * CV_CO, t0 = blockIdx.x * CV_T;
  const int tid = threadIdx.x, ty = tid / 16, tx = tid % 16;
  const int L = a.len ? a.len[b] : a.T;
  const int halo = (a.K - 1) * a.dil, W = CV_T + halo;
  const float* xb = a.x + (long long)b * a.xbs;
  float acc[2][4] = {};
  for (int ci0 = 0; ci0 < a.Cin; ci0 += CV_CI) {
    for (int i = tid; i < CV_CI * W; i += 256) {
      const int ci = i / W, tt = i % W, t = t0 + tt - a.pad;
      float v = 0.f;
      if (ci0 + ci < a.Cin && t >= 0 && t < a.T && !(a.in_mask && t >= L)) v = xb[(long long)(ci0 + ci) * a.T + t];
      xs[ci][tt] = v;
    }
    for (int i = tid; i < CV_CO * CV_CI * a.K; i += 256) {
      const int co = i / (CV_CI * a.K), r = i % (CV_CI * a.K), ci = r / a.K, j = r % a.K;
      float v = 0.f;
      if (co0 + co < a.Cout && ci0 + ci < a.Cin) v = a.w[((long long)(co0 + co) * a.Cin + ci0 + ci) * a.K + j];
      ws[co][ci * a.K + j] = v;
    }
    __syncthreads();
    for (int ci = 0; ci < CV_CI; ++ci)
      for (int j = 0; j < a.K; ++j) {
        const float w0 = ws[ty * 2][ci * a.K + j], w1 = ws[ty * 2 + 1][ci * a.K + j];
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const float xv = xs[ci][tx + 16 * q + j * a.dil];
          acc[0][q] += w0 * xv;
          acc[1][q] += w1 * xv;
        }
      }
    __syncthreads();
  }
  for (int r = 0; r < 2; ++r) {
    const int co = co0 + ty * 2 + r;
    if (co >= a.Cout) continue;
    const float bv = a.bias ? a.bias[co] : 0.f, gv = a.bbias ? a.bbias[(long long)b * a.bbs + co] : 0.f;
    for (int q = 0; q < 4; ++q) {
      const int t = t0 + tx + 16 * q;
      if (t >= a.T) continue;
      float v = acc[r][q] + bv;
      if (a.bbias) v = v + gv;
      if (a.relu) v = fmaxf(v, 0.f);
      float* yp = a.y + (long long)b * a.ybs + (long long)co * a.T + t;
      if (a.mode == EPI_ACC) v = *yp + v;
      else if (a.mode == EPI_SUB) v = *yp - v;
      if (a.out_mask) v = v * (t < L ? 1.f : 0.f);
      *yp = v;
    }
  }
}

// DDSConv's depthwise dilated k = 3 conv over x * mask (vits_modules.py:93)
__global__ void dwconv_kernel(const float* x, const float* w, const float* bias, float* y, int B, int C, int T, int K,
                              int dil, const int32_t* len) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)B * C * T) return;
  const int t = (int)(i % T), c = (int)((i / T) % C), b = (int)(i / ((long long)C * T));
  const int L = len[b], pad = (K * dil - dil) / 2;
  const float* xr = x + ((long long)b * C + c) * T;
  float acc = 0.f;
  for (int j = 0; j < K; ++j) {
    const int s = t + j * dil - pad;
    const float v = (s >= 0 && s < T && s < L) ? xr[s] : 0.f;
    acc += w[c * K + j] * v;
  }
  y[i] = acc + bias[c];
}

__device__ __forceinline__ float gelu_erf(float v) { return 0.5f * v * (1.f + erff(v * 0.70710678118654752f)); }

// out = res + act(LayerNorm_C(a + b2)) (* mask): channel LayerNorm (vits_modules.py:13-25, eps 1e-5), one thread per (b, t)
__global__ void layernorm_kernel(const float* a, const float* b2, const float* gamma, const float* beta, const float* res,
                                 float* out, int B, int C, int T, int gelu, const int32_t* len) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)B * T) return;
  const int t = (int)(i % T), b = (int)(i / T);
  const long long base = (long long)b * C * T + t;
  float s = 0.f;
  for (int c = 0; c < C; ++c) s += a[base + (long long)c * T] + (b2 ? b2[base + (long long)c * T] : 0.f);
  const float mean = s / C;
  float v2 = 0.f;
  for (int c = 0; c < C; ++c) {
    const float d = a[base + (long long)c * T] + (b2 ? b2[base + (long long)c * T] : 0.f) - mean;
    v2 += d * d;
  }
  const float rstd = 1.f / sqrtf(v2 / C + 1e-5f);
  const float m = (len && t >= len[b]) ? 0.f : 1.f;
  for (int c = 0; c < C; ++c) {
    const long long o = base + (long long)c * T;
    float v = ((a[o] + (b2 ? b2[o] : 0.f)) - mean) * rstd * gamma[c] + beta[c];
    if (gelu) v = gelu_erf(v);
    if (res) v = res[o] + v;
    if (len) v = v * m;
    out[o] = v;
  }
}

// x[b, :, t] = emb[id] * sqrt(H) + e[b] (emo_proj), masked (vits.py:168-173)
__global__ void embed_kernel(const int32_t* ids, const float* emb, const float* e, float* x, int B, int H, int T, int n_vocab,
                             const int32_t* len) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)B * H * T) return;
  const int t = (int)(i % T), c = (int)((i / T) % H), b = (int)(i / ((long long)H * T));
  int id = ids[(long long)b * T + t];
  if (id < 0 || id >= n_vocab) id = 0;
  const float v = emb[(long long)id * H + c] * sqrtf((float)H) + e[(long long)b * H + c];
  x[i] = v * (t < len[b] ? 1.f : 0.f);
}

// g[b] = emb_g[sid[b]]
__global__ void gather_rows_kernel(const float* table, const int32_t* idx, float* out, int B, int C, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * C) return;
  int r = idx[i / C];
  if (r < 0 || r >= n) r = 0;
  out[i] = table[(long long)r * C + i % C];
}

// Relative-position self-attention of one head for one query row (vits_modules.py:520-551, window 4, shared relative
// embeddings): scores = q/sqrt(dk) . (k_s + rel_k[s - t]) with rel_k zero beyond the window, -1e4 where query or key is
// padding, softmax, then sum_s p_s (v_s + rel_v[s - t]).
__global__ void __launch_bounds__(128) rel_attn_kernel(const float* q, const float* k, const float* v, const float* erk,
                                                       const float* erv, float* o, int H, int nh, int T, const int32_t* len) {
  __shared__ float qs[kMaxHead];
  __shared__ float sc[kMaxTokens];
  __shared__ float red[32];
  const int t = blockIdx.x, hd = blockIdx.y, b = blockIdx.z, dk = H / nh, tid = threadIdx.x;
  const int L = len[b];
  const long long base = (long long)b * H * T + (long long)hd * dk * T;
  const float scale = sqrtf((float)dk);
  for (int d = tid; d < dk; d += 128) qs[d] = q[base + (long long)d * T + t] / scale;
  __syncthreads();
  for (int s = tid; s < T; s += 128) {
    float acc = 0.f;
    for (int d = 0; d < dk; ++d) acc += qs[d] * k[base + (long long)d * T + s];
    const int r = s - t;
    if (r >= -kWindow && r <= kWindow) {
      float rel = 0.f;
      for (int d = 0; d < dk; ++d) rel += qs[d] * erk[(r + kWindow) * dk + d];
      acc = acc + rel;
    }
    if (t >= L || s >= L) acc = -1e4f;
    sc[s] = acc;
  }
  __syncthreads();
  float m = -INFINITY;
  for (int s = tid; s < T; s += 128) m = fmaxf(m, sc[s]);
  for (int off = 16; off; off >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, off));
  if ((tid & 31) == 0) red[tid >> 5] = m;
  __syncthreads();
  m = fmaxf(fmaxf(red[0], red[1]), fmaxf(red[2], red[3]));
  __syncthreads();
  float sum = 0.f;
  for (int s = tid; s < T; s += 128) {
    const float e = expf(sc[s] - m);
    sc[s] = e;
    sum += e;
  }
  for (int off = 16; off; off >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, off);
  if ((tid & 31) == 0) red[tid >> 5] = sum;
  __syncthreads();
  sum = (red[0] + red[1]) + (red[2] + red[3]);
  for (int d = tid; d < dk; d += 128) {
    float acc = 0.f;
    for (int s = 0; s < T; ++s) acc += (sc[s] / sum) * v[base + (long long)d * T + s];
    float rel = 0.f;
    for (int r = -kWindow; r <= kWindow; ++r) {
      const int s = t + r;
      if (s >= 0 && s < T) rel += (sc[s] / sum) * erv[(r + kWindow) * dk + d];
    }
    o[base + (long long)d * T + t] = acc + rel;
  }
}

// One ConvFlow in reverse (vits_modules.py:356-383, transforms.py): proj (C -> 29) of the DDSConv output, widths /
// heights / derivatives, the inverse rational-quadratic spline of z[c1] with linear tails at +-5, then z = z * mask.  One
// warp per (b, t).
__global__ void spline_flow_kernel(const float* h, const float* wp, const float* bp, float* z, int B, int C, int T, int c0,
                                   int c1, const int32_t* len) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= B * T) return;
  const int b = warp / T, t = warp % T;
  const float m = t < len[b] ? 1.f : 0.f;
  constexpr int NP = 3 * kBins - 1;
  float p = 0.f;
  if (lane < NP) {
    float acc = 0.f;
    for (int c = 0; c < C; ++c) acc += wp[lane * C + c] * h[((long long)b * C + c) * T + t];
    p = (acc + bp[lane]) * m;
  }
  float hv[NP];
#pragma unroll
  for (int j = 0; j < NP; ++j) hv[j] = __shfl_sync(0xffffffffu, p, j);
  if (lane != 0) return;
  float* zb = z + (long long)b * 2 * T;
  const float x0 = zb[(long long)c0 * T + t], x1 = zb[(long long)c1 * T + t];
  float out = x1;
  if (x1 >= -kTail && x1 <= kTail) {
    const float sq = sqrtf((float)C);
    const float minw = 1e-3f, minh = 1e-3f, mind = 1e-3f;
    float uw[kBins], uh[kBins], der[kBins + 1];
    for (int j = 0; j < kBins; ++j) uw[j] = hv[j] / sq, uh[j] = hv[kBins + j] / sq;
    const float cst = logf(expf(1.f - mind) - 1.f);
    float ud[kBins + 1];
    ud[0] = cst;
    ud[kBins] = cst;
    for (int j = 1; j < kBins; ++j) ud[j] = hv[2 * kBins + j - 1];
    for (int j = 0; j <= kBins; ++j) der[j] = mind + (ud[j] > 20.f ? ud[j] : log1pf(expf(ud[j])));
    float cw[kBins + 1], ch[kBins + 1];
    auto cum = [&](const float* u, float mn, float* cs) {
      float mx = u[0];
      for (int j = 1; j < kBins; ++j) mx = fmaxf(mx, u[j]);
      float e[kBins], s = 0.f;
      for (int j = 0; j < kBins; ++j) e[j] = expf(u[j] - mx), s += e[j];
      float run = 0.f;
      cs[0] = -kTail;
      for (int j = 0; j < kBins; ++j) {
        run += mn + (1.f - mn * kBins) * (e[j] / s);
        cs[j + 1] = 2.f * kTail * run - kTail;
      }
      cs[0] = -kTail;
      cs[kBins] = kTail;
    };
    cum(uw, minw, cw);
    cum(uh, minh, ch);
    // searchsorted(cumheights, x, eps=1e-6): the last edge is raised by eps
    int k = -1;
    for (int j = 0; j <= kBins; ++j) k += (x1 >= (j == kBins ? ch[j] + 1e-6f : ch[j])) ? 1 : 0;
    k = k < 0 ? 0 : (k > kBins - 1 ? kBins - 1 : k);
    const float w_k = cw[k + 1] - cw[k], h_k = ch[k + 1] - ch[k];
    const float delta = h_k / w_k, d0 = der[k], d1 = der[k + 1];
    const float dx = x1 - ch[k], sdd = d0 + d1 - 2.f * delta;
    const float qa = dx * sdd + h_k * (delta - d0);
    const float qb = h_k * d0 - dx * sdd;
    const float qc = -delta * dx;
    const float disc = qb * qb - 4.f * qa * qc;
    const float root = (2.f * qc) / (-qb - sqrtf(disc));
    out = root * w_k + cw[k];
  }
  zb[(long long)c0 * T + t] = x0 * m;
  zb[(long long)c1 * T + t] = out * m;
}

// ElementwiseAffine reverse on the SDP's z (vits_modules.py:287) followed by w = exp(logw) * mask * length_scale, w_ceil =
// ceil(w) for channel 0 (vits.py:511-513); z is the DurationPredictor's logw [B, 1, T] instead when ea_m == nullptr.
// logw_out [B, T] (nullable) receives the logw the durations were taken from.
__global__ void durations_kernel(const float* z, const float* ea_m, const float* ea_logs, int zC, float length_scale, int B,
                                 int T, const int32_t* len, int32_t* w_ceil, int32_t* y_len, float* logw_out) {
  const int b = blockIdx.x;
  __shared__ int tot[32];
  int s = 0;
  for (int t = threadIdx.x; t < T; t += blockDim.x) {
    const float m = t < len[b] ? 1.f : 0.f;
    float logw = z[(long long)b * zC * T + t];
    if (ea_m) logw = (logw - ea_m[0]) * expf(-ea_logs[0]) * m;
    if (logw_out) logw_out[(long long)b * T + t] = logw;
    const float w = expf(logw) * m * length_scale;
    const int c = (int)ceilf(w);
    w_ceil[(long long)b * T + t] = c;
    s += c;
  }
  for (int off = 16; off; off >>= 1) s += __shfl_xor_sync(0xffffffffu, s, off);
  if ((threadIdx.x & 31) == 0) tot[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    int a = 0;
    for (int i = 0; i < (int)(blockDim.x >> 5); ++i) a += tot[i];
    y_len[b] = a < 1 ? 1 : a;
  }
}

// per-row inclusive cumulative sum of w_ceil over the valid tokens (generate_path, utils/util.py:93-108)
__global__ void cumsum_kernel(const int32_t* w_ceil, const int32_t* x_len, int32_t* cum, int32_t* y_len, int B, int T) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  int s = 0;
  for (int t = 0; t < T; ++t) {
    s += t < x_len[b] ? w_ceil[(long long)b * T + t] : 0;
    cum[(long long)b * T + t] = s;
  }
  y_len[b] = s < 1 ? 1 : s;
}

// frame j of row b takes token i with cum[i-1] <= j < cum[i] (none past y_len or past the last token): m_p / logs_p
// gathered, z_p = m + eps * exp(logs) * noise_scale (vits.py:514-522); attn written when asked for
__global__ void expand_kernel(const float* m_p, const float* logs_p, const int32_t* cum, const int32_t* y_len, const float* eps,
                              float noise_scale, float* z_p, float* m_y, float* logs_y, float* attn, int B, int C, int Tx,
                              int Ty) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)B * Ty) return;
  const int j = (int)(i % Ty), b = (int)(i / Ty);
  const int32_t* cb = cum + (long long)b * Tx;
  int tok = -1;
  if (j < y_len[b] && j < cb[Tx - 1]) {
    int lo = 0, hi = Tx - 1;  // first i with cum[i] > j
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (cb[mid] > j) hi = mid;
      else lo = mid + 1;
    }
    tok = lo;
  }
  if (attn) {
    float* ar = attn + ((long long)b * Ty + j) * Tx;
    for (int t = 0; t < Tx; ++t) ar[t] = t == tok ? 1.f : 0.f;
  }
  for (int c = 0; c < C; ++c) {
    const long long src = ((long long)b * C + c) * Tx + tok, dst = ((long long)b * C + c) * Ty + j;
    const float m = tok >= 0 ? m_p[src] : 0.f, ls = tok >= 0 ? logs_p[src] : 0.f;
    if (m_y) m_y[dst] = m;
    if (logs_y) logs_y[dst] = ls;
    z_p[dst] = m + eps[dst] * expf(ls) * noise_scale;
  }
}

// out = a * s (+ bb[b, c] broadcast over t when bb is given)
__global__ void scale_bias_kernel(const float* a, float s, const float* bb, float* out, int B, int C, int T) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)B * C * T) return;
  const int c = (int)((i / T) % C), b = (int)(i / ((long long)C * T));
  float v = a[i] * s;
  if (bb) v = v + bb[(long long)b * C + c];
  out[i] = v;
}

// out = a + b
__global__ void add_kernel(const float* a, const float* b, float* out, long long n) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = a[i] + b[i];
}

// torch.flip(x, [1]) over C channels
__global__ void flip_kernel(const float* x, float* y, int B, int C, int T) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)B * C * T) return;
  const int t = (int)(i % T), c = (int)((i / T) % C), b = (int)(i / ((long long)C * T));
  y[((long long)b * C + (C - 1 - c)) * T + t] = x[i];
}

// WN gate: acts = tanh(x_in[:H] + g_l[:H]) * sigmoid(x_in[H:] + g_l[H:]) (utils/util.py:111-117); the g_l slice is already
// part of x_in (the in_layer's per-utterance bias)
__global__ void gate_kernel(const float* xin, float* acts, int B, int H, int T) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)B * H * T) return;
  const int t = (int)(i % T), c = (int)((i / T) % H), b = (int)(i / ((long long)H * T));
  const float a = xin[((long long)b * 2 * H + c) * T + t], s = xin[((long long)b * 2 * H + H + c) * T + t];
  acts[i] = tanhf(a) * (1.f / (1.f + expf(-s)));
}

// decoder input: (z * y_mask)[:, :, :t_dec] followed by g broadcast over time (cond(g) folded into conv_pre)
__global__ void dec_input_kernel(const float* z, const float* g, float* out, int B, int C, int G, int Ty, int Td,
                                 const int32_t* y_len) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)B * (C + G) * Td) return;
  const int t = (int)(i % Td), c = (int)((i / Td) % (C + G)), b = (int)(i / ((long long)(C + G) * Td));
  out[i] = c < C ? z[((long long)b * C + c) * Ty + t] * (!y_len || t < y_len[b] ? 1.f : 0.f) : g[(long long)b * G + (c - C)];
}

// conv_pre's weight over [z ; g] channels: w[:, :I, :] = conv_pre.weight, w[:, I:, centre] = cond.weight; bias = sum of both
__global__ void fold_cond_kernel(const float* wpre, const float* bpre, const float* wc, const float* bc, float* w, float* bias,
                                 int C0, int I, int G, int K) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long n = (long long)C0 * (I + G) * K;
  if (i < C0) bias[i] = bpre[i] + (bc ? bc[i] : 0.f);
  if (i >= n) return;
  const int j = (int)(i % K), c = (int)((i / K) % (I + G)), o = (int)(i / ((long long)(I + G) * K));
  w[i] = c < I ? wpre[((long long)o * I + c) * K + j] : (j == K / 2 ? wc[(long long)o * G + (c - I)] : 0.f);
}

inline unsigned blocks(long long n, int t = 256) { return (unsigned)((n + t - 1) / t); }

}  // namespace
}  // namespace mb

using namespace mb;

struct mb_vits {
  mb_vits_config cfg{};
  WeightTable w;
  mb_gan* gan = nullptr;
  float* arena = nullptr;
  size_t table_bytes = 0;
  bool finalized = false;
  int I = 0, H = 0, F = 0, G = 0, NH = 0, NL = 0, K = 0, C0 = 0, DPC = 0;

  const float* p(const std::string& n) const { return w.ptr(n); }
  const float* po(const std::string& n) const { return w.has(n) ? w.ptr(n) : nullptr; }
};

namespace {

using mb::ConvArgs;

int conv(const char* what, const float* x, long long xbs, int Cin, const float* wt, const float* bias, const float* bbias,
         int bbs, float* y, long long ybs, int Cout, int B, int T, int K, int dil, int pad, const int32_t* len, int in_mask,
         int out_mask, int relu, int mode, cudaStream_t st) {
  if (K > CV_MAXK || (K - 1) * dil > CV_MAXK + 7) return fail(MB_ERR_INVALID, "%s: conv k=%d dil=%d unsupported", what, K, dil);
  ConvArgs a{x, xbs, Cin, wt, bias, bbias, bbs, y, ybs, Cout, T, K, dil, pad, len, in_mask, out_mask, relu, mode};
  conv1d_kernel<<<dim3((T + CV_T - 1) / CV_T, (Cout + CV_CO - 1) / CV_CO, B), 256, 0, st>>>(a);
  MB_LAUNCH_CHECK(what);
  return MB_OK;
}

// 1x1 conv, NCL with the tensors' own channel counts as batch strides
int conv1x1(const char* what, const float* x, int Cin, const float* wt, const float* bias, float* y, int Cout, int B, int T,
            cudaStream_t st, const int32_t* len = nullptr, int in_mask = 0, int out_mask = 0) {
  return conv(what, x, (long long)Cin * T, Cin, wt, bias, nullptr, 0, y, (long long)Cout * T, Cout, B, T, 1, 1, 0, len,
              in_mask, out_mask, 0, EPI_STORE_, st);
}

int layernorm(const float* a, const float* b2, const float* gamma, const float* beta, const float* res, float* out, int B, int C,
              int T, int gelu, const int32_t* len, cudaStream_t st) {
  layernorm_kernel<<<blocks((long long)B * T, 128), 128, 0, st>>>(a, b2, gamma, beta, res, out, B, C, T, gelu, len);
  MB_LAUNCH_CHECK("layernorm_kernel");
  return MB_OK;
}

#define TRY(x)                 \
  do {                         \
    if (int _rc = (x)) return _rc; \
  } while (0)

// DDSConv (vits_modules.py:89-101): x = (x (+ g)) ; for each layer x += gelu(LN(1x1(gelu(LN(dwconv(x * mask)))))) ;
// x * mask.  y1 / y2 are scratch of x's size.
int ddsconv(const mb_vits* h, const std::string& pre, float* x, float* y1, float* y2, int B, int C, int T, const int32_t* len,
            cudaStream_t st) {
  for (int l = 0; l < kSdpLayers; ++l) {
    const std::string L = std::to_string(l);
    int dil = 1;
    for (int i = 0; i < l; ++i) dil *= 3;
    dwconv_kernel<<<blocks((long long)B * C * T), 256, 0, st>>>(x, h->p(pre + "convs_sep." + L + ".weight"),
                                                                 h->p(pre + "convs_sep." + L + ".bias"), y1, B, C, T, 3, dil, len);
    MB_LAUNCH_CHECK("dwconv_kernel");
    TRY(layernorm(y1, nullptr, h->p(pre + "norms_1." + L + ".gamma"), h->p(pre + "norms_1." + L + ".beta"), nullptr, y1, B, C, T,
                  1, nullptr, st));
    TRY(conv1x1("ddsconv 1x1", y1, C, h->p(pre + "convs_1x1." + L + ".weight"), h->p(pre + "convs_1x1." + L + ".bias"), y2, C, B,
                T, st));
    // x = x + gelu(LN(y)); the final * mask is applied on the last layer
    TRY(layernorm(y2, nullptr, h->p(pre + "norms_2." + L + ".gamma"), h->p(pre + "norms_2." + L + ".beta"), x, x, B, C, T, 1,
                  l == kSdpLayers - 1 ? len : nullptr, st));
  }
  return MB_OK;
}

// WN layer l of the coupling layer with prefix `e` ("flow.flows.N.enc."), vits_modules.py:148-168: x_in = in_layer(x) (+ the
// cond_layer slice of `cond` [B, 2H * 4]), acts = tanh * sigmoid, then x = (x + res) * mask and out += skip (out = skip for
// l = 0; the last layer has only the skip half)
int wn_layer(const mb_vits* h, const std::string& e, int l, float* hh, float* xin, float* acts, float* out, const float* cond, int B,
             int T, const int32_t* len, cudaStream_t st) {
  const int H = h->H;
  const long long hbs = (long long)H * T;
  const std::string L = std::to_string(l);
  TRY(conv("wn in_layer", hh, hbs, H, h->p(e + "in_layers." + L + ".weight"), h->p(e + "in_layers." + L + ".bias"),
           cond ? cond + 2 * H * l : nullptr, 2 * H * kWnLayers, xin, 2 * hbs, 2 * H, B, T, kWnK, 1, (kWnK - 1) / 2, nullptr, 0, 0,
           0, EPI_STORE_, st));
  gate_kernel<<<blocks((long long)B * H * T), 256, 0, st>>>(xin, acts, B, H, T);
  MB_LAUNCH_CHECK("gate_kernel");
  const float* rw = h->p(e + "res_skip_layers." + L + ".weight");
  const float* rb = h->p(e + "res_skip_layers." + L + ".bias");
  if (l < kWnLayers - 1) {
    TRY(conv("wn res", acts, hbs, H, rw, rb, nullptr, 0, hh, hbs, H, B, T, 1, 1, 0, len, 0, 1, 0, EPI_ACC, st));
    return conv("wn skip", acts, hbs, H, rw + (size_t)H * H, rb + H, nullptr, 0, out, hbs, H, B, T, 1, 1, 0, nullptr, 0, 0, 0,
                l == 0 ? EPI_STORE_ : EPI_ACC, st);
  }
  return conv("wn skip", acts, hbs, H, rw, rb, nullptr, 0, out, hbs, H, B, T, 1, 1, 0, nullptr, 0, 0, 0, EPI_ACC, st);
}

struct DurWs {
  size_t x, q, k, v, a, y, f, e, g, gb, s0, s1, s2, s3, z;
  size_t total;
};

DurWs dur_layout(const mb_vits* h, size_t B, size_t T) {
  WsLayout L;
  DurWs o;
  const size_t H = h->H;
  o.x = L.take<float>(B * H * T);
  o.q = L.take<float>(B * H * T);
  o.k = L.take<float>(B * H * T);
  o.v = L.take<float>(B * H * T);
  o.a = L.take<float>(B * H * T);
  o.y = L.take<float>(B * H * T);
  o.f = L.take<float>(B * std::max(h->F, h->DPC) * T);
  o.e = L.take<float>(B * H);
  o.g = L.take<float>(B * std::max(h->G, 1));
  o.gb = L.take<float>(B * H);
  o.s0 = L.take<float>(B * H * T);
  o.s1 = L.take<float>(B * H * T);
  o.s2 = L.take<float>(B * H * T);
  o.s3 = L.take<float>(B * std::max((size_t)h->DPC, H) * T);
  o.z = L.take<float>(B * 2 * T);
  o.total = L.total();
  return o;
}

struct DecWs {
  size_t cum, ylen, g, cond, za, zb, hh, xin, acts, out, din, gan;
  size_t total;
};

DecWs dec_layout(const mb_vits* h, size_t B, size_t Tx, size_t Ty, size_t Td) {
  WsLayout L;
  DecWs o;
  const size_t H = h->H, I = h->I;
  o.cum = L.take<int32_t>(B * Tx);
  o.ylen = L.take<int32_t>(B);
  o.g = L.take<float>(B * std::max(h->G, 1));
  o.cond = L.take<float>(B * 2 * H * kWnLayers);
  o.za = L.take<float>(B * I * Ty);
  o.zb = L.take<float>(B * I * Ty);
  o.hh = L.take<float>(B * H * Ty);
  o.xin = L.take<float>(B * 2 * H * Ty);
  o.acts = L.take<float>(B * H * Ty);
  o.out = L.take<float>(B * H * Ty);
  o.din = L.take<float>(B * (I + h->G) * Td);
  L.align = 1024;  // the tensor-core decoder's planes
  o.gan = L.take(mb_gan_workspace_bytes(h->gan, (int32_t)B, (int32_t)Td));
  o.total = L.total();
  return o;
}

// The stages below are shared by mb_vits_durations / mb_vits_decode and mb_vits_debug, so that the debug kinds run the
// shipped code.

// Text-encoder layer l (vits_modules.py:407-419) in place on X [B, H, T]: X = LN_1(X + conv_o(attn(q, k, v))), then
// X = LN_2(X + FFN(X)), masked after the last layer.  Scratch: the q, k, v, a, y and f planes of `o` in `ws`.
int enc_layer(const mb_vits* h, int l, float* X, const DurWs& o, char* ws, int B, int T, const int32_t* len, cudaStream_t st) {
  auto F = [&](size_t off) { return (float*)ws + off; };
  const int H = h->H, NH = h->NH;
  float *Q = F(o.q), *Kb = F(o.k), *V = F(o.v), *A = F(o.a), *Y = F(o.y), *FF = F(o.f);
  const std::string L = std::to_string(l), a = "enc_p.encoder.attn_layers." + L;
  TRY(conv1x1("conv_q", X, H, h->p(a + ".conv_q.weight"), h->p(a + ".conv_q.bias"), Q, H, B, T, st));
  TRY(conv1x1("conv_k", X, H, h->p(a + ".conv_k.weight"), h->p(a + ".conv_k.bias"), Kb, H, B, T, st));
  TRY(conv1x1("conv_v", X, H, h->p(a + ".conv_v.weight"), h->p(a + ".conv_v.bias"), V, H, B, T, st));
  rel_attn_kernel<<<dim3(T, NH, B), 128, 0, st>>>(Q, Kb, V, h->p(a + ".emb_rel_k"), h->p(a + ".emb_rel_v"), A, H, NH, T, len);
  MB_LAUNCH_CHECK("rel_attn_kernel");
  TRY(conv1x1("conv_o", A, H, h->p(a + ".conv_o.weight"), h->p(a + ".conv_o.bias"), Y, H, B, T, st));
  TRY(layernorm(X, Y, h->p("enc_p.encoder.norm_layers_1." + L + ".gamma"), h->p("enc_p.encoder.norm_layers_1." + L + ".beta"),
                nullptr, X, B, H, T, 0, nullptr, st));
  // FFN (vits_modules.py:649-657): conv_2(relu(conv_1(x * mask)) * mask) * mask, same padding
  const std::string f = "enc_p.encoder.ffn_layers." + L;
  TRY(conv("ffn conv_1", X, (long long)H * T, H, h->p(f + ".conv_1.weight"), h->p(f + ".conv_1.bias"), nullptr, 0, FF,
           (long long)h->F * T, h->F, B, T, h->K, 1, (h->K - 1) / 2, len, 1, 0, 1, EPI_STORE_, st));
  TRY(conv("ffn conv_2", FF, (long long)h->F * T, h->F, h->p(f + ".conv_2.weight"), h->p(f + ".conv_2.bias"), nullptr, 0, Y,
           (long long)H * T, H, B, T, h->K, 1, (h->K - 1) / 2, len, 1, 1, 0, EPI_STORE_, st));
  return layernorm(X, Y, h->p("enc_p.encoder.norm_layers_2." + L + ".gamma"), h->p("enc_p.encoder.norm_layers_2." + L + ".beta"),
                   nullptr, X, B, H, T, 0, l == h->NL - 1 ? len : nullptr, st);
}

// The duration predictor on the encoder output X [B, H, T] (vits.py:48-130, either kind), then w_ceil = ceil(exp(logw) *
// mask * length_scale) and y_len = max(1, sum w_ceil).  g = emb_g[sid] conditions it when sid is given; noise [B, 2, T] is
// the SDP's unscaled draw.  logw_out [B, T] (nullable) receives logw.  Scratch: the remaining planes of `o` in `ws`.
int duration_predictor(const mb_vits* h, const float* X, const int32_t* sid, const float* noise, float noise_scale_w,
                       float length_scale, int32_t* w_ceil, int32_t* y_lengths, float* logw_out, const DurWs& o, char* ws, int B,
                       int T, const int32_t* len, cudaStream_t st) {
  auto F = [&](size_t off) { return (float*)ws + off; };
  const int H = h->H;
  float* FF = F(o.f);
  const float* gb = nullptr;
  if (h->G && sid) {
    gather_rows_kernel<<<blocks((long long)B * h->G), 256, 0, st>>>(h->p("emb_g.weight"), sid, F(o.g), B, h->G, h->cfg.n_speakers);
    MB_LAUNCH_CHECK("gather_rows_kernel");
    TRY(conv("dp.cond", F(o.g), h->G, h->G, h->p("dp.cond.weight"), h->p("dp.cond.bias"), nullptr, 0, F(o.gb), H, H, B, 1, 1, 1, 0,
             nullptr, 0, 0, 0, EPI_STORE_, st));
    gb = F(o.gb);
  }
  float *S0 = F(o.s0), *S1 = F(o.s1), *S2 = F(o.s2), *S3 = F(o.s3), *Z = F(o.z);
  if (h->cfg.use_sdp) {
    // StochasticDurationPredictor reverse (vits.py:48-93): x = proj(DDS(pre(x) + cond(g))) * mask
    TRY(conv("dp.pre", X, (long long)H * T, H, h->p("dp.pre.weight"), h->p("dp.pre.bias"), gb, H, S0, (long long)H * T, H, B, T, 1,
             1, 0, nullptr, 0, 0, 0, EPI_STORE_, st));
    TRY(ddsconv(h, "dp.convs.", S0, S1, S2, B, H, T, len, st));
    TRY(conv1x1("dp.proj", S0, H, h->p("dp.proj.weight"), h->p("dp.proj.bias"), S3, H, B, T, st, len, 0, 1));
    // z = noise * noise_scale_w; flows: Flip, ConvFlow 7, Flip, ConvFlow 5, Flip, ConvFlow 3, Flip, ElementwiseAffine
    scale_bias_kernel<<<blocks(2LL * B * T), 256, 0, st>>>(noise, noise_scale_w, nullptr, Z, B, 2, T);
    MB_LAUNCH_CHECK("scale_bias_kernel");
    int c0 = 1, c1 = 0;  // after the first Flip, channel 1 is x0 and channel 0 is x1
    for (int f : {7, 5, 3}) {
      const std::string n = "dp.flows." + std::to_string(f);
      // ConvFlow: h = pre(x0); h = DDS(h + x); h = proj(h) * mask (fused into the spline kernel)
      TRY(conv("convflow pre", Z + (long long)c0 * T, 2LL * T, 1, h->p(n + ".pre.weight"), h->p(n + ".pre.bias"), nullptr, 0, S0,
               (long long)H * T, H, B, T, 1, 1, 0, nullptr, 0, 0, 0, EPI_STORE_, st));
      add_kernel<<<blocks((long long)B * H * T), 256, 0, st>>>(S0, S3, S0, (long long)B * H * T);
      MB_LAUNCH_CHECK("add_kernel");
      TRY(ddsconv(h, n + ".convs.", S0, S1, S2, B, H, T, len, st));
      spline_flow_kernel<<<blocks((long long)B * T * 32, 128), 128, 0, st>>>(S0, h->p(n + ".proj.weight"), h->p(n + ".proj.bias"),
                                                                              Z, B, H, T, c0, c1, len);
      MB_LAUNCH_CHECK("spline_flow_kernel");
      std::swap(c0, c1);  // Flip
    }
    durations_kernel<<<B, 256, 0, st>>>(Z, h->p("dp.flows.0.m"), h->p("dp.flows.0.logs"), 2, length_scale, B, T, len, w_ceil,
                                        y_lengths, logw_out);
    MB_LAUNCH_CHECK("durations_kernel");
    return MB_OK;
  }
  // DurationPredictor (vits.py:116-130)
  const int D = h->DPC;
  const float* xd = X;
  if (gb) {
    scale_bias_kernel<<<blocks((long long)B * H * T), 256, 0, st>>>(X, 1.f, gb, S0, B, H, T);
    MB_LAUNCH_CHECK("scale_bias_kernel");
    xd = S0;
  }
  TRY(conv("dp.conv_1", xd, (long long)H * T, H, h->p("dp.conv_1.weight"), h->p("dp.conv_1.bias"), nullptr, 0, S3,
           (long long)D * T, D, B, T, 3, 1, 1, len, 1, 0, 1, EPI_STORE_, st));
  TRY(layernorm(S3, nullptr, h->p("dp.norm_1.gamma"), h->p("dp.norm_1.beta"), nullptr, S3, B, D, T, 0, nullptr, st));
  TRY(conv("dp.conv_2", S3, (long long)D * T, D, h->p("dp.conv_2.weight"), h->p("dp.conv_2.bias"), nullptr, 0, FF,
           (long long)D * T, D, B, T, 3, 1, 1, len, 1, 0, 1, EPI_STORE_, st));
  TRY(layernorm(FF, nullptr, h->p("dp.norm_2.gamma"), h->p("dp.norm_2.beta"), nullptr, FF, B, D, T, 0, nullptr, st));
  TRY(conv1x1("dp.proj", FF, D, h->p("dp.proj.weight"), h->p("dp.proj.bias"), Z, 1, B, T, st, len, 1, 1));
  durations_kernel<<<B, 256, 0, st>>>(Z, nullptr, nullptr, 1, length_scale, B, T, len, w_ceil, y_lengths, logw_out);
  MB_LAUNCH_CHECK("durations_kernel");
  return MB_OK;
}

// ResidualCouplingLayer flow.flows.(2f) in reverse, mean only (vits_modules.py:317-336), in place on z [B, I, T]: h =
// pre(x0) * mask, WN (vits_modules.py:141-169) with the cond_layer(g) bias when g [B, G] is given, then x1 = (x1 -
// post(out * mask) * mask) * mask.  Scratch: hh, acts, out [B, H, T], xin [B, 2H, T], cond [B, 2H * 4].
int coupling_layer(const mb_vits* h, int f, float* z, const float* g, float* hh, float* xin, float* acts, float* out, float* cond,
                   int B, int T, const int32_t* len, cudaStream_t st) {
  const int H = h->H, Ih = h->I / 2;
  const long long zbs = (long long)h->I * T, hbs = (long long)H * T;
  const std::string n = "flow.flows." + std::to_string(2 * f), e = n + ".enc.";
  TRY(conv("coupling pre", z, zbs, Ih, h->p(n + ".pre.weight"), h->p(n + ".pre.bias"), nullptr, 0, hh, hbs, H, B, T, 1, 1, 0, len,
           0, 1, 0, EPI_STORE_, st));
  if (g)
    TRY(conv("cond_layer", g, h->G, h->G, h->p(e + "cond_layer.weight"), h->p(e + "cond_layer.bias"), nullptr, 0, cond,
             2LL * H * kWnLayers, 2 * H * kWnLayers, B, 1, 1, 1, 0, nullptr, 0, 0, 0, EPI_STORE_, st));
  for (int l = 0; l < kWnLayers; ++l) TRY(wn_layer(h, e, l, hh, xin, acts, out, g ? cond : nullptr, B, T, len, st));
  return conv("coupling post", out, hbs, H, h->p(n + ".post.weight"), h->p(n + ".post.bias"), nullptr, 0, z + (long long)Ih * T, zbs,
              Ih, B, T, 1, 1, 0, len, 1, 1, 0, EPI_SUB, st);
}

void declare(mb_vits* h) {
  WeightTable& w = h->w;
  const int64_t I = h->I, H = h->H, F = h->F, G = h->G, K = h->K, dk = H / h->NH;
  auto conv_w = [&](const std::string& n, int64_t co, int64_t ci, int64_t k) {
    w.add(n + ".weight", {co, ci, k});
    w.add(n + ".bias", {co});
  };
  auto ln = [&](const std::string& n, int64_t c) {
    w.add(n + ".gamma", {c});
    w.add(n + ".beta", {c});
  };
  w.add("enc_p.emb.weight", {h->cfg.n_vocab, H});
  w.add("enc_p.emo_proj.weight", {H, kEmo});
  w.add("enc_p.emo_proj.bias", {H});
  for (int l = 0; l < h->NL; ++l) {
    const std::string L = std::to_string(l), a = "enc_p.encoder.attn_layers." + L;
    for (const char* c : {".conv_q", ".conv_k", ".conv_v", ".conv_o"}) conv_w(a + c, H, H, 1);
    w.add(a + ".emb_rel_k", {1, 2 * kWindow + 1, dk});
    w.add(a + ".emb_rel_v", {1, 2 * kWindow + 1, dk});
    ln("enc_p.encoder.norm_layers_1." + L, H);
    conv_w("enc_p.encoder.ffn_layers." + L + ".conv_1", F, H, K);
    conv_w("enc_p.encoder.ffn_layers." + L + ".conv_2", H, F, K);
    ln("enc_p.encoder.norm_layers_2." + L, H);
  }
  conv_w("enc_p.proj", 2 * I, H, 1);
  if (G) w.add("emb_g.weight", {h->cfg.n_speakers, G});
  auto dds = [&](const std::string& n, int64_t c) {
    for (int l = 0; l < kSdpLayers; ++l) {
      const std::string L = std::to_string(l);
      conv_w(n + ".convs_sep." + L, c, 1, 3);
      conv_w(n + ".convs_1x1." + L, c, c, 1);
      ln(n + ".norms_1." + L, c);
      ln(n + ".norms_2." + L, c);
    }
  };
  if (h->cfg.use_sdp) {
    conv_w("dp.pre", H, H, 1);
    conv_w("dp.proj", H, H, 1);
    dds("dp.convs", H);
    if (G) conv_w("dp.cond", H, G, 1);
    w.add("dp.flows.0.m", {2, 1});
    w.add("dp.flows.0.logs", {2, 1});
    for (int f : {3, 5, 7}) {
      const std::string n = "dp.flows." + std::to_string(f);
      conv_w(n + ".pre", H, 1, 1);
      dds(n + ".convs", H);
      conv_w(n + ".proj", 3 * kBins - 1, H, 1);
    }
  } else {
    const int64_t D = h->DPC;
    conv_w("dp.conv_1", D, H, 3);
    ln("dp.norm_1", D);
    conv_w("dp.conv_2", D, D, 3);
    ln("dp.norm_2", D);
    conv_w("dp.proj", 1, D, 1);
    if (G) conv_w("dp.cond", H, G, 1);
  }
  for (int f = 0; f < 4; ++f) {
    const std::string n = "flow.flows." + std::to_string(2 * f);
    conv_w(n + ".pre", H, I / 2, 1);
    for (int l = 0; l < kWnLayers; ++l) {
      const std::string L = std::to_string(l);
      conv_w(n + ".enc.in_layers." + L, 2 * H, H, kWnK);
      conv_w(n + ".enc.res_skip_layers." + L, l < kWnLayers - 1 ? 2 * H : H, H, 1);
    }
    if (G) conv_w(n + ".enc.cond_layer", 2 * H * kWnLayers, G, 1);
    conv_w(n + ".post", I / 2, H, 1);
  }
  conv_w("dec.conv_pre", h->C0, I, 7);
  if (G) conv_w("dec.cond", h->C0, G, 1);
  w.add_derived("dec.conv_pre+cond.weight", (size_t)h->C0 * (I + G) * 7);
  w.add_derived("dec.conv_pre+cond.bias", (size_t)h->C0);
  w.ignored = [](const std::string& n) {
    return n.rfind("enc_q.", 0) == 0 || n.rfind("dp.post_", 0) == 0 || n.rfind("dp.flows.1.", 0) == 0 ||
           n.rfind("net_d.", 0) == 0 || n.rfind("discriminators.", 0) == 0;
  };
}

}  // namespace

extern "C" {

int32_t mb_vits_max_tokens(void) { return kMaxTokens; }

int mb_vits_create(const mb_vits_config* cfg, mb_vits** out) {
  if (!cfg || !out) return fail(MB_ERR_INVALID, "mb_vits_create: null argument");
  const mb_vits_config& c = *cfg;
  if (c.n_vocab < 1) return fail(MB_ERR_INVALID, "mb_vits_create: n_vocab %d", c.n_vocab);
  if (c.inter_channels < 2 || c.inter_channels % 2)
    return fail(MB_ERR_INVALID, "mb_vits_create: inter_channels %d must be even", c.inter_channels);
  if (c.hidden_channels < 1 || c.n_heads < 1 || c.hidden_channels % c.n_heads || c.hidden_channels / c.n_heads > kMaxHead)
    return fail(MB_ERR_INVALID, "mb_vits_create: hidden_channels %d / n_heads %d (head width <= %d)", c.hidden_channels, c.n_heads,
                kMaxHead);
  if (c.filter_channels < 1 || c.n_layers < 1) return fail(MB_ERR_INVALID, "mb_vits_create: filter_channels / n_layers");
  if (c.kernel_size < 1 || c.kernel_size % 2 == 0 || c.kernel_size > CV_MAXK)
    return fail(MB_ERR_INVALID, "mb_vits_create: kernel_size %d (odd, <= %d)", c.kernel_size, CV_MAXK);
  if (c.n_speakers == 1 || c.n_speakers < 0)
    return fail(MB_ERR_INVALID, "mb_vits_create: n_speakers %d (0, or > 1: Vits builds emb_g only for n_speakers > 1)", c.n_speakers);
  if ((c.n_speakers > 1) != (c.gin_channels > 0))
    return fail(MB_ERR_INVALID, "mb_vits_create: gin_channels %d with n_speakers %d", c.gin_channels, c.n_speakers);
  if (c.use_sdp != 0 && c.use_sdp != 1) return fail(MB_ERR_INVALID, "mb_vits_create: use_sdp %d", c.use_sdp);
  if (c.num_kernels < 1 || c.num_kernels > 4 || c.num_upsamples < 1 || c.num_upsamples > 8)
    return fail(MB_ERR_INVALID, "mb_vits_create: decoder lists");
  mb_gan_config g{};
  g.kind = MB_GAN_VITS;
  g.num_mels = c.inter_channels + c.gin_channels;
  g.upsample_initial_channel = c.upsample_initial_channel;
  g.num_upsamples = c.num_upsamples;
  for (int i = 0; i < 8; ++i) g.upsample_rates[i] = c.upsample_rates[i], g.upsample_kernel_sizes[i] = c.upsample_kernel_sizes[i];
  g.num_kernels = c.num_kernels;
  for (int i = 0; i < 4; ++i) {
    g.resblock_kernel_sizes[i] = c.resblock_kernel_sizes[i];
    for (int j = 0; j < 4; ++j) g.resblock_dilation_sizes[i][j] = c.resblock_dilation_sizes[i][j];
  }
  g.num_dilations = c.num_dilations;
  g.resblock_type = c.resblock_type;
  g.precision = c.precision;
  mb_gan* gan = nullptr;
  if (int rc = mb_gan_create(&g, &gan)) return rc;
  mb_vits* h = new mb_vits();
  h->cfg = c;
  h->gan = gan;
  h->I = c.inter_channels;
  h->H = c.hidden_channels;
  h->F = c.filter_channels;
  h->G = c.gin_channels;
  h->NH = c.n_heads;
  h->NL = c.n_layers;
  h->K = c.kernel_size;
  h->C0 = c.upsample_initial_channel;
  h->DPC = c.use_sdp ? c.hidden_channels : 256;  // DurationPredictor(hidden, 256, 3, ...) (vits.py:453)
  declare(h);
  h->table_bytes = align_up(h->w.floats() * sizeof(float), 256);
  *out = h;
  return MB_OK;
}

void mb_vits_destroy(mb_vits* h) {
  if (!h) return;
  mb_gan_destroy(h->gan);
  delete h;
}

size_t mb_vits_arena_bytes(const mb_vits* h) { return h ? h->table_bytes + mb_gan_arena_bytes(h->gan) : 0; }

int mb_vits_set_arena(mb_vits* h, void* arena, size_t bytes) {
  if (int rc = check_arena("mb_vits_set_arena", h, arena, bytes, mb_vits_arena_bytes(h), 256)) return rc;
  h->w.attach((float*)arena);
  h->arena = (float*)arena;
  h->finalized = false;
  return mb_gan_set_arena(h->gan, (char*)arena + h->table_bytes, bytes - h->table_bytes);
}

int mb_vits_set_weight(mb_vits* h, const char* name, const float* w, const int64_t* dims, int32_t ndim, void* stream) {
  if (!h || !name) return fail(MB_ERR_INVALID, "mb_vits_set_weight: null argument");
  const std::string n(name);
  h->finalized = false;
  // the decoder's layers but conv_pre / cond (folded at finalize) live in the generator
  if (n.rfind("dec.", 0) == 0 && n.rfind("dec.conv_pre.", 0) != 0 && n.rfind("dec.cond.", 0) != 0)
    return mb_gan_set_weight(h->gan, name + 4, w, dims, ndim, stream);
  return h->w.set("mb_vits_set_weight", name, w, dims, ndim, stream);
}

int mb_vits_finalize(mb_vits* h, void* stream) {
  if (!h) return fail(MB_ERR_INVALID, "mb_vits_finalize: null handle");
  if (!h->arena) return fail(MB_ERR_STATE, "mb_vits_finalize: set the arena first");
  if (int rc = h->w.check_all_set("mb_vits_finalize")) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  float* wf = h->w.ptr("dec.conv_pre+cond.weight");
  float* bf = h->w.ptr("dec.conv_pre+cond.bias");
  const long long n = (long long)h->C0 * (h->I + h->G) * 7;
  fold_cond_kernel<<<blocks(n), 256, 0, st>>>(h->p("dec.conv_pre.weight"), h->p("dec.conv_pre.bias"), h->po("dec.cond.weight"),
                                              h->po("dec.cond.bias"), wf, bf, h->C0, h->I, h->G, 7);
  MB_LAUNCH_CHECK("fold_cond_kernel");
  const int64_t dw[3] = {h->C0, h->I + h->G, 7}, db[1] = {h->C0};
  if (int rc = mb_gan_set_weight(h->gan, "conv_pre.weight", wf, dw, 3, stream)) return rc;
  if (int rc = mb_gan_set_weight(h->gan, "conv_pre.bias", bf, db, 1, stream)) return rc;
  if (int rc = mb_gan_finalize(h->gan)) return rc;
  h->finalized = true;
  return MB_OK;
}

int32_t mb_vits_hop(const mb_vits* h) { return h ? mb_gan_hop(h->gan) : 0; }

size_t mb_vits_durations_workspace_bytes(const mb_vits* h, int32_t batch, int32_t t_x) {
  if (!h || batch <= 0 || t_x <= 0) return 0;
  return dur_layout(h, batch, t_x).total;
}

int mb_vits_durations(mb_vits* h, const int32_t* x, const int32_t* x_lengths, int32_t B, int32_t T, const int32_t* sid,
                      const float* emo, const float* noise, float noise_scale_w, float length_scale, float* m_p, float* logs_p,
                      int32_t* w_ceil, int32_t* y_lengths, void* workspace, size_t workspace_bytes, void* stream) {
  const char* fn = "mb_vits_durations";
  if (!h || !x || !x_lengths || !emo || !m_p || !logs_p || !w_ceil || !y_lengths) return fail(MB_ERR_INVALID, "%s: null argument", fn);
  if (!h->finalized) return fail(MB_ERR_STATE, "%s: weights not finalized", fn);
  if (B <= 0 || T <= 0 || T > kMaxTokens) return fail(MB_ERR_INVALID, "%s: batch %d, t_x %d (1..%d)", fn, B, T, kMaxTokens);
  if (h->G && !sid) return fail(MB_ERR_INVALID, "%s: a multi-speaker model needs sid", fn);
  if (h->cfg.use_sdp && !noise) return fail(MB_ERR_INVALID, "%s: the stochastic duration predictor needs noise", fn);
  char* ws;
  const DurWs o = dur_layout(h, B, T);
  if (int rc = bind(fn, workspace, workspace_bytes, o.total, &ws)) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  auto F = [&](size_t off) { return (float*)ws + off; };
  const int H = h->H, I = h->I;
  const int32_t* len = x_lengths;
  float* X = F(o.x);
  // ---- text encoder (vits.py:167-177, vits_modules.py:407-419)
  TRY(conv("emo_proj", emo, kEmo, kEmo, h->p("enc_p.emo_proj.weight"), h->p("enc_p.emo_proj.bias"), nullptr, 0, F(o.e), H, H, B, 1,
           1, 1, 0, nullptr, 0, 0, 0, EPI_STORE_, st));
  embed_kernel<<<blocks((long long)B * H * T), 256, 0, st>>>(x, h->p("enc_p.emb.weight"), F(o.e), X, B, H, T, h->cfg.n_vocab, len);
  MB_LAUNCH_CHECK("embed_kernel");
  for (int l = 0; l < h->NL; ++l) TRY(enc_layer(h, l, X, o, ws, B, T, len, st));
  TRY(conv1x1("enc_p.proj m", X, H, h->p("enc_p.proj.weight"), h->p("enc_p.proj.bias"), m_p, I, B, T, st, len, 0, 1));
  TRY(conv1x1("enc_p.proj logs", X, H, h->p("enc_p.proj.weight") + (size_t)I * H, h->p("enc_p.proj.bias") + I, logs_p, I, B, T, st,
              len, 0, 1));
  // ---- speaker embedding, duration predictor
  return duration_predictor(h, X, sid, noise, noise_scale_w, length_scale, w_ceil, y_lengths, nullptr, o, ws, B, T, len, st);
}

size_t mb_vits_decode_workspace_bytes(const mb_vits* h, int32_t batch, int32_t t_x, int32_t t_y, int32_t t_dec) {
  if (!h || batch <= 0 || t_x <= 0 || t_y <= 0 || t_dec <= 0 || t_dec > t_y) return 0;
  return dec_layout(h, batch, t_x, t_y, t_dec).total;
}

int mb_vits_decode(mb_vits* h, const float* m_p, const float* logs_p, const int32_t* w_ceil, const int32_t* x_lengths,
                   const int32_t* sid, int32_t B, int32_t Tx, int32_t Ty, const float* eps, float noise_scale, int32_t Td,
                   int32_t ragged, float* wav, float* attn, float* z_p, float* z, float* m_p_y, float* logs_p_y, void* workspace,
                   size_t workspace_bytes, void* stream) {
  const char* fn = "mb_vits_decode";
  if (!h || !m_p || !logs_p || !w_ceil || !x_lengths || !eps || !wav) return fail(MB_ERR_INVALID, "%s: null argument", fn);
  if (!h->finalized) return fail(MB_ERR_STATE, "%s: weights not finalized", fn);
  if (B <= 0 || Tx <= 0 || Ty <= 0 || Td <= 0 || Td > Ty)
    return fail(MB_ERR_INVALID, "%s: batch %d, t_x %d, t_y %d, t_dec %d (1 <= t_dec <= t_y)", fn, B, Tx, Ty, Td);
  if (h->G && !sid) return fail(MB_ERR_INVALID, "%s: a multi-speaker model needs sid", fn);
  char* ws;
  const DecWs o = dec_layout(h, B, Tx, Ty, Td);
  if (int rc = bind(fn, workspace, workspace_bytes, o.total, &ws, 1024)) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  auto F = [&](size_t off) { return (float*)ws + off; };
  const int I = h->I, G = h->G;
  int32_t* cum = (int32_t*)ws + o.cum;
  int32_t* ylen = (int32_t*)ws + o.ylen;
  cumsum_kernel<<<blocks(B, 64), 64, 0, st>>>(w_ceil, x_lengths, cum, ylen, B, Tx);
  MB_LAUNCH_CHECK("cumsum_kernel");
  float* za = F(o.za);
  float* zb = F(o.zb);
  expand_kernel<<<blocks((long long)B * Ty), 256, 0, st>>>(m_p, logs_p, cum, ylen, eps, noise_scale, za, m_p_y, logs_p_y, attn, B,
                                                           I, Tx, Ty);
  MB_LAUNCH_CHECK("expand_kernel");
  if (z_p) MB_CUDA_CHECK(cudaMemcpyAsync(z_p, za, sizeof(float) * B * I * Ty, cudaMemcpyDeviceToDevice, st));
  float* g = nullptr;
  if (G) {
    g = F(o.g);
    gather_rows_kernel<<<blocks((long long)B * G), 256, 0, st>>>(h->p("emb_g.weight"), sid, g, B, G, h->cfg.n_speakers);
    MB_LAUNCH_CHECK("gather_rows_kernel");
  }
  // ---- reverse coupling flow (vits.py:203-210): Flip, layer 6, Flip, layer 4, Flip, layer 2, Flip, layer 0
  float *hh = F(o.hh), *xin = F(o.xin), *acts = F(o.acts), *out = F(o.out), *cond = F(o.cond);
  for (int f = 3; f >= 0; --f) {
    flip_kernel<<<blocks((long long)B * I * Ty), 256, 0, st>>>(za, zb, B, I, Ty);
    MB_LAUNCH_CHECK("flip_kernel");
    std::swap(za, zb);
    TRY(coupling_layer(h, f, za, g, hh, xin, acts, out, cond, B, Ty, ylen, st));
  }
  if (z) MB_CUDA_CHECK(cudaMemcpyAsync(z, za, sizeof(float) * B * I * Ty, cudaMemcpyDeviceToDevice, st));
  // ---- decoder: dec((z * y_mask)[:, :, :t_dec], g) with cond(g) folded into conv_pre over the extra g channels
  float* din = F(o.din);
  dec_input_kernel<<<blocks((long long)B * (I + G) * Td), 256, 0, st>>>(za, g, din, B, I, G, Ty, Td, ylen);
  MB_LAUNCH_CHECK("dec_input_kernel");
  return mb_gan_forward(h->gan, din, ragged ? ylen : nullptr, B, Td, wav, ws + o.gan, mb_gan_workspace_bytes(h->gan, B, Td), stream);
}

}  // extern "C"

namespace {
// mb_vits_debug's workspace: scratch planes (x_in / acts, DDSConv, the coupling layer's h / acts / out), the cond_layer
// output / decoder input, the text encoder's layout (ENC_LAYER, LOGW), LOGW's w_ceil / y_len, the generator's
struct DbgWs {
  size_t s0, s1, s2, s3, dur, ints, gan, total;
};
DbgWs dbg_layout(const mb_vits* h, const mb_vits_debug_spec* s) {
  const size_t B = s->batch, T = s->frames, H = h->H;
  const bool planes = s->kind <= MB_VITS_DBG_DECODER || s->kind == MB_VITS_DBG_COUPLING;
  const bool dur = s->kind == MB_VITS_DBG_ENC_LAYER || s->kind == MB_VITS_DBG_LOGW;
  WsLayout L;
  DbgWs o;
  o.s0 = L.take<float>(planes ? B * 2 * H * T : 0);
  o.s1 = L.take<float>(planes ? B * 2 * H * T : 0);
  o.s2 = L.take<float>(planes ? B * 2 * H * kWnLayers + B * (h->I + h->G) * T : 0);
  o.s3 = L.take<float>(s->kind == MB_VITS_DBG_COUPLING ? B * H * T : 0);
  o.dur = L.take(dur ? dur_layout(h, B, T).total : 0);
  o.ints = L.take<int32_t>(s->kind == MB_VITS_DBG_LOGW ? B * T + B : 0);
  L.align = 1024;
  o.gan = L.take(s->kind == MB_VITS_DBG_DECODER ? mb_gan_workspace_bytes(h->gan, (int32_t)B, (int32_t)T) : 0);
  o.total = L.total();
  return o;
}
}  // namespace

extern "C" {

size_t mb_vits_debug_workspace_bytes(const mb_vits* h, const mb_vits_debug_spec* s) {
  if (!h || !s || s->batch <= 0 || s->frames <= 0) return 0;
  return dbg_layout(h, s).total;
}

int mb_vits_debug(mb_vits* h, const mb_vits_debug_spec* s, void* workspace, size_t workspace_bytes, void* stream) {
  const char* fn = "mb_vits_debug";
  if (!h || !s || !s->x || !s->y) return fail(MB_ERR_INVALID, "%s: null argument", fn);
  if (!h->finalized) return fail(MB_ERR_STATE, "%s: weights not finalized", fn);
  const int B = s->batch, T = s->frames, H = h->H;
  if (B <= 0 || T <= 0) return fail(MB_ERR_INVALID, "%s: empty batch", fn);
  const bool unmasked = s->kind == MB_VITS_DBG_DECODER || s->kind == MB_VITS_DBG_CONV || s->kind == MB_VITS_DBG_LAYERNORM;
  if (!unmasked && !s->lengths) return fail(MB_ERR_INVALID, "%s: lengths required", fn);
  char* ws;
  const DbgWs o = dbg_layout(h, s);
  if (int rc = bind(fn, workspace, workspace_bytes, o.total, &ws, 1024)) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  float* s0 = (float*)ws + o.s0;
  float* s1 = (float*)ws + o.s1;
  float* s2 = (float*)ws + o.s2;
  const int32_t* len = s->lengths;
  const size_t n = (size_t)B * H * T;
  switch (s->kind) {
    case MB_VITS_DBG_SPLINE: {  // y = z [B, 2, T] (copied from x2) after ConvFlow `index`'s spline on h = x
      if (!s->x2 || (s->index != 3 && s->index != 5 && s->index != 7) || !h->cfg.use_sdp || (s->c0 | s->c1) != 1 || s->c0 == s->c1)
        return fail(MB_ERR_INVALID, "%s: spline needs z, a ConvFlow index 3 / 5 / 7 and channels {0, 1}", fn);
      MB_CUDA_CHECK(cudaMemcpyAsync(s->y, s->x2, sizeof(float) * 2 * B * T, cudaMemcpyDeviceToDevice, st));
      const std::string p = "dp.flows." + std::to_string(s->index) + ".proj";
      spline_flow_kernel<<<blocks((long long)B * T * 32, 128), 128, 0, st>>>(s->x, h->p(p + ".weight"), h->p(p + ".bias"), s->y, B,
                                                                              H, T, s->c0, s->c1, len);
      MB_LAUNCH_CHECK("spline_flow_kernel");
      return MB_OK;
    }
    case MB_VITS_DBG_ATTN: {  // y = attention of encoder layer `index` over q = x, k = x2, v = x3
      if (!s->x2 || !s->x3 || s->index < 0 || s->index >= h->NL || T > kMaxTokens)
        return fail(MB_ERR_INVALID, "%s: attention needs q, k, v, a layer index and T <= %d", fn, kMaxTokens);
      const std::string a = "enc_p.encoder.attn_layers." + std::to_string(s->index);
      rel_attn_kernel<<<dim3(T, h->NH, B), 128, 0, st>>>(s->x, s->x2, s->x3, h->p(a + ".emb_rel_k"), h->p(a + ".emb_rel_v"), s->y, H,
                                                          h->NH, T, len);
      MB_LAUNCH_CHECK("rel_attn_kernel");
      return MB_OK;
    }
    case MB_VITS_DBG_WN: {  // WN layer `sub` of coupling layer `index`: y = x after the residual update, y2 = skip stream in/out
      if (!s->y2 || s->index < 0 || s->index > 3 || s->sub < 0 || s->sub >= kWnLayers || (s->x2 && !h->G))
        return fail(MB_ERR_INVALID, "%s: WN needs y2, a coupling index 0..3 and a layer 0..3 (g only with speakers)", fn);
      const std::string e = "flow.flows." + std::to_string(2 * s->index) + ".enc.";
      MB_CUDA_CHECK(cudaMemcpyAsync(s->y, s->x, sizeof(float) * n, cudaMemcpyDeviceToDevice, st));
      if (s->x2)
        TRY(conv("cond_layer", s->x2, h->G, h->G, h->p(e + "cond_layer.weight"), h->p(e + "cond_layer.bias"), nullptr, 0, s2,
                 2LL * H * kWnLayers, 2 * H * kWnLayers, B, 1, 1, 1, 0, nullptr, 0, 0, 0, EPI_STORE_, st));
      return wn_layer(h, e, s->sub, s->y, s0, s1, s->y2, s->x2 ? s2 : nullptr, B, T, len, st);
    }
    case MB_VITS_DBG_DDSCONV: {  // y = DDSConv with prefix "dp.convs." (index 0) or "dp.flows.<index>.convs." on x
      if (!h->cfg.use_sdp || (s->index != 0 && s->index != 3 && s->index != 5 && s->index != 7))
        return fail(MB_ERR_INVALID, "%s: DDSConv index 0 / 3 / 5 / 7 of a stochastic duration predictor", fn);
      MB_CUDA_CHECK(cudaMemcpyAsync(s->y, s->x, sizeof(float) * n, cudaMemcpyDeviceToDevice, st));
      const std::string p = s->index ? "dp.flows." + std::to_string(s->index) + ".convs." : std::string("dp.convs.");
      return ddsconv(h, p, s->y, s0, s1, B, H, T, len, st);
    }
    case MB_VITS_DBG_DECODER: {  // y = dec(x, g) for z = x [B, inter, T], g = emb_g[sid] (sid in x2 as int32), no mask
      const int G = h->G, I = h->I;
      if (G && !s->x2) return fail(MB_ERR_INVALID, "%s: decoder of a multi-speaker model needs sid", fn);
      float* g = nullptr;
      if (G) {
        g = s2;
        gather_rows_kernel<<<blocks((long long)B * G), 256, 0, st>>>(h->p("emb_g.weight"), (const int32_t*)s->x2, g, B, G,
                                                                     h->cfg.n_speakers);
        MB_LAUNCH_CHECK("gather_rows_kernel");
      }
      float* din = s2 + (size_t)B * 2 * H * kWnLayers;
      dec_input_kernel<<<blocks((long long)B * (I + G) * T), 256, 0, st>>>(s->x, g, din, B, I, G, T, T, nullptr);
      MB_LAUNCH_CHECK("dec_input_kernel");
      return mb_gan_forward(h->gan, din, nullptr, B, T, s->y, ws + o.gan, mb_gan_workspace_bytes(h->gan, B, T), stream);
    }
    case MB_VITS_DBG_CONV: {  // one conv1d_kernel launch through conv(), whose limits it keeps
      if (!s->w || s->cin < 1 || s->cout < 1 || s->k < 1 || s->dil < 1 || s->pad < 0 || s->mode < EPI_STORE_ || s->mode > EPI_SUB ||
          (s->bbias && s->bbs < s->cout))
        return fail(MB_ERR_INVALID, "%s: conv needs a weight, cin, cout, k, dil >= 1, pad >= 0, mode 0..2, bbs >= cout", fn);
      return conv("mb_vits_debug conv", s->x, s->xbs, s->cin, s->w, s->bias, s->bbias, s->bbs, s->y, s->ybs, s->cout, B, T, s->k,
                  s->dil, s->pad, len, s->in_mask, s->out_mask, s->relu, s->mode, st);
    }
    case MB_VITS_DBG_LAYERNORM: {  // y = res + act(LN_cin(x + x2)) (* mask) with gamma = w, beta = bias
      if (!s->w || !s->bias || s->cin < 1) return fail(MB_ERR_INVALID, "%s: layernorm needs gamma, beta and cin", fn);
      return layernorm(s->x, s->x2, s->w, s->bias, s->res, s->y, B, s->cin, T, s->gelu, len, st);
    }
    case MB_VITS_DBG_ENC_LAYER: {  // y = text-encoder layer `index` on x
      if (s->index < 0 || s->index >= h->NL || T > kMaxTokens)
        return fail(MB_ERR_INVALID, "%s: encoder layer 0..%d and T <= %d", fn, h->NL - 1, kMaxTokens);
      MB_CUDA_CHECK(cudaMemcpyAsync(s->y, s->x, sizeof(float) * n, cudaMemcpyDeviceToDevice, st));
      return enc_layer(h, s->index, s->y, dur_layout(h, B, T), ws + o.dur, B, T, len, st);
    }
    case MB_VITS_DBG_LOGW: {  // y = logw [B, 1, T] of the duration predictor on the encoder output x, y2 = w_ceil, y_len
      if ((h->cfg.use_sdp && !s->x3) || (s->x2 && !h->G))
        return fail(MB_ERR_INVALID, "%s: logw needs the SDP noise in x3 (stochastic predictor) and sid only with speakers", fn);
      int32_t* wc = s->y2 ? (int32_t*)s->y2 : (int32_t*)ws + o.ints;
      return duration_predictor(h, s->x, (const int32_t*)s->x2, s->x3, s->noise_scale_w, s->length_scale, wc, wc + (size_t)B * T, s->y,
                                dur_layout(h, B, T), ws + o.dur, B, T, len, st);
    }
    case MB_VITS_DBG_COUPLING: {  // y = coupling layer flow.flows.(2 * index) in reverse on z = x
      if (s->index < 0 || s->index > 3 || (s->x2 && !h->G))
        return fail(MB_ERR_INVALID, "%s: coupling index 0..3 (g only with speakers)", fn);
      MB_CUDA_CHECK(cudaMemcpyAsync(s->y, s->x, sizeof(float) * B * h->I * T, cudaMemcpyDeviceToDevice, st));
      return coupling_layer(h, s->index, s->y, s->x2, s1, s0, s1 + n, (float*)ws + o.s3, s2, B, T, len, st);
    }
    default:
      return fail(MB_ERR_INVALID, "%s: unknown kind %d", fn, s->kind);
  }
}

}  // extern "C"
