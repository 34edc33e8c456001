// GAN generator plan + C ABI (mb_gan_*): HiFi-GAN Generator.forward (hifigan/models.py:134-150) and
// FreGAN.forward (fregan/generator.py:137-166) lowered to a list of tap-conv ops over a handful of
// workspace buffers.  See include/mockingbird_b200.h for the contract.
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include "gan_kernels.h"
#include "gan_tc.h"
#include "mb_common.h"

namespace mb {

namespace {

constexpr int BUF_NONE = -1;
constexpr int BUF_IN = 100;   // caller's mel
constexpr int BUF_OUT = 101;  // caller's wav

enum OpKind { OP_CONV = 0, OP_ADD = 1 };

struct Layer {
  OpKind kind = OP_CONV;
  std::string name;  // state_dict prefix ("ups.0", "resblocks.4.convs2.1", ...)
  int cin = 0, cout = 0, k = 1, dil = 1, stride = 1;
  int cin_w = 0, cout_w = 0;  // channel counts of the checkpoint tensors (cin / cout may be zero-padded, see pad_channels)
  bool transposed = false;
  int nearest = 1;  // nearest-neighbour upsample factor in front of a 1x1 conv (Fre-GAN res_output)
  float in_slope = 1.f;
  int src = BUF_NONE, dst = BUF_NONE, res = BUF_NONE, dst2 = BUF_NONE;
  int mode = EPI_STORE;
  float div = 1.f;
  int act_tanh = 0;
  int rate_in = 1, rate_out = 1;  // rows per mel frame at input / output
  size_t w_off = 0, b_off = 0;    // float offsets into the fp32 arena section
  bool w_set = false, b_set = false;
  TapConv taps{};                 // static part (B, Lin, Lout, lengths filled per call)
  TcLayer tc{};                   // tensor-core packing info (MB_PREC_F16TC)
};

void build_taps(Layer& L) {
  TapConv& t = L.taps;
  memset(&t, 0, sizeof(t));
  t.Cin = L.cin;
  t.Cout = L.cout;
  t.in_slope = L.in_slope;
  t.mode = L.mode;
  t.div = L.div;
  t.act_tanh = L.act_tanh;
  t.len_mul_in = L.rate_in;
  t.len_mul_out = L.rate_out;
  if (L.transposed) {
    // ConvTranspose1d(k, stride=s, padding=p=s/2+s%2, output_padding=s%2) (models.py:120-123):
    //   out[i*s - p + kk] += x[i] * w[:, :, kk]   ->   phase r = o mod s gathers taps kk == r+p (mod s)
    const int s = L.stride, p = s / 2 + s % 2;
    t.stride = s;
    for (int r = 0; r < s; ++r) {
      int n = 0;
      for (int kk = 0; kk < L.k; ++kk) {
        const int num = r + p - kk;
        if (((num % s) + s) % s != 0) continue;
        t.off[r][n] = num >= 0 ? num / s : -((-num) / s);
        t.slab[r][n] = kk;
        ++n;
      }
      t.ntaps[r] = n;
    }
  } else if (L.nearest > 1) {
    // nn.Upsample(scale_factor=u, 'nearest') + 1x1 conv: out[q*u + r] = W x[q]
    t.stride = L.nearest;
    for (int r = 0; r < L.nearest; ++r) {
      t.ntaps[r] = 1;
      t.off[r][0] = 0;
      t.slab[r][0] = 0;
    }
  } else {
    // Conv1d(k, dilation=d, padding=get_padding(k,d)=(k*d-d)/2) (utils/util.py:60-61)
    const int pad = (L.k * L.dil - L.dil) / 2;
    t.stride = 1;
    t.ntaps[0] = L.k;
    for (int kk = 0; kk < L.k; ++kk) {
      t.off[0][kk] = kk * L.dil - pad;
      t.slab[0][kk] = kk;
    }
  }
}

}  // namespace

}  // namespace mb

using namespace mb;

struct mb_gan {
  mb_gan_config cfg{};
  std::vector<Layer> layers;
  int hop = 1;
  // per-buffer max (channels * rows-per-frame); bytes = B * T * that * 4
  std::vector<size_t> buf_cr;
  float* arena = nullptr;
  size_t arena_bytes = 0;
  size_t f32_floats = 0;   // fp32 section of the arena (weights + biases)
  size_t tc_bytes = 0;     // tensor-core section (packed fp16 images)
  bool finalized = false;
};

namespace {

int new_buf(mb_gan* h) {
  h->buf_cr.push_back(0);
  return (int)h->buf_cr.size() - 1;
}

void touch(mb_gan* h, int buf, int c, int rate) {
  if (buf >= 0 && buf < (int)h->buf_cr.size()) {
    const size_t cr = (size_t)c * rate;
    if (cr > h->buf_cr[buf]) h->buf_cr[buf] = cr;
  }
}

// Tensor-core path: internal tensors with fewer than 32 channels (Fre-GAN's full-rate stage has 16) are carried with
// 32 channels, the extra ones identically zero (zero weight rows / columns and biases), so that the whole stage runs
// on the C = 32 tensor-core kernels instead of the FP32 FFMA kernels.  MB_GAN_PAD16=0 disables it.
int pad_channels(const mb_gan* h, int c) {
  static const bool env = [] {
    const char* e = getenv("MB_GAN_PAD16");
    return e ? atoi(e) != 0 : true;
  }();
  return (env && h->cfg.precision != MB_PREC_FP32 && c > 1 && c < 32) ? 32 : c;
}

// run-time switches of the Fre-GAN lowering on the tensor-core path (A/B measurements):
//   MB_FREGAN_SPLIT=0   keep "x += cond_up(mel)" fused as a second destination of the cond_up layer (FP32 kernel);
//                       default: cond_up is a plain (tensor-core) transposed conv followed by an add op
//   MB_GAN_NEAREST_TC=1 try the nearest-upsample + 1x1 layers (res_output) on the tensor cores (default 0: their source
//                       buffer is also read by `ups` with a different activation, which the plane analysis rejects)
bool env_flag(const char* name, bool dflt) {
  const char* e = getenv(name);
  return e ? atoi(e) != 0 : dflt;
}

Layer& add_conv(mb_gan* h, const std::string& name, int cin, int cout, int k, int dil, int stride,
                bool transposed, int nearest, float in_slope, int src, int dst, int res, int rate_in) {
  Layer L;
  L.kind = OP_CONV;
  L.name = name;
  L.cin_w = cin;
  L.cout_w = cout;
  if (src != BUF_IN) cin = pad_channels(h, cin);
  if (dst != BUF_OUT) cout = pad_channels(h, cout);
  L.cin = cin;
  L.cout = cout;
  L.k = k;
  L.dil = dil;
  L.stride = transposed ? stride : 1;
  L.transposed = transposed;
  L.nearest = nearest;
  L.in_slope = in_slope;
  L.src = src;
  L.dst = dst;
  L.res = res;
  L.rate_in = rate_in;
  L.rate_out = rate_in * (transposed ? stride : nearest);
  touch(h, src, cin, L.rate_in);
  touch(h, dst, cout, L.rate_out);
  h->layers.push_back(L);
  return h->layers.back();
}

// one multi-receptive-field stage (models.py:139-144): S = mean_j resblock_j(X)
void add_mrf(mb_gan* h, int stage, int ch, int rate, int X, int R, int T, int S) {
  const mb_gan_config& c = h->cfg;
  const int nk = c.num_kernels;
  for (int j = 0; j < nk; ++j) {
    const int k = c.resblock_kernel_sizes[j];
    const std::string base = "resblocks." + std::to_string(stage * nk + j);
    const int mode = (nk == 1 || j == 0) ? EPI_STORE : (j == nk - 1 ? EPI_ADD_DIV : EPI_ADD);
    const int nd = c.num_dilations;
    if (c.resblock_type == 1) {
      for (int m = 0; m < nd; ++m) {
        const int d = c.resblock_dilation_sizes[j][m];
        const int cur = (m == 0) ? X : R;
        add_conv(h, base + ".convs1." + std::to_string(m), ch, ch, k, d, 1, false, 1, 0.1f, cur, T, BUF_NONE, rate);
        const bool last = (m == nd - 1);
        Layer& c2 = add_conv(h, base + ".convs2." + std::to_string(m), ch, ch, k, 1, 1, false, 1, 0.1f, T,
                             last ? S : R, cur, rate);
        if (last) {
          c2.mode = mode;
          c2.div = (float)nk;
          if (nk == 1) c2.mode = EPI_STORE;
        }
      }
    } else {
      int cur = X, other = R;
      for (int m = 0; m < nd; ++m) {
        const int d = c.resblock_dilation_sizes[j][m];
        const bool last = (m == nd - 1);
        Layer& cc = add_conv(h, base + ".convs." + std::to_string(m), ch, ch, k, d, 1, false, 1, 0.1f, cur,
                             last ? S : other, cur, rate);
        if (last) {
          cc.mode = mode;
          cc.div = (float)nk;
          if (nk == 1) cc.mode = EPI_STORE;
        }
        cur = other;
        other = (cur == R) ? T : R;
      }
    }
  }
}

int build_plan(mb_gan* h) {
  const mb_gan_config& c = h->cfg;
  if (c.num_upsamples < 1 || c.num_upsamples > 8 || c.num_kernels < 1 || c.num_kernels > 4 ||
      c.num_dilations < 1 || c.num_dilations > 4 || (c.resblock_type != 1 && c.resblock_type != 2))
    return fail(MB_ERR_INVALID, "mb_gan_create: unsupported generator config");
  for (int j = 0; j < c.num_kernels; ++j)
    if (c.resblock_kernel_sizes[j] > kMaxTaps || c.resblock_kernel_sizes[j] % 2 == 0)
      return fail(MB_ERR_INVALID, "mb_gan_create: resblock kernel size %d unsupported (odd, <= %d)",
                  c.resblock_kernel_sizes[j], kMaxTaps);
  for (int j = 0; j < c.num_kernels; ++j)
    for (int m = 0; m < c.num_dilations; ++m)
      if ((c.resblock_kernel_sizes[j] - 1) * c.resblock_dilation_sizes[j][m] > 96)
        return fail(MB_ERR_INVALID, "mb_gan_create: receptive field of resblock kernel %d dilation %d too wide",
                    c.resblock_kernel_sizes[j], c.resblock_dilation_sizes[j][m]);
  for (int i = 0; i < c.num_upsamples; ++i) {
    const int u = c.upsample_rates[i], k = c.upsample_kernel_sizes[i];
    if (u < 1 || u > kMaxPhases) return fail(MB_ERR_INVALID, "mb_gan_create: upsample rate %d unsupported", u);
    // output length (L-1)u - 2p + k + op must equal u*L
    if (k - 2 * (u / 2 + u % 2) + (u % 2) != u)
      return fail(MB_ERR_INVALID, "mb_gan_create: upsample (k=%d,u=%d) does not produce u*L samples", k, u);
  }
  const int T = new_buf(h), X = new_buf(h), R = new_buf(h), S = new_buf(h);
  const int C0 = c.upsample_initial_channel;
  int rate = 1;
  if (c.kind == MB_GAN_HIFIGAN) {
    add_conv(h, "conv_pre", c.num_mels, C0, 7, 1, 1, false, 1, 1.f, BUF_IN, T, BUF_NONE, 1);
    int cur = T;
    int ch = C0;
    for (int i = 0; i < c.num_upsamples; ++i) {
      const int u = c.upsample_rates[i];
      add_conv(h, "ups." + std::to_string(i), ch, ch / 2, c.upsample_kernel_sizes[i], 1, u, true, 1, 0.1f, cur, X,
               BUF_NONE, rate);
      ch /= 2;
      rate *= u;
      add_mrf(h, i, ch, rate, X, R, T, S);
      cur = S;
    }
    Layer& post = add_conv(h, "conv_post", ch, 1, 7, 1, 1, false, 1, 0.01f, S, BUF_OUT, BUF_NONE, rate);
    post.act_tanh = 1;
  } else if (c.kind == MB_GAN_FREGAN) {
    const int cond_level = c.num_upsamples - c.fregan_top_k;
    if (cond_level < 1 || cond_level >= c.num_upsamples - 1)
      return fail(MB_ERR_INVALID, "mb_gan_create: fregan top_k=%d unsupported for %d upsamples", c.fregan_top_k,
                  c.num_upsamples);
    const int CA = new_buf(h), CB = new_buf(h), OA = new_buf(h), OB = new_buf(h);
    add_conv(h, "conv_pre", c.num_mels, C0, 7, 1, 1, false, 1, 1.f, BUF_IN, S, BUF_NONE, 1);
    int ch = C0;
    int cond = BUF_IN, cond_ch = c.num_mels, cond_rate = 1;
    int output = BUF_NONE, out_ch = 0, out_rate = 1;
    for (int i = 0; i < c.num_upsamples; ++i) {
      if (i >= cond_level) {
        const int j = i - cond_level;
        const int u = c.upsample_rates[i - 1], k = c.upsample_kernel_sizes[i - 1];
        const int dstc = (cond == CA) ? CB : CA;
        Layer& cu = add_conv(h, "cond_up." + std::to_string(j), cond_ch, ch, k, 1, u, true, 1, 1.f, cond, dstc,
                             BUF_NONE, cond_rate);
        const bool split = c.precision != MB_PREC_FP32 && j > 0 && env_flag("MB_FREGAN_SPLIT", true);
        if (!split) cu.dst2 = S;  // x += mel  (generator.py:143-144) fused as a second destination
        cond = dstc;
        cond_ch = ch;
        cond_rate *= u;
        if (cond_rate != rate) return fail(MB_ERR_INVALID, "mb_gan_create: fregan cond rate mismatch");
        if (split) {  // x += mel as its own op, so that cond_up itself is tensor-core capable
          Layer A;
          A.kind = OP_ADD;
          A.name = "x+=cond_up." + std::to_string(j);
          A.cin_w = A.cout_w = ch;
          A.cin = A.cout = pad_channels(h, ch);
          A.src = dstc;
          A.dst = S;
          A.rate_in = A.rate_out = rate;
          h->layers.push_back(A);
        }
      }
      if (i > cond_level) {
        const int j = i - cond_level - 1;
        const int u = c.upsample_rates[i];
        const int srcb = (output == BUF_NONE) ? S : output;
        const int srcc = (output == BUF_NONE) ? ch : out_ch;
        const int srcr = (output == BUF_NONE) ? rate : out_rate;
        const int dsto = (output == OA) ? OB : OA;
        add_conv(h, "res_output." + std::to_string(j) + ".1", srcc, ch / 2, 1, 1, 1, false, u, 1.f, srcb, dsto,
                 BUF_NONE, srcr);
        output = dsto;
        out_ch = ch / 2;
        out_rate = srcr * u;
      }
      const int u = c.upsample_rates[i];
      add_conv(h, "ups." + std::to_string(i), ch, ch / 2, c.upsample_kernel_sizes[i], 1, u, true, 1, 0.1f, S, X,
               BUF_NONE, rate);
      ch /= 2;
      rate *= u;
      add_mrf(h, i, ch, rate, X, R, T, S);
      if (output != BUF_NONE) {
        if (out_ch != ch || out_rate != rate) return fail(MB_ERR_INVALID, "mb_gan_create: fregan skip mismatch");
        Layer A;
        A.kind = OP_ADD;
        A.name = "output+=x";
        A.cin_w = A.cout_w = ch;
        A.cin = A.cout = pad_channels(h, ch);
        A.src = S;
        A.dst = output;
        A.rate_in = A.rate_out = rate;
        h->layers.push_back(A);
      }
    }
    if (output == BUF_NONE) return fail(MB_ERR_INVALID, "mb_gan_create: fregan without skip output");
    Layer& post = add_conv(h, "conv_post", ch, 1, 7, 1, 1, false, 1, 0.01f, output, BUF_OUT, BUF_NONE, rate);
    post.act_tanh = 1;
  } else {
    return fail(MB_ERR_INVALID, "mb_gan_create: unknown kind %d", c.kind);
  }
  h->hop = rate;
  // arena layout: fp32 slabs + biases
  size_t off = 0;
  for (Layer& L : h->layers) {
    if (L.kind != OP_CONV) continue;
    build_taps(L);
    L.w_off = off;
    off += (size_t)L.k * L.cin * L.cout;
    off = align_up(off, 64);
    L.b_off = off;
    off += (size_t)L.cout;
    off = align_up(off, 64);
  }
  h->f32_floats = off;
  return MB_OK;
}

float* buf_ptr(const mb_gan* h, int buf, const float* in, float* out, float* ws, size_t B, size_t T,
               const std::vector<size_t>& offs) {
  if (buf == BUF_NONE) return nullptr;
  if (buf == BUF_IN) return const_cast<float*>(in);
  if (buf == BUF_OUT) return out;
  (void)h;
  (void)B;
  (void)T;
  return ws + offs[buf];
}

std::vector<size_t> buf_offsets(const mb_gan* h, size_t B, size_t T, size_t* total) {
  std::vector<size_t> offs(h->buf_cr.size());
  size_t o = 0;
  for (size_t i = 0; i < h->buf_cr.size(); ++i) {
    offs[i] = o;
    o += align_up(B * T * h->buf_cr[i], 64);
  }
  *total = o;
  return offs;
}

TRef ncl(const void* p, int C, int L) {
  TRef t;
  t.p = const_cast<void*>(p);
  t.layout = p ? LAYOUT_NCL : LAYOUT_NONE;
  t.C = C;
  t.L = L;
  return t;
}

TcOp tc_op(const mb_gan* h, const Layer& L) {
  TcOp o{};
  o.is_conv = (L.kind == OP_CONV);
  o.taps = L.taps;
  o.tc = L.tc;
  o.name = L.name.c_str();
  o.src = L.src;
  o.dst = L.dst;
  o.res = L.res;
  o.dst2 = L.dst2;
  o.cin = L.cin;
  o.cout = L.cout;
  o.rate_in = L.rate_in;
  o.rate_out = L.rate_out;
  o.w32 = h->arena ? h->arena + L.w_off : nullptr;  // (the plan query runs before an arena is set)
  o.b32 = h->arena ? h->arena + L.b_off : nullptr;
  return o;
}

std::vector<TcOp> tc_ops(const mb_gan* h) {
  std::vector<TcOp> ops;
  for (const Layer& L : h->layers) ops.push_back(tc_op(h, L));
  return ops;
}

int run_layer_f32(mb_gan* h, const Layer& L, const float* src, const float* res, float* dst, float* dst2,
                  const int32_t* lengths, int B, int T, cudaStream_t st) {
  if (L.kind == OP_ADD) {
    cudaError_t e = launch_add_inplace_f32(ncl(dst, L.cout, L.rate_out * T), ncl(src, L.cout, L.rate_out * T),
                                           TRef{}, 1.f, B, st);
    if (e != cudaSuccess) return fail(MB_ERR_CUDA, "add kernel: %s", cudaGetErrorString(e));
    count_launch();
    return MB_OK;
  }
  TapConv p = L.taps;
  p.B = B;
  p.Lin = T * L.rate_in;
  p.Lout = T * L.rate_out;
  p.lengths = lengths;
  TapConvIO io;
  io.x = ncl(src, L.cin, p.Lin);
  io.res = ncl(res, L.cout, p.Lout);
  io.y32 = ncl(dst, L.cout, p.Lout);
  io.y2_32 = ncl(dst2, L.cout, p.Lout);
  cudaError_t e = (L.cout == 1 && p.stride == 1)
                      ? launch_tapconv_cout1_f32(p, io, h->arena + L.w_off, h->arena + L.b_off, st)
                      : launch_tapconv_f32(p, io, h->arena + L.w_off, h->arena + L.b_off, st);
  if (e != cudaSuccess) return fail(MB_ERR_CUDA, "tapconv_f32 (%s): %s", L.name.c_str(), cudaGetErrorString(e));
  count_launch();
  return MB_OK;
}

}  // namespace

extern "C" {

int mb_gan_create(const mb_gan_config* cfg, mb_gan** out) {
  if (!cfg || !out) return fail(MB_ERR_INVALID, "mb_gan_create: null argument");
  if (cfg->precision != MB_PREC_FP32 && cfg->precision != MB_PREC_F16TC && cfg->precision != MB_PREC_F16X3)
    return fail(MB_ERR_INVALID, "mb_gan_create: unknown precision %d", cfg->precision);
  mb_gan* h = new mb_gan();
  h->cfg = *cfg;
  int rc = build_plan(h);
  if (rc == MB_OK && cfg->precision != MB_PREC_FP32) {
    std::vector<TcLayerDesc> descs;
    for (Layer& L : h->layers) {
      TcLayerDesc d{};
      d.is_conv = (L.kind == OP_CONV);
      // (res_output reads its source un-activated while ups reads the same buffer through leaky-relu: one fp16 plane
      //  cannot serve both, so the nearest-upsample layers stay on the FP32 kernel unless explicitly requested)
      // Fre-GAN res_output: the first one reads S, which `ups` reads through leaky-relu (one fp16 plane cannot serve both): FP32
      // kernel.  The later ones read the running `output` buffer, which nothing else consumes: they run on the tensor cores with
      // the 3-term split over an un-activated hi/lo plane written by the preceding "output += x" op (MB_GAN_NEAREST_TC=0: FP32).
      const bool nearest_f32 = L.nearest > 1 && (L.name.rfind("res_output.0.", 0) == 0 || !env_flag("MB_GAN_NEAREST_TC", true));
      d.force_f32 = (L.dst2 != BUF_NONE) || nearest_f32;
      // 3-term split (FP32-equivalent operands): every layer in MB_PREC_F16X3; in MB_PREC_F16TC the serial layers nothing
      // downstream averages out - the transposed convs `ups.*` / `cond_up.*` (DESIGN.md 3.4; MB_TC_UPS_X3=0 disables)
      d.want_x3 = cfg->precision == MB_PREC_F16X3 ||
                  (env_flag("MB_TC_UPS_X3", true) &&
                   (L.name.rfind("ups.", 0) == 0 || L.name.rfind("cond_up.", 0) == 0 || L.name.rfind("res_output.", 0) == 0));
      d.taps = &L.taps;
      d.k = L.k;
      d.tc = &L.tc;
      descs.push_back(d);
    }
    rc = tc_plan_layers(descs, &h->tc_bytes);
  }
  if (rc != MB_OK) {
    delete h;
    return rc;
  }
  *out = h;
  return MB_OK;
}

void mb_gan_destroy(mb_gan* h) { delete h; }

size_t mb_gan_arena_bytes(const mb_gan* h) {
  if (!h) return 0;
  return align_up(h->f32_floats * sizeof(float), 256) + h->tc_bytes;
}

int mb_gan_set_arena(mb_gan* h, void* arena, size_t bytes) {
  if (!h || !arena) return fail(MB_ERR_INVALID, "mb_gan_set_arena: null argument");
  if (bytes < mb_gan_arena_bytes(h)) return fail(MB_ERR_WORKSPACE, "mb_gan_set_arena: need %zu bytes, got %zu",
                                                 mb_gan_arena_bytes(h), bytes);
  if (((uintptr_t)arena & 255) != 0) return fail(MB_ERR_INVALID, "mb_gan_set_arena: arena must be 256-byte aligned");
  h->arena = (float*)arena;
  h->arena_bytes = bytes;
  return MB_OK;
}

int mb_gan_set_weight(mb_gan* h, const char* name, const float* w, const int64_t* dims, int32_t ndim, void* stream) {
  if (!h || !name || !w || !dims) return fail(MB_ERR_INVALID, "mb_gan_set_weight: null argument");
  if (!h->arena) return fail(MB_ERR_STATE, "mb_gan_set_weight: call mb_gan_set_arena first");
  cudaStream_t st = (cudaStream_t)stream;
  const std::string n(name);
  const size_t dot = n.rfind('.');
  if (dot == std::string::npos) return fail(MB_ERR_INVALID, "mb_gan_set_weight: bad name '%s'", name);
  const std::string base = n.substr(0, dot), leaf = n.substr(dot + 1);
  for (Layer& L : h->layers) {
    if (L.kind != OP_CONV || L.name != base) continue;
    if (leaf == "bias") {
      if (ndim != 1 || dims[0] != L.cout_w)
        return fail(MB_ERR_INVALID, "mb_gan_set_weight: %s expects [%d]", name, L.cout_w);
      if (L.cout != L.cout_w) MB_CUDA_CHECK(cudaMemsetAsync(h->arena + L.b_off, 0, sizeof(float) * L.cout, st));
      MB_CUDA_CHECK(cudaMemcpyAsync(h->arena + L.b_off, w, sizeof(float) * L.cout_w, cudaMemcpyDeviceToDevice, st));
      L.b_set = true;
      return MB_OK;
    }
    if (leaf == "weight") {
      const int64_t d0 = L.transposed ? L.cin_w : L.cout_w, d1 = L.transposed ? L.cout_w : L.cin_w;
      if (ndim != 3 || dims[0] != d0 || dims[1] != d1 || dims[2] != L.k)
        return fail(MB_ERR_INVALID, "mb_gan_set_weight: %s expects [%lld,%lld,%d]", name, (long long)d0,
                    (long long)d1, L.k);
      cudaError_t e = launch_pack_slabs_f32(w, h->arena + L.w_off, L.cout_w, L.cin_w, L.k, L.transposed, st, L.cout, L.cin);
      if (e != cudaSuccess) return fail(MB_ERR_CUDA, "pack_slabs: %s", cudaGetErrorString(e));
      count_launch();
      if (h->cfg.precision != MB_PREC_FP32) {
        char* tcbase = (char*)h->arena + align_up(h->f32_floats * sizeof(float), 256);
        int rc = tc_pack_weights(L.tc, L.taps, h->arena + L.w_off, tcbase, st);
        if (rc != MB_OK) return rc;
      }
      L.w_set = true;
      return MB_OK;
    }
    return fail(MB_ERR_INVALID, "mb_gan_set_weight: unknown leaf '%s' (weight-norm must be folded by the host)", name);
  }
  return fail(MB_ERR_INVALID, "mb_gan_set_weight: no layer named '%s' in this config", base.c_str());
}

int mb_gan_finalize(mb_gan* h) {
  if (!h) return fail(MB_ERR_INVALID, "mb_gan_finalize: null handle");
  for (const Layer& L : h->layers) {
    if (L.kind != OP_CONV) continue;
    if (!L.w_set || !L.b_set)
      return fail(MB_ERR_STATE, "mb_gan_finalize: tensor %s.%s was never set", L.name.c_str(),
                  L.w_set ? "bias" : "weight");
  }
  h->finalized = true;
  return MB_OK;
}

int32_t mb_gan_hop(const mb_gan* h) { return h ? h->hop : 0; }

size_t mb_gan_workspace_bytes(const mb_gan* h, int32_t batch, int32_t frames) {
  if (!h || batch <= 0 || frames <= 0) return 0;
  if (h->cfg.precision != MB_PREC_FP32) {
    std::vector<TcBufReq> req;
    for (size_t i = 0; i < h->buf_cr.size(); ++i) req.push_back({h->buf_cr[i]});
    return tc_workspace_bytes(req, batch, frames, h->cfg.num_mels, h->hop);
  }
  size_t total = 0;
  buf_offsets(h, (size_t)batch, (size_t)frames, &total);
  return total * sizeof(float) + 256;
}

static int gan_forward_impl(mb_gan* h, const float* mel, const int32_t* lengths, int32_t batch, int32_t frames,
                            float* wav, void* workspace, size_t workspace_bytes, void* stream, cudaEvent_t* events) {
  if (!h || !mel || !wav || !workspace) return fail(MB_ERR_INVALID, "mb_gan_forward: null argument");
  if (!h->finalized) return fail(MB_ERR_STATE, "mb_gan_forward: weights not finalized");
  if (batch <= 0 || frames <= 0) return fail(MB_ERR_INVALID, "mb_gan_forward: empty batch");
  const size_t need = mb_gan_workspace_bytes(h, batch, frames);
  if (workspace_bytes < need)
    return fail(MB_ERR_WORKSPACE, "mb_gan_forward: workspace %zu < %zu bytes", workspace_bytes, need);
  cudaStream_t st = (cudaStream_t)stream;
  if (h->cfg.precision != MB_PREC_FP32) {
    const std::vector<TcOp> ops = tc_ops(h);
    std::vector<TcBufReq> req;
    for (size_t i = 0; i < h->buf_cr.size(); ++i) req.push_back({h->buf_cr[i]});
    char* tcbase = (char*)h->arena + align_up(h->f32_floats * sizeof(float), 256);
    return tc_forward(ops, req, tcbase, mel, lengths, batch, frames, h->cfg.num_mels, h->hop, wav, workspace, st,
                      events);
  }
  size_t total = 0;
  const std::vector<size_t> offs = buf_offsets(h, (size_t)batch, (size_t)frames, &total);
  float* ws = (float*)(((uintptr_t)workspace + 255) & ~(uintptr_t)255);
  for (const Layer& L : h->layers) {
    const float* src = buf_ptr(h, L.src, mel, wav, ws, batch, frames, offs);
    const float* res = buf_ptr(h, L.res, mel, wav, ws, batch, frames, offs);
    float* dst = buf_ptr(h, L.dst, mel, wav, ws, batch, frames, offs);
    float* dst2 = buf_ptr(h, L.dst2, mel, wav, ws, batch, frames, offs);
    if (events) MB_CUDA_CHECK(cudaEventRecord(events[&L - &h->layers[0]], st));
    int rc = run_layer_f32(h, L, src, res, dst, dst2, lengths, batch, frames, st);
    if (rc != MB_OK) return rc;
  }
  if (events) MB_CUDA_CHECK(cudaEventRecord(events[h->layers.size()], st));
  return MB_OK;
}

int mb_gan_forward(mb_gan* h, const float* mel, const int32_t* lengths, int32_t batch, int32_t frames, float* wav,
                   void* workspace, size_t workspace_bytes, void* stream) {
  return gan_forward_impl(h, mel, lengths, batch, frames, wav, workspace, workspace_bytes, stream, nullptr);
}

int mb_gan_forward_profiled(mb_gan* h, const float* mel, const int32_t* lengths, int32_t batch, int32_t frames,
                            float* wav, void* workspace, size_t workspace_bytes, void* stream, float* ms) {
  if (!h || !ms) return fail(MB_ERR_INVALID, "mb_gan_forward_profiled: null argument");
  const size_t n = h->layers.size();
  std::vector<cudaEvent_t> ev(n + 1);
  for (auto& e : ev) MB_CUDA_CHECK(cudaEventCreate(&e));
  int rc = gan_forward_impl(h, mel, lengths, batch, frames, wav, workspace, workspace_bytes, stream, ev.data());
  if (rc == MB_OK) {
    cudaError_t e = cudaEventSynchronize(ev[n]);
    if (e != cudaSuccess) rc = fail(MB_ERR_CUDA, "mb_gan_forward_profiled: %s", cudaGetErrorString(e));
  }
  if (rc == MB_OK)
    for (size_t i = 0; i < n; ++i) cudaEventElapsedTime(&ms[i], ev[i], ev[i + 1]);
  for (auto& e : ev) cudaEventDestroy(e);
  return rc;
}

int mb_gan_layer_work(const mb_gan* h, int32_t i, int32_t batch, int32_t frames, double* macs, double* bytes) {
  if (!h || i < 0 || i >= (int32_t)h->layers.size()) return fail(MB_ERR_INVALID, "mb_gan_layer_work: bad index");
  const Layer& L = h->layers[i];
  const double rows_in = (double)batch * frames * L.rate_in, rows_out = (double)batch * frames * L.rate_out;
  if (L.kind == OP_CONV) {
    // every output row receives k/stride taps of Cin x Cout (transposed), or k taps (conv)
    const double taps = L.transposed ? (double)L.k / L.stride : (double)L.k;
    if (macs) *macs = rows_out * taps * L.cin_w * L.cout_w;  // algorithmic work: the checkpoint's channel counts
    if (bytes) *bytes = 4.0 * (rows_in * L.cin_w + rows_out * L.cout_w);
  } else {
    if (macs) *macs = 0;
    if (bytes) *bytes = 4.0 * 3.0 * rows_out * L.cout_w;
  }
  return MB_OK;
}

int32_t mb_gan_num_layers(const mb_gan* h) { return h ? (int32_t)h->layers.size() : 0; }

int mb_gan_layer_info(const mb_gan* h, int32_t i, char* buf, size_t buflen) {
  if (!h || !buf || i < 0 || i >= (int32_t)h->layers.size()) return fail(MB_ERR_INVALID, "mb_gan_layer_info: bad index");
  const Layer& L = h->layers[i];
  snprintf(buf, buflen, "%s %s cin=%d cout=%d k=%d dil=%d stride=%d rate_in=%d res=%d mode=%d",
           L.kind == OP_CONV ? "conv" : "add", L.name.c_str(), L.cin, L.cout, L.k, L.dil,
           L.transposed ? L.stride : L.nearest, L.rate_in, L.res != BUF_NONE, L.mode);
  return MB_OK;
}

int mb_gan_debug_layer(mb_gan* h, int32_t i, const float* x, const float* residual, int32_t batch,
                       int32_t frames_in, float* y, void* workspace, size_t workspace_bytes, void* stream) {
  if (!h || !x || !y || i < 0 || i >= (int32_t)h->layers.size())
    return fail(MB_ERR_INVALID, "mb_gan_debug_layer: bad argument");
  const Layer& L0 = h->layers[i];
  if (L0.kind != OP_CONV) return fail(MB_ERR_INVALID, "mb_gan_debug_layer: layer %d is not a conv", i);
  if (!L0.w_set || !L0.b_set) return fail(MB_ERR_STATE, "mb_gan_debug_layer: weights of %s not set", L0.name.c_str());
  // frames_in = input rows; run with rate_in = 1, STORE epilogue semantics kept except MRF modes
  Layer L = L0;
  const int mult = L.rate_out / L.rate_in;
  L.rate_in = 1;
  L.rate_out = mult;
  L.taps.len_mul_in = 1;
  L.taps.len_mul_out = mult;
  L.mode = EPI_STORE;
  L.taps.mode = EPI_STORE;
  cudaStream_t st = (cudaStream_t)stream;
  if (h->cfg.precision != MB_PREC_FP32) {
    TcOp o{};
    o.is_conv = true;
    o.taps = L.taps;
    o.tc = L.tc;
    o.name = L.name.c_str();
    o.cin = L.cin;
    o.cout = L.cout;
    o.rate_in = 1;
    o.rate_out = mult;
    o.w32 = h->arena + L.w_off;
    o.b32 = h->arena + L.b_off;
    char* tcbase = (char*)h->arena + align_up(h->f32_floats * sizeof(float), 256);
    return tc_debug_layer(o, tcbase, x, residual, batch, frames_in, y, workspace, workspace_bytes, st);
  }
  return run_layer_f32(h, L, x, residual, y, nullptr, nullptr, batch, frames_in, st);
}

int mb_gan_tc_plan_info(const mb_gan* h, int32_t i, char* buf, size_t buflen) {
  if (!h || !buf || i < 0 || i >= (int32_t)h->layers.size()) return fail(MB_ERR_INVALID, "mb_gan_tc_plan_info: bad index");
  if (h->cfg.precision == MB_PREC_FP32) return fail(MB_ERR_INVALID, "mb_gan_tc_plan_info: fp32 handle has no tensor-core plan");
  const std::vector<TcOp> ops = tc_ops(h);
  const std::vector<char> fuse = tc_fusion_plan(ops, (int)h->buf_cr.size());
  TcOpPlan p;
  int rc = tc_op_plan(ops, fuse, i, &p);
  if (rc != MB_OK) return rc;
  snprintf(buf, buflen,
           "%s use_tc=%d x3=%d split3=%d kc=%d n_cchunks=%d mt=%d rows_item=%d resident=%d wstages=%d omin=%d omax=%d "
           "fuse_next=%d fused_prev=%d pair_mt=%d pair_rows_item=%d pair_resident=%d pair_wstages=%d pair_omin=%d "
           "kernel=%d,%d,%d,%d",
           h->layers[i].name.c_str(), p.use_tc, p.x3, p.split3, p.kc, p.n_cchunks, p.mt, p.rows_item, p.resident, p.wstages,
           p.omin, p.omax, p.fuse_next, p.fused_prev, p.pair_mt, p.pair_rows_item, p.pair_resident, p.pair_wstages, p.pair_omin,
           p.kn, p.kmt, p.kcw, p.kpair);
  return MB_OK;
}

int mb_gan_debug_launch(mb_gan* h, const mb_gan_debug_spec* s, void* workspace, size_t workspace_bytes, void* stream,
                        char* report, size_t report_len) {
  if (!h || !s || !workspace || !s->x) return fail(MB_ERR_INVALID, "mb_gan_debug_launch: null argument");
  const int32_t i = s->layer_index;
  const int32_t n = (int32_t)h->layers.size();
  if (h->cfg.precision == MB_PREC_FP32) return fail(MB_ERR_INVALID, "mb_gan_debug_launch: fp32 handle has no tensor-core layers");
  if (i < 0 || i >= n || s->pair < 0 || s->pair > 2 || (s->pair && i + 1 >= n))
    return fail(MB_ERR_INVALID, "mb_gan_debug_launch: bad layer %d / pair %d", i, s->pair);
  if (s->mode < EPI_STORE || s->mode > EPI_ADD_DIV) return fail(MB_ERR_INVALID, "mb_gan_debug_launch: bad mode %d", s->mode);
  if (s->batch <= 0 || s->frames_in <= 0) return fail(MB_ERR_INVALID, "mb_gan_debug_launch: empty batch");
  const int nl = s->pair ? 2 : 1;
  for (int k = 0; k < nl; ++k) {
    const Layer& L = h->layers[i + k];
    if (L.kind != OP_CONV) return fail(MB_ERR_INVALID, "mb_gan_debug_launch: layer %d is not a conv", i + k);
    if (!L.w_set || !L.b_set) return fail(MB_ERR_STATE, "mb_gan_debug_launch: weights of %s not set", L.name.c_str());
  }
  if (s->pair) {
    const std::vector<char> fuse = tc_fusion_plan(tc_ops(h), (int)h->buf_cr.size());
    if (!fuse[i])
      return fail(MB_ERR_INVALID, "mb_gan_debug_launch: %s and %s are not a fused pair", h->layers[i].name.c_str(),
                  h->layers[i + 1].name.c_str());
  }
  // run at rate_in = 1 (frames_in = input rows); the last op takes the requested accumulate mode
  TcOp o[2];
  for (int k = 0; k < nl; ++k) {
    const Layer& L = h->layers[i + k];
    o[k] = tc_op(h, L);
    const int mult = L.rate_out / L.rate_in;
    o[k].rate_in = 1;
    o[k].rate_out = mult;
    o[k].taps.len_mul_in = 1;
    o[k].taps.len_mul_out = mult;
  }
  o[nl - 1].taps.mode = s->mode;
  o[nl - 1].taps.div = s->div;
  TcDebugSpec d;
  d.B = s->batch;
  d.Lin = s->frames_in;
  d.x = s->x;
  d.res = s->residual;
  d.res_kind = s->res_kind;
  d.res_slope = s->res_slope;
  d.lengths = s->lengths;
  d.red_add = s->red_add != 0;
  d.y = s->y;
  d.out16 = s->out16;
  d.out_slope = s->out_slope;
  d.y16 = s->y16;
  d.two_launches = s->pair == 2;
  char* tcbase = (char*)h->arena + align_up(h->f32_floats * sizeof(float), 256);
  TcLaunchInfo info[2];
  int launches = 0;
  int rc = tc_debug_launch(o[0], s->pair ? &o[1] : nullptr, d, tcbase, workspace, workspace_bytes, (cudaStream_t)stream, info,
                           &launches);
  if (rc != MB_OK) return rc;
  if (report && report_len) {
    size_t used = 0;
    report[0] = 0;
    for (int k = 0; k < launches && used < report_len; ++k) {
      const TcLaunchInfo& f = info[k];
      const int w = snprintf(report + used, report_len - used,
                             "kernel=%d,%d,%d,%d rows_item=%d resident=%d wstages=%d n_work=%d grid=%d red_add=%d\n", f.n, f.mt,
                             f.cw, f.pair, f.rows_item, f.resident, f.wstages, f.n_work, f.grid, f.red_add);
      if (w < 0) break;
      used += (size_t)w;
    }
  }
  return MB_OK;
}

}  // extern "C"
