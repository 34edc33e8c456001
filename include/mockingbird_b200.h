/*
 * mockingbird_b200 - C ABI of the H100-native (sm_90a) vocoder / mel-synthesizer hot path.
 *
 * This is the drop-in boundary (SURVEY.md section 8b).  The reference (babysor/MockingBird) has no
 * FFI of its own: its callers talk to duck-typed Python module singletons.  The Python host layer
 * in mockingbird_b200/ presents exactly those surfaces and binds the entry points below through
 * ctypes (INTEGRATION.md shows the stub).  Each group cites the reference interface it replaces.
 *
 * Conventions
 *   - every function returns an int status: 0 = OK, non-zero = error; mb_last_error() gives the
 *     message for the calling thread.  No exceptions cross the ABI.
 *   - handles are opaque; one handle must not be used from two threads at once.
 *   - all tensor arguments are caller-owned DEVICE pointers unless the name ends in _host.
 *   - no hidden device allocation after *_create: packed weights live in a caller-provided arena
 *     (mb_*_arena_bytes), temporaries in a caller-provided workspace (mb_*_workspace_bytes).
 *     Derived weight images are (re)packed inside that arena at finalize, or - for the large-M GEMMs of the Tacotron CBHG
 *     stacks and the encoder's input projections - at the first use of a layer after any set_arena / set_weight (no
 *     cudaMalloc: the packers' scratch is a slot of the arena).  Exceptions (no device memory): mb_tacotron owns two
 *     streams and ten events (created at its first generate call), mb_mtstream its pinned host ring, a side stream and events.
 *   - weights: mb_*_set_arena, then mb_*_set_weight once per checkpoint tensor, then mb_*_finalize.  A tensor is fp32,
 *     contiguous, device-resident and has exactly its reference shape (a transposed or flattened tensor is refused).
 *     Derived tensors (packed images, folded BatchNorm, scratch) are not settable.  set_arena forgets every tensor set
 *     before it: finalize and the compute calls return MB_ERR_STATE until all are set again and finalized.  set_weight
 *     reports argument errors (NULL pointers, unknown name, wrong shape: MB_ERR_INVALID) before call-order errors (no
 *     arena: MB_ERR_STATE).
 *   - every launch goes to the cudaStream_t passed as `stream` (void* here so that the header
 *     needs no CUDA include); functions are asynchronous with respect to the host unless stated.
 *   - multi-GPU: the library links no communication library and has no global state.  The packed arena of every model
 *     is ONE contiguous device buffer precisely so that the host layer can ship it with a single collective of whatever
 *     it already uses - torch.distributed.broadcast(model.packed_arena(), src=0) over NCCL/NVLink in this repo
 *     (SURVEY.md 8b listed an `mb_nccl_broadcast_weights` entry point; it would only wrap that one call and force an NCCL
 *     link dependency on single-GPU users, so the contract is: arena = broadcast unit, collective = the host's).  Every
 *     rank still loads the checkpoint itself (host-side pack scales are per handle), see INTEGRATION.md section 4.
 */
#ifndef MOCKINGBIRD_B200_H
#define MOCKINGBIRD_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MB_OK 0
#define MB_ERR_INVALID 1   /* bad argument / unknown weight name / shape mismatch */
#define MB_ERR_STATE 2     /* call order violated (e.g. forward before finalize) */
#define MB_ERR_CUDA 3      /* a CUDA runtime call or kernel launch failed        */
#define MB_ERR_WORKSPACE 4 /* workspace / arena too small                        */

/* library-wide ----------------------------------------------------------------------------- */
const char* mb_last_error(void);
/* "mockingbird_b200 <ver> sm_90a"; never NULL */
const char* mb_version(void);
/* number of kernel launches issued by this library since load (all handles); used by bench.py
 * to report gpu_launches from a counter rather than from a guess */
uint64_t mb_launch_count(void);

/* ---------------------------------------------------------------------------------------------
 * GAN vocoder generators: HiFi-GAN and Fre-GAN
 *   replaces  models/vocoder/hifigan/models.py:96-162  Generator.{__init__,forward,remove_weight_norm}
 *             models/vocoder/fregan/generator.py:79-179 FreGAN.{__init__,forward,remove_weight_norm}
 *   driven by models/vocoder/hifigan/inference.py:22-73 and fregan/inference.py:22-73
 * ------------------------------------------------------------------------------------------- */
#define MB_GAN_HIFIGAN 0
#define MB_GAN_FREGAN 1
/* HiFi-GAN as the reference builds it for h.sampling_rate == 24000 (models.py:107-118): each upsampling layer is
 * InterpolationBlock(u) (nearest) + Conv1d(k, padding=(k-1)//2), checkpoint keys "ups.{i}.1.*"; k must be odd.  Lowered
 * to a polyphase tap conv with folded weights (DESIGN.md 3.6); same mb_gan_config fields as MB_GAN_HIFIGAN. */
#define MB_GAN_HIFIGAN_INTERP 2

/* arithmetic of the channel-mixing convolutions */
#define MB_PREC_FP32 0      /* FP32 FFMA everywhere (parity anchor, ~1e-6 of the reference)     */
#define MB_PREC_F16TC 1     /* wgmma tensor cores: fp16 operands, fp32 accumulate, fp32
                               residual stream; conv_post in fp32 (tolerance 1e-3, see DESIGN.md) */
#define MB_PREC_F16X3 2     /* wgmma tensor cores with the 3-term fp16 split on EVERY layer
                               (x*w = hi*hi + lo*hi + hi*lo, fp32 accumulate): FP32-equivalent results
                               (~1e-5 of the reference) at 3x the MMA work of MB_PREC_F16TC            */

typedef struct mb_gan_config {
  int32_t kind;                 /* MB_GAN_HIFIGAN | MB_GAN_FREGAN | MB_GAN_HIFIGAN_INTERP          */
  int32_t num_mels;             /* 80 (models.py:99 hard-codes 80)                                 */
  int32_t upsample_initial_channel;
  int32_t num_upsamples;        /* len(h.upsample_rates) <= 8                                      */
  int32_t upsample_rates[8];
  int32_t upsample_kernel_sizes[8];
  int32_t num_kernels;          /* len(h.resblock_kernel_sizes) <= 4                               */
  int32_t resblock_kernel_sizes[4];
  int32_t num_dilations;        /* dilations per resblock <= 4                                     */
  int32_t resblock_dilation_sizes[4][4];
  int32_t resblock_type;        /* 1 = ResBlock1 (models.py:11), 2 = ResBlock2 (models.py:50)      */
  int32_t fregan_top_k;         /* FreGAN(h, top_k=4); ignored for HiFi-GAN                        */
  int32_t precision;            /* MB_PREC_*                                                       */
} mb_gan_config;

typedef struct mb_gan mb_gan;

int mb_gan_create(const mb_gan_config* cfg, mb_gan** out);
void mb_gan_destroy(mb_gan* h);

/* bytes of device memory the packed weights need; pass such a buffer to mb_gan_set_arena */
size_t mb_gan_arena_bytes(const mb_gan* h);
int mb_gan_set_arena(mb_gan* h, void* arena, size_t bytes);

/* Feed one tensor of ckpt['generator'] (hifigan/inference.py:51) AFTER weight-norm folding
 * (w = g*v/||v||, models.py:152-162 - the host layer folds): name as in state_dict
 * ("conv_pre.weight", "ups.0.bias", "resblocks.3.convs1.0.weight", "cond_up.1.weight",
 * "res_output.0.1.weight" ...).  Packs into the arena on `stream`.  */
int mb_gan_set_weight(mb_gan* h, const char* name, const float* w, const int64_t* dims, int32_t ndim,
                      void* stream);
/* verifies that every tensor the config needs has been set */
int mb_gan_finalize(mb_gan* h);

/* samples produced per mel frame = prod(upsample_rates) */
int32_t mb_gan_hop(const mb_gan* h);
size_t mb_gan_workspace_bytes(const mb_gan* h, int32_t batch, int32_t frames);

/* Generator.forward (models.py:134-150):  mel [B, num_mels, T] fp32  ->  wav [B, 1, T*hop] fp32.
 * lengths (optional, int32 [B], device): valid frames per utterance; rows beyond are treated as
 * zero padding at every layer so each utterance equals its own batch-1 reference call, and
 * wav[b, lengths[b]*hop:] = 0.   */
int mb_gan_forward(mb_gan* h, const float* mel, const int32_t* lengths, int32_t batch, int32_t frames,
                   float* wav, void* workspace, size_t workspace_bytes, void* stream);

/* Measurement hook for bench.py's roofline: same as mb_gan_forward, but brackets every layer launch
 * with CUDA events on `stream`, synchronises, and writes the device time of layer i (milliseconds)
 * to ms_per_layer_host[i] (host array of mb_gan_num_layers entries). */
int mb_gan_forward_profiled(mb_gan* h, const float* mel, const int32_t* lengths, int32_t batch,
                            int32_t frames, float* wav, void* workspace, size_t workspace_bytes,
                            void* stream, float* ms_per_layer_host);
/* algorithmic work of layer i for a [batch, frames] call: multiply-accumulates, and fp32
 * layer-granular bytes (input elements read + output elements written, x4; SURVEY.md section 8d) */
int mb_gan_layer_work(const mb_gan* h, int32_t layer_index, int32_t batch, int32_t frames,
                      double* macs, double* layer_bytes);

/* test hook: run ONE convolution layer of the plan in isolation through the selected precision
 * path.  Used only by tests/ to compare the tensor-core kernels with the FP32 kernels layer by
 * layer.  x/y are [B, C, L] fp32 (reference layout). */
int mb_gan_debug_layer(mb_gan* h, int32_t layer_index, const float* x, const float* residual,
                       int32_t batch, int32_t frames_in, float* y, void* workspace,
                       size_t workspace_bytes, void* stream);
int32_t mb_gan_num_layers(const mb_gan* h);
/* fills a short description "name Cin Cout k dil stride" for layer i; returns 0 on success */
int mb_gan_layer_info(const mb_gan* h, int32_t layer_index, char* buf, size_t buflen);

/* Host-only (no GPU needed, like mb_gan_create): how the tensor-core forward runs op i of a
 * MB_PREC_F16TC / MB_PREC_F16X3 handle, as "name key=value ...":
 *   use_tc x3 split3 kc n_cchunks mt rows_item resident wstages omin omax   (the op launched alone)
 *   fuse_next fused_prev             1: first / second op of a resblock pair run as ONE fused launch
 *   pair_mt pair_rows_item pair_resident pair_wstages pair_omin   (fuse_next: the pair's launch)
 *   kernel=N,MT,CW,PAIR              the tc_conv_kernel instance this op launches (0,0,0,0: none) */
int mb_gan_tc_plan_info(const mb_gan* h, int32_t op_index, char* buf, size_t buflen);

/* test hook: one tensor-core launch of the plan with caller-chosen epilogue inputs and outputs.
 * All tensors are device memory; x [B, Cin, L], residual / y [B, Cout, L*stride], y16 [B, C16, L*stride]
 * fp32 NCL.  The layers run at one input row per frame (lengths count input rows). */
typedef struct mb_gan_debug_spec {
  int32_t layer_index;
  int32_t pair;        /* 0: layer alone; 1: layers (i, i+1) as one fused launch (error if the
                          forward does not fuse them); 2: the same pair as two launches */
  int32_t mode;        /* epilogue of the (last) layer: 0 store, 1 y += v, 2 y = (y + v) / div */
  float div;
  int32_t red_add;     /* 1: mode 1 without fp16 output accumulates by red.global.add */
  int32_t res_kind;    /* residual: 0 none, 1 fp32 plane, 2 activated fp16 plane, 3 hi/lo plane */
  float res_slope;     /* leaky-relu slope of the fp16 residual planes */
  int32_t out16;       /* fp16 output plane: 0 none, 1 plain, 2 hi/lo */
  float out_slope;     /* leaky-relu slope of the fp16 output plane */
  int32_t batch, frames_in;
  const float* x;
  const float* residual;
  const int32_t* lengths; /* [B] or NULL */
  float* y;            /* running sum in (modes 1, 2), result out; may be NULL in mode 0 */
  float* y16;          /* out16: the plane read back, C16 = Cout (plain) or the hi/lo plane's
                          channels (2 Cout, at least 64): hi channels first, then lo */
} mb_gan_debug_spec;
/* writes one line per kernel launch into `report`:
 * "kernel=N,MT,CW,PAIR rows_item= resident= wstages= n_work= grid= red_add=" */
int mb_gan_debug_launch(mb_gan* h, const mb_gan_debug_spec* spec, void* workspace, size_t workspace_bytes,
                        void* stream, char* report, size_t report_len);

/* ---------------------------------------------------------------------------------------------
 * fatchord WaveRNN
 *   replaces  models/vocoder/wavernn/models/fatchord_version.py:88-257 (WaveRNN.generate and the
 *             UpsampleNetwork/MelResNet conditioning :27-85), driven by wavernn/inference.py:8-64
 * ------------------------------------------------------------------------------------------- */
typedef struct mb_wavernn_config {
  int32_t rnn_dims;      /* 512 hparams.voc_rnn_dims */
  int32_t fc_dims;       /* 512 */
  int32_t bits;          /* 9 -> 512 classes */
  int32_t pad;           /* 2 */
  int32_t num_upsample;  /* 3 */
  int32_t upsample_factors[4]; /* (5,5,8) */
  int32_t feat_dims;     /* 80 */
  int32_t compute_dims;  /* 128 */
  int32_t res_out_dims;  /* 128 */
  int32_t res_blocks;    /* 10 */
} mb_wavernn_config;

typedef struct mb_wavernn mb_wavernn;

int mb_wavernn_create(const mb_wavernn_config* cfg, mb_wavernn** out);
void mb_wavernn_destroy(mb_wavernn* h);
size_t mb_wavernn_arena_bytes(const mb_wavernn* h);
int mb_wavernn_set_arena(mb_wavernn* h, void* arena, size_t bytes);
/* tensors of ckpt['model_state'] (wavernn/inference.py:36-37) under their reference names (SURVEY.md appendix B) */
int mb_wavernn_set_weight(mb_wavernn* h, const char* name, const float* w, const int64_t* dims,
                          int32_t ndim, void* stream);
int mb_wavernn_finalize(mb_wavernn* h, void* stream);

size_t mb_wavernn_workspace_bytes(const mb_wavernn* h, int32_t frames, int32_t folds, int32_t steps);

/* UpsampleNetwork.forward on the padded mel (fatchord_version.py:168-170): mel [80, T] fp32
 * (already divided by mel_max_abs_value, inference.py:60-61) -> frame-rate conditioning kept in
 * the workspace (aux [T,128]; the mel FIR ladder is evaluated on the fly by the sample loop's
 * conditioning stage, the 200x upsampled tensors are never materialised in full). */
int mb_wavernn_condition(mb_wavernn* h, const float* mel, int32_t frames, void* workspace,
                         size_t workspace_bytes, void* stream);

/* The sample loop (fatchord_version.py:190-234) over `folds` independent rows, each `steps` long,
 * row r starting at upsampled-time offset fold_starts[r] (fold_with_overlap, :288-338; positions
 * past the end of the conditioning read zeros like the reference's zero padding).
 *   noise  : Exp(1) draws, fp32 [steps_in_call, folds, 512] in the reference's draw order
 *            (Categorical.sample == argmax(p/q), SURVEY.md fact 5), or NULL to use the built-in
 *            counter-based generator seeded by `seed`.
 *   step0/nsteps: run steps [step0, step0+nsteps) - state (h1,h2,x) persists in the workspace
 *            between calls so the host can call the progress callback every 100 steps
 *            (fatchord_version.py:232-234); step0 == 0 resets the state to zeros (:178-185).
 *   out_idx: int16 [folds, steps] class indices (row-major, written at [r, step0+i]).      */
int mb_wavernn_generate(mb_wavernn* h, const int32_t* fold_starts_host, int32_t folds, int32_t steps,
                        int32_t step0, int32_t nsteps, const float* noise, uint64_t seed,
                        int16_t* out_idx, void* workspace, size_t workspace_bytes, void* stream);

/* Same, for a contiguous subset of an utterance's folds (fold sharding across GPUs, SURVEY.md 8e row 2): this call's
 * local rows are the global folds [row0, row0+folds); `noise` holds all `noise_folds` rows per step
 * ([steps_in_call, noise_folds, 512]) and the built-in generator is keyed by the global fold index, so the samples of
 * a fold do not depend on how the folds are dealt to GPUs.  out_idx is local: int16 [folds, steps]. */
int mb_wavernn_generate_rows(mb_wavernn* h, const int32_t* fold_starts_host, int32_t folds, int32_t steps,
                             int32_t step0, int32_t nsteps, const float* noise, int32_t noise_folds, int32_t row0,
                             uint64_t seed, int16_t* out_idx, void* workspace, size_t workspace_bytes, void* stream);

/* The float64 tail of WaveRNN.generate on the device (fatchord_version.py:236-253, :340-402; wavernn/audio.py:92-107):
 * class indices int16 [folds, steps] (device) -> sample = 2*idx/(n_classes-1) - 1 -> equal-power cross-fade + unfold
 * (batched) -> mu-law decode -> de-emphasis y[n] = x[n] + preemphasis*y[n-1] (0 = off) -> out[:wave_len] ->
 * linear fade-out over the last fade_len samples.  `out` (device, float64) must hold
 * min(wave_len, folds*(target+overlap)+overlap | steps) samples; *n_out receives that count. */
size_t mb_wavernn_postprocess_workspace_bytes(int32_t folds, int32_t steps, int32_t batched, int32_t target, int32_t overlap);
int mb_wavernn_postprocess(const int16_t* idx, int32_t folds, int32_t steps, int32_t batched, int32_t target,
                           int32_t overlap, int32_t n_classes, int32_t mu_law, double preemphasis, int64_t wave_len,
                           int32_t fade_len, double* out, int64_t* n_out, void* workspace, size_t workspace_bytes,
                           void* stream);

/* debug/test hook: logits [folds, 512] fp32 of the LAST step executed by mb_wavernn_generate */
int mb_wavernn_last_logits(mb_wavernn* h, float* logits, int32_t folds, void* workspace, void* stream);

/* ---------------------------------------------------------------------------------------------
 * monotonic alignment search (SURVEY.md 8f row N4; csrc/monotonic.cu)
 *   replaces  monotonic_align/core.pyx:7-42 (maximum_path_c) + the host round trip of monotonic_align/__init__.py:6-19
 *   values float32 [b, T_y, T_x] (device, updated in place like the reference), paths int32 [b, T_y, T_x] (device),
 *   t_ys / t_xs int32 [b] (device): valid lengths per item.
 * ------------------------------------------------------------------------------------------- */
int mb_monotonic_path(float* values, int32_t* paths, const int32_t* t_ys, const int32_t* t_xs, int32_t batch, int32_t T_y,
                      int32_t T_x, void* stream);

/* ---------------------------------------------------------------------------------------------
 * DeepMind-style dual-softmax WaveRNN (SURVEY.md 8f row N3; csrc/deepmind.cu)
 *   replaces  models/vocoder/wavernn/models/deepmind_version.py:75-162 (WaveRNN.generate: one unconditioned row, per sample a
 *             coarse and a dependent fine 256-way draw) and :8-34 (the parameters, reference names: R.weight [2688,896],
 *             O1..O4.{weight,bias}, I_coarse.weight [1344,2], I_fine.weight [1344,3], bias_u/r/e [896])
 * ------------------------------------------------------------------------------------------- */
typedef struct mb_deepmind mb_deepmind;
int mb_deepmind_create(int32_t hidden_size, int32_t quantisation, mb_deepmind** out);
void mb_deepmind_destroy(mb_deepmind* h);
size_t mb_deepmind_arena_bytes(const mb_deepmind* h);
int mb_deepmind_set_arena(mb_deepmind* h, void* arena, size_t bytes);
int mb_deepmind_set_weight(mb_deepmind* h, const char* name, const float* w, const int64_t* dims, int32_t ndim, void* stream);
int mb_deepmind_finalize(mb_deepmind* h, void* stream);
size_t mb_deepmind_workspace_bytes(const mb_deepmind* h);
/* samples [step0, step0+nsteps) of one generate(seq_len = steps); step0 == 0 resets hidden state / previous outputs to zero.
 * noise: Exp(1) draws fp32 [nsteps][2][256] (coarse then fine, the order Categorical.sample() consumes the torch generator)
 * or NULL (built-in counter-based generator, `seed`).  coarse / fine: int16 [steps] class ids (device). */
int mb_deepmind_generate(mb_deepmind* h, int32_t steps, int32_t step0, int32_t nsteps, const float* noise, uint64_t seed,
                         int16_t* coarse, int16_t* fine, void* workspace, size_t workspace_bytes, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Reference-identical sampling noise (mt_stream.cu)
 *   replaces  the per-step `Categorical(...).sample()` draw of fatchord_version.py:223-226, i.e. ATen's CPU
 *             `exponential_` on the global torch generator: serial MT19937, two 32-bit draws per element,
 *             q = (float)(-log1p(-((hi<<32|lo) & (2^53-1)) * 2^-53)).
 *   A host worker thread continues the generator's MT19937 sequence from its exact state into a ring of pinned
 *   buffers (allocated at create); per chunk the raw draws are copied on a side stream and converted on the device
 *   into the fp32 noise tensor `mb_wavernn_generate` consumes; `finish` returns the advanced generator state.
 * ------------------------------------------------------------------------------------------- */
typedef struct mb_mtstream mb_mtstream;
/* ring of `nslots` (2..8) pinned slots of `slot_words` 32-bit draws each; one side stream; current device */
int mb_mtstream_create(uint64_t slot_words, int32_t nslots, mb_mtstream** out);
void mb_mtstream_destroy(mb_mtstream* ms);
/* start producing `total_words` draws in chunks of `words_per_chunk` from the at::mt19937 position
 * (state[624], left_, next_) */
int mb_mtstream_begin(mb_mtstream* ms, const uint32_t* state624, int32_t left, int32_t next, uint64_t total_words,
                      uint64_t words_per_chunk);
/* next chunk: H2D into dev_raw (2*n_elems words) + conversion into dev_noise (n_elems fp32) on the side stream;
 * `main_stream` is made to wait for the result */
int mb_mtstream_next(mb_mtstream* ms, uint64_t n_elems, void* dev_raw, float* dev_noise, void* main_stream);
/* mark the chunk handed out last as consumed by the work enqueued on main_stream so far */
int mb_mtstream_consumed(mb_mtstream* ms, void* main_stream);
int mb_mtstream_finish(mb_mtstream* ms, uint32_t* state624_out, int32_t* left_out, int32_t* next_out);
/* host-only: n raw draws continuing from (state, left, next), which are advanced in place */
int mb_mt19937_fill(uint32_t* state624, int32_t* left, int32_t* next, uint32_t* out, uint64_t n);
/* device conversion alone: raw draws [n_elems][2] (device) -> Exp(1) fp32 [n_elems] */
int mb_mt_to_exp(const void* dev_raw, float* dev_noise, uint64_t n_elems, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Tacotron mel synthesizer
 *   replaces  models/synthesizer/models/tacotron.py:140-298 (Tacotron.forward / generate: Encoder + CBHG,
 *             global style token, attention decoder loop, postnet CBHG + post_proj),
 *             driven by models/synthesizer/inference.py:75-142 (Synthesizer.synthesize_spectrograms)
 * ------------------------------------------------------------------------------------------- */
typedef struct mb_tacotron_config {
  int32_t num_chars;              /* len(symbols) = 75 */
  int32_t embed_dims;             /* 512 tts_embed_dims */
  int32_t encoder_dims;           /* 256 */
  int32_t decoder_dims;           /* 128 */
  int32_t n_mels;                 /* 80  */
  int32_t postnet_dims;           /* 512 */
  int32_t encoder_K;              /* 5   */
  int32_t lstm_dims;              /* 1024 */
  int32_t postnet_K;              /* 5   */
  int32_t num_highways;           /* 4   */
  int32_t speaker_embedding_size; /* 256 */
  int32_t gst_E;                  /* 512 gst_hyperparameters.E */
  int32_t gst_tokens;             /* 10  */
  int32_t gst_heads;              /* 8   */
  int32_t max_r;                  /* 20  Decoder.max_r */
} mb_tacotron_config;

typedef struct mb_tacotron mb_tacotron;

int mb_tacotron_create(const mb_tacotron_config* cfg, mb_tacotron** out);
void mb_tacotron_destroy(mb_tacotron* h);
size_t mb_tacotron_arena_bytes(const mb_tacotron* h);
int mb_tacotron_set_arena(mb_tacotron* h, void* arena, size_t bytes);
/* tensors of ckpt['model_state'] under their reference names (SURVEY.md appendix B), plus one
 * derived tensor "gst.const_enc" [gst_E/2]: the GST ReferenceEncoder applied to the all-zero input of
 * tacotron.py:251 - input independent, folded at load time by the host layer */
int mb_tacotron_set_weight(mb_tacotron* h, const char* name, const float* w, const int64_t* dims, int32_t ndim,
                           void* stream);
int mb_tacotron_finalize(mb_tacotron* h, void* stream);
size_t mb_tacotron_workspace_bytes(const mb_tacotron* h, int32_t batch, int32_t chars, int32_t steps, int32_t r);

/* Tacotron.generate (tacotron.py:295-298) for one padded batch:
 *   chars  int32 [B][Tc] (pad id 0), spk fp32 [B][speaker_embedding_size]
 *   steps / r / style_idx / min_stop_token as the reference's arguments (r = decoder.r)
 *   enc_masks uint8 [2][B*Tc][encoder_dims], dec_masks uint8 [ceil(steps/r)][2][B][2*decoder_dims]:
 *     PreNet dropout keep-flags (pre_net.py:23,26 hard-wires training=True) to inject; NULL -> drawn
 *     on the device from `seed`
 *   mel / linear fp32 [B][n_mels][ceil(steps/r)*r] (first *frames_out_host frames valid, caller strides
 *     by *frames_out_host: the arrays are written densely as [B][n_mels][frames]), attn fp32
 *     [B][frames/r][Tc] or NULL.
 * The work runs on an internal non-blocking stream that is ordered after everything already enqueued on `stream`
 * and that `stream` waits for before the call returns (events) - the decoder loop is replayed from a CUDA graph
 * (groups of 8 steps; the step index lives in device memory) and capture is not legal on the legacy default
 * stream.  Inside the loop a second internal stream carries the parts of a step that the next step does not wait for
 * (W_hh h of both LSTM cells and the context half of the attention GRU's input projection for the NEXT step, the stop
 * projection); it forks from and joins the first one with events, also inside the captured graph.
 * The call blocks the host while polling the early-stop rule of tacotron.py:275 every 16 decoder steps. */
int mb_tacotron_generate(mb_tacotron* h, const int32_t* chars, const float* spk, int32_t batch, int32_t n_chars,
                         int32_t steps, int32_t r, int32_t style_idx, float min_stop_token, const uint8_t* enc_masks,
                         const uint8_t* dec_masks, uint64_t seed, float* mel, float* linear, float* attn,
                         int32_t* frames_out_host, void* workspace, size_t workspace_bytes, void* stream);

/* test hook: ONE launch of a 3-term-split tensor-core GEMM of the Tacotron / speaker-encoder family on caller-provided fp32
 * device tensors (no model handle), through the functions the forward uses, in its order: tc_skinny_absmax -> tc_weight_scale ->
 * tc_skinny_pack / pack_big_w -> act_split / im2col_split -> launch_tc_{skinny,gru,lstm_seq,big}.  Tensors are row-major. */
#define MB_TACO_TC_SKINNY_PLAIN 0 /* y[M][N] = [x0 | x1] . [w0 | w1]^T + b0 + b1 (+ pre), at y + step * y_step                   */
#define MB_TACO_TC_SKINNY_LSTM 1  /* gates of [x0 | x1] . [w0 | w1]^T + b0 + b1, w [4H][K] (i|f|g|o): c in/out, h out, xres += h */
#define MB_TACO_TC_GRU 2          /* per direction d: gh = h_d . w[d]^T + b[d] (w [3H][H]), GRU cell with gi[d]: hst[d] in/out, out[d] */
#define MB_TACO_TC_LSTM_SEQ 3     /* gates = x0 . w0^T + gi[0] (w0 [4H][H], x0 = h_{t-1}, any M): c in/out, h_t -> out[0] */
#define MB_TACO_TC_BIG 4          /* y = res + BN(act(sum_s x_s[row + shift_s] . W_s^T + b0)), W_s[n][k] = w0[n*ldw + w_off_s + k*w_stride_s] */
typedef struct mb_taco_tc_debug_spec {
  int32_t kind;              /* MB_TACO_TC_* */
  int32_t M, N, H;           /* rows; output columns (PLAIN, BIG); hidden units (LSTM, GRU, LSTM_SEQ) */
  int32_t K0, K1;            /* SKINNY: the two K segments (K1 may be 0); GRU / LSTM_SEQ: K0 = H; BIG: K of every segment */
  const float* w[2];         /* SKINNY: w0 [rows][K0], w1 [rows][K1]; GRU: W_hh of direction d; LSTM_SEQ / BIG: w[0] */
  const float* b[2];         /* SKINNY: biases summed (either may be NULL); GRU: b_hh of direction d; BIG: b[0] [N] or NULL */
  int32_t ldw;               /* BIG */
  int32_t nseg, T;           /* BIG: segments (taps, <= 5), rows per sequence (shift bounds) */
  const float* x[5];         /* SKINNY: x0 [M][ldx0], x1; GRU: h_{t-1} of direction d; LSTM_SEQ: x[0]; BIG: segment inputs */
  int32_t ldx[5], shift[5], w_off[5], w_stride[5];
  int32_t kb0, kb_count;     /* SKINNY: only k-blocks [kb0, kb0 + kb_count) of the image (kb_count 0: all) */
  const float* pre;          /* SKINNY: partial sum [M][ldpre] in tile column order, or NULL */
  int32_t ldpre;
  const int32_t* step_ptr;   /* PLAIN: output slab step = (*step_ptr or 0) + step_j */
  int32_t step_j;
  int64_t y_step;
  float* y;                  /* PLAIN / BIG output, row stride ldy */
  int32_t ldy;
  float* c;                  /* LSTM / LSTM_SEQ cell state [M][H] */
  float* h;                  /* LSTM: h' out [M][H] */
  float* xres;               /* LSTM: residual stream [M][H] in/out */
  const float* gi[2];        /* GRU / LSTM_SEQ: input projections, row m at gi[d] + m * ldgi */
  int32_t ldgi;
  float* hst[2];             /* GRU: state [M][H] in/out of direction d */
  float* out[2];             /* GRU / LSTM_SEQ: h' also at out[d] + m * ldout */
  int32_t ldout, ndir;
  void* s_hi[2];             /* fused hi/lo outputs (fp16 tiles [KB][rows_pad][64]) at columns s_k0[slot] + n, or NULL: */
  void* s_lo[2];             /*   SKINNY slot 0 = y (PLAIN) / xres (LSTM), slot 1 = h (LSTM); GRU slot 0 = direction 0's h' */
  int32_t s_k0[2];
  void* nxt_hi[2];           /* GRU / LSTM_SEQ: the next step's operand tiles of h' (direction d), or NULL */
  void* nxt_lo[2];
  int32_t act;               /* BIG: 0 none, 1 ReLU */
  const float* bn_scale;     /* BIG: y = act(.) * bn_scale + bn_shift, or NULL */
  const float* bn_shift;
  const float* res;          /* BIG: residual [M][ldres] or NULL */
  int32_t ldres;
  int32_t compact;           /* SKINNY: compact 8-stage ring for <= 64 rows: 0 / 1, -1 = MB_TACO_RING8 */
  int32_t cluster;           /* SKINNY: activation multicast cluster 1 / 2 / 4 / 8, 0 = MB_TACO_MC */
  int32_t pdl;               /* 0 / 1, -1 = MB_TACO_PDL */
  void* a_tiles;             /* optional out: the activation operand tiles, hi plane then lo plane (direction 0) */
  void* w_tiles;             /* optional out: the packed weight image (direction 0) */
} mb_taco_tc_debug_spec;
/* device workspace the spec needs */
size_t mb_taco_tc_debug_workspace_bytes(const mb_taco_tc_debug_spec* spec);
/* synchronises `stream` (the pack scale is read back); writes one line into `report`:
 * "kernel=K grid=X,Y cluster=C compact=0|1 rows_pad=R mma_groups=G,G_last inv_scale=S a_bytes=A w_bytes=W" */
int mb_taco_tc_debug(const mb_taco_tc_debug_spec* spec, void* workspace, size_t workspace_bytes, void* stream, char* report,
                     size_t report_len);

/* ---------------------------------------------------------------------------------------------
 * Speaker encoder (cfg 5 front half)
 *   replaces  models/encoder/model.py:41-61 (SpeakerEncoder.forward: 3 x LSTM(40 -> 256), last hidden of
 *             the top layer -> Linear -> ReLU -> L2), driven by models/encoder/inference.py:51-64
 *             (embed_frames_batch) and :157-166 (mean of the partial embeddings, L2 normalised)
 * ------------------------------------------------------------------------------------------- */
typedef struct mb_encoder_config {
  int32_t mel_n_channels; /* 40  params_data.py mel_n_channels */
  int32_t hidden_size;    /* 256 params_model.py model_hidden_size */
  int32_t num_layers;     /* 3   model_num_layers */
  int32_t embedding_size; /* 256 model_embedding_size */
} mb_encoder_config;

typedef struct mb_encoder mb_encoder;

int mb_encoder_create(const mb_encoder_config* cfg, mb_encoder** out);
void mb_encoder_destroy(mb_encoder* h);
size_t mb_encoder_arena_bytes(const mb_encoder* h);
int mb_encoder_set_arena(mb_encoder* h, void* arena, size_t bytes);
/* tensors of ckpt['model_state'] under their reference names: lstm.weight_ih_l{0..}, lstm.weight_hh_l*,
 * lstm.bias_ih_l*, lstm.bias_hh_l*, linear.weight, linear.bias (similarity_weight/bias are loss-only) */
int mb_encoder_set_weight(mb_encoder* h, const char* name, const float* w, const int64_t* dims, int32_t ndim,
                          void* stream);
int mb_encoder_finalize(mb_encoder* h, void* stream);
size_t mb_encoder_workspace_bytes(const mb_encoder* h, int32_t rows, int32_t n_frames);
/* SpeakerEncoder.forward: frames fp32 [rows][n_frames][mel_n_channels] -> embeds fp32 [rows][embedding_size]
 * (L2 normalised with the reference's +1e-5) */
int mb_encoder_embed_frames(mb_encoder* h, const float* frames, int32_t rows, int32_t n_frames, float* embeds,
                            void* workspace, size_t workspace_bytes, void* stream);
/* embed_utterance's reduction (inference.py:164-166): utterance u owns partial rows
 * [offsets[u], offsets[u+1]) (int32 device array [n_utterances+1]); out = L2(mean of those rows) */
int mb_encoder_reduce_partials(mb_encoder* h, const float* partial_embeds, const int32_t* offsets,
                               int32_t n_utterances, float* utterance_embeds, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Mel-spectrogram front-ends (SURVEY.md 8f rows N1 / N2)
 *   replaces  models/encoder/audio.py:53-65 (wav_to_mel_spectrogram: librosa.feature.melspectrogram, power, [frames][40])
 *             models/synthesizer/audio.py:59-65,115-121,156-206 (melspectrogram: preemphasis, librosa.stft,
 *             librosa.filters.mel, amp_to_db, symmetric normalisation to +-4)
 * ------------------------------------------------------------------------------------------- */
typedef struct mb_melspec_config {
  int32_t sample_rate;
  int32_t n_fft;          /* <= 2048 */
  int32_t hop_length;
  int32_t win_length;     /* periodic Hann, zero padded (centered) to n_fft */
  int32_t n_mels;
  float fmin, fmax;       /* Slaney mel scale, area-normalised triangles (librosa.filters.mel defaults) */
  int32_t pad_mode;       /* centered frames: 0 = reflect padding, 1 = zero padding */
  float preemphasis;      /* 0: none; else y[n] = x[n] - k x[n-1] before framing (synthesizer/audio.py:19-22) */
  int32_t power;          /* 1: magnitude, 2: power spectrogram before the mel projection */
  int32_t to_db;          /* 1: 20 log10(max(10^(min_level_db/20), x)) - ref_level_db (audio.py:133-135) */
  float min_level_db, ref_level_db;
  int32_t normalize;      /* 1: clip((2 A) (S - min_level_db) / (-min_level_db) - A, -A, A) if symmetric, else [0, A] */
  float max_abs_value;
  int32_t symmetric;
  int32_t transpose_out;  /* 1: out [frames][n_mels] (encoder), 0: out [n_mels][frames] (synthesizer) */
} mb_melspec_config;

typedef struct mb_melspec mb_melspec;

int mb_melspec_create(const mb_melspec_config* cfg, mb_melspec** out);
void mb_melspec_destroy(mb_melspec* h);
size_t mb_melspec_arena_bytes(const mb_melspec* h);
/* uploads the window, the DFT twiddles and the mel basis (computed on the host at create time) */
int mb_melspec_set_arena(mb_melspec* h, void* arena, size_t bytes, void* stream);
int32_t mb_melspec_num_frames(const mb_melspec* h, int32_t n_samples);   /* 1 + n_samples / hop_length */
/* wav fp32 [n_samples] (device) -> out fp32 [frames][n_mels] or [n_mels][frames] (device) */
int mb_melspec_forward(mb_melspec* h, const float* wav, int32_t n_samples, float* out, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Voice-conversion mel decoder (ppg2mel)
 *   replaces  models/ppg2mel/__init__.py:166-192 (MelDecoderMOLv2.inference: PPG / pitch encoder, reduce_proj with the
 *             normalised speaker embedding), models/ppg2mel/rnn_decoder_mol.py:267-315 (Decoder.inference: PreNet with
 *             dropout always on, attention LSTMCell, MoL attention, decoder LSTMCell, projection + stop layer) and
 *             models/ppg2mel/utils/cnn_postnet.py (Postnet, eval BatchNorm)
 * ------------------------------------------------------------------------------------------- */
typedef struct mb_ppg2mel_config {
  int32_t bottle_neck_feature_dim;     /* 144 PPG dim (any 1..1024) */
  int32_t spk_embed_dim;               /* 256 (any 1..1024) */
  int32_t encoder_dim;                 /* 256 */
  int32_t encoder_downsample_rates[2]; /* 2, 2 */
  int32_t attention_rnn_dim;           /* 512 */
  int32_t decoder_rnn_dim;             /* 512 */
  int32_t num_decoder_rnn_layer;       /* 1 */
  int32_t concat_context_to_last;      /* 1 */
  int32_t prenet_dims[2];              /* 256, 128 */
  int32_t num_mixtures;                /* 5 */
  int32_t frames_per_step;             /* 2 */
  int32_t num_mels;                    /* 80 */
} mb_ppg2mel_config;

typedef struct mb_ppg2mel mb_ppg2mel;

/* every field but the two input dims must hold the value shown (the kernels specialise on them): MB_ERR_INVALID else */
int mb_ppg2mel_create(const mb_ppg2mel_config* cfg, mb_ppg2mel** out);
void mb_ppg2mel_destroy(mb_ppg2mel* h);
size_t mb_ppg2mel_arena_bytes(const mb_ppg2mel* h);
int mb_ppg2mel_set_arena(mb_ppg2mel* h, void* arena, size_t bytes);
/* tensors of ckpt['model'] under their reference names (decoder.prenet_pitch.* is accepted and ignored; the postnet's
 * num_batches_tracked is ignored); finalize repacks them and folds the postnet BatchNorm into its convolutions */
int mb_ppg2mel_set_weight(mb_ppg2mel* h, const char* name, const float* w, const int64_t* dims, int32_t ndim,
                          void* stream);
int mb_ppg2mel_finalize(mb_ppg2mel* h, void* stream);
/* 0 when frames < 4, when the device query fails, or when T_enc = frames / 4 needs more shared memory than the MoL
 * attention kernel can have (the message names the limit: 29 039 on an H100 80GB HBM3) */
size_t mb_ppg2mel_workspace_bytes(const mb_ppg2mel* h, int32_t batch, int32_t frames);

/* MelDecoderMOLv2.inference for a padded batch of 1..128 rows, each row computed as its own B = 1 call:
 *   ppg fp32 [B][frames][bottle_neck_feature_dim], lf0_uv fp32 [B][frames][2], spk fp32 [B][spk_embed_dim] (device)
 *   lengths int32 [B] (host): valid PPG frames of each row, 4 <= lengths[b] <= frames; T_enc[b] = lengths[b] / 4
 *   mask1 uint8 [S][B][256], mask2 uint8 [S][B][128] (device): PreNet keep flags of decoder step s, S = 2 * (frames / 4);
 *     both NULL -> drawn on the device from `seed` (Philox, keyed by step, row and unit)
 *   outputs (device, zero-filled past each row's end): mel / mel_post fp32 [B][2 S][80], align fp32 [B][S][frames / 4],
 *     stop fp32 [B][S] (stop logits, may be NULL); steps_host int32 [B] (host): decoder steps n of each row (2 n mel
 *     frames, n alignment rows).
 * frames / 4 above the attention's shared-memory limit (see mb_ppg2mel_workspace_bytes) is MB_ERR_INVALID, before anything is
 * queued.
 * Row b stops after step n when sigmoid(stop) > 0.5 and n >= 2 T_enc[b] - 5, or when n = 2 T_enc[b]; a finished row
 * is frozen while the others run on.  The decoder steps are replayed from a CUDA graph of 16 steps on an internal
 * stream ordered after `stream` (events); the host polls the finished rows once per graph replay. */
int mb_ppg2mel_inference(mb_ppg2mel* h, const float* ppg, const float* lf0_uv, const float* spk, const int32_t* lengths,
                         int32_t batch, int32_t frames, const uint8_t* mask1, const uint8_t* mask2, uint64_t seed,
                         float* mel, float* mel_post, float* align, float* stop, int32_t* steps_host, void* workspace,
                         size_t workspace_bytes, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Voice-conversion PPG extractor (Conformer ASR encoder)
 *   replaces  models/ppg_extractor/__init__.py:25-39 (PPGModel.forward: DefaultFrontend STFT + log-mel, UtteranceMVN,
 *             ConformerEncoder with a Conv2d input layer, relative or absolute positional attention, macaron FFN and
 *             convolution module)
 * Every config value comes from the caller (the reference's args.frontend_conf / normalize_conf / encoder_conf); options
 * the kernels do not implement are rejected by create with MB_ERR_INVALID and a message.
 * ------------------------------------------------------------------------------------------- */
#define MB_PPGX_INPUT_CONV2D 0        /* input_layer: "conv2d" (only this); 1 "linear", 2 "vgg2l", 3 "embed" */
#define MB_PPGX_POS_ABS 0             /* pos_enc_layer_type "abs_pos" */
#define MB_PPGX_POS_SCALED_ABS 1      /*   "scaled_abs_pos" (rejected) */
#define MB_PPGX_POS_REL 2             /*   "rel_pos" */
#define MB_PPGX_ATTN_SELF 0           /* selfattention_layer_type "selfattn" */
#define MB_PPGX_ATTN_REL 1            /*   "rel_selfattn" */
#define MB_PPGX_FF_LINEAR 0           /* positionwise_layer_type "linear"; 1 "conv1d", 2 "conv1d-linear" (rejected) */
#define MB_PPGX_ACT_SWISH 0           /* activation_type "swish" */
#define MB_PPGX_ACT_RELU 1            /*   "relu" */
typedef struct mb_ppgx_config {
  int32_t n_fft, win_length, hop_length, n_mels;  /* frontend_conf (n_fft <= 1024, win_length <= n_fft) */
  int32_t kaldi_padding_mode, downsample_rate;    /* frontend_conf: 0 and 1 only */
  int32_t norm_means, norm_vars;                  /* normalize_conf */
  int32_t attention_dim, attention_heads, linear_units, num_blocks;
  int32_t input_layer, no_subsample, subsample_by_2;
  int32_t normalize_before, concat_after, positionwise_layer_type;
  int32_t macaron_style, pos_enc_layer_type, selfattention_layer_type, activation_type;
  int32_t use_cnn_module, cnn_module_kernel;
} mb_ppgx_config;

typedef struct mb_ppgx mb_ppgx;

int mb_ppgx_create(const mb_ppgx_config* cfg, mb_ppgx** out);
void mb_ppgx_destroy(mb_ppgx* h);
size_t mb_ppgx_arena_bytes(const mb_ppgx* h);
int mb_ppgx_set_arena(mb_ppgx* h, void* arena, size_t bytes);
/* tensors of PPGModel.state_dict() under their reference names (frontend.logmel.melmat [n_fft / 2 + 1][n_mels] is an input
 * weight; inv_melmat and num_batches_tracked are accepted and ignored); finalize packs the tensor-core weight images */
int mb_ppgx_set_weight(mb_ppgx* h, const char* name, const float* w, const int64_t* dims, int32_t ndim, void* stream);
int mb_ppgx_finalize(mb_ppgx* h, void* stream);
/* PPG frames of an n-sample utterance: 1 + n / hop_length, halved by each stride-2 conv of the input layer */
int32_t mb_ppgx_num_frames(const mb_ppgx* h, int32_t n_samples);
size_t mb_ppgx_workspace_bytes(const mb_ppgx* h, int32_t batch, int32_t n_samples_max);
/* PPGModel.forward for a padded batch of 1..128 rows, each row computed as its own B = 1 call (bitwise):
 *   wav fp32 [B][n_max] (device); n_samples int32 [B] (host): n_fft / 2 < n_samples[b] <= n_max
 *   pe_len: rows of the positional table the module instance holds (max(5000, longest T it has seen)); pos_table fp32
 *     [T_max][attention_dim] (device): rows [0, T_max) of that table as the reference builds it (rel_pos: row k encodes
 *     position pe_len - 1 - k; abs_pos: position k), T_max = mb_ppgx_num_frames(h, n_max)
 *   out fp32 [B][T_max][attention_dim] (device), zero past each row's frames;
 *   taps fp32 [num_blocks + 1][B][T_max][attention_dim] or NULL: the embed output and each block's output */
int mb_ppgx_forward(mb_ppgx* h, const float* wav, const int32_t* n_samples, int32_t batch, int32_t n_max, int32_t pe_len,
                    const float* pos_table, float* out, float* taps, void* workspace, size_t workspace_bytes, void* stream);

/* test hook: ONE launch of a PPG-extractor kernel on caller-provided device tensors (no model handle), through the launch
 * helpers the forward uses; CONV2D_TC also packs w as finalize does (absmax -> tc_weight_scale -> conv2d_tc_pack).  Row b of a
 * padded batch has len[b] valid entries of T.  "Operand tiles" are fp16 hi / lo planes [ceil(cols / 64)][rows_total][64] with
 * 16-byte chunk c of row m at c ^ (m & 7), the layout every tensor-core GEMM of the extractor reads. */
#define MB_PPGX_DBG_FRONTEND 0  /* log-mel of wav x [B][n_max] (len: samples, len2: frames) -> y [B][T][F]; w = melmat        */
#define MB_PPGX_DBG_MVN 1       /* y [B][T][F] in place over len frames; flags 1 norm_means | 2 norm_vars                      */
#define MB_PPGX_DBG_CONV0 2     /* relu(conv k/stride/pad of x [B][T][F], len frames; w [N][1][k][k]) -> y_hi / y_lo planes    */
                                /*   [B][T_out][F_out][N] channels-last                                                        */
#define MB_PPGX_DBG_CONV2D_TC 3 /* relu(conv of the planes x_hi + x_lo [B][T][F][C], len frames; w [N][C][k][k]) -> operand     */
                                /*   tiles of [B T_out][N F_out] (column n F_out + f), zeroed first                            */
#define MB_PPGX_DBG_LN_TILES 4  /* LayerNorm (w, bias) of x [M][D] -> operand tiles of [rows_total][D]                         */
#define MB_PPGX_DBG_ACT_TILES 5 /* act of x [M][ld] columns [0, D) -> operand tiles of [rows_total][D]                         */
#define MB_PPGX_DBG_LN_ROWS 6   /* LayerNorm (w, bias) of x [B T][D] -> y (may be x); flags 4: zero_pad rows t >= len[b]       */
#define MB_PPGX_DBG_DW 7        /* GLU of x [B T][2 D], depthwise conv w [D][k] + bias, BatchNorm bn[4], act -> operand tiles  */
#define MB_PPGX_DBG_ATTN 8      /* attention of x = qkv [B T][3 D], heads H x dk, rel: P [T][ldp], pos biases pu / pv [H][dk] */
                                /*   -> y = ctx [B T][D]                                                                       */
typedef struct mb_ppgx_debug_spec {
  int32_t kind;                  /* MB_PPGX_DBG_* */
  int32_t B, T;                  /* rows; padded frames of each row (FRONTEND: STFT frames of n_max; CONV*: input frames) */
  const int32_t* len;            /* device [B]: valid samples (FRONTEND) / frames of each row */
  const int32_t* len2;           /* FRONTEND: device [B] STFT frames of each row */
  int32_t n_max, n_fft, win_length, hop_length;  /* FRONTEND */
  int32_t F;                     /* mel bins (FRONTEND, MVN, CONV0); input plane width (CONV2D_TC) */
  int32_t C, N;                  /* CONV2D_TC input channels; CONV0 / CONV2D_TC output channels */
  int32_t k, stride, pad;        /* CONV0 / CONV2D_TC: k x k kernel; DW: kernel size (odd) */
  int32_t M, D, ld, rows_total;  /* LN_TILES / ACT_TILES rows; features; ACT_TILES row stride; operand tile rows (x 128) */
  int32_t act;                   /* ACT_TILES / DW: 0 none, 1 ReLU, 2 swish */
  int32_t flags;                 /* MVN: 1 norm_means | 2 norm_vars; LN_ROWS: 4 zero_pad */
  int32_t H, dk, ldp, rel;       /* ATTN */
  const float* x;
  const void* x_hi;              /* CONV2D_TC input planes (fp16) */
  const void* x_lo;
  const float* w;
  const float* bias;
  const float* bn[4];            /* DW: weight, bias, running_mean, running_var */
  const float* P;
  const float* pu;
  const float* pv;
  float* y;
  void* y_hi;                    /* CONV0 planes / operand tiles (fp16) */
  void* y_lo;
} mb_ppgx_debug_spec;
/* device workspace the spec needs */
size_t mb_ppgx_debug_workspace_bytes(const mb_ppgx_debug_spec* spec);
/* synchronises `stream` (CONV2D_TC reads the pack scale back); writes one line into `report`:
 * "kernel=K inst=I grid=X,Y,Z inv_scale=S" (inst: NT of conv2d_tc, DK of attn_kernel, 0 otherwise) */
int mb_ppgx_debug(const mb_ppgx_debug_spec* spec, void* workspace, size_t workspace_bytes, void* stream, char* report,
                  size_t report_len);

#ifdef __cplusplus
}
#endif
#endif /* MOCKINGBIRD_B200_H */
