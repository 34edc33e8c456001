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
 *   - workspaces: a compute call takes any alignment of `workspace` and needs at least the bytes its mb_*_workspace_bytes
 *     reports, a figure that includes the slack for aligning the pointer inside the library.  A NULL workspace is
 *     MB_ERR_INVALID and a shorter one MB_ERR_WORKSPACE, both reported before anything is queued.  Its contents do not
 *     persist from one call to the next, except where an entry point says so: the sample-loop state of
 *     mb_wavernn_generate* and mb_deepmind_generate, and what mb_wavernn_last_logits reads.
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
/* The VITS decoder (models/synthesizer/models/vits.py:245-290, `Vits.dec`): HiFi-GAN's plan with num_mels input channels,
 * ConvTranspose1d(k, u, padding=(k-u)//2) without output padding ((k-u) even), and conv_post without bias (its checkpoint
 * has no "conv_post.bias"; the layer adds zero).  The per-utterance cond(g) of Generator.forward is not part of this kind:
 * mb_vits feeds it as extra, time-constant input channels of conv_pre (see mb_vits_decode). */
#define MB_GAN_VITS 3

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
  /* mb_gan_debug_f32 only (zero / NULL: NCL everywhere, no second destination).  The layouts say how
   * the kernel sees its tensors; the caller's tensors are fp32 NCL either way and are converted. */
  int32_t x_layout;    /* 0 / 1 NCL fp32, 2 channel-quad blocked fp32, 3 fp16 plane (activated
                          with the layer's input slope when converted, as the forward writes it) */
  int32_t y_layout;    /* residual / y / y2 as the kernel sees them: 0 / 1 NCL fp32, 2 blocked fp32 */
  float* y2;           /* second destination [B, Cout, L*stride]: running sum in, y2 + v out (NULL: none) */
  int32_t y2_out16;    /* fp16 plane of the second destination: 0 none, 1 plain, 2 hi/lo */
  float y2_slope;      /* leaky-relu slope of that plane */
  float* y2_16;        /* y2_out16: the plane read back (mb_gan_debug_f32 sizes both y16 and y2_16 as the
                          forward sizes the planes of its FP32 layers: Cout plain, 2 Cout hi/lo) */
} mb_gan_debug_spec;
/* writes one line per kernel launch into `report`:
 * "kernel=N,MT,CW,PAIR rows_item= resident= wstages= n_work= grid= red_add=" */
int mb_gan_debug_launch(mb_gan* h, const mb_gan_debug_spec* spec, void* workspace, size_t workspace_bytes,
                        void* stream, char* report, size_t report_len);

/* test hook: op `layer_index` of any handle (fp32, f16tc, f16x3) run once on the FP32 kernels, with the
 * caller's epilogue inputs and outputs (pair, red_add and res_kind 2 / 3 are refused).  An add op
 * (mb_gan_layer_info "add ...") computes y += x and refreshes the fp16 plane out16 = lrelu(y, out_slope).
 * post_variant picks the Cout = 1 kernel: MB_GAN_POST_DEFAULT (the MB_POST_* switches), 1 / 2 / 4
 * output rows per thread, or MB_GAN_POST_TILE; other ops take MB_GAN_POST_DEFAULT.  Writes
 * "kernel=NAME" into `report`: tapconv_f32, cout1<R>, post_tile<7,CQ>, add or add_dst16. */
#define MB_GAN_POST_DEFAULT 0
#define MB_GAN_POST_TILE (-1)
int mb_gan_debug_f32(mb_gan* h, const mb_gan_debug_spec* spec, int32_t post_variant, void* workspace,
                     size_t workspace_bytes, void* stream, char* report, size_t report_len);

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

/* sampler of a handle (hparams.voc_mode), fixed at create */
#define MB_WAVERNN_RAW 0 /* fc3 [512, 512]: softmax + Categorical over 2^bits classes */
#define MB_WAVERNN_MOL 1 /* fc3 [30, 512]: 10-component discretized mixture of logistics (models/vocoder/distribution.py:87-123) */

int mb_wavernn_create(const mb_wavernn_config* cfg, mb_wavernn** out); /* == mb_wavernn_create_mode(cfg, MB_WAVERNN_RAW, out) */
int mb_wavernn_create_mode(const mb_wavernn_config* cfg, int32_t mode, mb_wavernn** out);
void mb_wavernn_destroy(mb_wavernn* h);
size_t mb_wavernn_arena_bytes(const mb_wavernn* h);
int mb_wavernn_set_arena(mb_wavernn* h, void* arena, size_t bytes);
/* tensors of ckpt['model_state'] (wavernn/inference.py:36-37) under their reference names (SURVEY.md appendix B) */
int mb_wavernn_set_weight(mb_wavernn* h, const char* name, const float* w, const int64_t* dims,
                          int32_t ndim, void* stream);
int mb_wavernn_finalize(mb_wavernn* h, void* stream);

size_t mb_wavernn_workspace_bytes(const mb_wavernn* h, int32_t frames, int32_t folds, int32_t steps);

/* UpsampleNetwork.forward on the padded mel (fatchord_version.py:168-170): mel [80, T] fp32
 * (already divided by mel_max_abs_value, inference.py:60-61) -> the conditioning the sample loop reads, kept in
 * the workspace: aux [T,128], the mel ladder's output melup [200T,80] and three frame-rate tables of the aux
 * contributions (DESIGN.md section 4.1).  This is mb_wavernn_condition_multi with one utterance: T + 4 frames
 * must stay below 2^31 / (200 * 80), i.e. T <= 134 213 (about 28 min at 16 kHz); a longer mel is refused with
 * MB_ERR_INVALID and mb_wavernn_workspace_bytes returns 0 for it. */
int mb_wavernn_condition(mb_wavernn* h, const float* mel, int32_t frames, void* workspace,
                         size_t workspace_bytes, void* stream);

/* The sample loop (fatchord_version.py:190-234) over `folds` independent rows, each `steps` long,
 * row r starting at upsampled-time offset fold_starts[r] (fold_with_overlap, :288-338; positions
 * past the end of the conditioning read zeros like the reference's zero padding).  A fold start must be
 * >= 0 and fold_starts[r] + steps must fit in int32; otherwise the call is refused with MB_ERR_INVALID.
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

/* The sample loop of a MOL handle (fatchord_version.py:211-221): per step and row, 10 mixture uniforms pick the component
 * argmax(logit_probs - log(-log(temp))), one more uniform draws x = clip(mean + exp(max(log_scale, log(1e-14))) *
 * (log(u) - log(1 - u)), -1, 1); x is the output sample and the next step's input.  Rows, steps and fold sharding as in
 * mb_wavernn_generate_rows.
 *   uniforms: fp32 [steps_in_call][11 * noise_folds], per step the noise_folds x 10 mixture uniforms (row-major) and then the
 *             noise_folds logistic uniforms, all in [1e-5, 1 - 1e-5] - the order the reference draws them from the torch
 *             generator - or NULL for the built-in counter-based generator keyed by (seed, step, global fold, slot).
 *   out_x   : fp32 [folds, steps] samples (local rows). */
int mb_wavernn_generate_rows_mol(mb_wavernn* h, const int32_t* fold_starts_host, int32_t folds, int32_t steps,
                                 int32_t step0, int32_t nsteps, const float* uniforms, int32_t noise_folds, int32_t row0,
                                 uint64_t seed, float* out_x, void* workspace, size_t workspace_bytes, void* stream);

/* Several utterances of different lengths in one sample loop (the loop costs about the same per step for 1 row as for 64:
 * DESIGN.md section 4.7).  Utterance u's samples are those of mb_wavernn_condition + mb_wavernn_generate_rows[_mol] on it alone.
 *
 * mb_wavernn_condition_multi: mels [80, frames[u]] fp32 back to back in `mel_concat`; the conditioning tables of all
 * utterances are kept concatenated in the workspace (one launch per layer whatever n_utts is).
 *
 * mb_wavernn_generate_multi[_mol]: `rows` rows, row r = (row_utt[r], row_start[r] offset in upsampled time, row_steps[r],
 * row_fold[r] = index of the row among the folds of its utterance), all host arrays.  The folds 0 .. n-1 of an utterance are
 * adjacent rows of one length and the rows are ordered longest first, so that the rows alive at any step are a prefix:
 *   max_steps   : steps of row 0; out_idx / out_x is [rows, max_steps], row r written at [r, 0 .. row_steps[r])
 *   step0/nsteps: as in mb_wavernn_generate; step0 == 0 resets the state and uploads the row table
 *   n_live      : number of rows with row_steps > step0; only the 64-row blocks that hold one of them run
 *   noise       : RAW: Exp(1) fp32 [nsteps][n_live][512].  MOL: uniforms fp32 [nsteps][11 * n_live], per step and per live
 *                 utterance of n folds its n x 10 mixture uniforms and then its n logistic uniforms (each utterance's draws
 *                 of a step are contiguous, as one generator per utterance produces them).  NULL: the built-in generator
 *                 keyed by (utt_seeds[row_utt[r]], step, row_fold[r], slot) - what the single call draws for that utterance
 *                 under that seed.
 *   utt_seeds   : one per conditioned utterance; may be NULL when noise is given */
size_t mb_wavernn_workspace_bytes_multi(const mb_wavernn* h, int32_t n_utts, const int32_t* frames, int32_t rows,
                                        int32_t max_steps);
int mb_wavernn_condition_multi(mb_wavernn* h, const float* mel_concat, const int32_t* frames, int32_t n_utts, void* workspace,
                               size_t workspace_bytes, void* stream);
int mb_wavernn_generate_multi(mb_wavernn* h, const int32_t* row_utt, const int32_t* row_start, const int32_t* row_steps,
                              const int32_t* row_fold, int32_t rows, const uint64_t* utt_seeds, int32_t max_steps,
                              int32_t step0, int32_t nsteps, int32_t n_live, const float* noise, int16_t* out_idx,
                              void* workspace, size_t workspace_bytes, void* stream);
int mb_wavernn_generate_multi_mol(mb_wavernn* h, const int32_t* row_utt, const int32_t* row_start, const int32_t* row_steps,
                                  const int32_t* row_fold, int32_t rows, const uint64_t* utt_seeds, int32_t max_steps,
                                  int32_t step0, int32_t nsteps, int32_t n_live, const float* uniforms, float* out_x,
                                  void* workspace, size_t workspace_bytes, void* stream);

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
/* the same tail for the float samples of a MOL handle: fp32 [folds, steps] (device), cast to float64; no mu-law */
int mb_wavernn_postprocess_f32(const float* samples, int32_t folds, int32_t steps, int32_t batched, int32_t target,
                               int32_t overlap, double preemphasis, int64_t wave_len, int32_t fade_len, double* out,
                               int64_t* n_out, void* workspace, size_t workspace_bytes, void* stream);

/* debug/test hook: logits [folds, 512] (RAW) or [folds, 30] (MOL) fp32 of the LAST step executed by mb_wavernn_generate */
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
/* host-only: one chunk of noise from several independent streams (one generator position per utterance of a multi-utterance
 * sample loop).  Source s continues from (states[s][624], left[s], next[s]) - advanced in place - and writes, for each of the
 * first steps[s] steps j of the chunk, words_per_step[s] finished draws at out[j * stride + col[s]]; a source whose utterance
 * ends inside the chunk has fewer steps than the others.  n_threads host threads share the sources. */
int mb_mt19937_fill_sources(int32_t n_src, uint32_t* states, int32_t* left, int32_t* next, const uint64_t* words_per_step,
                            const uint64_t* col, const int32_t* steps, uint32_t* out, uint64_t stride, int32_t n_threads);
/* device conversion alone: raw draws [n_elems][2] (device) -> Exp(1) fp32 [n_elems] */
int mb_mt_to_exp(const void* dev_raw, float* dev_noise, uint64_t n_elems, void* stream);
/* The uniforms of the MOL sampler: ATen's CPU float `uniform_(1e-5, 1 - 1e-5)` takes ONE 32-bit draw per element,
 * u = fma((w & (2^24-1)) * 2^-24, float(1-1e-5) - float(1e-5), float(1e-5)) in float.  `next_uniform` is mb_mtstream_next
 * for such a stream: n_elems words -> n_elems fp32; `mb_mt_to_uniform` converts finished (tempered) draws. */
int mb_mtstream_next_uniform(mb_mtstream* ms, uint64_t n_elems, void* dev_raw, float* dev_noise, void* main_stream);
int mb_mt_to_uniform(const void* dev_raw, float* dev_noise, uint64_t n_elems, void* stream);

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
/* 0 for a shape generate would refuse, including more characters than mb_tacotron_max_chars() (when a device can be asked) */
size_t mb_tacotron_workspace_bytes(const mb_tacotron* h, int32_t batch, int32_t chars, int32_t steps, int32_t r);
/* the longest input (characters per utterance) generate accepts on the current device: the attention step keeps
 * 4 * (5438 + 38 * chars) bytes in shared memory, within the per-block opt-in limit (1386 on an H100); 0 without a device */
int32_t mb_tacotron_max_chars(void);

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

/* Many utterances as independent rows (Tacotron.generate_many): row b is computed as that utterance's own B = 1 generate.
 *   chars int32 [B][Tc] (row b's first row_chars[b] entries are its text; the rest is never read as input), spk [B][256],
 *   B <= 128.  Row b stops at its own stop rule (stop * 10 > min_stop_token and frame t > 10) or at its cap of
 *   ceil(row_steps[b] / r) decoder steps; a finished row keeps computing until every row is done, and nothing it computes
 *   after its stop reaches its outputs or another row.  Its frames, (done step + 1) * r, go to row_frames_host[b].
 *   Outputs: mel, linear [B][80][F] and attn [B][F / r][Tc] with F = *frames_out_host = the largest row_frames_host[b];
 *   row b's part is [:, :row_frames_host[b]] (attn [:row_frames_host[b] / r, :row_chars[b]]).  Buffers are sized for
 *   F = ceil(max row_steps / r) * r.
 *   Dropout: enc_masks [2][B][Tc][256] and dec_masks [ceil(max row_steps / r)][2][B][256] as for mb_tacotron_generate,
 *   or, when null, drawn on the device with Philox keyed by row_seeds[b] and counted by (unit, character or step, layer):
 *   an utterance draws the same masks whatever its row or its neighbours.
 *   Every layer takes a route chosen from something other than the row count (DESIGN.md section 4b), so a row's outputs are
 *   bitwise the same in any batch.  The call blocks the host like mb_tacotron_generate. */
size_t mb_tacotron_ragged_workspace_bytes(const mb_tacotron* h, int32_t batch, int32_t n_chars, int32_t max_steps, int32_t r);
int mb_tacotron_generate_ragged(mb_tacotron* h, const int32_t* chars, const float* spk, int32_t batch, int32_t n_chars,
                                const int32_t* row_chars, const int32_t* row_steps, const uint64_t* row_seeds, int32_t r,
                                int32_t style_idx, float min_stop_token, const uint8_t* enc_masks, const uint8_t* dec_masks,
                                float* mel, float* linear, float* attn, int32_t* frames_out_host, int32_t* row_frames_host,
                                void* workspace, size_t workspace_bytes, void* stream);

/* Streamed decoding (Tacotron.generate_stream): a decoder loop over `slots` (<= 128) rows that texts enter when a row is free
 * and leave when their row stops.  Each text's mel, linear and attention are bitwise those mb_tacotron_generate_ragged gives it.
 *   workspace_bytes / open: texts of at most n_chars characters and max_steps frames; 0 / MB_ERR_INVALID as generate would refuse.
 *     The workspace holds the encoder's scratch, the decoder loop, the postnet's scratch, a staging pool of 2 x slots encoded
 *     texts and a pool of 2 x slots finished rows; it must outlive the stream.  open captures the 8-step decoder graph once.
 *   encode: n texts (chars int32 device [n][n_chars], zero past each text's row_chars[i]; spk device [n][256]; enc_masks device
 *     [2][n][n_chars][256] or NULL: drawn from row_seeds) into staging-pool rows [pool_row, pool_row + n), inside one half of the
 *     pool, on an internal encoder stream that runs while the decoder does; it waits for the admissions before it.  `stream`
 *     does not wait for the encode (only the admissions that copy these rows do), so the inputs must stay allocated until
 *     the stream is closed.
 *   admit: texts from the staging pool into free slots, between graph replays (one launch: the slot's state reset to a fresh row's,
 *     its encoder rows copied, its dropout masks copied from dec_masks[i] (device [>= ceil(row_steps / r)][2][256]) or drawn).
 *   run: replays the decoder graph 16 steps at a time until at least one occupied row has stopped (at once when none is
 *     occupied), copies each stopped row's frames and alignment to the finished-row pool and frees its slot; returns their text
 *     ids and frames in the order found (steps_run: decoder steps run so far).  Blocks the host while it polls.
 *   harvest: the postnet over the n oldest finished rows not harvested yet, on `stream`: mel, linear [n][80][frames] and attn
 *     [n][frames / r][n_chars], frames = the longest of their frames; row i's part is its own frames.  Every harvest of a stream
 *     must use the same `stream`.  run refuses when finished rows would overflow their pool: harvest at least every `slots` rows.
 *   close: waits for the stream's work and frees it; the model handle stays usable. */
typedef struct mb_taco_stream mb_taco_stream;
/* test hook: the per-slot regions of an open stream (device addresses into its workspace).  Admission zeroes slot b's row of
 * every region with reset = 1 and writes slot b's row of seq, proj, chars, lens, caps, done, start and dmask; pool_* are the
 * staging pool the encoder writes.  Layouts by kind: */
#define MB_TACO_REGION_F32 0  /* fp32 [rows][width] */
#define MB_TACO_REGION_TILE 1 /* fp16 operand tile plane [ceil(width / 64)][rows][64], 16-byte chunks XOR (row & 7) */
#define MB_TACO_REGION_U8 2   /* uint8 [depth][2][rows][width] (decoder dropout masks: ring steps, layers, slots, units) */
#define MB_TACO_REGION_I32 3  /* int32 [rows][width] */
typedef struct mb_taco_stream_region {
  char name[24];
  void* ptr;
  int32_t kind, rows, width, depth, reset;
} mb_taco_stream_region;
/* fills up to `max` entries of out (may be NULL) and returns how many regions there are, or a negative error */
int32_t mb_tacotron_stream_regions(const mb_taco_stream* s, mb_taco_stream_region* out, int32_t max);
size_t mb_tacotron_stream_workspace_bytes(const mb_tacotron* h, int32_t slots, int32_t n_chars, int32_t max_steps, int32_t r);
int mb_tacotron_stream_open(mb_tacotron* h, int32_t slots, int32_t n_chars, int32_t max_steps, int32_t r, int32_t style_idx,
                            float min_stop_token, void* workspace, size_t workspace_bytes, void* stream, mb_taco_stream** out);
int mb_tacotron_stream_encode(mb_taco_stream* s, int32_t pool_row, int32_t n, const int32_t* chars, const float* spk,
                              const int32_t* row_chars, const uint64_t* row_seeds, const uint8_t* enc_masks, void* stream);
int mb_tacotron_stream_admit(mb_taco_stream* s, int32_t n, const int32_t* slot, const int32_t* pool_row, const int64_t* text_id,
                             const int32_t* row_chars, const int32_t* row_steps, const uint64_t* row_seeds,
                             const uint8_t* const* dec_masks, void* stream);
int mb_tacotron_stream_run(mb_taco_stream* s, int32_t* n_done, int64_t* done_ids, int32_t* done_frames, int64_t* steps_run);
int mb_tacotron_stream_harvest(mb_taco_stream* s, int32_t n, int32_t frames, float* mel, float* linear, float* attn, void* stream);
void mb_tacotron_stream_close(mb_taco_stream* s);

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
  const int32_t* len;        /* ragged rows, or NULL (the padded path).  BIG: device [ceil(M / T)] valid length of each length-T
                                sequence: a shifted tap reads zeros at and past it (TcIm2col::len).  GRU: device [M] valid
                                length of each row: direction 1 keeps h = 0 (state, out[1], nxt tiles) while t1 >= len[m] */
  int32_t t1;                /* GRU with len: the time index direction 1 is at in this step (TcGruArgs::t1) */
  const int32_t* row_start;  /* PLAIN: device [M] per-row step origin, or NULL: row m writes at y + ((step - row_start[m]) % ring) * y_step */
  int32_t ring;
} mb_taco_tc_debug_spec;
/* device workspace the spec needs */
size_t mb_taco_tc_debug_workspace_bytes(const mb_taco_tc_debug_spec* spec);
/* synchronises `stream` (the pack scale is read back); writes one line into `report`:
 * "kernel=K grid=X,Y cluster=C compact=0|1 rows_pad=R mma_groups=G,G_last inv_scale=S a_bytes=A w_bytes=W" */
int mb_taco_tc_debug(const mb_taco_tc_debug_spec* spec, void* workspace, size_t workspace_bytes, void* stream, char* report,
                     size_t report_len);

/* test hook: ONE launch of an FP32 kernel of the Tacotron path (csrc/tacotron_kernels.cu, csrc/tacotron.cu) on caller-provided
 * device tensors (no model handle), through the launcher the forward uses.  GEMM and STOP_STEP read the GemmArgs fields; the
 * other kinds read in[] / out[] / n[] as listed (n[] entries are sizes, strides and flags in the order given).  Every kind
 * honours step_ptr / step_j where its kernel takes them. */
#define MB_TACO_DBG_GEMM 0             /* launch_gemm: the GemmArgs fields below                                              */
#define MB_TACO_DBG_PRENET 1           /* in: x, x_first, W1, b1, W2, b2, m1, m2  out: y, s_hi, s_lo
                                          n: B, K, H, ldy, x_ld, x_step, mask_step, s_k0, s_rows_pad                         */
#define MB_TACO_DBG_GRU_CELL 2         /* in: gi, gh  out: h, out2  n: M, H, ldgi, ldh, ldout2                                 */
#define MB_TACO_DBG_LSTM_CELL 3        /* in: g  out: c, h, x (x += h, or NULL)  n: M, H                                        */
#define MB_TACO_DBG_HIGHWAY 4          /* in: x12  out: y  n: M, C                                                              */
#define MB_TACO_DBG_MAXPOOL2 5         /* in: x  out: y  n: B, T, C                                                             */
#define MB_TACO_DBG_EMBEDDING 6        /* in: ids (int32), table  out: y  n: M, D                                               */
#define MB_TACO_DBG_COPY_COLS 7        /* in: src  out: dst  n: M, n, ldsrc, rows_per_src, lddst, off                           */
#define MB_TACO_DBG_LSA_STEP 8         /* in: pq, proj, seq, chars, conv_w, conv_b, L, v, q_in, Wq, bq  out: cum, scores, ctx
                                          n: B, Tc, seq_dim, scores_ld, threads (256 | 512); q_in NULL: pq is read
                                          row_len: the kernel's lens (row b ends at row_len[b] <= Tc), or NULL              */
#define MB_TACO_DBG_LSA_CTX 9          /* in: scores, seq  out: ctx, sa_hi, sa_lo, sb_hi, sb_lo
                                          n: B, Tc, seq_dim (a multiple of 256), scores_ld, s_rows_pad
                                          row_len: the kernel's lens (only t < row_len[b] is read), or NULL                 */
#define MB_TACO_DBG_GST_ATTENTION 10   /* in: q, keys, values  out: y  n: B, ntok (<= 16), E, heads (<= 8)                      */
#define MB_TACO_DBG_STOP_STEP 11       /* GemmArgs (x, W, bias, y, ldy; N = 1) and out: flags, ticket  n: B, r  fval: min_stop
                                          row_done / row_caps: the per-row rule of ragged batches, or NULL (both or neither) */
#define MB_TACO_DBG_STOP_FLAG 12       /* in: stopv  out: flags  n: B, r  fval: min_stop_token  row_done / row_caps as above   */
#define MB_TACO_DBG_FILL_MASKS 13      /* out: m  n: count, stream_id  seed (step_ptr: stream_id += *step_ptr)                  */
#define MB_TACO_DBG_FILL_MASKS_STEPS 14 /* out: m  n: per_step, steps  seed                                                     */
#define MB_TACO_DBG_PACK_MELPROJ 15    /* in: W  out: dst  n: n_mels, max_r, r, K                                               */
#define MB_TACO_DBG_TO_NCL 16          /* in: x  out: y  n: steps, B, C, frames                                                 */
#define MB_TACO_DBG_BN_FOLD 17         /* in: gamma, beta, mean, var  out: scale, shift  n: count                               */
#define MB_TACO_DBG_FILL_MASKS_SEEDED 18 /* out: m  n: B, npos, units, dec (0: m [2][B][npos][units], 1: m [npos][2][B][units])
                                            row_seeds: device [B] Philox key of each row                                     */
typedef struct mb_taco_debug_spec {
  int32_t kind;                /* MB_TACO_DBG_* */
  /* GemmArgs (csrc/tacotron_kernels.cuh) */
  int32_t nseg;
  const float* x[5];
  int32_t K[5], ld[5], shift[5], w_off[5], w_stride[5];
  const float* W;
  int32_t ldw;
  const float* bias;
  int32_t M, N, T, act;
  const float* bn_scale;
  const float* bn_shift;
  const uint8_t* mask;
  const float* res;
  int32_t ldres;
  float* y;
  int32_t ldy;
  int32_t step_mode;
  const int32_t* step_ptr;     /* every kind: step = (*step_ptr or 0) + step_j */
  int32_t step_j;
  int64_t x_step;
  const float* x_first;
  int64_t mask_step;
  /* the other kinds */
  const void* in[12];
  void* out[6];
  int64_t n[10];
  float fval;
  uint64_t seed;
  /* ragged rows (all NULL / 0: the padded path) */
  const int32_t* row_len;      /* LSA_STEP / LSA_CTX: device [B] characters of each row */
  int32_t* row_done;           /* STOP_STEP / STOP_FLAG: device [B] done step of each row (-1 while running), in/out */
  const int32_t* row_caps;     /* STOP_STEP / STOP_FLAG: device [B] decoder-step cap of each row */
  const uint64_t* row_seeds;   /* FILL_MASKS_SEEDED: device [B] */
  int32_t fma_chain;           /* GEMM / STOP_STEP: into GemmArgs::fma_chain (launch_gemm keeps to gemm32 / gemm64 / gemm_big) */
  /* per-row step origin of streamed decoding (NULL: every row's step is the global step) */
  const int32_t* row_start;    /* PRENET / LSA_STEP / LSA_CTX / STOP_STEP / STOP_FLAG: device [B] global step row b started at; its
                                  step is the global step minus it.  PRENET reads x and the masks, LSA_STEP writes and LSA_CTX reads
                                  the scores at that step modulo `ring`; the stop kinds apply the rule at it, need row_done /
                                  row_caps and take flags = NULL */
  int32_t ring;                /* steps the per-step buffers hold (>= 1 with row_start) */
} mb_taco_debug_spec;
/* device workspace the spec needs (no kind needs scratch: a nominal 256 bytes), 0 for a spec mb_taco_debug refuses */
size_t mb_taco_debug_workspace_bytes(const mb_taco_debug_spec* spec);
/* enqueues the launch on `stream` (no synchronisation); writes one line into `report`: "kernel=K grid=X,Y block=T smem=S" */
int mb_taco_debug(const mb_taco_debug_spec* spec, void* workspace, size_t workspace_bytes, void* stream, char* report,
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
/* device workspace of mb_encoder_embed_rows for `rows` rows of at most max_len frames; 0 for a non-positive argument */
size_t mb_encoder_rows_workspace_bytes(const mb_encoder* h, int32_t rows, int32_t max_len);
/* SpeakerEncoder.forward on rows cut straight out of a ragged frame buffer (many utterances in one call):
 *   frames fp32 [n_frames][mel_n_channels] (device): e.g. the utterances' mels of mb_melspec_forward_ragged back to back
 *   row_start_host, row_len_host int32 [rows] (host): row r is frames [row_start[r], row_start[r] + row_len[r])
 *   embeds fp32 [rows][embedding_size] (device, out)
 * The LSTM runs to max_len = max row_len over inputs that are zero past each row's end; row r's embedding comes from the top
 * layer's hidden state at its own step row_len[r] - 1, which the LSTM being causal makes exactly the row alone.  Every launch
 * takes a route chosen without looking at the row count (tensor-core input projections at any rows * frames and tc_lstm_seq
 * steps; with MB_ENC_TC=0 the FP32 GEMMs of one fmaf chain per output; the final Linear always the latter), so a row's result
 * is bitwise the same whatever rows share the call.  MB_ERR_INVALID before anything is queued for an empty row or a row
 * outside [0, n_frames); the message names the row.  The row table is copied from pageable host memory into the workspace. */
int mb_encoder_embed_rows(mb_encoder* h, const float* frames, int64_t n_frames, const int32_t* row_start_host,
                          const int32_t* row_len_host, int32_t rows, float* embeds, void* workspace, size_t workspace_bytes,
                          void* stream);

/* ---------------------------------------------------------------------------------------------
 * Mel-spectrogram front-ends (SURVEY.md 8f rows N1 / N2)
 *   replaces  models/encoder/audio.py:53-65 (wav_to_mel_spectrogram: librosa.feature.melspectrogram, power, [frames][40])
 *             models/synthesizer/audio.py:59-65,115-121,156-206 (melspectrogram: preemphasis, librosa.stft,
 *             librosa.filters.mel, amp_to_db, symmetric normalisation to +-4)
 * ------------------------------------------------------------------------------------------- */
typedef struct mb_melspec_config {
  int32_t sample_rate;
  int32_t n_fft;          /* even, 16 .. 2048 (bin k at k sr / n_fft; odd n_fft is refused: librosa's grid for it
                             depends on the librosa version) */
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
/* device workspace of mb_melspec_forward_ragged for `batch` utterances (its utterance table); 0 when batch < 1 */
size_t mb_melspec_ragged_workspace_bytes(const mb_melspec* h, int32_t batch);
/* the mels of many utterances in one launch:
 *   wavs fp32: the utterances back to back (device), lengths_host[b] > 0 samples each (host)
 *   signal_lengths_host int32 [batch] (host) or NULL: utterance b is framed as a signal of signal_lengths_host[b] >=
 *     lengths_host[b] samples whose tail past lengths_host[b] is zero, bitwise as if the zeros were stored (np.pad); NULL:
 *     the stored lengths.  Reflect padding needs more than n_fft/2 signal samples.
 *   out fp32 (device): utterance b has F_b = 1 + signal_b / hop_length frames, stored from out + n_mels * (F_0 + .. + F_{b-1})
 *     as [F_b][n_mels] or [n_mels][F_b] (transpose_out)
 * Padding, pre-emphasis and the output layout use each utterance's own indices, so utterance b's frames are bitwise
 * mb_melspec_forward of it alone.  MB_ERR_INVALID before anything is queued for an empty or too short utterance; the message
 * names it.  The utterance table is copied from pageable host memory into the workspace. */
int mb_melspec_forward_ragged(mb_melspec* h, const float* wavs, const int32_t* lengths_host,
                              const int32_t* signal_lengths_host, int32_t batch, float* out, void* workspace,
                              size_t workspace_bytes, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Griffin-Lim inversion of normalised dB mel spectrograms (DESIGN.md section 4i; csrc/griffinlim.cu)
 *   replaces  models/synthesizer/audio.py:84-99 (inv_mel_spectrogram), :105-124 (_griffin_lim with librosa.stft / istft),
 *             :162-166 (_mel_to_linear), :177-206 (_db_to_amp, _denormalize), :25-28 (inv_preemphasis)
 * librosa's contract: centred frames (n_fft / 2 padding), periodic Hann window of win_length centred in n_fft, ISTFT by
 * overlap-add divided by the window sum-square where it exceeds FLT_MIN and trimmed to hop (T - 1) samples, angle(0) = 0,
 * the imaginary parts of the DC and Nyquist bins ignored by the inverse transform.
 * ------------------------------------------------------------------------------------------- */
typedef struct mb_griffinlim_config {
  int32_t n_fft;                /* 256, 512, 1024 or 2048 */
  int32_t hop_length;           /* 1 .. win_length */
  int32_t win_length;           /* 1 .. n_fft */
  int32_t n_mels;               /* 1 .. 1024 */
  int32_t pad_mode;             /* centred frames of the STFT: 0 = reflect, 1 = constant (zeros) */
  float power;                  /* S = max(1e-10, inv_mel_basis @ amp) ** power (hparams.power, 1.5) */
  double preemphasis;           /* 0: off; else out = lfilter([1], [1, -k], y), 0 < k with k^W < 2^-30 for W <= 4096 */
  int32_t signal_normalization; /* 1: _denormalize the input first */
  int32_t allow_clipping;       /* allow_clipping_in_normalization: clip to [-A, A] (symmetric) or [0, A] first */
  int32_t symmetric;            /* symmetric_mels */
  float max_abs_value;          /* A */
  float min_level_db, ref_level_db;
} mb_griffinlim_config;

typedef struct mb_griffinlim mb_griffinlim;

/* MB_ERR_INVALID, with a message, for a non-power-of-two or out-of-range n_fft, win_length > n_fft, hop_length >
 * win_length, and a pre-emphasis whose inverse filter needs a warm-up of more than 4096 samples */
int mb_griffinlim_create(const mb_griffinlim_config* cfg, mb_griffinlim** out);
void mb_griffinlim_destroy(mb_griffinlim* h);
size_t mb_griffinlim_arena_bytes(const mb_griffinlim* h);
int mb_griffinlim_set_arena(mb_griffinlim* h, void* arena, size_t bytes);
/* one tensor, "inv_mel_basis" [n_fft / 2 + 1][n_mels] (the caller's pseudo-inverse of the mel basis); finalize writes the
 * window and the FFT twiddles (computed on the host in float64 at create) into the arena and synchronises `stream` */
int mb_griffinlim_set_weight(mb_griffinlim* h, const char* name, const float* w, const int64_t* dims, int32_t ndim,
                             void* stream);
int mb_griffinlim_finalize(mb_griffinlim* h, void* stream);
/* frames_host int32 [batch] (host); 0 when batch < 1 or a length is < 1 */
size_t mb_griffinlim_workspace_bytes(const mb_griffinlim* h, int32_t batch, const int32_t* frames_host);
/* inv_mel_spectrogram for `batch` utterances of frames_host[b] frames in one sequence of 2 n_iters + 4 launches:
 *   mels fp32: one [n_mels][T_b] row-major block per utterance, back to back (device)
 *   uniforms float64: one [n_fft / 2 + 1][T_b] block per utterance, back to back (device), the initial phases exp(2 pi i u);
 *     or NULL and seeds_host uint64 [batch] (host): u drawn on the device from Philox keyed by (seed_b, bin, frame).
 *     Exactly one of the two is given.
 *   out fp32 [sum_b hop (T_b - 1)] (device)
 * Each utterance's output is bitwise what a batch of that utterance alone gives.  MB_ERR_INVALID before anything is queued
 * for n_iters < 0 and for an utterance too short for the pad mode (reflect: hop (T - 1) > n_fft / 2; constant: T >= 2);
 * the message names the utterance.  The row tables are copied from pageable host memory into the workspace. */
int mb_griffinlim_forward(mb_griffinlim* h, const float* mels, const int32_t* frames_host, int32_t batch,
                          const double* uniforms, const uint64_t* seeds_host, int32_t n_iters, float* out, void* workspace,
                          size_t workspace_bytes, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Log-MMSE speech enhancement (DESIGN.md section 4j; csrc/logmmse.cu)
 *   replaces  utils/logmmse.py:36-69 (profile_noise), :72-133 (denoise), as models/synthesizer/inference.py:145-159
 *             (load_preprocess_wav) calls them
 * The reference's contract: samples + DBL_EPSILON times the caller's window, zero-padded n_fft-point FFTs; the profile averages
 * |X| over the non-overlapping frames of the noise and squares it; the denoiser runs nframes = L // len2 - W // len2 frames
 * at hop len2 with the gain recursion of utils/logmmse.py, overlap-adds the first W samples of each Re(IFFT(hw X)) and
 * leaves the samples past nframes * len2 at zero.  All float64; the output is rounded once to fp32.
 * ------------------------------------------------------------------------------------------- */
typedef struct mb_logmmse_config {
  int32_t window_size; /* W: even, 2 .. n_fft (NoiseProfile.window_size, 320 at 16 kHz) */
  int32_t len1, len2;  /* both W / 2 */
  int32_t n_fft;       /* 2^a or 5 * 2^a in [64, 2048] (2 W in the reference) */
} mb_logmmse_config;

typedef struct mb_logmmse mb_logmmse;

/* MB_ERR_INVALID, with a message naming the field, for any other n_fft, W or len1 / len2 */
int mb_logmmse_create(const mb_logmmse_config* cfg, mb_logmmse** out);
void mb_logmmse_destroy(mb_logmmse* h);
/* the handle holds no checkpoint tensor: its arena is the FFT twiddles (float64, computed on the host at create), which
 * finalize writes and then synchronises `stream` */
size_t mb_logmmse_arena_bytes(const mb_logmmse* h);
int mb_logmmse_set_arena(mb_logmmse* h, void* arena, size_t bytes);
int mb_logmmse_finalize(mb_logmmse* h, void* stream);
/* lengths_host int32 [batch] (host); 0 when batch < 1 or a length is < 2 len2.  Also what mb_logmmse_profile needs for
 * the same lengths. */
size_t mb_logmmse_workspace_bytes(const mb_logmmse* h, int32_t batch, const int32_t* lengths_host);
/* profile_noise for `batch` noise signals in one launch:
 *   noise fp32: the signals back to back (device), lengths_host[b] >= W samples each (host)
 *   window float64 [W] (device): NoiseProfile.win
 *   noise_mu2 float64 [batch][n_fft] (device, out)
 * MB_ERR_INVALID before anything is queued for a signal shorter than W; the message names it. */
int mb_logmmse_profile(mb_logmmse* h, const float* noise, const int32_t* lengths_host, int32_t batch, const double* window,
                       double* noise_mu2, void* workspace, size_t workspace_bytes, void* stream);
/* denoise for `batch` utterances in one sequence of 4 launches:
 *   x fp32: the utterances back to back (device), lengths_host[b] >= 2 len2 samples each (host)
 *   window float64 [W], noise_mu2 float64 [batch][n_fft] (device): each utterance's NoiseProfile (bins 0 .. n_fft / 2 read)
 *   eta: the VAD threshold below which noise_mu2 is updated (0 disables the update)
 *   out fp32 [sum_b L_b] (device)
 *   vad_out float64 [sum_b nframes_b] (device) or NULL: each frame's VAD statistic
 * Each utterance's output is bitwise what a batch of that utterance alone gives.  MB_ERR_INVALID before anything is queued
 * for an utterance shorter than 2 len2 (the reference fails on it); the message names the utterance.  The row tables are
 * copied from pageable host memory into the workspace. */
int mb_logmmse_denoise(mb_logmmse* h, const float* x, const int32_t* lengths_host, int32_t batch, const double* window,
                       const double* noise_mu2, double eta, float* out, double* vad_out, void* workspace,
                       size_t workspace_bytes, void* stream);
/* E1(x) = expint(1, x) for x > 0, the device function the gains use: x, y float64 [n] (device) */
int mb_logmmse_exp1(const double* x, double* y, int64_t n, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Harvest F0 tracking (DESIGN.md section 4n; csrc/f0.cu)
 *   replaces  pyworld.harvest(wav, 16000, frame_period=10, f0_floor=80, f0_ceil=600), as utils/f0_utils.py:14-20
 *             (compute_f0) calls it
 * The contract is oracle/harvest_oracle.py: 16 kHz float64 input decimated by 2, 128 band-pass channels, events and
 * official candidates per 1 ms frame, refinement, FixStep1-4 and smoothing, then every 10th frame.  All float64.
 * ------------------------------------------------------------------------------------------- */
typedef struct mb_f0 mb_f0;

/* Optional outputs for tests, per 1 ms frame of every clip back to back (T_b = int(1000 L_b / 16000) + 1 frames); any
 * member may be NULL:
 *   raw_count int32 [sum T_b]: channels with a raw candidate
 *   official_count int32 [sum T_b]: official candidates of the frame itself
 *   refined, scores float64 [sum T_b][91]: slot s < 7 nc_b (nc_b the clip's largest official count) after refinement,
 *     before the unreliable-candidate removal; 0 in the other slots
 *   contour float64 [sum T_b]: after FixStep4, before smoothing */
typedef struct mb_f0_debug {
  int32_t* raw_count;
  int32_t* official_count;
  double* refined;
  double* scores;
  double* contour;
} mb_f0_debug;

int mb_f0_create(mb_f0** out);
void mb_f0_destroy(mb_f0* h);
/* the handle holds no checkpoint tensor: its arena is the channel table, the band-pass taps and the DFT twiddles (float64,
 * computed on the host at create), which finalize writes and then synchronises `stream` */
size_t mb_f0_arena_bytes(const mb_f0* h);
int mb_f0_set_arena(mb_f0* h, void* arena, size_t bytes);
int mb_f0_finalize(mb_f0* h, void* stream);
/* lengths_host int32 [batch] (host); 0 when batch < 1 or a length is outside 1 .. 2^28.  About 8 MB per second of audio. */
size_t mb_f0_workspace_bytes(const mb_f0* h, int32_t batch, const int32_t* lengths_host);
/* Harvest of `batch` clips in one sequence of five launches:
 *   x float64: the 16 kHz clips back to back (device), lengths_host[b] samples each (host)
 *   f0_out float64 [sum_b int(L_b / 160) + 1] (device): each clip's F0 every 10 ms, 0 where unvoiced
 * Each clip's outputs are bitwise what a batch of that clip alone gives.  MB_ERR_INVALID before anything is queued for an
 * empty clip or one longer than 2^28 samples; the message names the clip.  The clip table is copied from pageable host
 * memory into the workspace. */
int mb_f0_harvest(mb_f0* h, const double* x, const int32_t* lengths_host, int32_t batch, double* f0_out,
                  const mb_f0_debug* debug, void* workspace, size_t workspace_bytes, void* stream);

/* The shared Stockham FFT of Griffin-Lim and log-MMSE (csrc/mb_fft.cuh) on its own, for tests: y[r] = sum_j x[r][j]
 * exp(-+2 pi i j k / n) for each of `rows` rows of n complex points, unscaled in both directions, over the handles' twiddle
 * table.  x, y [rows][n] (device) of float2 (dtype 0) or double2 (dtype 1); inverse != 0 takes the + sign.  n is 2^a or 5 * 2^a
 * in [64, 2048]; MB_ERR_INVALID before anything is queued otherwise.  Synchronises the stream. */
int mb_fft_debug(const void* x, void* y, int32_t n, int32_t rows, int32_t dtype, int32_t inverse, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Polyphase resampling and per-clip levelling (DESIGN.md section 4k; csrc/resample.cu)
 *   replaces  scipy.signal.resample_poly(x, up, down) as synthesizer/audio_host.py load_wav and preprocess_wav call it
 *             (librosa.load's resampling in the reference), normalize_volume (models/encoder/audio.py:108-117) and the
 *             rescale of load_preprocess_wav (models/synthesizer/inference.py:145-150)
 * scipy's float32 contract, bitwise: the filter is firwin(20 max(up, down) + 1, 1 / max(up, down), ('kaiser', 5.0)) cast
 * to float32 and multiplied by up in float32 (designed by the caller, one per reduced ratio); output sample j is the sum,
 * over input samples in ascending order, of one rounded float32 multiply tap * x and one rounded float32 add, from zero;
 * ceil(n up / down) samples.  up == down == 1 is a copy.
 * ------------------------------------------------------------------------------------------- */
#define MB_RESAMPLE_F32 0 /* float32 samples */
#define MB_RESAMPLE_I16 1 /* int16 PCM, converted on the device as x / 32768.0f (exact, what load_wav does) */

typedef struct mb_resample mb_resample;

/* filter_smem_bytes: the largest polyphase table [up][ceil(taps / up)] (fp32) staged in shared memory per work item; larger
 * tables are read through L2.  < 0: the default (64 KB); at most 128 KB. */
int mb_resample_create(int32_t filter_smem_bytes, mb_resample** out);
void mb_resample_destroy(mb_resample* h);
/* register the filter of a reduced ratio (gcd(up, down) == 1, not 1 / 1): taps_host fp32 [20 max(up, down) + 1] (host),
 * already multiplied by up.  Returns its index (the same index for a ratio added before).  A new filter forgets the arena:
 * set_arena and finalize again.  MB_ERR_INVALID for a ratio whose tile would read more input than shared memory holds. */
int mb_resample_add_filter(mb_resample* h, int32_t up, int32_t down, const float* taps_host, int32_t n_taps, int32_t* index_out);
/* the polyphase tables of every filter added so far; 16-byte aligned */
size_t mb_resample_arena_bytes(const mb_resample* h);
int mb_resample_set_arena(mb_resample* h, void* arena, size_t bytes);
/* writes the tables into the arena and synchronises `stream` */
int mb_resample_finalize(mb_resample* h, void* stream);
/* 1: filter `index` is staged in shared memory, 0: read through L2, -1: no such filter (host only) */
int mb_resample_filter_in_smem(const mb_resample* h, int32_t index);
/* ceil(n up / down); -1 for a bad argument (host only) */
int64_t mb_resample_output_length(int32_t up, int32_t down, int64_t n);
/* the work items of a mb_resample_forward call with these clips (host only): tile0_host int32 [batch + 1] gets the first work
 * item of every clip and the number of work items, out_offsets_host int64 [batch + 1] the first output sample of every clip
 * and the output length.  MB_ERR_INVALID, naming the clip, for what forward refuses. */
int mb_resample_work_items(const mb_resample* h, const int32_t* lengths_host, const int32_t* filters_host, int32_t batch,
                           int32_t* tile0_host, int64_t* out_offsets_host);
/* device workspace of mb_resample_forward (its clip table); 0 when batch < 1 */
size_t mb_resample_workspace_bytes(const mb_resample* h, int32_t batch);
/* resample_poly of `batch` clips in one launch, one work item per (clip, tile of 512 output samples):
 *   x: the clips back to back (device, 16-byte aligned), dtype MB_RESAMPLE_F32 or MB_RESAMPLE_I16, lengths_host[b] >= 1
 *   filters_host int32 [batch] (host): the add_filter index of clip b's ratio, or -1 for a copy
 *   out fp32 (device): clip b's ceil(n_b up_b / down_b) samples after those of clips 0 .. b-1
 * Each clip's output is bitwise what a batch of that clip alone gives.  MB_ERR_INVALID before anything is queued for an
 * empty clip or an unknown filter; the message names the clip.  The clip table is copied from pageable host memory. */
int mb_resample_forward(mb_resample* h, const void* x, int32_t dtype, const int32_t* lengths_host, const int32_t* filters_host,
                        int32_t batch, float* out, void* workspace, size_t workspace_bytes, void* stream);
/* device workspace of the three levelling calls below (their clip table); 0 when batch < 1 */
size_t mb_resample_level_workspace_bytes(int32_t batch);
/* x fp32: `batch` clips back to back (device), lengths_host[b] >= 1 (host).  sumsq fp32 [batch] (device): the float32 sum of
 * x * x in numpy's pairwise order, bitwise np.add.reduce(x ** 2) (np.mean(x ** 2) is that sum / n, rounded once) */
int mb_resample_sumsq(const float* x, const int32_t* lengths_host, int32_t batch, float* sumsq, void* workspace,
                      size_t workspace_bytes, void* stream);
/* y = x * gains[b] (one rounded fp32 multiply; gains fp32 [batch], device); y may be x */
int mb_resample_scale(const float* x, const int32_t* lengths_host, int32_t batch, const float* gains, float* y, void* workspace,
                      size_t workspace_bytes, void* stream);
/* y = (x / max |x|) * peak per clip (two rounded fp32 operations); y may be x */
int mb_resample_rescale(const float* x, const int32_t* lengths_host, int32_t batch, float peak, float* y, void* workspace,
                        size_t workspace_bytes, void* stream);
/* The same three calls on float64 clips (the text-to-speech chain's levelling, gen_voice.py), same workspace:
 *   sumsq_f64    the float64 sum of x * x in numpy's pairwise order, bitwise np.add.reduce(x ** 2) on float64
 *   scale_f64    y = x * gains[b] (one rounded fp64 multiply; gains fp64 [batch], device); y may be x
 *   rescale_f64  y = (x / max |x|) * peak (two rounded fp64 operations); a NaN sample makes max |x| NaN, as np.abs(x).max()
 *                does, so the clip comes out all NaN; y may be x */
int mb_resample_sumsq_f64(const double* x, const int32_t* lengths_host, int32_t batch, double* sumsq, void* workspace,
                          size_t workspace_bytes, void* stream);
int mb_resample_scale_f64(const double* x, const int32_t* lengths_host, int32_t batch, const double* gains, double* y,
                          void* workspace, size_t workspace_bytes, void* stream);
int mb_resample_rescale_f64(const double* x, const int32_t* lengths_host, int32_t batch, double peak, double* y,
                            void* workspace, size_t workspace_bytes, void* stream);

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

/* mb_ppg2mel_inference with one dropout stream per row, so that a row's result does not depend on the batch around it:
 *   seeds uint64 [B] (device): row b draws its PreNet keep flags exactly as the only row of a B = 1 mb_ppg2mel_inference
 *     call with seed = seeds[b] (Philox keyed by step, row 0 and unit).  The table is copied into the workspace before
 *     the decoder runs (the workspace holds room for it: mb_ppg2mel_workspace_bytes counts B seeds); the captured decoder
 *     steps read it from there.
 * Every other argument, output and error is mb_ppg2mel_inference's; a NULL seed table is MB_ERR_INVALID. */
int mb_ppg2mel_inference_rows(mb_ppg2mel* h, const float* ppg, const float* lf0_uv, const float* spk,
                              const int32_t* lengths, int32_t batch, int32_t frames, const uint64_t* seeds, float* mel,
                              float* mel_post, float* align, float* stop, int32_t* steps_host, void* workspace,
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

/* ---------------------------------------------------------------------------------------------
 * VITS synthesizer: token ids -> waveform
 *   replaces  models/synthesizer/models/vits.py:389-527  Vits.{__init__,infer} (enc_p, emb_g, dp, flow, dec)
 *   driven by vits.ipynb: model.infer(x, x_lengths, sid=sid, noise_scale=.667, noise_scale_w=.8, length_scale=1, emo=emo)
 * Two calls, because the frame count T_y is known only after the durations: mb_vits_durations (text encoder, speaker
 * embedding, duration predictor, ceil(exp(logw) * mask * length_scale)), then - once the caller has read y_lengths back -
 * mb_vits_decode (prior expansion along the monotonic path, prior noise, reverse coupling flow, decoder).  FP32 kernels
 * everywhere but the decoder, which is an MB_GAN_VITS generator in `precision`.  Layout NCL; every T axis is padded to the
 * call's T_x / T_y, rows past x_lengths / y_lengths are masked as the reference masks them.
 * ------------------------------------------------------------------------------------------- */
typedef struct mb_vits_config {
  int32_t n_vocab, inter_channels, hidden_channels, filter_channels, n_heads, n_layers, kernel_size;
  int32_t resblock_type;         /* 1 = ResBlock1, 2 = ResBlock2 (vits_modules.py:180-249) */
  int32_t num_kernels;           /* len(resblock_kernel_sizes) <= 4 */
  int32_t resblock_kernel_sizes[4];
  int32_t num_dilations;
  int32_t resblock_dilation_sizes[4][4];
  int32_t num_upsamples;         /* <= 8 */
  int32_t upsample_rates[8];
  int32_t upsample_kernel_sizes[8];
  int32_t upsample_initial_channel;
  int32_t n_speakers;            /* 0: no speaker embedding; > 1: emb_g [n_speakers, gin_channels]; 1 is refused */
  int32_t gin_channels;          /* must be > 0 exactly when n_speakers > 1 */
  int32_t use_sdp;               /* 1: StochasticDurationPredictor, 0: DurationPredictor */
  int32_t precision;             /* MB_PREC_* of the decoder */
} mb_vits_config;

typedef struct mb_vits mb_vits;

/* MB_ERR_INVALID, with a message naming the field, for a config the kernels do not cover (odd kernel_size, hidden %
 * n_heads, inter_channels odd, head width > 256, the decoder constraints of MB_GAN_VITS) */
int mb_vits_create(const mb_vits_config* cfg, mb_vits** out);
void mb_vits_destroy(mb_vits* h);
size_t mb_vits_arena_bytes(const mb_vits* h);
int mb_vits_set_arena(mb_vits* h, void* arena, size_t bytes);
/* One tensor of Vits.state_dict() after weight-norm folding ("...weight_g" / "...weight_v" -> "...weight").  enc_q.*, the
 * discriminators, dp.post_* and dp.flows.1.* (the flow reverse inference drops) are accepted and ignored. */
int mb_vits_set_weight(mb_vits* h, const char* name, const float* w, const int64_t* dims, int32_t ndim, void* stream);
/* MB_ERR_STATE naming the first tensor never set; combines dec.conv_pre and dec.cond into the decoder's input layer */
int mb_vits_finalize(mb_vits* h, void* stream);
int32_t mb_vits_hop(const mb_vits* h);
/* largest T_x the attention kernel takes (its scores row lives in shared memory) */
int32_t mb_vits_max_tokens(void);

size_t mb_vits_durations_workspace_bytes(const mb_vits* h, int32_t batch, int32_t t_x);
/* x int32 [B, T_x] token ids, x_lengths int32 [B] in [1, T_x], sid int32 [B] (NULL without speakers), emo [B, 1024],
 * noise [B, 2, T_x] (the SDP's torch.randn draw, unscaled; ignored and may be NULL when use_sdp == 0).  Writes m_p and
 * logs_p [B, inter, T_x], w_ceil int32 [B, T_x] and y_lengths int32 [B] = max(1, sum w_ceil).  A token id or sid out of
 * range reads as id 0 (the host layer checks them). */
int mb_vits_durations(mb_vits* h, const int32_t* x, const int32_t* x_lengths, int32_t batch, int32_t t_x, const int32_t* sid,
                      const float* emo, const float* noise, float noise_scale_w, float length_scale, float* m_p, float* logs_p,
                      int32_t* w_ceil, int32_t* y_lengths, void* workspace, size_t workspace_bytes, void* stream);

size_t mb_vits_decode_workspace_bytes(const mb_vits* h, int32_t batch, int32_t t_x, int32_t t_y, int32_t t_dec);
/* m_p, logs_p, w_ceil, x_lengths and sid as mb_vits_durations took / wrote them; t_y >= max(y_lengths); eps [B, inter, T_y]
 * the prior noise (torch.randn_like of the expanded m_p).  t_dec <= t_y frames are decoded (Vits.infer's max_len):
 * wav [B, 1, t_dec * hop].  ragged == 0 decodes every row over all t_dec frames as the reference does (z * y_mask, no mask
 * inside the decoder); ragged != 0 masks the decoder at min(y_length, t_dec), so that each row is bitwise the row decoded
 * alone.  Optional outputs (NULL: not written): attn [B, 1, T_y, T_x], z_p / z / m_p_y / logs_p_y [B, inter, T_y]. */
int mb_vits_decode(mb_vits* h, const float* m_p, const float* logs_p, const int32_t* w_ceil, const int32_t* x_lengths,
                   const int32_t* sid, int32_t batch, int32_t t_x, int32_t t_y, const float* eps, float noise_scale, int32_t t_dec,
                   int32_t ragged, float* wav, float* attn, float* z_p, float* z, float* m_p_y, float* logs_p_y, void* workspace,
                   size_t workspace_bytes, void* stream);

/* One kernel stage of a finalized handle on its own weights, for tests against float64 references.  lengths int32 [B] masks
 * as the compute calls do.  Kinds:
 *   SPLINE   ConvFlow `index` (3 / 5 / 7) reverse: x = the DDSConv output h [B, hidden, T], x2 = z [B, 2, T]; y = z with
 *            channel c1 through the inverse spline that proj(h) parametrises, channel c0 kept, both masked
 *   ATTN     encoder layer `index`: x, x2, x3 = q, k, v [B, hidden, T]; y = attention output [B, hidden, T]
 *   WN       WN layer `sub` of coupling layer flow.flows.(2 * index): x = h [B, hidden, T], x2 = g [B, gin] or NULL;
 *            y = h after the residual update, y2 = the skip stream [B, hidden, T] (read unless sub == 0, then written)
 *   DDSCONV  DDSConv "dp.convs." (index 0) or "dp.flows.<index>.convs.": x [B, hidden, T] -> y
 *   DECODER  dec(x, g) on z = x [B, inter, T] unmasked, x2 = sid int32 [B] (multi-speaker); y = wav [B, 1, T * hop]
 *   CONV     one launch of the FP32 conv kernel through its host wrapper (MB_ERR_INVALID, nothing launched, for k > 7 or
 *            (k - 1) * dil > 14): y[b, co, t] = epi(bias[co] + bbias[b * bbs + co] + sum_{ci, j} w[co, ci, j] *
 *            x[b * xbs + ci * T + t + j * dil - pad]), x read as 0 outside [0, T) and, with in_mask, at t >= lengths[b];
 *            epi: relu, then mode (0 store, 1 y += v, 2 y -= v), then * mask with out_mask.  y's batch stride is ybs and
 *            its channel stride T.  lengths, bias and bbias may be NULL
 *   LAYERNORM y = res + act(LayerNorm_cin(x + x2) * w + bias) (* mask when lengths is given) over [B, cin, T]; x2 and
 *            res may be NULL, act = GELU when gelu != 0
 *   ENC_LAYER text-encoder layer `index` on x [B, hidden, T] -> y (attention, conv_o, LN 1, FFN, LN 2; the last layer
 *            masks its output)
 *   LOGW     the duration predictor's logw [B, 1, T] (before exp and ceil) on the encoder output x [B, hidden, T];
 *            x2 = sid int32 [B] (NULL: no g), x3 = the SDP's unscaled noise [B, 2, T]; y2 (nullable) receives what
 *            mb_vits_durations derives from it at length_scale: w_ceil int32 [B, T] followed by y_lengths int32 [B]
 *   COUPLING ResidualCouplingLayer flow.flows.(2 * index) in reverse on z = x [B, inter, T] -> y, masked at lengths;
 *            x2 = g [B, gin] or NULL (only with speakers) */
#define MB_VITS_DBG_SPLINE 0
#define MB_VITS_DBG_ATTN 1
#define MB_VITS_DBG_WN 2
#define MB_VITS_DBG_DDSCONV 3
#define MB_VITS_DBG_DECODER 4
#define MB_VITS_DBG_CONV 5
#define MB_VITS_DBG_LAYERNORM 6
#define MB_VITS_DBG_ENC_LAYER 7
#define MB_VITS_DBG_LOGW 8
#define MB_VITS_DBG_COUPLING 9
typedef struct mb_vits_debug_spec {
  int32_t kind, batch, frames, index, sub, c0, c1;
  const int32_t* lengths;
  const float* x;
  const float* x2;
  const float* x3;
  float* y;
  float* y2;
  /* CONV / LAYERNORM operands: w = weight or gamma, bias = bias or beta */
  const float* w;
  const float* bias;
  const float* bbias;
  const float* res;
  int64_t xbs, ybs;
  int32_t bbs, cin, cout, k, dil, pad, in_mask, out_mask, relu, mode, gelu;
  float noise_scale_w, length_scale; /* LOGW */
} mb_vits_debug_spec;
size_t mb_vits_debug_workspace_bytes(const mb_vits* h, const mb_vits_debug_spec* spec);
int mb_vits_debug(mb_vits* h, const mb_vits_debug_spec* spec, void* workspace, size_t workspace_bytes, void* stream);

/* ---- wav2vec2 emotion model (models/synthesizer/models/wav2emo.py EmotionExtractorModel, the model of extract_emo) ----------
 * Wav2Vec2Config fields as the caller parsed them.  create refuses what the kernels do not implement: feat_extract_norm
 * "group", do_stable_layer_norm False, activations other than "gelu", adapters, a head size other than 64, widths that are not
 * multiples of 64, conv layers 1.. with more than 5 taps, and positional-conv groups that are not a multiple of 64 wide. */
#define MB_EMO_NORM_LAYER 0           /* feat_extract_norm "layer"; MB_EMO_NORM_GROUP "group" (rejected) */
#define MB_EMO_NORM_GROUP 1
#define MB_EMO_ACT_GELU 0             /* feat_extract_activation / hidden_act "gelu"; MB_EMO_ACT_OTHER anything else (rejected) */
#define MB_EMO_ACT_OTHER 1
typedef struct mb_emo_config {
  int32_t hidden_size, num_hidden_layers, num_attention_heads, intermediate_size;
  int32_t num_conv_layers;                            /* len(conv_dim), 1..8 */
  int32_t conv_dim[8], conv_kernel[8], conv_stride[8];
  int32_t conv_bias;
  int32_t num_conv_pos_embeddings, num_conv_pos_embedding_groups;
  float layer_norm_eps;
  int32_t feat_extract_norm, do_stable_layer_norm, feat_extract_activation, hidden_act, add_adapter;
  int32_t num_labels;
} mb_emo_config;

typedef struct mb_emo mb_emo;

int mb_emo_create(const mb_emo_config* cfg, mb_emo** out);
void mb_emo_destroy(mb_emo* h);
size_t mb_emo_arena_bytes(const mb_emo* h);
int mb_emo_set_arena(mb_emo* h, void* arena, size_t bytes);
/* tensors of EmotionExtractorModel.state_dict() under their reference names, except the positional conv: its weight norm is
 * folded by the caller into "wav2vec2.encoder.pos_conv_embed.conv.weight" [hidden][hidden / groups][taps] (g v / ||v|| with
 * one norm per tap).  wav2vec2.masked_spec_embed is accepted and ignored.  finalize packs the tensor-core weight images. */
int mb_emo_set_weight(mb_emo* h, const char* name, const float* w, const int64_t* dims, int32_t ndim, void* stream);
int mb_emo_finalize(mb_emo* h, void* stream);
/* encoder frames of an n-sample clip: floor((n - k) / s) + 1 per conv layer; 0 when the clip is too short for one */
int32_t mb_emo_num_frames(const mb_emo* h, int32_t n_samples);
size_t mb_emo_workspace_bytes(const mb_emo* h, int32_t batch, int32_t n_samples_max);
/* EmotionExtractorModel.forward of 1..128 clips, each computed as its own B = 1 call (bitwise):
 *   wav fp32 (device): the clips' raw samples concatenated; n_samples int32 [B] (host), each with at least one frame
 *   emb fp32 [B][hidden]: the mean of the last hidden state over the clip's frames; logits fp32 [B][num_labels]
 *   normalize: 1 runs the feature extractor's zero-mean unit-variance normalisation (numpy's float32 order) on each clip
 *     first; 0 takes wav as the model's input_values
 *   normed fp32 like wav, or NULL (ignored unless normalize): the normalised input
 *   hidden fp32 [B][T_max][hidden], or NULL: the last hidden state, zero past each clip's frames,
 *     T_max = mb_emo_num_frames(h, max n_samples); the workspace is mb_emo_workspace_bytes(h, B, max n_samples) */
int mb_emo_forward(mb_emo* h, const float* wav, const int32_t* n_samples, int32_t batch, int32_t normalize, float* emb,
                   float* logits, float* normed, float* hidden, void* workspace, size_t workspace_bytes, void* stream);

/* test hook: ONE launch of an emotion-model kernel on caller-provided device tensors (no model handle), through the launch
 * helpers the forward uses.  lengths int32 [batch] (host): per clip, samples (NORM, CONV0) or valid frames of `frames`
 * (every other kind); rows [B][frames] are padded per clip.  Kinds:
 *   NORM     x: the clips' samples concatenated -> y like x, normalised
 *   CONV0    x: normalised samples concatenated, w [dim][1][kernel], bias [dim] or NULL, stride -> y [B][frames][dim]
 *   LN_ACT   x [B][frames][dim] -> y: LayerNorm (eps, gamma, beta) then act (0 none, 3 gelu); y may be x
 *   POSCONV  x [B][frames][dim], w [dim][dim / groups][kernel] (folded), bias [dim] -> y = x + gelu(conv) (packs w as finalize)
 *   ATTN     x = qkv [B][frames][3 dim], heads of 64 -> y = context [B][frames][dim]
 *   MEAN     x [B][frames][dim] -> y [B][dim]
 *   HEAD     x [B][dim], w [n_out][dim], bias [n_out], act (0 none, 1 tanh) -> y [B][n_out]
 * Rows past each clip's frames are written as zeros where the forward writes them (CONV0, LN_ACT, POSCONV, ATTN). */
#define MB_EMO_DBG_NORM 0
#define MB_EMO_DBG_CONV0 1
#define MB_EMO_DBG_LN_ACT 2
#define MB_EMO_DBG_POSCONV 3
#define MB_EMO_DBG_ATTN 4
#define MB_EMO_DBG_MEAN 5
#define MB_EMO_DBG_HEAD 6
typedef struct mb_emo_debug_spec {
  int32_t kind, batch, frames, dim, n_out, groups, kernel, stride, heads, act;
  float eps;
  const int32_t* lengths;
  const float* x;
  const float* w;
  const float* bias;
  const float* gamma;
  const float* beta;
  float* y;
} mb_emo_debug_spec;
size_t mb_emo_debug_workspace_bytes(const mb_emo_debug_spec* spec);
int mb_emo_debug(const mb_emo_debug_spec* spec, void* workspace, size_t workspace_bytes, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Text-to-speech chain (gen_voice.py): DESIGN.md section 4p
 * ------------------------------------------------------------------------------------------- */
/* device workspace of mb_tacotron_trim_frames (its row table); 0 when batch < 1 */
size_t mb_tacotron_trim_workspace_bytes(int32_t batch);
/* The trailing-silence trim of Tacotron rows (synthesizer/inference.py:135-138) in one launch:
 *   linear fp32 [batch][n_mels][frames] (device): a ragged chunk's postnet output, row b valid for row_frames_host[b] frames
 *   (host, 0 <= row_frames_host[b] <= frames)
 *   trimmed int32 [batch] (device): the largest t <= row_frames_host[b] for which max_c linear[b][c][t - 1] < threshold is
 *   false (0 when every frame is silent).  A frame holding a NaN is not silent.  Exact.
 * MB_ERR_INVALID before anything is queued for a row length out of range. */
int mb_tacotron_trim_frames(const float* linear, int32_t batch, int32_t n_mels, int32_t frames, const int32_t* row_frames_host,
                            float threshold, int32_t* trimmed, void* workspace, size_t workspace_bytes, void* stream);

/* One piece of a document: the slice src[start:end] of a vocoder row of src_len samples, with numpy's clamping
 * (start and end are cut to src_len; 0 <= start <= end), followed by `zeros` zeros. */
typedef struct mb_tts_piece {
  const float* src; /* device: the row's first sample (may be NULL when src_len is 0) */
  int64_t src_len;
  int64_t start, end;
  int32_t zeros;
  int32_t pad;
} mb_tts_piece;
/* offsets_host int64 [n_pieces + 1] (host): the first output sample of every piece of mb_tts_join and the total.
 * MB_ERR_INVALID for a malformed piece (the message names it). */
int mb_tts_join_plan(const mb_tts_piece* pieces_host, int32_t n_pieces, int64_t* offsets_host);
/* device workspace of mb_tts_join (its piece table); 0 when n_pieces < 1 */
size_t mb_tts_join_workspace_bytes(int32_t n_pieces);
/* gen_one_wav's break assembly (gen_voice.py:30-34) for every piece of pieces_host in one launch: out fp64 (device) receives
 * the pieces back to back at mb_tts_join_plan's offsets, each one's float32 samples widened exactly, then its zeros. */
int mb_tts_join(const mb_tts_piece* pieces_host, int32_t n_pieces, double* out, void* workspace, size_t workspace_bytes,
                void* stream);

#ifdef __cplusplus
}
#endif
#endif /* MOCKINGBIRD_B200_H */
