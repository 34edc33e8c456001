"""ctypes binding of libmockingbird_b200.so (the C ABI declared in include/mockingbird_b200.h).

There is no fallback: if the shared library cannot be loaded (and cannot be built with nvcc), or
a call returns a non-zero status, this module raises.  PyTorch is used by the host layer only for
device memory, streams and torch.distributed.
"""
from __future__ import annotations

import ctypes as C
from typing import Optional

from . import build as _build

MB_OK = 0
MB_GAN_HIFIGAN = 0
MB_GAN_FREGAN = 1
MB_GAN_HIFIGAN_INTERP = 2  # 24 kHz HiFi-GAN: nearest upsample + Conv1d per stage (hifigan/models.py:107-118)
MB_PREC_FP32 = 0
MB_PREC_F16TC = 1
MB_PREC_F16X3 = 2

PRECISIONS = {"fp32": MB_PREC_FP32, "f16tc": MB_PREC_F16TC, "f16x3": MB_PREC_F16X3}


class MbError(RuntimeError):
    pass


class GanConfig(C.Structure):
    _fields_ = [
        ("kind", C.c_int32),
        ("num_mels", C.c_int32),
        ("upsample_initial_channel", C.c_int32),
        ("num_upsamples", C.c_int32),
        ("upsample_rates", C.c_int32 * 8),
        ("upsample_kernel_sizes", C.c_int32 * 8),
        ("num_kernels", C.c_int32),
        ("resblock_kernel_sizes", C.c_int32 * 4),
        ("num_dilations", C.c_int32),
        ("resblock_dilation_sizes", (C.c_int32 * 4) * 4),
        ("resblock_type", C.c_int32),
        ("fregan_top_k", C.c_int32),
        ("precision", C.c_int32),
    ]


class GanDebugSpec(C.Structure):
    _fields_ = [
        ("layer_index", C.c_int32),
        ("pair", C.c_int32),
        ("mode", C.c_int32),
        ("div", C.c_float),
        ("red_add", C.c_int32),
        ("res_kind", C.c_int32),
        ("res_slope", C.c_float),
        ("out16", C.c_int32),
        ("out_slope", C.c_float),
        ("batch", C.c_int32),
        ("frames_in", C.c_int32),
        ("x", C.c_void_p),
        ("residual", C.c_void_p),
        ("lengths", C.c_void_p),
        ("y", C.c_void_p),
        ("y16", C.c_void_p),
    ]


MB_TACO_TC_SKINNY_PLAIN = 0
MB_TACO_TC_SKINNY_LSTM = 1
MB_TACO_TC_GRU = 2
MB_TACO_TC_LSTM_SEQ = 3
MB_TACO_TC_BIG = 4


class TacoTcDebugSpec(C.Structure):
    _fields_ = [
        ("kind", C.c_int32), ("M", C.c_int32), ("N", C.c_int32), ("H", C.c_int32), ("K0", C.c_int32), ("K1", C.c_int32),
        ("w", C.c_void_p * 2), ("b", C.c_void_p * 2), ("ldw", C.c_int32), ("nseg", C.c_int32), ("T", C.c_int32),
        ("x", C.c_void_p * 5), ("ldx", C.c_int32 * 5), ("shift", C.c_int32 * 5), ("w_off", C.c_int32 * 5),
        ("w_stride", C.c_int32 * 5), ("kb0", C.c_int32), ("kb_count", C.c_int32), ("pre", C.c_void_p), ("ldpre", C.c_int32),
        ("step_ptr", C.c_void_p), ("step_j", C.c_int32), ("y_step", C.c_int64), ("y", C.c_void_p), ("ldy", C.c_int32),
        ("c", C.c_void_p), ("h", C.c_void_p), ("xres", C.c_void_p), ("gi", C.c_void_p * 2), ("ldgi", C.c_int32),
        ("hst", C.c_void_p * 2), ("out", C.c_void_p * 2), ("ldout", C.c_int32), ("ndir", C.c_int32),
        ("s_hi", C.c_void_p * 2), ("s_lo", C.c_void_p * 2), ("s_k0", C.c_int32 * 2), ("nxt_hi", C.c_void_p * 2),
        ("nxt_lo", C.c_void_p * 2), ("act", C.c_int32), ("bn_scale", C.c_void_p), ("bn_shift", C.c_void_p),
        ("res", C.c_void_p), ("ldres", C.c_int32), ("compact", C.c_int32), ("cluster", C.c_int32), ("pdl", C.c_int32),
        ("a_tiles", C.c_void_p), ("w_tiles", C.c_void_p),
    ]


MB_PPGX_DBG_FRONTEND = 0
MB_PPGX_DBG_MVN = 1
MB_PPGX_DBG_CONV0 = 2
MB_PPGX_DBG_CONV2D_TC = 3
MB_PPGX_DBG_LN_TILES = 4
MB_PPGX_DBG_ACT_TILES = 5
MB_PPGX_DBG_LN_ROWS = 6
MB_PPGX_DBG_DW = 7
MB_PPGX_DBG_ATTN = 8


class PpgxDebugSpec(C.Structure):
    _fields_ = [
        ("kind", C.c_int32), ("B", C.c_int32), ("T", C.c_int32), ("len", C.c_void_p), ("len2", C.c_void_p),
        ("n_max", C.c_int32), ("n_fft", C.c_int32), ("win_length", C.c_int32), ("hop_length", C.c_int32), ("F", C.c_int32),
        ("C", C.c_int32), ("N", C.c_int32), ("k", C.c_int32), ("stride", C.c_int32), ("pad", C.c_int32), ("M", C.c_int32),
        ("D", C.c_int32), ("ld", C.c_int32), ("rows_total", C.c_int32), ("act", C.c_int32), ("flags", C.c_int32),
        ("H", C.c_int32), ("dk", C.c_int32), ("ldp", C.c_int32), ("rel", C.c_int32), ("x", C.c_void_p), ("x_hi", C.c_void_p),
        ("x_lo", C.c_void_p), ("w", C.c_void_p), ("bias", C.c_void_p), ("bn", C.c_void_p * 4), ("P", C.c_void_p),
        ("pu", C.c_void_p), ("pv", C.c_void_p), ("y", C.c_void_p), ("y_hi", C.c_void_p), ("y_lo", C.c_void_p),
    ]


class WaveRNNConfig(C.Structure):
    _fields_ = [
        ("rnn_dims", C.c_int32),
        ("fc_dims", C.c_int32),
        ("bits", C.c_int32),
        ("pad", C.c_int32),
        ("num_upsample", C.c_int32),
        ("upsample_factors", C.c_int32 * 4),
        ("feat_dims", C.c_int32),
        ("compute_dims", C.c_int32),
        ("res_out_dims", C.c_int32),
        ("res_blocks", C.c_int32),
    ]


class TacotronConfig(C.Structure):
    _fields_ = [(n, C.c_int32) for n in (
        "num_chars", "embed_dims", "encoder_dims", "decoder_dims", "n_mels", "postnet_dims", "encoder_K", "lstm_dims",
        "postnet_K", "num_highways", "speaker_embedding_size", "gst_E", "gst_tokens", "gst_heads", "max_r")]


class EncoderConfig(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("mel_n_channels", "hidden_size", "num_layers", "embedding_size")]


class Ppg2MelConfig(C.Structure):
    _fields_ = [("bottle_neck_feature_dim", C.c_int32), ("spk_embed_dim", C.c_int32), ("encoder_dim", C.c_int32),
                ("encoder_downsample_rates", C.c_int32 * 2), ("attention_rnn_dim", C.c_int32),
                ("decoder_rnn_dim", C.c_int32), ("num_decoder_rnn_layer", C.c_int32), ("concat_context_to_last", C.c_int32),
                ("prenet_dims", C.c_int32 * 2), ("num_mixtures", C.c_int32), ("frames_per_step", C.c_int32),
                ("num_mels", C.c_int32)]


class PpgxConfig(C.Structure):
    _fields_ = [(n, C.c_int32) for n in (
        "n_fft", "win_length", "hop_length", "n_mels", "kaldi_padding_mode", "downsample_rate", "norm_means", "norm_vars",
        "attention_dim", "attention_heads", "linear_units", "num_blocks", "input_layer", "no_subsample", "subsample_by_2",
        "normalize_before", "concat_after", "positionwise_layer_type", "macaron_style", "pos_enc_layer_type",
        "selfattention_layer_type", "activation_type", "use_cnn_module", "cnn_module_kernel")]


class MelSpecConfig(C.Structure):
    _fields_ = [("sample_rate", C.c_int32), ("n_fft", C.c_int32), ("hop_length", C.c_int32), ("win_length", C.c_int32),
                ("n_mels", C.c_int32), ("fmin", C.c_float), ("fmax", C.c_float), ("pad_mode", C.c_int32),
                ("preemphasis", C.c_float), ("power", C.c_int32), ("to_db", C.c_int32), ("min_level_db", C.c_float),
                ("ref_level_db", C.c_float), ("normalize", C.c_int32), ("max_abs_value", C.c_float),
                ("symmetric", C.c_int32), ("transpose_out", C.c_int32)]


# name -> (restype, argtypes); every symbol include/mockingbird_b200.h declares
SIGNATURES = {
    "mb_last_error": (C.c_char_p, []),
    "mb_version": (C.c_char_p, []),
    "mb_launch_count": (C.c_uint64, []),
    "mb_gan_create": (C.c_int, [C.POINTER(GanConfig), C.POINTER(C.c_void_p)]),
    "mb_gan_destroy": (None, [C.c_void_p]),
    "mb_gan_arena_bytes": (C.c_size_t, [C.c_void_p]),
    "mb_gan_set_arena": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t]),
    "mb_gan_set_weight": (C.c_int, [C.c_void_p, C.c_char_p, C.c_void_p, C.POINTER(C.c_int64), C.c_int32,
                                    C.c_void_p]),
    "mb_gan_finalize": (C.c_int, [C.c_void_p]),
    "mb_gan_hop": (C.c_int32, [C.c_void_p]),
    "mb_gan_workspace_bytes": (C.c_size_t, [C.c_void_p, C.c_int32, C.c_int32]),
    "mb_gan_forward": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p,
                                 C.c_void_p, C.c_size_t, C.c_void_p]),
    "mb_gan_forward_profiled": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p,
                                          C.c_void_p, C.c_size_t, C.c_void_p, C.POINTER(C.c_float)]),
    "mb_gan_layer_work": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.POINTER(C.c_double),
                                    C.POINTER(C.c_double)]),
    "mb_gan_debug_layer": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32,
                                     C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "mb_gan_num_layers": (C.c_int32, [C.c_void_p]),
    "mb_gan_layer_info": (C.c_int, [C.c_void_p, C.c_int32, C.c_char_p, C.c_size_t]),
    "mb_gan_tc_plan_info": (C.c_int, [C.c_void_p, C.c_int32, C.c_char_p, C.c_size_t]),
    "mb_gan_debug_launch": (C.c_int, [C.c_void_p, C.POINTER(GanDebugSpec), C.c_void_p, C.c_size_t, C.c_void_p, C.c_char_p,
                                      C.c_size_t]),
    "mb_wavernn_create": (C.c_int, [C.POINTER(WaveRNNConfig), C.POINTER(C.c_void_p)]),
    "mb_wavernn_destroy": (None, [C.c_void_p]),
    "mb_wavernn_arena_bytes": (C.c_size_t, [C.c_void_p]),
    "mb_wavernn_set_arena": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t]),
    "mb_wavernn_set_weight": (C.c_int, [C.c_void_p, C.c_char_p, C.c_void_p, C.POINTER(C.c_int64), C.c_int32,
                                        C.c_void_p]),
    "mb_wavernn_finalize": (C.c_int, [C.c_void_p, C.c_void_p]),
    "mb_wavernn_workspace_bytes": (C.c_size_t, [C.c_void_p, C.c_int32, C.c_int32, C.c_int32]),
    "mb_wavernn_condition": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_size_t, C.c_void_p]),
    "mb_wavernn_generate": (C.c_int, [C.c_void_p, C.POINTER(C.c_int32), C.c_int32, C.c_int32, C.c_int32,
                                      C.c_int32, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_size_t,
                                      C.c_void_p]),
    "mb_wavernn_generate_rows": (C.c_int, [C.c_void_p, C.POINTER(C.c_int32), C.c_int32, C.c_int32, C.c_int32,
                                           C.c_int32, C.c_void_p, C.c_int32, C.c_int32, C.c_uint64, C.c_void_p, C.c_void_p,
                                           C.c_size_t, C.c_void_p]),
    "mb_wavernn_postprocess_workspace_bytes": (C.c_size_t, [C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32]),
    "mb_wavernn_postprocess": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                         C.c_double, C.c_int64, C.c_int32, C.c_void_p, C.POINTER(C.c_int64), C.c_void_p, C.c_size_t,
                                         C.c_void_p]),
    "mb_wavernn_last_logits": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p]),
    "mb_monotonic_path": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p]),
    "mb_deepmind_create": (C.c_int, [C.c_int32, C.c_int32, C.POINTER(C.c_void_p)]),
    "mb_deepmind_destroy": (None, [C.c_void_p]),
    "mb_deepmind_arena_bytes": (C.c_size_t, [C.c_void_p]),
    "mb_deepmind_set_arena": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t]),
    "mb_deepmind_set_weight": (C.c_int, [C.c_void_p, C.c_char_p, C.c_void_p, C.POINTER(C.c_int64), C.c_int32, C.c_void_p]),
    "mb_deepmind_finalize": (C.c_int, [C.c_void_p, C.c_void_p]),
    "mb_deepmind_workspace_bytes": (C.c_size_t, [C.c_void_p]),
    "mb_deepmind_generate": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p,
                                       C.c_void_p, C.c_size_t, C.c_void_p]),
    "mb_mtstream_create": (C.c_int, [C.c_uint64, C.c_int32, C.POINTER(C.c_void_p)]),
    "mb_mtstream_destroy": (None, [C.c_void_p]),
    "mb_mtstream_begin": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_uint64, C.c_uint64]),
    "mb_mtstream_next": (C.c_int, [C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p]),
    "mb_mtstream_consumed": (C.c_int, [C.c_void_p, C.c_void_p]),
    "mb_mtstream_finish": (C.c_int, [C.c_void_p, C.c_void_p, C.POINTER(C.c_int32), C.POINTER(C.c_int32)]),
    "mb_mt19937_fill": (C.c_int, [C.c_void_p, C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.c_void_p, C.c_uint64]),
    "mb_mt_to_exp": (C.c_int, [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p]),
    "mb_tacotron_create": (C.c_int, [C.POINTER(TacotronConfig), C.POINTER(C.c_void_p)]),
    "mb_tacotron_destroy": (None, [C.c_void_p]),
    "mb_tacotron_arena_bytes": (C.c_size_t, [C.c_void_p]),
    "mb_tacotron_set_arena": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t]),
    "mb_tacotron_set_weight": (C.c_int, [C.c_void_p, C.c_char_p, C.c_void_p, C.POINTER(C.c_int64), C.c_int32,
                                         C.c_void_p]),
    "mb_tacotron_finalize": (C.c_int, [C.c_void_p, C.c_void_p]),
    "mb_tacotron_workspace_bytes": (C.c_size_t, [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32]),
    "mb_tacotron_generate": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                       C.c_int32, C.c_float, C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p,
                                       C.c_void_p, C.POINTER(C.c_int32), C.c_void_p, C.c_size_t, C.c_void_p]),
    "mb_taco_tc_debug_workspace_bytes": (C.c_size_t, [C.POINTER(TacoTcDebugSpec)]),
    "mb_taco_tc_debug": (C.c_int, [C.POINTER(TacoTcDebugSpec), C.c_void_p, C.c_size_t, C.c_void_p, C.c_char_p, C.c_size_t]),
    "mb_encoder_create": (C.c_int, [C.POINTER(EncoderConfig), C.POINTER(C.c_void_p)]),
    "mb_encoder_destroy": (None, [C.c_void_p]),
    "mb_encoder_arena_bytes": (C.c_size_t, [C.c_void_p]),
    "mb_encoder_set_arena": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t]),
    "mb_encoder_set_weight": (C.c_int, [C.c_void_p, C.c_char_p, C.c_void_p, C.POINTER(C.c_int64), C.c_int32,
                                        C.c_void_p]),
    "mb_encoder_finalize": (C.c_int, [C.c_void_p, C.c_void_p]),
    "mb_encoder_workspace_bytes": (C.c_size_t, [C.c_void_p, C.c_int32, C.c_int32]),
    "mb_encoder_embed_frames": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p,
                                          C.c_size_t, C.c_void_p]),
    "mb_encoder_reduce_partials": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p]),
    "mb_melspec_create": (C.c_int, [C.POINTER(MelSpecConfig), C.POINTER(C.c_void_p)]),
    "mb_melspec_destroy": (None, [C.c_void_p]),
    "mb_melspec_arena_bytes": (C.c_size_t, [C.c_void_p]),
    "mb_melspec_set_arena": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "mb_melspec_num_frames": (C.c_int32, [C.c_void_p, C.c_int32]),
    "mb_melspec_forward": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p]),
    "mb_ppg2mel_create": (C.c_int, [C.POINTER(Ppg2MelConfig), C.POINTER(C.c_void_p)]),
    "mb_ppg2mel_destroy": (None, [C.c_void_p]),
    "mb_ppg2mel_arena_bytes": (C.c_size_t, [C.c_void_p]),
    "mb_ppg2mel_set_arena": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t]),
    "mb_ppg2mel_set_weight": (C.c_int, [C.c_void_p, C.c_char_p, C.c_void_p, C.POINTER(C.c_int64), C.c_int32, C.c_void_p]),
    "mb_ppg2mel_finalize": (C.c_int, [C.c_void_p, C.c_void_p]),
    "mb_ppg2mel_workspace_bytes": (C.c_size_t, [C.c_void_p, C.c_int32, C.c_int32]),
    "mb_ppg2mel_inference": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_int32), C.c_int32,
                                       C.c_int32, C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p,
                                       C.c_void_p, C.POINTER(C.c_int32), C.c_void_p, C.c_size_t, C.c_void_p]),
    "mb_ppgx_create": (C.c_int, [C.POINTER(PpgxConfig), C.POINTER(C.c_void_p)]),
    "mb_ppgx_destroy": (None, [C.c_void_p]),
    "mb_ppgx_arena_bytes": (C.c_size_t, [C.c_void_p]),
    "mb_ppgx_set_arena": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t]),
    "mb_ppgx_set_weight": (C.c_int, [C.c_void_p, C.c_char_p, C.c_void_p, C.POINTER(C.c_int64), C.c_int32, C.c_void_p]),
    "mb_ppgx_finalize": (C.c_int, [C.c_void_p, C.c_void_p]),
    "mb_ppgx_num_frames": (C.c_int32, [C.c_void_p, C.c_int32]),
    "mb_ppgx_workspace_bytes": (C.c_size_t, [C.c_void_p, C.c_int32, C.c_int32]),
    "mb_ppgx_forward": (C.c_int, [C.c_void_p, C.c_void_p, C.POINTER(C.c_int32), C.c_int32, C.c_int32, C.c_int32, C.c_void_p,
                                  C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "mb_ppgx_debug_workspace_bytes": (C.c_size_t, [C.POINTER(PpgxDebugSpec)]),
    "mb_ppgx_debug": (C.c_int, [C.POINTER(PpgxDebugSpec), C.c_void_p, C.c_size_t, C.c_void_p, C.c_char_p, C.c_size_t]),
}

_lib: Optional[C.CDLL] = None


def lib() -> C.CDLL:
    """Load (building first if stale and nvcc is present) the shared library; raise if impossible."""
    global _lib
    if _lib is not None:
        return _lib
    path = _build.LIB_PATH
    if not _build.is_fresh():
        if _build.find_nvcc() is not None:
            path = _build.build()
        elif not path.is_file():
            raise MbError(f"{path} is missing and nvcc is not available: the CUDA extension is required "
                          "(mockingbird_b200 has no CPU fallback)")
    try:
        handle = C.CDLL(str(path))
    except OSError as e:  # pragma: no cover
        raise MbError(f"cannot load {path}: {e} (mockingbird_b200 has no CPU fallback)") from e
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(handle, name)  # AttributeError if the library lacks a declared symbol
        fn.restype = res
        fn.argtypes = args
    _lib = handle
    return handle


def check(status: int) -> None:
    if status != MB_OK:
        msg = lib().mb_last_error()
        raise MbError(f"mockingbird_b200 error {status}: {msg.decode() if msg else '?'}")


def require_cuda():
    import torch

    if not torch.cuda.is_available():
        raise MbError("mockingbird_b200 needs a CUDA device (sm_90a); there is no CPU fallback")
    return torch.device("cuda", torch.cuda.current_device())


def upload_weights(model: str, handle, weights, device, align: int = 256):
    """The weight protocol of a model handle: a zeroed arena of mb_<model>_arena_bytes aligned to `align`, set_arena,
    set_weight for every tensor of `weights` (name -> tensor, already filtered to what the model takes), finalize, then a
    synchronise.  Returns the arena as one uint8 device tensor (what multi-GPU start-up broadcasts)."""
    import torch

    L = lib()
    nbytes = int(getattr(L, f"mb_{model}_arena_bytes")(handle))
    with torch.cuda.device(device):
        arena = torch.zeros(nbytes + align, dtype=torch.uint8, device=device)
        base = (arena.data_ptr() + align - 1) // align * align
        check(getattr(L, f"mb_{model}_set_arena")(handle, C.c_void_p(base), nbytes))
        stream = torch.cuda.current_stream(device)
        sp = C.c_void_p(stream.cuda_stream)
        keep = []  # the copies are asynchronous: the converted tensors live until the synchronise
        for name, t in weights.items():
            d = t.to(device=device, dtype=torch.float32).contiguous()
            keep.append(d)
            dims = (C.c_int64 * max(1, d.dim()))(*d.shape)
            check(getattr(L, f"mb_{model}_set_weight")(handle, name.encode(), C.c_void_p(d.data_ptr()), dims, d.dim(), sp))
        finalize = getattr(L, f"mb_{model}_finalize")
        # mb_gan_finalize only checks that every tensor was set (the GAN packs in set_weight): it takes no stream
        check(finalize(handle) if len(finalize.argtypes) == 1 else finalize(handle, sp))
        stream.synchronize()
    return arena
