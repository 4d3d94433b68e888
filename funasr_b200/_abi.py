"""ctypes mirror of include/funasr_b200.h and loader of the in-tree CUDA library.

The product path has NO fallback: if ``libfunasr_b200.so`` is missing or a call fails, an exception is raised.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libfunasr_b200.so")

FA_OK = 0
GEMM_F32_SIMT, GEMM_F16X1, GEMM_F16X3, GEMM_F16X6 = 0, 1, 3, 6
GEMM_MODES = {"fp32": GEMM_F32_SIMT, "fp16": GEMM_F16X1, "fp16x3": GEMM_F16X3, "fp16x6": GEMM_F16X6}

c_f32p = C.POINTER(C.c_float)
c_i32p = C.POINTER(C.c_int32)


class FaLinear(C.Structure):
    _fields_ = [("w", C.c_void_p), ("b", C.c_void_p), ("w_planes", C.c_void_p),
                ("out_f", C.c_int32), ("in_f", C.c_int32), ("in_pad", C.c_int32), ("_pad", C.c_int32)]


class FaNorm(C.Structure):
    _fields_ = [("g", C.c_void_p), ("b", C.c_void_p), ("n", C.c_int32), ("eps", C.c_float)]


class FaEncLayer(C.Structure):
    _fields_ = [("norm1", FaNorm), ("qkv", FaLinear), ("fsmn_w", C.c_void_p), ("out", FaLinear),
                ("norm2", FaNorm), ("w1", FaLinear), ("w2", FaLinear)]


class FaEncoder(C.Structure):
    _fields_ = [("layers", C.POINTER(FaEncLayer)), ("n_layers", C.c_int32), ("heads", C.c_int32),
                ("fsmn_k", C.c_int32), ("_pad", C.c_int32), ("after_norm", FaNorm),
                ("pe_inv_timescales", C.c_void_p)]


class FaPredictor(C.Structure):
    _fields_ = [("conv", FaLinear), ("out_w", C.c_void_p), ("out_b", C.c_void_p), ("threshold", C.c_float),
                ("tail_threshold", C.c_float), ("smooth_factor", C.c_float), ("noise_threshold", C.c_float),
                ("cif_variant", C.c_int32), ("_pad", C.c_int32)]


class FaDecLayer(C.Structure):
    _fields_ = [("norm1", FaNorm), ("ffn_w1", FaLinear), ("ffn_norm", FaNorm), ("ffn_w2", FaLinear),
                ("norm2", FaNorm), ("fsmn_w", C.c_void_p), ("norm3", FaNorm), ("q", FaLinear), ("kv", FaLinear),
                ("out", FaLinear)]


class FaDecoder(C.Structure):
    _fields_ = [("layers", C.POINTER(FaDecLayer)), ("n_layers", C.c_int32), ("heads", C.c_int32),
                ("fsmn_k", C.c_int32), ("vocab", C.c_int32), ("last", FaDecLayer), ("after_norm", FaNorm),
                ("output", FaLinear), ("has_bias", C.c_int32), ("n_hotwords", C.c_int32), ("bias_last", FaDecLayer),
                ("bias_norm3", FaNorm), ("bias_q", FaLinear), ("bias_kv", FaLinear), ("bias_out", FaLinear),
                ("bias_output", FaLinear), ("hw_embed", C.c_void_p), ("hw_lens", C.c_void_p), ("clas_scale", C.c_float),
                ("_pad2", C.c_int32)]


class FaTimestampHead(C.Structure):
    _fields_ = [("upsample", FaLinear), ("blstm_ih", FaLinear), ("w_hh_fwd", C.c_void_p), ("w_hh_bwd", C.c_void_p), ("out2_w", C.c_void_p),
                ("out2_b", C.c_void_p), ("up_times", C.c_int32), ("smooth2", C.c_float), ("noise2", C.c_float), ("threshold", C.c_float)]


class FaHotwordEncoder(C.Structure):
    _fields_ = [("embed", C.c_void_p), ("vocab", C.c_int32), ("n_layers", C.c_int32), ("ih", C.POINTER(FaLinear)), ("hh", C.POINTER(FaLinear))]


class FaVadLayer(C.Structure):
    _fields_ = [("lin", FaLinear), ("conv_w", C.c_void_p), ("affine", FaLinear)]


class FaVadEncoder(C.Structure):
    _fields_ = [("in1", FaLinear), ("in2", FaLinear), ("layers", C.POINTER(FaVadLayer)), ("n_layers", C.c_int32), ("lorder", C.c_int32),
                ("out1", FaLinear), ("out2", FaLinear), ("sil_ids", C.c_int32 * 4), ("n_sil", C.c_int32), ("_pad", C.c_int32)]


class FaVadOptions(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("sample_rate", "detect_mode", "max_end_silence_time", "max_start_silence_time", "window_size_ms",
                                         "sil_to_speech_time_thres", "speech_to_sil_time_thres", "do_extend", "lookback_time_start_point",
                                         "lookahead_time_end_point", "max_single_segment_time", "noise_frame_num_used_for_snr", "frame_in_ms",
                                         "frame_length_ms")] + \
               [(n, C.c_double) for n in ("speech_2_noise_ratio", "snr_thres", "decibel_thres", "speech_noise_thres", "fe_prior_thres")]


class FaVadRunOptions(C.Structure):
    _fields_ = [("dynamic_silence", C.c_int32), ("max_end_silence_time", C.c_int32), ("speech_noise_thres", C.c_double)]


class FaLongAudioOptions(C.Structure):
    _fields_ = [("batch_size_s", C.c_int32), ("batch_size_threshold_s", C.c_int32), ("merge_vad", C.c_int32), ("merge_length_s", C.c_int32),
                ("vad", FaVadRunOptions)]


class FaAudioFormat(C.Structure):
    _fields_ = [("sample_format", C.c_int32), ("channels", C.c_int32), ("sample_rate", C.c_int32), ("resampler", C.c_int32)]


RESAMPLE_LOADER, RESAMPLE_RUNTIME = 0, 1
RESAMPLERS = {"loader": RESAMPLE_LOADER, "runtime": RESAMPLE_RUNTIME}


class FaIngestTable(C.Structure):
    _fields_ = [("mode", C.c_int32), ("in_unit", C.c_int32), ("out_unit", C.c_int32), ("width", C.c_int32), ("taps", C.c_int32),
                ("_pad", C.c_int32), ("weights", C.c_void_p), ("first", C.c_void_p), ("n_taps", C.c_void_p)]


class FaCamConv2d(C.Structure):
    _fields_ = [("w", C.c_void_p), ("b", C.c_void_p), ("c_in", C.c_int32), ("c_out", C.c_int32), ("ksize", C.c_int32), ("stride_f", C.c_int32)]


class FaCamLayer(C.Structure):
    _fields_ = [("bn1_scale", C.c_void_p), ("bn1_shift", C.c_void_p), ("linear1", FaLinear), ("local_w", C.c_void_p), ("w1", C.c_void_p),
                ("b1", C.c_void_p), ("w2", C.c_void_p), ("b2", C.c_void_p)]


class FaCamTransit(C.Structure):
    _fields_ = [("scale", C.c_void_p), ("shift", C.c_void_p), ("linear", FaLinear)]


class FaCampplus(C.Structure):
    _fields_ = [("fcm", FaCamConv2d * 12), ("tdnn", FaLinear), ("layers", C.POINTER(FaCamLayer)), ("n_layers", C.c_int32 * 3),
                ("dilation", C.c_int32 * 3), ("transit", FaCamTransit * 3), ("out_scale", C.c_void_p), ("out_shift", C.c_void_p),
                ("dense", FaLinear)]


_vp, _i32, _i64, _sz, _f = C.c_void_p, C.c_int32, C.c_int64, C.c_size_t, C.c_float

# fa_punc_score_fn: (ctx, ids, lens, batch, t_max, punc_out) -> 0 on success
PUNC_SCORE_FN = C.CFUNCTYPE(_i32, _vp, c_i32p, c_i32p, _i32, _i32, c_i32p)

# name -> (restype, argtypes); every symbol include/funasr_b200.h declares
SIGNATURES = {
    "fa_version": (C.c_char_p, []),
    "fa_launch_count": (C.c_uint64, []),
    "fa_status_string": (C.c_char_p, [C.c_int]),
    "fa_fbank_tables_bytes": (_sz, []),
    "fa_fbank_make_tables": (C.c_int, [_vp, _vp, _vp, _vp]),
    "fa_fbank_lfr_cmvn_tables": (C.c_int, [_vp, _vp, _i32, _i64, _vp, _vp, _i32, _i32, _vp, _i64, _vp, _i32, _vp]),
    "fa_fbank_short": (C.c_int, [_vp, _i32, _vp, _vp, _i32, _vp, _i32, _vp, _vp]),
    "fa_broadcast_rows": (C.c_int, [_vp, _i32, _i32, _vp, _i64, _i32, _vp]),
    "fa_sv_query_rows": (C.c_int, [_vp, _i32, _i32, _vp, _i32, _vp, _i64, _vp]),
    "fa_ctc_greedy_workspace_bytes": (_sz, [_i32, _i32, _i32, _i32]),
    "fa_ctc_greedy_forward": (C.c_int, [C.POINTER(FaLinear), _vp, _vp, _i32, _i32, _i32, _vp, _vp, _vp, _vp, _i32, _vp, _sz, _vp]),
    "fa_layernorm": (C.c_int, [_vp, _i64, C.POINTER(FaNorm), _vp, _vp, _f, _i32, _vp]),
    "fa_linear": (C.c_int, [_vp, _i64, _i64, C.POINTER(FaLinear), _i32, _vp, _i64, _vp, _i64, _vp, _i64, _i32, _vp, _sz, _vp]),
    "fa_linear_workspace_bytes": (_sz, [_i64, _i32, _i32]),
    "fa_split_rows": (C.c_int, [_vp, _i64, _i64, _i32, _i32, _i32, _vp, _vp]),
    "fa_linear_planes": (C.c_int, [_vp, _i64, C.POINTER(FaLinear), _i32, _vp, _i64, _vp, _i64, _vp, _i64, _i32, _vp]),
    "fa_linear_planes_to_planes": (C.c_int, [_vp, _i64, C.POINTER(FaLinear), _i32, _vp, _i64, _i32, _vp]),
    "fa_linear_planes_view": (C.c_int, [_vp, _i64, _i64, _i64, C.POINTER(FaLinear), _i32, _vp, _i64, _i32, _vp]),
    "fa_layernorm_planes": (C.c_int, [_vp, _i64, C.POINTER(FaNorm), _vp, _vp, _i32, _i32, _vp, _f, _i32, _vp, _vp]),
    "fa_linear_attn_sinks": (C.c_int, [_vp, _i64, C.POINTER(FaLinear), _i32, _i32, _i32, _i32, _i32, _i32, _f, _vp, _vp, _vp, _vp, _i64,
                                       _i32, _vp]),
    "fa_fsmn": (C.c_int, [_vp, _i64, _vp, _i32, _i32, _i32, _vp, _i32, _vp, _i64, _vp, _i64, _vp]),
    "fa_fsmn_tma": (C.c_int, [_vp, _i64, _vp, _i32, _i32, _i32, _vp, _i32, _vp, _i64, _vp, _i64, _vp]),
    "fa_fsmn_simt": (C.c_int, [_vp, _i64, _vp, _i32, _i32, _i32, _vp, _i32, _vp, _i64, _vp, _i64, _vp]),
    "fa_attention": (C.c_int, [_vp, _i64, _vp, _i64, _vp, _i64, _vp, _i32, _i32, _i32, _i32, _vp, _i64, _vp]),
    "fa_attention_tc_workspace_bytes": (_sz, [_i32, _i32, _i32, _i32, _i32]),
    "fa_attention_tc": (C.c_int, [_vp, _i64, _vp, _i64, _vp, _i64, _vp, _i32, _i32, _i32, _i32, _vp, _i64, _i32, _vp, _sz, _vp]),
    "fa_attention_tc_planes": (C.c_int, [_vp, _vp, _vp, _vp, _i32, _i32, _i32, _i32, _vp, _i64, _vp, _i64, _i32, _i32, _i32, _vp]),
    "fa_attention_tc_planes_ex": (C.c_int, [_vp, _vp, _vp, _vp, _i32, _i32, _i32, _i32, _i32, _vp, _i64, _vp, _i64, _i32, _i32, _i32, _vp]),
    "fa_attention_f32_ex": (C.c_int, [_vp, _i64, _vp, _i64, _vp, _i64, _vp, _i32, _i32, _i32, _i32, _i32, _vp, _i64, _i32, _vp]),
    "fa_attention_grouped_workspace_bytes": (_sz, [_i32, _i32, _i32, _i32, _i32, _i32]),
    "fa_attention_grouped": (C.c_int, [_vp, _i64, _vp, _i64, _vp, _i64, _vp, _vp, _i32, _i32, _i32, _i32, _i32, _i32, _vp, _i64, _i32, _vp, _sz,
                                       _vp]),
    "fa_sanm_encoder_workspace_bytes": (_sz, [_i32, _i32, _i32]),
    "fa_sanm_encoder_forward": (C.c_int, [C.POINTER(FaEncoder), _vp, _vp, _i32, _i32, _vp, _i32, _vp, _sz, _vp]),
    "fa_cif_predictor_workspace_bytes": (_sz, [_i32, _i32, _i32]),
    "fa_cif_predictor_forward": (C.c_int, [C.POINTER(FaPredictor), _vp, _vp, _i32, _i32, _vp, _i32, _vp, _vp, _vp, _i32, _vp, _sz, _vp]),
    "fa_cif_predictor_ext_workspace_bytes": (_sz, [_i32, _i32, _i32]),
    "fa_cif_predictor_forward_ext": (C.c_int, [C.POINTER(FaPredictor), _vp, _vp, _i32, _i32, _vp, _i32, _vp, _vp, _vp, _i32, _vp, _sz, _vp,
                                               _vp, _vp]),
    "fa_paraformer_decoder_workspace_bytes_hw": (_sz, [_i32, _i32, _i32, _i32, _i32, _i32]),
    "fa_paraformer_decoder_forward": (C.c_int, [C.POINTER(FaDecoder), _vp, _vp, _i32, _i32, _vp, _i64, _vp, _i32, _vp, _vp, _vp, _i32, _i32, _vp, _sz, _vp]),
    "fa_row_sum_f32": (C.c_int, [_vp, _i64, _i32, _i32, _vp, _vp]),
    "fa_paraformer_decoder_forward_hidden": (C.c_int, [C.POINTER(FaDecoder), _vp, _vp, _i32, _i32, _vp, _i64, _vp, _i32, _vp, _vp, _vp, _i32, _vp, _i32, _vp, _sz, _vp]),
    "fa_sanm_decoder_stack_workspace_bytes": (_sz, [_i32, _i32, _i32, _i32]),
    "fa_sanm_decoder_stack_forward": (C.c_int, [C.POINTER(FaDecoder), _vp, _vp, _i32, _i32, _i32, _vp, _i64, _vp, _i32, _i32, _i32, _vp, _vp, _i32, _vp, _sz, _vp]),
    "fa_paraformer_decoder_grouped_workspace_bytes": (_sz, [_i32, _i32, _i32, _i32, _i32, _i32, _i32]),
    "fa_paraformer_decoder_forward_grouped": (C.c_int, [C.POINTER(FaDecoder), _vp, _vp, _i32, _i32, _vp, _i64, _vp, _i32, _vp, _vp, _vp, _i32, _vp,
                                                        _vp, _vp, _vp, _i32, _i32, _i32, _vp, _sz, _vp]),
    "fa_sanm_decoder_stack_grouped_workspace_bytes": (_sz, [_i32, _i32, _i32, _i32, _i32, _i32]),
    "fa_sanm_decoder_stack_forward_grouped": (C.c_int, [C.POINTER(FaDecoder), _vp, _vp, _vp, _i32, _i32, _i32, _vp, _i64, _vp, _i32, _i32, _i32,
                                                        _vp, _vp, _vp, _i32, _i32, _vp, _sz, _vp]),
    "fa_linear_argmax_workspace_bytes": (_sz, [_i64, _i32, _i32]),
    "fa_linear_argmax": (C.c_int, [C.POINTER(FaLinear), _vp, _vp, _i64, _vp, _vp, _vp, _i32, _vp, _sz, _vp]),
    "fa_seaco_merge": (C.c_int, [_vp, _vp, _vp, _vp, _i64, _i32, _vp, _vp, _vp, _vp, _vp, _i32, _vp]),
    "fa_seaco_asf_select_host": (_i32, [_vp, _i32, _i32, _i32, _i32, _vp]),
    "fa_hotword_encoder_workspace_bytes": (_sz, [_i32, _i64, _i32]),
    "fa_hotword_encoder_forward": (C.c_int, [C.POINTER(FaHotwordEncoder), _vp, _vp, _i32, _vp, _i32, _vp, _sz, _vp]),
    "fa_cif_upsample_alphas": (C.c_int, [_vp, _i32, _vp, _vp, _vp, _vp, _i32, _i32, _f, _f, _f, _vp, _vp, _vp]),
    "fa_blstm_tc_scratch_bytes": (_sz, [_i32]),
    "fa_blstm_tc_ext_scratch_bytes": (_sz, [_i32]),
    "fa_blstm_forward_tc_ext": (C.c_int, [_vp, _vp, _vp, _i32, _i32, _i32, _vp, _vp, _sz, _vp, _vp]),
    "fa_blstm_forward_tc": (C.c_int, [_vp, _vp, _vp, _i32, _i32, _i32, _vp, _vp, _sz, _vp]),
    "fa_timestamp_head_workspace_bytes": (_sz, [_i32, _i32, _i32, _i32, _i32]),
    "fa_timestamp_head_ext_workspace_bytes": (_sz, [_i32, _i32, _i32, _i32, _i32]),
    "fa_timestamp_head_forward_ext": (C.c_int, [C.POINTER(FaTimestampHead), _vp, _vp, _vp, _i32, _i32, _vp, _vp, _i32, _vp, _sz, _vp, _vp, _vp]),
    "fa_timestamp_head_forward": (C.c_int, [C.POINTER(FaTimestampHead), _vp, _vp, _vp, _i32, _i32, _vp, _vp, _i32, _vp, _sz, _vp]),
    "fa_fsmn_vad_workspace_bytes": (_sz, [C.POINTER(FaVadEncoder), _i32]),
    "fa_fsmn_vad_forward": (C.c_int, [C.POINTER(FaVadEncoder), _vp, _i64, _i32, _vp, _vp, _vp, _sz, _vp]),
    "fa_frame_decibels": (C.c_int, [_vp, _i64, _i32, _vp, _vp]),
    "fa_fsmn_vad_batch_workspace_bytes": (_sz, [C.POINTER(FaVadEncoder), _i32, _i32]),
    "fa_fsmn_vad_forward_batch": (C.c_int, [C.POINTER(FaVadEncoder), _vp, _i64, _vp, _i32, _i32, _vp, _vp, _sz, _vp]),
    "fa_frame_decibels_batch": (C.c_int, [_vp, _i64, _vp, _i32, _i32, _vp, _vp]),
    "fa_cif_wo_hidden_host": (C.c_int, [_vp, _i64, C.c_float, _vp]),
    "fa_ts_stamps_host": (_i64, [_vp, _vp, _i64, _i64, _i32, C.c_double, _vp, _i64]),
    "fa_vad_detect_segments": (_i64, [_vp, _vp, _i64, _i64, C.POINTER(FaVadOptions), _i32, _i32, _vp, _i32, C.c_double, _vp, _i64]),
    "fa_greedy_filter": (C.c_int, [_vp, _vp, _i32, _i32, _i32, _i32, _i32, _vp, _vp, _vp]),
    "fa_split_planes": (C.c_int, [_vp, _i64, _i64, _i32, _i32, _vp, _vp]),
    "fa_embedding": (C.c_int, [_vp, _vp, _i32, _i32, _i64, _vp, _vp]),
    "fa_pcm_decode": (C.c_int, [_vp, _i32, _i32, _i64, _vp, _vp]),
    "fa_resample": (C.c_int, [_vp, _vp, _i32, _i64, _vp, _i32, _i32, _i32, _vp, _i64, _i32, _vp, _vp]),
    # audio at any rate and PCM layout: the host tables (host_ops.cpp), the ingest kernel (resample.cu) and the handle entries
    "fa_loader_resample_table_host": (_i64, [_i32, _i32, c_i32p, c_i32p, c_i32p, _vp, _i64]),
    "fa_runtime_resample_table_host": (_i64, [_i32, _i32, c_i32p, c_i32p, c_i32p, _vp, _vp, _vp, _i64]),
    "fa_runtime_resample_out_len_host": (_i64, [_i32, _i32, _i64]),
    "fa_ingest_pcm": (C.c_int, [_vp, _vp, _i32, _i32, _i32, C.POINTER(FaIngestTable), _vp, _i64, _vp]),
    "fa_offline_infer_audio": (_vp, [_vp, C.POINTER(_vp), C.POINTER(_i64), _i32, C.POINTER(FaAudioFormat), _vp, _i32, _vp, _vp]),
    "fa_offline_infer_vad_audio": (_vp, [_vp, _vp, _vp, C.POINTER(_vp), C.POINTER(_i64), _i32, C.POINTER(FaAudioFormat), _vp, _i32, _vp, _vp,
                                         C.POINTER(FaLongAudioOptions), _i32]),
    "fa_vad_infer_audio": (_vp, [_vp, _vp, _i64, C.POINTER(FaAudioFormat), C.POINTER(FaVadRunOptions)]),
    "fa_spk_embed_audio": (C.c_int, [_vp, C.POINTER(_vp), C.POINTER(_i64), _i32, C.POINTER(FaAudioFormat), _vp]),
    # CAM++ speaker embedding (campplus.cu)
    "fa_campplus_features": (C.c_int, [_vp, _vp, _i32, _i64, _vp, _vp, _vp, _i32, _vp]),
    "fa_campplus_workspace_bytes": (_sz, [C.POINTER(FaCampplus), _i32, _i32, _i32]),
    "fa_campplus_forward": (C.c_int, [C.POINTER(FaCampplus), _vp, _i32, _i32, _vp, _i32, _vp, _sz, _vp]),
    "fa_campplus_ext_workspace_bytes": (_sz, [C.POINTER(FaCampplus), _i32, _i32, _i32]),
    "fa_campplus_forward_ext": (C.c_int, [C.POINTER(FaCampplus), _vp, _i32, _i32, _vp, _i32, _vp, _sz, _vp, _vp]),
    "fa_campplus_conv2d": (C.c_int, [C.POINTER(FaCamConv2d), _vp, _i32, _i32, _i32, _vp, _vp, _i32, _vp]),
    "fa_campplus_cam": (C.c_int, [_vp, _i32, _i32, _i32, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i64, _vp]),
    "fa_campplus_stats_pool": (C.c_int, [_vp, _i32, _i32, _i32, _vp, _vp, _vp, _vp]),
    # handle-style offline recogniser (funasrruntime.h:100-116 counterpart; offline_asr.cu)
    "fa_offline_init": (_vp, [C.c_char_p, _i32, _i32]),
    "fa_offline_infer": (_vp, [_vp, C.POINTER(_vp), C.POINTER(_i64), _i32, _i32]),
    "fa_offline_infer_hw": (_vp, [_vp, C.POINTER(_vp), C.POINTER(_i64), _i32, _i32, _vp, _i32]),
    "fa_offline_is_contextual": (_i32, [_vp]),
    "fa_offline_has_timestamps": (_i32, [_vp]),
    "fa_offline_pool_stats": (C.c_int, [_vp, C.POINTER(_i64), C.POINTER(_i64)]),
    "fa_offline_host_tensor": (_vp, [_vp, C.c_char_p, C.POINTER(_i64)]),
    "fa_offline_result_count": (_i32, [_vp]),
    "fa_offline_result_ids": (C.POINTER(_i32), [_vp, _i32, C.POINTER(_i32)]),
    "fa_offline_result_audio_seconds": (C.c_float, [_vp]),
    "fa_offline_result_stamps": (C.POINTER(_i32), [_vp, _i32, C.POINTER(_i32)]),
    "fa_offline_is_sensevoice": (_i32, [_vp]),
    "fa_offline_is_seaco": (_i32, [_vp]),
    "fa_offline_hotword_embed": (C.c_int, [_vp, _vp, _vp, _i32, _vp]),
    "fa_offline_infer_sv": (_vp, [_vp, C.POINTER(_vp), C.POINTER(_i64), _i32, _i32, _vp, _vp]),
    "fa_sv_ctc_text_host": (_i64, [_vp, _i32, C.POINTER(C.c_char_p), _i32, C.c_char_p, _i64]),
    "fa_offline_free_result": (None, [_vp]),
    "fa_offline_uninit": (None, [_vp]),
    "fa_offline_last_error": (C.c_char_p, []),
    # handle-style FSMN-VAD and long-audio recognition (offline_vad.cu, offline_long.cu; fa_pack_segments / fa_merge_vad: vad_detector.cpp)
    "fa_vad_init": (_vp, [C.c_char_p, _i32]),
    "fa_vad_uninit": (None, [_vp]),
    "fa_vad_infer": (_vp, [_vp, _vp, _i64, _i32, C.POINTER(FaVadRunOptions)]),
    "fa_vad_result_segments": (C.POINTER(_i32), [_vp, C.POINTER(_i64)]),
    "fa_vad_result_frames": (C.POINTER(C.c_float), [_vp, C.POINTER(_i64)]),
    "fa_vad_result_audio_seconds": (C.c_float, [_vp]),
    "fa_vad_free_result": (None, [_vp]),
    "fa_offline_infer_vad": (_vp, [_vp, _vp, C.POINTER(_vp), C.POINTER(_i64), _i32, _i32, _vp, _i32, C.POINTER(FaLongAudioOptions)]),
    "fa_offline_infer_vad_sv": (_vp, [_vp, _vp, C.POINTER(_vp), C.POINTER(_i64), _i32, _i32, _vp, _vp, C.POINTER(FaLongAudioOptions)]),
    "fa_offline_result_segments": (C.POINTER(_i32), [_vp, _i32, C.POINTER(_i32)]),
    "fa_gather_segments": (C.c_int, [_vp, _i64, _vp, _vp, _i32, _i64, _vp, _vp]),
    "fa_pack_segments": (_i64, [_vp, _i64, _i32, _i32, _vp, _vp]),
    "fa_merge_vad": (_i64, [_vp, _i64, _i32, _i32, _vp]),
    # speaker diarization: the CAM++ handle (offline_spk.cu) and long audio (offline_long.cu), the clustering kernels (spk_cluster.cu), host routines (host_ops.cpp)
    "fa_spk_init": (_vp, [C.c_char_p, _i32, _i32]),
    "fa_spk_uninit": (None, [_vp]),
    "fa_spk_embed": (C.c_int, [_vp, C.POINTER(_vp), C.POINTER(_i64), _i32, _i32, _vp]),
    "fa_spk_cluster": (C.c_int, [_vp, _vp, _i32, _i32, _vp]),
    "fa_spk_pool_stats": (C.c_int, [_vp, C.POINTER(_i64), C.POINTER(_i64)]),
    "fa_offline_infer_vad_spk": (_vp, [_vp, _vp, _vp, C.POINTER(_vp), C.POINTER(_i64), _i32, _i32, _vp, _i32, _vp, _vp,
                                       C.POINTER(FaLongAudioOptions), _i32]),
    "fa_offline_result_spk": (C.POINTER(_i32), [_vp, _i32, C.POINTER(_i32)]),
    "fa_spk_effective_pval": (C.c_double, [_i32, C.c_double]),
    "fa_spk_laplacian_workspace_bytes": (_sz, [_i32, _i32]),
    "fa_spk_laplacian": (C.c_int, [_vp, _i32, _i32, C.c_double, _vp, _vp, _sz, _vp]),
    "fa_spk_tridiagonalize_workspace_bytes": (_sz, [_i32]),
    "fa_spk_tridiagonalize": (C.c_int, [_vp, _i32, _vp, _vp, _vp, _vp, _sz, _vp]),
    "fa_spk_back_transform": (C.c_int, [_vp, _vp, _i32, _vp, _i32, _vp]),
    "fa_spk_laplacian_batch_workspace_bytes": (_sz, [_vp, _i32, _i32]),
    "fa_spk_laplacian_batch": (C.c_int, [_vp, _vp, _i32, _i32, C.c_double, _vp, _vp, _sz, _vp]),
    "fa_spk_tridiagonalize_batch_workspace_bytes": (_sz, [_vp, _i32]),
    "fa_spk_tridiagonalize_batch": (C.c_int, [_vp, _vp, _i32, _vp, _vp, _vp, _vp, _sz, _vp]),
    "fa_spk_back_transform_batch": (C.c_int, [_vp, _vp, _vp, _vp, _i32, _vp, _vp]),
    "fa_sym_tridiag_smallest_host": (C.c_int, [_vp, _vp, _i32, _i32, _i32, _vp, _vp]),
    "fa_spk_kmeans_host": (C.c_int, [_vp, _i64, _i32, _i32, C.c_uint64, _i32, _i32, _vp]),
    "fa_spk_merge_by_cos_host": (C.c_int, [_vp, _vp, _i64, _i32, C.c_double]),
    "fa_spk_postprocess_host": (_i64, [_vp, _vp, _i64, _vp]),
    "fa_spk_distribute_host": (C.c_int, [_vp, _i64, _vp, _i64, _vp]),
    # handle-style MonotonicAligner forced alignment (offline_align.cu); results through the fa_offline_result_* accessors
    "fa_align_init": (_vp, [C.c_char_p, _i32, _i32]),
    "fa_align_infer": (_vp, [_vp, C.POINTER(_vp), C.POINTER(_i64), _i32, C.POINTER(FaAudioFormat), C.POINTER(_vp), C.POINTER(_i32)]),
    "fa_align_uninit": (None, [_vp]),
    # handle-style CT-Transformer punctuation (offline_punc.cu; the text walk: punc_text.cpp)
    "fa_punc_init": (_vp, [C.c_char_p, _i32]),
    "fa_punc_infer": (_vp, [_vp, C.POINTER(C.c_char_p), _i32]),
    "fa_punc_result_text": (C.c_char_p, [_vp, _i32]),
    "fa_punc_result_ids": (C.POINTER(_i32), [_vp, _i32, C.POINTER(_i32)]),
    "fa_punc_result_steps": (_i64, [_vp]),
    "fa_punc_free_result": (None, [_vp]),
    "fa_punc_uninit": (None, [_vp]),
    "fa_punc_walk_host": (_vp, [C.POINTER(C.c_char_p), _i32, C.POINTER(C.c_char_p), _i32, C.POINTER(C.c_char_p), _i32, _i32, _i32, _i64,
                                PUNC_SCORE_FN, _vp]),
    "fa_punc_init_host": (_vp, [C.POINTER(C.c_char_p), _i32, C.POINTER(C.c_char_p), _i32, _i32, _i32, _i64, PUNC_SCORE_FN, _vp]),
    "fa_punc_pool_stats": (C.c_int, [_vp, C.POINTER(_i64), C.POINTER(_i64)]),
}


_lib = None


class FunasrB200Error(RuntimeError):
    pass


def load():
    """Load (once) and return the CUDA library; raises loudly when it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise FunasrB200Error(
            "funasr_b200: %s not found — build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(or funasr_b200/csrc/build.sh). There is no CPU/PyTorch fallback." % LIB_PATH)
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError if the header and the library disagree
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def check(status: int, what: str):
    if status != FA_OK:
        raise FunasrB200Error("%s failed: %s (%d)" % (what, load().fa_status_string(status).decode(), status))
