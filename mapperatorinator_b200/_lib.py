"""ctypes binding of libmapperatorinator_b200.so (the C ABI in include/mapperatorinator_b200.h).

There is deliberately no fallback: if the shared library has not been built (`python -c "import __graft_entry__ as g;
g.build()"` or `mapperatorinator_b200/csrc/build.sh`) every compute entry point raises.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Optional

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libmapperatorinator_b200.so")


class MelConfigC(C.Structure):
    _fields_ = [("n_fft", C.c_int32), ("hop_length", C.c_int32), ("n_mels", C.c_int32), ("pad_reflect", C.c_int32),
                ("log_scale", C.c_int32)]


class ModelConfigC(C.Structure):
    _fields_ = [("d_model", C.c_int32), ("encoder_layers", C.c_int32), ("decoder_layers", C.c_int32), ("heads", C.c_int32),
                ("ffn_dim", C.c_int32), ("src_seq_len", C.c_int32), ("tgt_seq_len", C.c_int32), ("vocab_size_in", C.c_int32),
                ("vocab_size_out", C.c_int32), ("mel", MelConfigC), ("max_windows", C.c_int32), ("max_batch", C.c_int32)]


class GenerateParamsC(C.Structure):
    _fields_ = [("cfg_scale", C.c_float), ("timeshift_bias", C.c_float), ("types_first", C.c_int32),
                ("temperature", C.c_float), ("timing_temperature", C.c_float), ("mania_column_temperature", C.c_float),
                ("taiko_hit_temperature", C.c_float), ("lookback_on", C.c_int32), ("lookback_start", C.c_int32),
                ("lookback_end", C.c_int32), ("do_sample", C.c_int32), ("top_k", C.c_int32), ("top_p", C.c_float),
                ("max_length", C.c_int32), ("min_new_tokens", C.c_int32), ("pad_token_id", C.c_int32), ("seed", C.c_uint64),
                ("time_shift_start", C.c_int32), ("time_shift_end", C.c_int32), ("n_cond", C.c_int32),
                ("cond_temp", C.c_float * 3), ("cond_offset", C.c_int32 * 3), ("cond_flag", C.c_int32 * 3),
                ("position_rule", C.c_int32), ("top_p_cut", C.c_float)]


class DitConfigC(C.Structure):
    _fields_ = [("hidden", C.c_int32), ("depth", C.c_int32), ("heads", C.c_int32), ("mlp_ratio", C.c_int32),
                ("in_channels", C.c_int32), ("context_size", C.c_int32), ("class_size", C.c_int32), ("pos_freq_dim", C.c_int32),
                ("t_freq_dim", C.c_int32), ("max_seq_len", C.c_int32), ("max_batch", C.c_int32)]


class GemvSegC(C.Structure):
    _fields_ = [("out", C.c_void_p), ("out_bs", C.c_int64), ("pos_stride", C.c_int64), ("n_begin", C.c_int32), ("n_end", C.c_int32),
                ("alpha", C.c_float), ("act", C.c_int32)]


class RowMapC(C.Structure):
    _fields_ = [("ptr", C.c_void_p), ("ld", C.c_int64), ("rpb", C.c_int32), ("bstride", C.c_int64)]


class DitMaskC(C.Structure):
    _fields_ = [("mask_mode", C.c_int32), ("band", C.c_int32), ("dense_mask", C.c_void_p)]


# every symbol include/mapperatorinator_b200.h declares (tests/test_abi.py checks the library exports each one)
ABI_SYMBOLS = [
    "mb200_abi_version", "mb200_last_error",
    "mb200_mel_create", "mb200_mel_destroy", "mb200_mel_forward",
    "mb200_model_create", "mb200_model_destroy", "mb200_model_set_weight", "mb200_model_set_weight_bf16", "mb200_model_finalize",
    "mb200_model_token_weight_bytes", "mb200_model_encode",
    "mb200_model_generate", "mb200_model_generate_beams", "mb200_model_generate_ragged", "mb200_model_forward_logits",
    "mb200_stream_open", "mb200_stream_admit", "mb200_stream_run", "mb200_stream_take", "mb200_stream_close",
    "mb200_model_score_tokens",
    "mb200_dit_create", "mb200_dit_destroy", "mb200_dit_set_weight", "mb200_dit_finalize", "mb200_dit_forward_with_cfg",
    "mb200_dit_sample_loop", "mb200_dit_set_option", "mb200_dit_set_sliders", "mb200_dit_apply_sliders",
    "mb200_launch_count", "mb200_wbf16_launch_count", "mb200_model_set_option", "mb200_model_profile_step", "mb200_model_read_trace", "mb200_model_mega_stats", "mb200_model_logits_chain",
    "mb200_model_beam_step",
    "mb200_op_gemm_mapped", "mb200_set_tensor_cores", "mb200_op_layernorm", "mb200_op_attention", "mb200_op_decode_attention", "mb200_op_gemv", "mb200_op_gemv_bf16", "mb200_set_attention_tc", "mb200_audio_out_frames", "mb200_audio_ingest",
]

_lib: Optional[C.CDLL] = None


def load() -> C.CDLL:
    """Load the engine library; raises (never falls back) when it is missing."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            f"{LIB_PATH} is not built. mapperatorinator_b200 has no CPU fallback: build the sm_90a engine with "
            "`python -c 'import __graft_entry__ as g; g.build()'` (or mapperatorinator_b200/csrc/build.sh).")
    lib = C.CDLL(LIB_PATH)
    lib.mb200_last_error.restype = C.c_char_p
    vp, i32, i64, f32 = C.c_void_p, C.c_int32, C.c_int64, C.c_float
    lib.mb200_mel_create.argtypes = [C.POINTER(vp), C.POINTER(MelConfigC), vp]
    lib.mb200_mel_destroy.argtypes = [vp]; lib.mb200_mel_destroy.restype = None
    lib.mb200_mel_forward.argtypes = [vp, vp, i32, i32, vp, vp]
    lib.mb200_model_create.argtypes = [C.POINTER(vp), C.POINTER(ModelConfigC), vp]
    lib.mb200_model_destroy.argtypes = [vp]; lib.mb200_model_destroy.restype = None
    lib.mb200_model_set_weight.argtypes = [vp, C.c_char_p, vp, i64]
    lib.mb200_model_set_weight_bf16.argtypes = [vp, C.c_char_p, vp, i64]
    lib.mb200_model_finalize.argtypes = [vp]
    lib.mb200_model_token_weight_bytes.argtypes = [vp, C.POINTER(i32)]
    lib.mb200_model_encode.argtypes = [vp, vp, i32, i32, vp, vp]
    lib.mb200_model_generate.argtypes = [vp, vp, i32, vp, vp, i32, vp, vp, vp, C.POINTER(GenerateParamsC), vp, C.POINTER(i32), vp]
    lib.mb200_model_generate_beams.argtypes = [vp, vp, i32, vp, vp, i32, vp, vp, vp, C.POINTER(GenerateParamsC), i32, i64, vp,
                                               C.POINTER(i32), vp, vp]
    lib.mb200_model_generate_ragged.argtypes = [vp, i32, vp, vp, vp, vp, vp, vp, vp, i32, vp, vp]
    lib.mb200_stream_open.argtypes = [vp, i32, i32, i32, C.POINTER(vp), vp]
    lib.mb200_stream_admit.argtypes = [vp, i32, vp, vp, vp, vp, vp, vp, vp, vp]
    lib.mb200_stream_run.argtypes = [vp, i32, vp, vp, C.POINTER(i32), C.POINTER(i32), vp]
    lib.mb200_stream_take.argtypes = [vp, i32, vp, i32, vp]
    lib.mb200_stream_close.argtypes = [vp]; lib.mb200_stream_close.restype = None
    lib.mb200_model_forward_logits.argtypes = [vp, vp, i32, vp, vp, i32, i32, vp, vp]
    lib.mb200_model_score_tokens.argtypes = [vp, vp, i32, vp, vp, i32, i32, vp, vp, vp, vp, vp]
    lib.mb200_model_set_option.argtypes = [vp, C.c_char_p, i32]
    lib.mb200_launch_count.restype = i64
    lib.mb200_wbf16_launch_count.restype = i64
    lib.mb200_model_profile_step.argtypes = [vp, i32, i32, i32, i32, vp, vp]
    lib.mb200_model_read_trace.argtypes = [vp, vp, i32]
    lib.mb200_model_mega_stats.argtypes = [vp, vp, i32]
    lib.mb200_dit_create.argtypes = [C.POINTER(vp), C.POINTER(DitConfigC)]
    lib.mb200_dit_destroy.argtypes = [vp]; lib.mb200_dit_destroy.restype = None
    lib.mb200_dit_set_weight.argtypes = [vp, C.c_char_p, vp, i64]
    lib.mb200_dit_finalize.argtypes = [vp]
    lib.mb200_dit_forward_with_cfg.argtypes = [vp, vp, vp, vp, vp, i32, i32, f32, C.POINTER(DitMaskC), vp, vp]
    lib.mb200_dit_sample_loop.argtypes = [vp, vp, vp, vp, vp, i32, i32, f32, C.POINTER(DitMaskC), vp, i32, vp, vp, vp]
    lib.mb200_model_logits_chain.argtypes = [vp, vp, i32, i32, vp, i32, i32, vp, C.POINTER(GenerateParamsC), i32, i32, vp, vp, vp]
    lib.mb200_model_beam_step.argtypes = [vp, vp, i32, i32, i32, vp, i32, i32, vp, C.POINTER(GenerateParamsC), vp, i32, i32, vp, vp,
                                          vp, vp, vp, vp, vp, vp, vp, vp]
    lib.mb200_dit_set_option.argtypes = [vp, C.c_char_p, i32]
    lib.mb200_dit_set_sliders.argtypes = [vp, i32, vp, vp, vp, vp, vp]
    lib.mb200_dit_apply_sliders.argtypes = [vp, vp, i32, i32, vp]
    rm = C.POINTER(RowMapC)
    lib.mb200_op_gemm_mapped.argtypes = [rm, vp, i64, rm, vp, i32, f32, rm, vp, i64, i32, i32, i32, i32, i32, vp]
    lib.mb200_set_tensor_cores.argtypes = [i32]
    lib.mb200_op_layernorm.argtypes = [vp, vp, vp, vp, vp, vp, i64, i32, i32, i32, f32, vp]
    lib.mb200_op_attention.argtypes = [vp, i64, i64, vp, i64, i64, vp, i64, i64, vp, i64, i64, i32, i32, i32, i32, f32, i32, i32, vp, i64,
                                       i32, vp, vp, vp]
    lib.mb200_set_attention_tc.argtypes = [i32, i32]
    lib.mb200_op_decode_attention.argtypes = [vp, vp, i32, i32, i32, i32, vp, i32, i32, vp, i64, i32, i32, vp, i64, vp, vp, i32, vp, vp]
    lib.mb200_op_gemv.argtypes = [vp, i64, i32, i32, i32, vp, vp, f32, vp, i64, i32, vp, vp, i64, C.POINTER(GemvSegC), i32, i32, vp, vp,
                                  i32, i32, vp]
    lib.mb200_op_gemv_bf16.argtypes = lib.mb200_op_gemv.argtypes
    lib.mb200_audio_out_frames.argtypes = [i64, i32, i32]
    lib.mb200_audio_out_frames.restype = i64
    lib.mb200_audio_ingest.argtypes = [vp, i64, i32, i32, i32, i32, vp, vp, vp]
    _lib = lib
    return lib


def check(status: int) -> None:
    if status != 0:
        msg = load().mb200_last_error()
        raise RuntimeError(f"mapperatorinator_b200 engine error {status}: {msg.decode() if msg else '?'}")
