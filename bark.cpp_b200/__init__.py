"""ctypes binding of libbark_b200.so — the H100-native drop-in for bark.cpp's hot path.

The product is the C-ABI shared library (include/bark.h, include/bark_b200.h); this module only
loads it and mirrors the reference's call sequence (bark_context_default_params -> bark_load_model
-> bark_generate_audio -> bark_get_audio_data -> bark_free, examples/main/main.cpp:49-91) for the
Python-side tests and the benchmark.  There is no CPU path: loading fails loudly when the CUDA
extension has not been built, and bark_load_model fails when no sm_90 (H100) device is present.

The directory name contains a dot, so import it through `__graft_entry__.load_package()`.
"""
from __future__ import annotations

import ctypes as C
import math
import os
import re

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libbark_b200.so")

PROGRESS_CB = C.CFUNCTYPE(None, C.c_void_p, C.c_int, C.c_int, C.c_void_p)


class BarkContextParams(C.Structure):
    """struct bark_context_params (include/bark.h; reference bark.h:81-141) — passed by value."""
    _fields_ = [
        ("verbosity", C.c_int), ("temp", C.c_float), ("fine_temp", C.c_float), ("min_eos_p", C.c_float),
        ("sliding_window_size", C.c_int32), ("max_coarse_history", C.c_int32), ("sample_rate", C.c_int32),
        ("target_bandwidth", C.c_int32), ("cls_token_id", C.c_int32), ("sep_token_id", C.c_int32),
        ("n_steps_text_encoder", C.c_int32), ("text_pad_token", C.c_int32), ("text_encoding_offset", C.c_int32),
        ("semantic_rate_hz", C.c_float), ("semantic_pad_token", C.c_int32), ("semantic_vocab_size", C.c_int32),
        ("semantic_infer_token", C.c_int32), ("coarse_rate_hz", C.c_float), ("coarse_infer_token", C.c_int32),
        ("coarse_semantic_pad_token", C.c_int32), ("n_coarse_codebooks", C.c_int32), ("n_fine_codebooks", C.c_int32),
        ("codebook_size", C.c_int32), ("progress_callback", PROGRESS_CB), ("progress_callback_user_data", C.c_void_p),
    ]


class BarkStatistics(C.Structure):
    _fields_ = [("t_load_us", C.c_int64), ("t_eval_us", C.c_int64), ("t_semantic_us", C.c_int64), ("t_coarse_us", C.c_int64),
                ("t_fine_us", C.c_int64), ("n_sample_semantic", C.c_int32), ("n_sample_coarse", C.c_int32), ("n_sample_fine", C.c_int32)]


class EncodecStatistics(C.Structure):
    """struct encodec_statistics (include/encodec.h)."""
    _fields_ = [("t_load_us", C.c_int64), ("t_compute_us", C.c_int64)]


class HistoryPromptStruct(C.Structure):
    """struct bark_b200_history_prompt (include/bark_b200.h)."""
    _fields_ = [("semantic", C.c_void_p), ("n_semantic", C.c_int), ("coarse", C.c_void_p), ("n_coarse_frames", C.c_int),
                ("fine", C.c_void_p), ("n_fine_frames", C.c_int)]


HISTORY_KEYS = ("semantic_prompt", "coarse_prompt", "fine_prompt")


def load_history_prompt(src) -> dict:
    """A speaker history prompt from an upstream Bark voice file (.npz path) or a mapping with its three keys: semantic_prompt [n_s],
    coarse_prompt [2][n_c] and fine_prompt [8][n_f] (n_f may be 0).  Returns the three as contiguous int32 arrays; raises ValueError on
    a missing key or a wrong rank or shape.  Id ranges and the semantic / coarse alignment are checked by bark_b200_set_history_prompt."""
    if isinstance(src, (str, bytes, os.PathLike)):
        with np.load(src) as f:
            return load_history_prompt({k: f[k] for k in f.files})
    out = {}
    for k, lead in zip(HISTORY_KEYS, (None, 2, 8)):
        try:
            a = np.asarray(src[k])
        except KeyError:
            raise ValueError(f"history prompt: missing {k}") from None
        if a.dtype.kind not in "iu":
            raise ValueError(f"history prompt: {k} holds {a.dtype} values, not integer ids")
        if lead is None and a.ndim != 1:
            raise ValueError(f"history prompt: {k} has shape {a.shape}, expected [n]")
        if lead is not None and (a.ndim != 2 or a.shape[0] != lead):
            raise ValueError(f"history prompt: {k} has shape {a.shape}, expected [{lead}][n]")
        out[k] = np.ascontiguousarray(a, np.int32)
    return out


class SamplingStruct(C.Structure):
    """struct bark_b200_sampling (include/bark_b200.h)"""
    _fields_ = [("top_k", C.c_int32), ("use_top_p", C.c_int32), ("top_p", C.c_float)]


SAMPLING_STAGES = {"semantic": 0, "coarse": 1}


def _sampling_struct(top_k=None, top_p=None):
    """struct bark_b200_sampling for top_k (None or 0: off) and top_p (None: off)."""
    return SamplingStruct(int(top_k or 0), int(top_p is not None), float(top_p) if top_p is not None else 1.0)


def _history_struct(p):
    """(struct bark_b200_history_prompt, the arrays it points into) for a prompt as load_history_prompt accepts it."""
    p = load_history_prompt(p)
    s, c, f = (p[k] for k in HISTORY_KEYS)
    return HistoryPromptStruct(_p(s), s.size, _p(c), c.shape[1], _p(f) if f.size else None, f.shape[1]), p


class LongFormStruct(C.Structure):
    """struct bark_b200_long_form (include/bark_b200.h)"""
    _fields_ = [("voice", C.c_int32), ("max_chunk_ids", C.c_int32), ("gap_samples", C.c_int32)]


VOICES = {"chain": 0, "fixed": 1}             # BARK_B200_VOICE_CHAIN / _FIXED
LONG_FORM_DEFAULTS = dict(max_chunk_ids=48, gap_samples=6000)


# every symbol the two public headers declare (tests check the library exports exactly these)
EXPORTS = [
    "bark_context_default_params", "bark_load_model", "bark_generate_audio", "bark_get_audio_data", "bark_get_audio_data_size",
    "bark_get_load_time", "bark_get_eval_time", "bark_reset_statistics", "bark_model_quantize", "bark_free",
    "bark_b200_set_device", "bark_b200_version", "bark_b200_gpt_eval", "bark_b200_fine_eval", "bark_b200_encodec_decode",
    "bark_b200_encodec_encode", "bark_b200_rvq_encode",
    "bark_b200_sample", "bark_b200_sample_rows", "bark_b200_reseed", "bark_b200_tokenize", "bark_b200_forward_text_encoder",
    "bark_b200_forward_coarse_encoder", "bark_b200_forward_fine_encoder", "bark_b200_get_tokens", "bark_b200_set_tokens",
    "bark_b200_get_stats", "bark_b200_get_hparams", "bark_b200_kernel_launches", "bark_b200_layernorm_fallbacks",
    "bark_b200_profile_enable", "bark_b200_profile_report", "bark_b200_io_counters", "bark_b200_decode_timing",
    "bark_b200_shard_init", "bark_b200_shard_connect", "bark_b200_shard_nvlink_bytes",
    "bark_b200_fast_mode", "bark_b200_fast_gemm", "bark_b200_fast_attention", "bark_b200_parity_attention", "bark_b200_batch_attention", "bark_b200_parity_gemm",
    "bark_b200_parity_rows", "bark_b200_sample_given_u", "bark_b200_generate_batch", "bark_b200_batch_audio", "bark_b200_batch_tokens", "bark_b200_gpt_eval_slot", "bark_b200_gpt_step_batch",
    "bark_b200_set_history_prompt", "bark_b200_generate_batch_prompted", "bark_b200_set_sampling", "bark_b200_sample_filtered_given_u",
    "bark_b200_quant_matmul", "bark_b200_fast_convert",
    "bark_b200_codec_conv1d", "bark_b200_codec_convtr1d", "bark_b200_codec_lstm", "bark_b200_codec_rvq_decode", "bark_b200_device_math",
    "bark_b200_encodec_compress_batch", "bark_b200_encodec_decompress_batch", "bark_b200_encodec_reconstruct_batch",
    "bark_b200_encodec_batch_codes", "bark_b200_encodec_batch_audio",
    "bark_b200_encodec_compress_resampled", "bark_b200_encodec_reconstruct_resampled", "bark_b200_encodec_compress_batch_resampled",
    "bark_b200_encodec_reconstruct_batch_resampled", "bark_b200_encodec_encode_resampled", "bark_b200_resample",
    "bark_b200_set_tokenizer", "bark_b200_text_ids", "bark_b200_bert_tokenize",
    "bark_b200_set_long_form", "bark_b200_long_chunks", "bark_b200_long_chunk_text", "bark_b200_long_chunk_tokens", "bark_b200_split_text",
    "bark_b200_encodec_stream_open", "bark_b200_encodec_stream_push", "bark_b200_encodec_stream_push_batch", "bark_b200_encodec_stream_read",
    "bark_b200_encodec_stream_finish", "bark_b200_encodec_stream_ready", "bark_b200_encodec_stream_codebooks", "bark_b200_encodec_stream_close",
    "bark_b200_codec_conv1d_window", "bark_b200_codec_convtr1d_window", "bark_b200_codec_lstm_state",
    "bark_b200_encodec_stream_open_resampled", "bark_b200_encodec_stream_ready_resampled", "bark_b200_resample_window",
    "ggml_time_init", "ggml_time_us", "ggml_time_ms", "ggml_init", "ggml_free",
]

# encodec.cpp's API (include/encodec.h), exported by the same library; kept apart from EXPORTS, which lists the bark headers' symbols
ENCODEC_EXPORTS = [
    "encodec_load_model", "encodec_set_target_bandwidth", "encodec_set_sample_rate", "encodec_reconstruct_audio", "encodec_compress_audio",
    "encodec_decompress_audio", "encodec_get_audio", "encodec_get_audio_size", "encodec_get_codes", "encodec_get_codes_size",
    "encodec_get_statistics", "encodec_reset_statistics", "encodec_free",
]

_lib = None


def lib() -> C.CDLL:
    """Load libbark_b200.so (built by `make -C bark.cpp_b200` / __graft_entry__.build())."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(f"{LIB_PATH} is missing: build the CUDA extension first (python -c 'import __graft_entry__ as g; g.build()'). "
                           "There is no CPU fallback.")
    L = C.CDLL(LIB_PATH)
    vp, i32p, f32p = C.c_void_p, C.c_void_p, C.c_void_p
    L.bark_context_default_params.restype = BarkContextParams
    L.bark_load_model.restype = vp
    L.bark_load_model.argtypes = [C.c_char_p, BarkContextParams, C.c_uint32]
    L.bark_generate_audio.restype = C.c_bool
    L.bark_generate_audio.argtypes = [vp, C.c_char_p, C.c_int]
    L.bark_get_audio_data.restype = C.POINTER(C.c_float)
    L.bark_get_audio_data.argtypes = [vp]
    L.bark_get_audio_data_size.restype = C.c_int
    L.bark_get_audio_data_size.argtypes = [vp]
    for n in ("bark_get_load_time", "bark_get_eval_time"):
        getattr(L, n).restype = C.c_int64
        getattr(L, n).argtypes = [vp]
    L.bark_reset_statistics.argtypes = [vp]
    L.bark_model_quantize.restype = C.c_bool
    L.bark_model_quantize.argtypes = [C.c_char_p, C.c_char_p, C.c_int]
    L.bark_free.argtypes = [vp]
    L.bark_b200_set_device.argtypes = [C.c_int]
    L.bark_b200_version.restype = C.c_char_p
    L.bark_b200_gpt_eval.restype = C.c_int
    L.bark_b200_gpt_eval.argtypes = [vp, C.c_int, i32p, C.c_int, C.POINTER(C.c_int), C.c_int, f32p]
    L.bark_b200_fine_eval.restype = C.c_int
    L.bark_b200_fine_eval.argtypes = [vp, i32p, C.c_int, f32p]
    L.bark_b200_encodec_decode.restype = C.c_int
    L.bark_b200_encodec_decode.argtypes = [vp, i32p, C.c_int, f32p, C.c_int]
    L.bark_b200_encodec_encode.restype = C.c_int
    L.bark_b200_encodec_encode.argtypes = [vp, f32p, C.c_int, i32p, C.c_int, f32p, C.c_int]
    L.bark_b200_rvq_encode.restype = C.c_int
    L.bark_b200_rvq_encode.argtypes = [f32p, C.c_int, f32p, C.c_int, C.c_int, C.c_int, i32p]
    L.bark_b200_sample.restype = C.c_int
    L.bark_b200_sample.argtypes = [vp, C.c_int, f32p, C.c_int, C.c_float, C.POINTER(C.c_float)]
    L.bark_b200_sample_rows.restype = C.c_int
    L.bark_b200_sample_rows.argtypes = [vp, f32p, C.c_int, C.c_int, C.c_float, i32p, f32p]
    L.bark_b200_reseed.argtypes = [vp, C.c_uint32]
    L.bark_b200_tokenize.argtypes = [vp, C.c_char_p, i32p]
    for n in ("bark_b200_forward_text_encoder", "bark_b200_forward_coarse_encoder", "bark_b200_forward_fine_encoder"):
        getattr(L, n).restype = C.c_bool
        getattr(L, n).argtypes = [vp, C.c_int]
    L.bark_b200_get_tokens.restype = C.c_int
    L.bark_b200_get_tokens.argtypes = [vp, C.c_int, i32p, C.c_int]
    L.bark_b200_set_tokens.argtypes = [vp, C.c_int, i32p, C.c_int]
    L.bark_b200_get_stats.argtypes = [vp, C.POINTER(BarkStatistics), C.c_void_p]
    L.bark_b200_get_hparams.argtypes = [vp, C.c_int, i32p]
    L.bark_b200_kernel_launches.restype = C.c_ulonglong
    L.bark_b200_layernorm_fallbacks.restype = C.c_uint
    L.bark_b200_layernorm_fallbacks.argtypes = [vp]
    L.bark_b200_profile_enable.argtypes = [C.c_int]
    L.bark_b200_profile_report.restype = C.c_int
    L.bark_b200_profile_report.argtypes = [C.c_char_p, C.c_int]
    L.bark_b200_io_counters.argtypes = [C.POINTER(C.c_ulonglong), C.POINTER(C.c_ulonglong), C.c_int]
    L.bark_b200_decode_timing.restype = C.c_int
    L.bark_b200_decode_timing.argtypes = [vp, C.c_void_p, C.c_int]
    L.bark_b200_shard_init.restype = C.c_int
    L.bark_b200_shard_init.argtypes = [vp, C.c_int, C.c_int, vp]
    L.bark_b200_shard_connect.restype = C.c_int
    L.bark_b200_shard_connect.argtypes = [vp, vp]
    L.bark_b200_shard_nvlink_bytes.restype = C.c_ulonglong
    L.bark_b200_shard_nvlink_bytes.argtypes = [vp, C.c_int]
    L.bark_b200_fast_mode.restype = C.c_int
    L.bark_b200_fast_mode.argtypes = [vp]
    L.bark_b200_fast_gemm.restype = C.c_int
    L.bark_b200_fast_gemm.argtypes = [vp, vp, vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int]
    L.bark_b200_fast_convert.restype = C.c_int
    L.bark_b200_fast_convert.argtypes = [C.c_int, vp, C.c_int, C.c_int, vp, C.POINTER(C.c_int)]
    L.bark_b200_fast_attention.restype = C.c_int
    L.bark_b200_fast_attention.argtypes = [vp, vp, vp, vp, C.c_int, C.c_int, C.c_int]
    L.bark_b200_parity_attention.restype = C.c_int
    L.bark_b200_parity_attention.argtypes = [vp, vp, vp, vp] + [C.c_int] * 7
    L.bark_b200_batch_attention.restype = C.c_int
    L.bark_b200_batch_attention.argtypes = [f32p, f32p, f32p, f32p, f32p, i32p] + [C.c_int] * 5 + [vp]
    L.bark_b200_parity_gemm.restype = C.c_int
    L.bark_b200_parity_gemm.argtypes = [vp, vp, vp] + [C.c_int] * 6 + [vp]
    L.bark_b200_quant_matmul.restype = C.c_int
    L.bark_b200_quant_matmul.argtypes = [C.c_int, vp, vp, vp] + [C.c_int] * 5 + [vp, vp, vp, vp]
    L.bark_b200_codec_conv1d.restype = C.c_int
    L.bark_b200_codec_conv1d.argtypes = [f32p, C.c_int, vp, C.c_int, vp, f32p] + [C.c_int] * 4 + [f32p, f32p]
    L.bark_b200_codec_convtr1d.restype = C.c_int
    L.bark_b200_codec_convtr1d.argtypes = [f32p, C.c_int, vp, C.c_int, vp, f32p, C.c_int, C.c_int, f32p]
    L.bark_b200_codec_lstm.restype = C.c_int
    L.bark_b200_codec_lstm.argtypes = [f32p, C.c_int, vp, C.c_int, vp, vp, f32p, f32p, f32p, f32p]
    L.bark_b200_codec_conv1d_window.restype = C.c_int
    L.bark_b200_codec_conv1d_window.argtypes = [f32p, C.c_int, vp, C.c_int, vp, vp, vp, vp, f32p] + [C.c_int] * 4 + [f32p, f32p]
    L.bark_b200_codec_convtr1d_window.restype = C.c_int
    L.bark_b200_codec_convtr1d_window.argtypes = [f32p, C.c_int, vp, C.c_int, vp, vp, vp, vp, f32p, C.c_int, C.c_int, f32p]
    L.bark_b200_codec_lstm_state.restype = C.c_int
    L.bark_b200_codec_lstm_state.argtypes = [f32p, C.c_int, vp, C.c_int, vp, vp, f32p, f32p, f32p, f32p, f32p]
    L.bark_b200_encodec_stream_open.restype = vp
    L.bark_b200_encodec_stream_open.argtypes = [vp, C.c_int]
    for n in ("bark_b200_encodec_stream_push", "bark_b200_encodec_stream_read"):
        getattr(L, n).restype = C.c_int
        getattr(L, n).argtypes = [vp, vp, C.c_int]
    L.bark_b200_encodec_stream_push_batch.restype = C.c_int
    L.bark_b200_encodec_stream_push_batch.argtypes = [vp, vp, vp, C.c_int]
    for n in ("bark_b200_encodec_stream_finish", "bark_b200_encodec_stream_codebooks"):
        getattr(L, n).restype = C.c_int
        getattr(L, n).argtypes = [vp]
    L.bark_b200_encodec_stream_ready.restype = C.c_longlong
    L.bark_b200_encodec_stream_ready.argtypes = [C.c_int, C.c_longlong]
    L.bark_b200_encodec_stream_open_resampled.restype = vp
    L.bark_b200_encodec_stream_open_resampled.argtypes = [vp, C.c_int, C.c_int, C.c_int]
    L.bark_b200_encodec_stream_ready_resampled.restype = C.c_longlong
    L.bark_b200_encodec_stream_ready_resampled.argtypes = [C.c_int, C.c_int, C.c_longlong]
    L.bark_b200_resample_window.restype = C.c_int
    L.bark_b200_resample_window.argtypes = [f32p, vp, vp, vp, vp, vp, vp, vp, vp, C.c_int, f32p]
    L.bark_b200_encodec_stream_close.restype = None
    L.bark_b200_encodec_stream_close.argtypes = [vp]
    L.bark_b200_codec_rvq_decode.restype = C.c_int
    L.bark_b200_codec_rvq_decode.argtypes = [i32p, C.c_int, vp, C.c_int, f32p, C.c_int, C.c_int, f32p]
    L.bark_b200_device_math.restype = C.c_int
    L.bark_b200_device_math.argtypes = [C.c_int, C.c_uint32, C.c_uint32, C.c_uint32, f32p]
    L.bark_b200_parity_rows.restype = C.c_int
    L.bark_b200_parity_rows.argtypes = [C.c_int, C.c_int, vp, C.c_int, C.c_int, vp, vp, vp, C.POINTER(C.c_uint)]
    L.bark_b200_sample_given_u.restype = C.c_int
    L.bark_b200_sample_given_u.argtypes = [f32p, C.c_int, C.c_int, C.c_float, vp, C.c_int, i32p, i32p, i32p, f32p]
    L.bark_b200_generate_batch.restype = C.c_bool
    L.bark_b200_generate_batch.argtypes = [vp, C.POINTER(C.c_char_p), C.POINTER(C.c_uint32), C.c_int, C.c_int]
    L.bark_b200_batch_audio.restype = C.c_int
    L.bark_b200_batch_audio.argtypes = [vp, C.c_int, f32p, C.c_int]
    L.bark_b200_batch_tokens.restype = C.c_int
    L.bark_b200_batch_tokens.argtypes = [vp, C.c_int, C.c_int, i32p, C.c_int]
    L.bark_b200_gpt_eval_slot.restype = C.c_int
    L.bark_b200_gpt_eval_slot.argtypes = [vp, C.c_int, C.c_int, i32p, C.c_int, C.POINTER(C.c_int), C.c_int, f32p]
    L.bark_b200_gpt_step_batch.restype = C.c_int
    L.bark_b200_gpt_step_batch.argtypes = [vp, C.c_int, C.c_int, i32p, i32p, i32p, f32p]
    L.bark_b200_set_sampling.restype = C.c_int
    L.bark_b200_set_sampling.argtypes = [vp, C.c_int, C.POINTER(SamplingStruct)]
    L.bark_b200_sample_filtered_given_u.restype = C.c_int
    L.bark_b200_sample_filtered_given_u.argtypes = [f32p, C.c_int, C.c_int, C.c_float, C.POINTER(SamplingStruct), vp, C.c_int, i32p, i32p, i32p, f32p, i32p]
    L.bark_b200_set_history_prompt.restype = C.c_int
    L.bark_b200_set_history_prompt.argtypes = [vp, C.POINTER(HistoryPromptStruct)]
    L.bark_b200_generate_batch_prompted.restype = C.c_bool
    L.bark_b200_generate_batch_prompted.argtypes = [vp, C.POINTER(C.c_char_p), C.POINTER(C.c_uint32), C.POINTER(C.POINTER(HistoryPromptStruct)),
                                                    C.c_int, C.c_int]
    for n in ("bark_b200_encodec_compress_batch", "bark_b200_encodec_decompress_batch", "bark_b200_encodec_reconstruct_batch"):
        getattr(L, n).restype = C.c_bool
        getattr(L, n).argtypes = [vp, vp, vp, C.c_int]
    for n in ("bark_b200_encodec_batch_codes", "bark_b200_encodec_batch_audio"):
        getattr(L, n).restype = C.c_int
        getattr(L, n).argtypes = [vp, C.c_int, vp, C.c_int]
    for n in ("bark_b200_encodec_compress_resampled", "bark_b200_encodec_reconstruct_resampled"):
        getattr(L, n).restype = C.c_bool
        getattr(L, n).argtypes = [vp, f32p, C.c_int, C.c_int, C.c_int]
    for n in ("bark_b200_encodec_compress_batch_resampled", "bark_b200_encodec_reconstruct_batch_resampled"):
        getattr(L, n).restype = C.c_bool
        getattr(L, n).argtypes = [vp, vp, vp, vp, vp, C.c_int]
    L.bark_b200_encodec_encode_resampled.restype = C.c_int
    L.bark_b200_encodec_encode_resampled.argtypes = [vp, f32p, C.c_int, C.c_int, C.c_int, i32p, C.c_int, f32p, C.c_int]
    L.bark_b200_resample.restype = C.c_int
    L.bark_b200_resample.argtypes = [f32p, C.c_int, C.c_int, C.c_int, C.c_int, f32p, C.c_int]
    L.bark_b200_set_tokenizer.restype = C.c_int
    L.bark_b200_set_tokenizer.argtypes = [vp, C.c_int]
    L.bark_b200_text_ids.restype = C.c_int
    L.bark_b200_text_ids.argtypes = [vp, C.c_int, C.c_char_p, i32p, C.c_int]
    L.bark_b200_bert_tokenize.restype = C.c_int
    L.bark_b200_bert_tokenize.argtypes = [C.POINTER(C.c_char_p), C.c_int, C.c_char_p, i32p, C.c_int]
    L.bark_b200_set_long_form.restype = C.c_int
    L.bark_b200_set_long_form.argtypes = [vp, C.POINTER(LongFormStruct)]
    L.bark_b200_long_chunks.restype = C.c_int
    L.bark_b200_long_chunks.argtypes = [vp]
    L.bark_b200_long_chunk_text.restype = C.c_int
    L.bark_b200_long_chunk_text.argtypes = [vp, C.c_int, C.c_char_p, C.c_int]
    L.bark_b200_long_chunk_tokens.restype = C.c_int
    L.bark_b200_long_chunk_tokens.argtypes = [vp, C.c_int, C.c_int, i32p, C.c_int]
    L.bark_b200_split_text.restype = C.c_int
    L.bark_b200_split_text.argtypes = [C.POINTER(C.c_char_p), C.c_int, C.c_int, C.c_char_p, C.c_int, i32p, C.c_int]
    L.ggml_time_us.restype = C.c_int64
    L.encodec_load_model.restype = vp
    L.encodec_load_model.argtypes = [C.c_char_p, C.c_int, C.c_int]
    L.encodec_set_target_bandwidth.argtypes = [vp, C.c_int]
    L.encodec_set_sample_rate.argtypes = [vp, C.c_int]
    for n in ("encodec_reconstruct_audio", "encodec_compress_audio"):
        getattr(L, n).restype = C.c_bool
        getattr(L, n).argtypes = [vp, f32p, C.c_int, C.c_int]
    L.encodec_decompress_audio.restype = C.c_bool
    L.encodec_decompress_audio.argtypes = [vp, i32p, C.c_int, C.c_int]
    L.encodec_get_audio.restype = C.POINTER(C.c_float)
    L.encodec_get_codes.restype = C.POINTER(C.c_int32)
    L.encodec_get_statistics.restype = C.POINTER(EncodecStatistics)
    for n in ("encodec_get_audio_size", "encodec_get_codes_size"):
        getattr(L, n).restype = C.c_int
    for n in ("encodec_get_audio", "encodec_get_audio_size", "encodec_get_codes", "encodec_get_codes_size", "encodec_get_statistics",
              "encodec_reset_statistics", "encodec_free"):
        getattr(L, n).argtypes = [vp]
    _lib = L
    return L


def _p(a: np.ndarray):
    return a.ctypes.data_as(C.c_void_p)


CODEC_RATE = 24000          # the EnCodec model's sample rate


def _frames(audio):
    """(interleaved float32 frames [n][C] flattened, n, C) of mono samples [n] or of [channels][n_frames], the layout torchaudio.load
    returns and upstream EnCodec's convert_audio takes."""
    a = np.asarray(audio, np.float32)
    if a.ndim == 1:
        return np.ascontiguousarray(a), a.size, 1
    if a.ndim != 2:
        raise ValueError(f"audio of shape {a.shape}: [n_frames] or [channels][n_frames]")
    return np.ascontiguousarray(a.T).ravel(), a.shape[1], a.shape[0]


def resampled_length(n_frames: int, sr: int, new_sr: int = CODEC_RATE) -> int:
    """L = ceil(new_sr n / sr), exactly: the samples of n frames at sr resampled to new_sr (0 for a rate below 1, which the library
    refuses)."""
    if sr < 1 or new_sr < 1:
        return 0
    g = math.gcd(sr, new_sr)
    return -(-(new_sr // g) * n_frames // (sr // g))


def resample(audio, sr: int, new_sr: int) -> np.ndarray:
    """audio (mono [n] or [channels][n]) at sr Hz down-mixed and resampled to new_sr Hz on the GPU (bark_b200_resample, DESIGN.md
    §16): torchaudio.functional.resample's default filter with an exact summation order, bit-reproducible.  Both rates in [4000,
    384000].  Returns float32 [ceil(new_sr n / sr)]."""
    x, n, ch = _frames(audio)
    out = np.zeros(max(resampled_length(n, int(sr), int(new_sr)), 1), np.float32)
    r = lib().bark_b200_resample(_p(x), n, ch, int(sr), int(new_sr), _p(out), out.size)
    if r < 0:
        raise RuntimeError(f"bark_b200_resample ({n} frames of {ch} channels, {sr} -> {new_sr} Hz) failed (see stderr)")
    return out[:r]


TOKENIZERS = {"reference": 0, "bert": 1}      # BARK_B200_TOKENIZER_REFERENCE / _BERT (include/bark_b200.h, DESIGN.md §17)


def _tokenizer_kind(name: str) -> int:
    if name not in TOKENIZERS:
        raise ValueError(f"tokenizer {name!r}: 'reference' (bark.cpp's, the default) or 'bert' (upstream Bark's)")
    return TOKENIZERS[name]


def _text_bytes(text) -> bytes:
    """text (str, or UTF-8 bytes) as the C string the library reads, which ends at a NUL: a text holding one is refused here."""
    b = text if isinstance(text, bytes) else text.encode()
    if b"\0" in b:
        raise ValueError("text holds a NUL byte, where the library's C string would end")
    return b


def _ids(run, what: str) -> np.ndarray:
    """The ids a (out, cap) -> count call returns, asked for twice: once for the count, once for the ids."""
    n = run(None, 0)
    if n < 0:
        raise ValueError(f"{what} refused the text (see stderr)")
    a = np.zeros(max(n, 1), np.int32)
    run(_p(a), n)
    return a[:n]


def bert_tokenize(vocab, text) -> np.ndarray:
    """Upstream Bark's text ids (bark_b200_bert_tokenize, DESIGN.md §17) of text (str, or UTF-8 bytes) over vocab, a list of WordPiece
    entries whose ids are their indices (a later duplicate wins); no context or device needed.  Raises ValueError for invalid UTF-8."""
    entries = [_text_bytes(v) for v in vocab]
    arr = (C.c_char_p * max(len(entries), 1))(*entries)
    t = _text_bytes(text)
    return _ids(lambda out, cap: lib().bark_b200_bert_tokenize(arr, len(entries), t, out, cap), "bark_b200_bert_tokenize")


def _normalize_whitespace(text: str) -> str:
    """Upstream Bark's _normalize_whitespace: every run of \\s one space, both ends stripped (long-form rule 1)."""
    return re.sub(r"\s+", " ", text).strip()


def split_text(vocab, text, tokenizer: str = "reference", max_chunk_ids: int = 48) -> list:
    """The chunks long-form generation makes of text (str, or UTF-8 bytes) under tokenizer over vocab, a list of WordPiece entries
    whose ids are their indices (bark_b200_split_text, DESIGN.md §18); no context or device needed.  Returns the chunk texts, pieces of
    the whitespace-normalised text.  Raises ValueError for a text or budget the library refuses."""
    entries = [_text_bytes(v) for v in vocab]
    arr = (C.c_char_p * max(len(entries), 1))(*entries)
    t = _text_bytes(text)
    run = lambda out, cap: lib().bark_b200_split_text(arr, len(entries), _tokenizer_kind(tokenizer), t, int(max_chunk_ids), out, cap)
    n = run(None, 0)
    if n < 0:
        raise ValueError("bark_b200_split_text refused the text (see stderr)")
    b = np.zeros((n, 2), np.int32)
    run(_p(b), n)
    norm = _normalize_whitespace(t.decode()).encode()
    return [norm[s:e].decode() for s, e in b]


class Bark:
    """One bark_context on one GPU.  Mirrors how examples/main/main.cpp uses bark.h."""

    def __init__(self, model_path: str, seed: int = 0, n_steps_text_encoder: int | None = None, temp=None, fine_temp=None,
                 min_eos_p=None, device: int | None = None, progress=None, tokenizer: str | None = None):
        """tokenizer: "reference" (bark.cpp's) or "bert" (upstream Bark's, for text in any of its languages); None keeps what
        BARK_B200_TOKENIZER chose at load (the reference's when it is unset)."""
        L = lib()
        p = L.bark_context_default_params()
        if n_steps_text_encoder is not None:
            p.n_steps_text_encoder = n_steps_text_encoder
        if temp is not None:
            p.temp = temp
        if fine_temp is not None:
            p.fine_temp = fine_temp
        if min_eos_p is not None:
            p.min_eos_p = min_eos_p
        self._cb = PROGRESS_CB(progress) if progress else PROGRESS_CB()
        p.progress_callback = self._cb
        if device is not None:
            L.bark_b200_set_device(device)
        self.params = p
        self.ctx = L.bark_load_model(os.fsencode(model_path), p, seed)
        if not self.ctx:
            raise RuntimeError(f"bark_load_model failed for {model_path} (see stderr); no CPU fallback exists")
        self.ctx = C.c_void_p(self.ctx)
        self.tokenizer = os.environ.get("BARK_B200_TOKENIZER") or "reference"     # what bark_load_model read (it refuses anything else)
        voice = os.environ.get("BARK_B200_LONG_FORM") or "off"                      # likewise
        self.long_form = None if voice == "off" else dict(voice=voice, **LONG_FORM_DEFAULTS)
        if tokenizer is not None:
            self.set_tokenizer(tokenizer)

    def close(self):
        if getattr(self, "ctx", None):
            lib().bark_free(self.ctx)
            self.ctx = None

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    # ---- bark.h ----
    def generate(self, text: str, n_threads: int = 1, history_prompt=None) -> np.ndarray:
        """The waveform for `text`.  history_prompt (a voice file or mapping, see load_history_prompt) conditions this call only: it
        is set before and cleared after, also on failure.  Without it the context's prompt (set_history_prompt) applies."""
        if history_prompt is not None:
            self.set_history_prompt(history_prompt)
            try:
                return self.generate(text, n_threads)
            finally:
                self.set_history_prompt(None)
        if not lib().bark_generate_audio(self.ctx, text.encode(), n_threads):
            raise RuntimeError("bark_generate_audio failed")
        n = lib().bark_get_audio_data_size(self.ctx)
        return np.ctypeslib.as_array(lib().bark_get_audio_data(self.ctx), shape=(n,)).copy()

    def set_history_prompt(self, prompt):
        """Speaker history prompt of the later generations on this context (bark_b200_set_history_prompt); None clears it.  Raises
        ValueError for a prompt the library rejects (the message is on stderr); the previous prompt then stays."""
        if prompt is None:
            lib().bark_b200_set_history_prompt(self.ctx, None)
            return
        st, _keep = _history_struct(prompt)
        if not lib().bark_b200_set_history_prompt(self.ctx, C.byref(st)):
            raise ValueError("bark_b200_set_history_prompt rejected the prompt (see stderr)")

    def set_long_form(self, voice: str | None = "chain", max_chunk_ids: int = 48, gap_samples: int = 6000):
        """Long-form generation for the later generate calls on this context (bark_b200_set_long_form, DESIGN.md §18): the text split
        into sentences, each generated on a prompt that keeps one voice ("chain": the previous chunk's ids; "fixed": the context's
        history prompt, or none), joined with gap_samples zeros.  voice None turns it off.  Raises ValueError for settings the library
        rejects; the previous ones then stay."""
        if voice is None:
            lib().bark_b200_set_long_form(self.ctx, None)
            self.long_form = None
            return
        if voice not in VOICES:
            raise ValueError(f"voice {voice!r}: 'chain', 'fixed' or None")
        st = LongFormStruct(VOICES[voice], int(max_chunk_ids), int(gap_samples))
        if not lib().bark_b200_set_long_form(self.ctx, C.byref(st)):
            raise ValueError(f"bark_b200_set_long_form rejected max_chunk_ids={max_chunk_ids!r}, gap_samples={gap_samples!r} (see stderr)")
        self.long_form = dict(voice=voice, max_chunk_ids=int(max_chunk_ids), gap_samples=int(gap_samples))

    def long_chunks(self) -> list:
        """The chunks of the last long-form generation ([] after a generation without it): per chunk a dict of its text, its ids as
        tokens() shapes them (prompt: the 513 prompt ids, semantic, coarse [T][2], fine [T][8]), and start / n_samples, its span in the
        joined waveform (with the gap of the current long-form settings)."""
        L = lib()
        gap = self.long_form["gap_samples"] if self.long_form else 0
        out, start = [], 0
        for k in range(L.bark_b200_long_chunks(self.ctx)):
            t = C.create_string_buffer(max(L.bark_b200_long_chunk_text(self.ctx, k, None, 0), 1))
            n_text = L.bark_b200_long_chunk_text(self.ctx, k, t, len(t))
            ids = {}
            for stage, name in ((3, "prompt"), (0, "semantic"), (1, "coarse"), (2, "fine")):
                a = _ids(lambda o, cap: L.bark_b200_long_chunk_tokens(self.ctx, k, stage, o, cap), "bark_b200_long_chunk_tokens")
                ids[name] = a.reshape(-1, 2) if stage == 1 else a.reshape(-1, 8) if stage == 2 else a
            n = 320 * ids["fine"].shape[0]
            out.append(dict(text=t.raw[:n_text].decode(), **ids, start=start, n_samples=n))
            start += n + gap
        return out

    def set_sampling(self, stage: str, top_k=None, top_p=None):
        """Top-k / top-p filter of the "semantic" or "coarse" stage for the later generations and batches on this context
        (bark_b200_set_sampling, DESIGN.md §14).  top_k: None or 0 for off, else k >= 1; top_p: None for off, else in [0, 1].  Both None
        turn the stage's filter off.  Raises ValueError for settings the library rejects; the previous ones then stay."""
        if stage not in SAMPLING_STAGES:
            raise ValueError(f"stage {stage!r}: 'semantic' or 'coarse' (the fine stage has no filter)")
        st = _sampling_struct(top_k, top_p)
        if not lib().bark_b200_set_sampling(self.ctx, SAMPLING_STAGES[stage], C.byref(st)):
            raise ValueError(f"bark_b200_set_sampling rejected top_k={top_k!r}, top_p={top_p!r} (see stderr)")

    def last_generation_prompt(self) -> dict:
        """The last generation's ids as a history prompt: semantic_prompt [n], coarse_prompt [2][T], fine_prompt [8][T].  np.savez of it
        writes a voice file upstream Bark also reads."""
        return {"semantic_prompt": self.tokens(0).copy(), "coarse_prompt": np.ascontiguousarray(self.tokens(1).T),
                "fine_prompt": np.ascontiguousarray(self.tokens(2).T)}

    @property
    def load_time_us(self):
        return lib().bark_get_load_time(self.ctx)

    @property
    def eval_time_us(self):
        return lib().bark_get_eval_time(self.ctx)

    # ---- bark_b200.h ----
    def hparams(self, which: int) -> np.ndarray:
        a = np.zeros(10, np.int32)
        lib().bark_b200_get_hparams(self.ctx, which, _p(a))
        return a

    def tokens(self, stage: int) -> np.ndarray:
        n = lib().bark_b200_get_tokens(self.ctx, stage, None, 0)
        a = np.zeros(max(n, 1), np.int32)
        lib().bark_b200_get_tokens(self.ctx, stage, _p(a), n)
        a = a[:n]
        return a.reshape(-1, 2) if stage == 1 else a.reshape(-1, 8) if stage == 2 else a

    def set_tokens(self, stage: int, arr):
        a = np.ascontiguousarray(arr, np.int32).ravel()
        lib().bark_b200_set_tokens(self.ctx, stage, _p(a), a.size)

    def tokenize(self, text: str) -> np.ndarray:
        a = np.zeros(513, np.int32)
        lib().bark_b200_tokenize(self.ctx, text.encode(), _p(a))
        return a

    def set_tokenizer(self, kind: str):
        """The text tokenizer of the later generations and batches on this context (bark_b200_set_tokenizer): "reference" or "bert"."""
        if not lib().bark_b200_set_tokenizer(self.ctx, _tokenizer_kind(kind)):
            raise ValueError(f"bark_b200_set_tokenizer rejected {kind!r} (see stderr)")
        self.tokenizer = kind

    def text_ids(self, text, tokenizer: str | None = None) -> np.ndarray:
        """The raw WordPiece ids of text (str, or UTF-8 bytes) under tokenizer (None: this context's), before truncation, offset and
        padding (bark_b200_text_ids).  Raises ValueError for a text the tokenizer refuses."""
        k = _tokenizer_kind(tokenizer or self.tokenizer)
        t = _text_bytes(text)
        return _ids(lambda out, cap: lib().bark_b200_text_ids(self.ctx, k, t, out, cap), "bark_b200_text_ids")

    def gpt_eval(self, which: int, tokens, n_past: int, merge_ctx: bool):
        t = np.ascontiguousarray(tokens, np.int32)
        out = np.zeros(int(self.hparams(which)[6]), np.float32)
        np_ = C.c_int(n_past)
        if not lib().bark_b200_gpt_eval(self.ctx, which, _p(t), t.size, C.byref(np_), int(merge_ctx), _p(out)):
            raise RuntimeError("bark_b200_gpt_eval failed")
        return out, np_.value

    def gpt_eval_slot(self, which: int, slot: int, tokens, n_past: int, merge_ctx: bool):
        """gpt_eval on batch slot `slot`'s KV cache (0..7) instead of the model's own; returns (logits, n_past)."""
        t = np.ascontiguousarray(tokens, np.int32)
        out = np.zeros(int(self.hparams(which)[6]), np.float32)
        np_ = C.c_int(n_past)
        if not lib().bark_b200_gpt_eval_slot(self.ctx, which, slot, _p(t), t.size, C.byref(np_), int(merge_ctx), _p(out)):
            raise RuntimeError("bark_b200_gpt_eval_slot failed")
        return out, np_.value

    def gpt_step_batch(self, which: int, slots, tokens, n_past):
        """One batched decode step: row r feeds tokens[r] at position n_past[r] through slot slots[r]'s cache.
        Returns (logits [B][n_out], the advanced n_past)."""
        sl = np.ascontiguousarray(slots, np.int32); t = np.ascontiguousarray(tokens, np.int32)
        npa = np.array(n_past, np.int32, copy=True)
        assert sl.size == t.size == npa.size
        out = np.zeros((sl.size, int(self.hparams(which)[6])), np.float32)
        if not lib().bark_b200_gpt_step_batch(self.ctx, which, sl.size, _p(sl), _p(t), _p(npa), _p(out)):
            raise RuntimeError("bark_b200_gpt_step_batch failed")
        return out, npa

    def generate_batch(self, texts, seeds, n_threads: int = 1, history_prompts=None) -> list:
        """Up to 8 prompts decoded together; item i equals a fresh context's generate(texts[i], history_prompt=history_prompts[i])
        with seed seeds[i].  history_prompts: None, or one prompt or None per item; the context's own prompt does not apply.
        Returns the waveforms; batch_tokens(i, stage) gives the ids."""
        n = len(texts)
        if len(seeds) != n:
            raise RuntimeError(f"generate_batch: {n} prompts but {len(seeds)} seeds")
        arr = (C.c_char_p * max(n, 1))(*[t.encode() for t in texts])
        sd = (C.c_uint32 * max(n, 1))(*[int(s) for s in seeds])
        if history_prompts is None:
            ok = lib().bark_b200_generate_batch(self.ctx, arr, sd, n, n_threads)
        else:
            if len(history_prompts) != n:
                raise RuntimeError(f"generate_batch: {n} prompts but {len(history_prompts)} history prompts")
            structs = [None if p is None else _history_struct(p) for p in history_prompts]
            ptrs = (C.POINTER(HistoryPromptStruct) * max(n, 1))(*[C.pointer(s[0]) if s else None for s in structs])
            ok = lib().bark_b200_generate_batch_prompted(self.ctx, arr, sd, ptrs, n, n_threads)
        if not ok:
            raise RuntimeError("bark_b200_generate_batch failed")
        out = []
        for i in range(n):
            m = lib().bark_b200_batch_audio(self.ctx, i, None, 0)
            a = np.zeros(max(m, 1), np.float32)
            lib().bark_b200_batch_audio(self.ctx, i, _p(a), m)
            out.append(a[:m])
        return out

    def batch_tokens(self, i: int, stage: int) -> np.ndarray:
        """Ids of item i of the last batch, shaped like tokens(stage)."""
        n = lib().bark_b200_batch_tokens(self.ctx, i, stage, None, 0)
        if n < 0:
            raise IndexError(f"no batch item {i}")
        a = np.zeros(max(n, 1), np.int32)
        lib().bark_b200_batch_tokens(self.ctx, i, stage, _p(a), n)
        a = a[:n]
        return a.reshape(-1, 2) if stage == 1 else a.reshape(-1, 8) if stage == 2 else a

    def fine_eval(self, in_buffer, nn: int) -> np.ndarray:
        t = np.ascontiguousarray(in_buffer, np.int32)
        assert t.size == 8 * 1024
        out = np.zeros((1024, int(self.hparams(2)[6])), np.float32)
        if not lib().bark_b200_fine_eval(self.ctx, _p(t), nn, _p(out)):
            raise RuntimeError("bark_b200_fine_eval failed")
        return out

    def encodec_decode(self, codes_8xT) -> np.ndarray:
        c = np.ascontiguousarray(codes_8xT, np.int32)
        T = c.shape[1]
        out = np.zeros(320 * T, np.float32)
        n = lib().bark_b200_encodec_decode(self.ctx, _p(c), T, _p(out), out.size)
        if n < 0:
            raise RuntimeError("bark_b200_encodec_decode failed")
        return out[:n]

    def encodec_encode(self, audio, return_latent: bool = False, sample_rate: int | None = None):
        """Mono 24 kHz float32 samples (finite, at least 1921) -> codes [8][T] int32, T = ceil(n / 320), the layout encodec_decode
        takes; with return_latent also the encoder output before quantisation, [128][T] float32.  With sample_rate, audio is mono [n] or
        [channels][n] at that rate, down-mixed and resampled to 24 kHz on the GPU first (bark_b200_encodec_encode_resampled): a fine
        prompt from a speaker clip; T then counts the resampled samples."""
        if sample_rate is None:
            a = np.ascontiguousarray(audio, np.float32).ravel()
            n = a.size
        else:
            a, nf, ch = _frames(audio)
            n = resampled_length(nf, int(sample_rate))
        T = (n + 319) // 320
        codes = np.zeros((8, max(T, 1)), np.int32); lat = np.zeros((128, max(T, 1)), np.float32)
        if sample_rate is None:
            r = lib().bark_b200_encodec_encode(self.ctx, _p(a), a.size, _p(codes), codes.size, _p(lat), lat.size)
        else:
            r = lib().bark_b200_encodec_encode_resampled(self.ctx, _p(a), nf, ch, int(sample_rate), _p(codes), codes.size, _p(lat), lat.size)
        if r < 0:
            raise RuntimeError(f"bark_b200_encodec_encode{'' if sample_rate is None else '_resampled'} failed (see stderr)")
        assert r == T, (r, T)
        return (codes, lat) if return_latent else codes

    def sample(self, which: int, logits, temp: float):
        l = np.ascontiguousarray(logits, np.float32)
        e = C.c_float(0)
        return lib().bark_b200_sample(self.ctx, which, _p(l), l.size, temp, C.byref(e)), e.value

    def sample_rows(self, logits_rows, temp: float):
        """Device sampler over [rows][n] logits; returns (tokens, eos_p, n_rows_replayed_on_host)."""
        l = np.ascontiguousarray(logits_rows, np.float32)
        rows, n = l.shape
        tok = np.zeros(rows, np.int32); eos = np.zeros(rows, np.float32)
        r = lib().bark_b200_sample_rows(self.ctx, _p(l), n, rows, temp, _p(tok), _p(eos))
        if r < 0:
            raise RuntimeError("bark_b200_sample_rows failed")
        return tok, eos, r

    def reseed(self, seed: int):
        lib().bark_b200_reseed(self.ctx, seed)

    def forward(self, stage: int):
        f = [lib().bark_b200_forward_text_encoder, lib().bark_b200_forward_coarse_encoder, lib().bark_b200_forward_fine_encoder][stage]
        if not f(self.ctx, 1):
            raise RuntimeError("stage failed")

    def stats(self):
        s = BarkStatistics()
        pm = np.zeros(9, np.int64)
        lib().bark_b200_get_stats(self.ctx, C.byref(s), _p(pm))
        return s, pm.reshape(3, 3)

    def shard_init(self, rank: int, world: int) -> bytes:
        """Row-sharded fine stage, step 1: returns this rank's 64-byte CUDA IPC handle."""
        h = C.create_string_buffer(64)
        if not lib().bark_b200_shard_init(self.ctx, rank, world, C.cast(h, C.c_void_p)):
            raise RuntimeError("bark_b200_shard_init failed")
        return h.raw

    def shard_connect(self, all_handles: bytes):
        """step 2: all ranks' handles, rank order (world * 64 bytes)."""
        buf = C.create_string_buffer(all_handles, len(all_handles))
        if not lib().bark_b200_shard_connect(self.ctx, C.cast(buf, C.c_void_p)):
            raise RuntimeError("bark_b200_shard_connect failed")

    def shard_nvlink_bytes(self, reset: bool = False) -> int:
        return int(lib().bark_b200_shard_nvlink_bytes(self.ctx, int(reset)))

    @property
    def fast_mode(self) -> bool:
        return bool(lib().bark_b200_fast_mode(self.ctx))

    def layernorm_fallbacks(self) -> int:
        return int(lib().bark_b200_layernorm_fallbacks(self.ctx))


FAST_EPILOGUES = {"f32": 0, "resid": 1, "gelu16": 2, "qkv16": 4}      # FEPI_* (csrc/gpt_kernels.h)


class GuardBandError(RuntimeError):
    """The GEMM stored outside its output."""


def _gemm(what: str, run, epilogue: str, resid: np.ndarray | None, shape, dtype, parts=None):
    """What the GEMM wrappers share: run(out) calls the hook on out, a float32 copy of resid [M][N] for the "resid" epilogue, else
    zeros of shape and dtype.  Returns (out, the hook's return value); with parts, out is split into arrays of those shapes (the Q / K
    / V blocks).  Raises GuardBandError when the hook stored outside its output, RuntimeError when it failed."""
    if epilogue == "resid":
        out = np.array(resid, np.float32, order="C", copy=True)
        assert out.shape == shape, out.shape
    else:
        out = np.zeros(shape, dtype)
    r = run(out)
    if r == -1:
        raise GuardBandError(f"{what} wrote outside its output")
    if r <= 0:
        raise RuntimeError(f"{what} failed")
    if parts:
        flat, o, blocks = out.reshape(-1), 0, []
        for p in parts:
            blocks.append(flat[o:o + p[0] * p[1]].reshape(p))
            o += p[0] * p[1]
        out = tuple(blocks)
    return out, r


def fast_gemm(A: np.ndarray, W: np.ndarray, epilogue: str = "f32", bn: int = 0, resid: np.ndarray | None = None, return_bn: bool = False):
    """A W^T on the wgmma path through one of the fine pass's epilogues; A [M][K], W [N][K] float16, K % 64 == 0.

    Returns float32 [M][N] for "f32" and for "resid" (resid [M][N] float32 + A W^T), float16 [M][N] for "gelu16", and for "qkv16"
    (N % 6 == 0) the pair (float16 [M][2N/3], the V columns transposed: float16 [N/3][M]).  bn = 0 lets the cost model pick the tile
    width, 64 / 128 / 256 force it; with return_bn the result is (outputs, the tile width that ran)."""
    A = np.ascontiguousarray(A, np.float16); W = np.ascontiguousarray(W, np.float16)
    M, K = A.shape; N = W.shape[0]
    assert W.shape[1] == K, (A.shape, W.shape)
    if epilogue == "qkv16":
        assert N % 6 == 0, N
    out, r = _gemm(f"bark_b200_fast_gemm ({epilogue}, {M}x{N}x{K}, bn {bn})",
                   lambda out: lib().bark_b200_fast_gemm(_p(A), _p(W), _p(out), M, N, K, FAST_EPILOGUES[epilogue], bn), epilogue, resid,
                   (M, N), np.float16 if epilogue in ("gelu16", "qkv16") else np.float32, ((M, 2 * N // 3), (N // 3, M)) if epilogue == "qkv16" else None)
    return (out, r) if return_bn else out


def fast_attention(q: np.ndarray, k: np.ndarray, v: np.ndarray, n_head: int) -> np.ndarray:
    """Non-causal attention on the wgmma path; q, k, v [n][E] float16 -> [n][E] float16."""
    q, k, v = (np.ascontiguousarray(a, np.float16) for a in (q, k, v))
    n, E = q.shape
    out = np.zeros((n, E), np.float16)
    if not lib().bark_b200_fast_attention(_p(q), _p(k), _p(v), _p(out), n, E, n_head):
        raise RuntimeError("bark_b200_fast_attention failed")
    return out


ATTN_PATHS = {"auto": 0, "fused": 1, "tiled": 2}


def parity_attention(q: np.ndarray, k: np.ndarray, v: np.ndarray, n_head: int, n_past: int = 0, causal: bool = False, path: str = "auto") -> np.ndarray:
    """Bit-exact multi-row attention; q [N][E], k, v [n_kv][E] float32 -> [N][E] float32.  causal masks key j for query i when
    j > n_past + i.  path: "auto" (what the library picks for the shape), "fused" or "tiled" (three kernels, few rows only)."""
    q, k, v = (np.ascontiguousarray(a, np.float32) for a in (q, k, v))
    N, E = q.shape
    n_kv = k.shape[0]
    assert k.shape == v.shape == (n_kv, E), (q.shape, k.shape, v.shape)
    out = np.zeros((N, E), np.float32)
    if not lib().bark_b200_parity_attention(_p(q), _p(k), _p(v), _p(out), N, n_kv, n_past, E, n_head, int(causal), ATTN_PATHS[path]):
        raise RuntimeError("bark_b200_parity_attention failed")
    return out


BATCH_ACTS = {"f32": 0, "f16": 1, "f32_gm": 2}      # the result's operand format: f32 rows, f16 / f32 group-major


def batch_attention(q: np.ndarray, k_new: np.ndarray, v_new: np.ndarray, k_cache: np.ndarray, v_cache: np.ndarray, pos, n_head: int,
                    act: str = "f32"):
    """The batched decode step's attention (attention_batch) for B <= 8 rows of different sequences; q, k_new, v_new [B][E] float32,
    k_cache, v_cache [B][cap][E] float32 (cap <= 1024), pos [B] with 0 <= pos[b] < cap.  Row b appends k_new[b] / v_new[b] at row
    pos[b] of its caches and attends over its pos[b] + 1 keys.  Returns (out [B][E], k_cache, v_cache): out float32, or float16 for
    act "f16" ("f32" is stored as f32 rows, "f16" / "f32_gm" as the group-major operand; every form comes back row-major), and copies
    of the caches after the call, NaN from row pos[b] + 1 on.  Raises GuardBandError when a store landed outside the output or a
    cache, RuntimeError when the hook failed or rejected its arguments."""
    q, k_new, v_new = (np.ascontiguousarray(a, np.float32) for a in (q, k_new, v_new))
    kc = np.array(k_cache, np.float32, order="C", copy=True); vc = np.array(v_cache, np.float32, order="C", copy=True)
    pos = np.ascontiguousarray(pos, np.int32)
    B, E = q.shape
    cap = kc.shape[1]
    assert k_new.shape == v_new.shape == (B, E) and kc.shape == vc.shape == (B, cap, E) and pos.shape == (B,), \
        (q.shape, k_new.shape, v_new.shape, kc.shape, vc.shape, pos.shape)
    out = np.zeros((B, E), np.float16 if act == "f16" else np.float32)
    r = lib().bark_b200_batch_attention(_p(q), _p(k_new), _p(v_new), _p(kc), _p(vc), _p(pos), B, cap, E, n_head, BATCH_ACTS[act], _p(out))
    if r == -1:
        raise GuardBandError(f"bark_b200_batch_attention ({B} rows, E {E}, {n_head} heads) wrote outside its output or a cache")
    if r != 1:
        raise RuntimeError(f"bark_b200_batch_attention ({B} rows, E {E}, {n_head} heads, cap {cap}) failed")
    return out, kc, vc


PARITY_EPILOGUES = {"store": 0, "resid": 1, "gelu": 2, "qkv": 3}      # EPI_* (csrc/gpt_kernels.h)


def _gelu_table(epilogue: str, gelu_tab):
    """gelu_tab as the hooks take it for the "gelu" epilogue, 65536 uint16 f16 bits; None for the others."""
    if epilogue != "gelu":
        return None
    tab = np.ascontiguousarray(gelu_tab, np.uint16)
    assert tab.shape == (65536,), tab.shape
    return tab


GEMM_VARIANTS = {"auto": 0, "tile32x16": 1, "tile32x32": 2, "rows": 3}


def parity_gemm(A: np.ndarray, W: np.ndarray, epilogue: str = "store", variant: int | str = 0, resid: np.ndarray | None = None,
                gelu_tab: np.ndarray | None = None, return_variant: bool = False):
    """Bit-exact A W^T on the parity path's dense mat-muls; A [M][K], W [N][K] both float16 or both float32, K % 32 == 0.

    Returns float32 [M][N] for "store" and for "resid" (resid [M][N] float32 + A W^T), [M][N] in the operands' dtype for "gelu"
    (GELU through gelu_tab, 65536 uint16 f16 bits), and for "qkv" (N % 3 == 0) the triple Q, K, V of float32 [M][N/3].
    variant = 0 ("auto") runs what the library picks for M rows (the few-row kernel below 16 rows, else the tiled GEMM's tile), 1
    ("tile32x16") / 2 ("tile32x32") force a tiled GEMM block tile, 3 ("rows") the few-row kernel at any M; with return_variant the
    result is (outputs, the variant that ran)."""
    variant = GEMM_VARIANTS.get(variant, variant)
    dt = np.float16 if np.asarray(A).dtype == np.float16 else np.float32
    A = np.ascontiguousarray(A, dt); W = np.ascontiguousarray(W, dt)
    M, K = A.shape; N = W.shape[0]
    assert W.shape[1] == K, (A.shape, W.shape)
    tab = _gelu_table(epilogue, gelu_tab)
    out, r = _gemm(f"bark_b200_parity_gemm ({epilogue}, {M}x{N}x{K}, variant {variant})",
                   lambda out: lib().bark_b200_parity_gemm(_p(A), _p(W), _p(out), M, N, K, 1 if dt == np.float16 else 0, PARITY_EPILOGUES[epilogue],
                                                           variant, None if tab is None else _p(tab)),
                   epilogue, resid, (M, N), dt if epilogue == "gelu" else np.float32, ((M, N // 3),) * 3 if epilogue == "qkv" else None)
    return (out, r) if return_variant else out


QUANT_TYPES = {"q4_0": 2, "q4_1": 3, "q5_0": 6, "q5_1": 7, "q8_0": 8}     # enum ggml_type
QUANT_BLOCK_BYTES = {"q4_0": 18, "q4_1": 20, "q5_0": 22, "q5_1": 24, "q8_0": 34}
QUANT_PATHS = {"auto": 0, "decode_staged": 1, "decode_global": 2}


def quant_matmul(qtype: str, W: np.ndarray, A: np.ndarray, epilogue: str = "store", path: str = "auto", resid: np.ndarray | None = None,
                 gelu_tab: np.ndarray | None = None, return_q8: bool = False):
    """Bit-exact A W^T on a quantised mat-mul; W [N][K/32 * block bytes] uint8, the weight rows as the model file stores them, A [M][K]
    float32, K % 32 == 0.  Returns float32 [M][N] for "store", "resid" (resid + A W^T) and "gelu" (GELU through gelu_tab, 65536 uint16
    f16 bits), the triple Q, K, V of [M][N/3] for "qkv".  path: "auto" (the per-op kernels the library runs for M rows), or for q4_0 with
    M == 1 the decode step's kernels with the rows staged in shared memory ("decode_staged") or read from global memory ("decode_global").
    With return_q8 the result is (outputs, q int8 [M][K], d float16 [M][K/32], s float16 [M][K/32] or None): the quantised activation."""
    A = np.ascontiguousarray(A, np.float32); W = np.ascontiguousarray(W, np.uint8)
    M, K = A.shape; N = W.shape[0]
    assert K % 32 == 0 and W.shape[1] == K // 32 * QUANT_BLOCK_BYTES[qtype], (qtype, A.shape, W.shape)
    tab = _gelu_table(epilogue, gelu_tab)
    q = np.zeros((M, K), np.int8); d = np.zeros((M, K // 32), np.float32)
    s = np.zeros((M, K // 32), np.float32) if qtype in ("q4_1", "q5_1") else None
    out, _ = _gemm(f"bark_b200_quant_matmul ({qtype}, {epilogue}, {M}x{N}x{K}, {path})",
                   lambda out: lib().bark_b200_quant_matmul(QUANT_TYPES[qtype], _p(W), _p(A), _p(out), M, N, K, PARITY_EPILOGUES[epilogue],
                                                            QUANT_PATHS[path], None if tab is None else _p(tab), _p(q), _p(d), None if s is None else _p(s)),
                   epilogue, resid, (M, N), np.float32, ((M, N // 3),) * 3 if epilogue == "qkv" else None)
    if not return_q8:
        return out
    return out, q, d.astype(np.float16), None if s is None else s.astype(np.float16)


def _codec_call(what: str, r: int):
    """The value a codec hook returned; GuardBandError when it stored outside its output, RuntimeError when it refused or failed."""
    if r == -1:
        raise GuardBandError(f"{what} wrote outside its output")
    if r <= 0:
        raise RuntimeError(f"{what} failed or refused the shape (see stderr)")
    return r


def _items(xs, C: int, dtype=np.float32):
    """Items [C][L_b] -> (their concatenation, int32 lengths)."""
    xs = [np.asarray(x, dtype).reshape(C, -1) for x in xs]
    return np.ascontiguousarray(np.concatenate([x.ravel() for x in xs])), np.array([x.shape[1] for x in xs], np.int32)


def _split(flat: np.ndarray, C: int, lengths):
    out, o = [], 0
    for L in lengths:
        out.append(flat[o:o + C * L].reshape(C, L))
        o += C * L
    return out


def codec_conv1d(xs, w: np.ndarray, bias: np.ndarray, stride: int = 1, elu_in: bool = False, resid=None, return_kernel: bool = False):
    """The EnCodec convolution launcher (bark_b200_codec_conv1d) on the items xs, each float32 [Cin][L_b]; w float16 [Cout][Cin][k] as the
    file stores it, bias float32 [Cout], resid (stride 1) a list of [Cout][L_b] or None.  Returns the items' outputs [Cout][T_b], and with
    return_kernel the id of the kernel that ran (include/bark_b200.h)."""
    w = np.ascontiguousarray(w, np.float16); Cout, Cin, k = w.shape
    x, L = _items(xs, Cin)
    T = [conv1d_out_len(int(l), k, stride) for l in L]
    y = np.zeros(Cout * sum(T), np.float32)
    r_flat = None if resid is None else _items(resid, Cout)[0]
    r = _codec_call(f"bark_b200_codec_conv1d (Cin {Cin}, Cout {Cout}, k {k}, stride {stride}, L {L.tolist()})",
                    lib().bark_b200_codec_conv1d(_p(x), Cin, _p(L), L.size, _p(w), _p(np.ascontiguousarray(bias, np.float32)), Cout, k, stride,
                                                 int(elu_in), None if r_flat is None else _p(r_flat), _p(y)))
    out = _split(y, Cout, T)
    return (out, r) if return_kernel else out


def conv1d_out_len(L: int, k: int, stride: int) -> int:
    """strided_conv_1d's output length: get_extra_padding_for_conv_1d evaluated in float32, as the reference does."""
    f32 = np.float32
    n_frames = (f32(L) - f32(k) + f32(k - stride)) / f32(stride) + f32(1)
    ideal = int((np.ceil(n_frames) - f32(1)) * f32(stride) + (f32(k) - f32(k - stride)))
    extra = int(f32(ideal) - f32(L))
    return (L + (k - stride) + extra - k) // stride + 1


def codec_convtr1d(xs, w: np.ndarray, bias: np.ndarray, stride: int, return_kernel: bool = False):
    """ELU and the transposed convolution (bark_b200_codec_convtr1d) on items [Cin][T_b]; w float16 [Cin][Cout][2 stride] as stored.
    Returns the items' outputs [Cout][T_b stride] (and the NG of the kernel that ran)."""
    w = np.ascontiguousarray(w, np.float16); Cin, Cout, k = w.shape
    assert k == 2 * stride, (w.shape, stride)
    x, T = _items(xs, Cin)
    y = np.zeros(Cout * int(T.sum()) * stride, np.float32)
    r = _codec_call(f"bark_b200_codec_convtr1d (Cin {Cin}, Cout {Cout}, stride {stride}, T {T.tolist()})",
                    lib().bark_b200_codec_convtr1d(_p(x), Cin, _p(T), T.size, _p(w), _p(np.ascontiguousarray(bias, np.float32)), Cout, stride, _p(y)))
    out = _split(y, Cout, [int(t) * stride for t in T])
    return (out, r) if return_kernel else out


def codec_lstm(xs, wih: np.ndarray, whh: np.ndarray, bih: np.ndarray, bhh: np.ndarray, skip=None, return_kernel: bool = False):
    """One LSTM layer (bark_b200_codec_lstm) on items [C][T_b]; wih, whh float16 [4C][C], bih, bhh float32 [4C], skip a list of [C][T_b]
    added to the output, or None.  Returns the items' outputs (and 1 / 2: the one-item / batched recurrence ran)."""
    wih = np.ascontiguousarray(wih, np.float16); whh = np.ascontiguousarray(whh, np.float16)
    C = wih.shape[1]
    x, T = _items(xs, C)
    s_flat = None if skip is None else _items(skip, C)[0]
    out = np.zeros(x.size, np.float32)
    r = _codec_call(f"bark_b200_codec_lstm (C {C}, T {T.tolist()})",
                    lib().bark_b200_codec_lstm(_p(x), C, _p(T), T.size, _p(wih), _p(whh), _p(np.ascontiguousarray(bih, np.float32)),
                                               _p(np.ascontiguousarray(bhh, np.float32)), None if s_flat is None else _p(s_flat), _p(out)))
    res = _split(out, C, T)
    return (res, r) if return_kernel else res


def resample_window(items) -> list:
    """resample_kernel over windows (bark_b200_resample_window), all items in one launch.  items: dicts with frames (mono [n] or
    interleaved [n][channels] float32, the global frames org ..), sr, new_sr, org, first, n_out and optionally end (the signal's
    length; frames at or past it read as zeros).  Returns each item's outputs first .. first + n_out - 1, float32."""
    fr = [np.ascontiguousarray(it["frames"], np.float32) for it in items]
    n = len(items)
    flat = np.ascontiguousarray(np.concatenate([f.ravel() for f in fr] + [np.zeros(1, np.float32)]))
    ints = lambda v: np.ascontiguousarray(v, np.int32)          # noqa: E731
    longs = lambda v: np.ascontiguousarray(v, np.int64)         # noqa: E731
    nf = ints([f.shape[0] for f in fr])
    ch = ints([1 if f.ndim == 1 else f.shape[1] for f in fr])
    sr, nsr = ints([it["sr"] for it in items]), ints([it["new_sr"] for it in items])
    o, f, no = _window([it["org"] for it in items], [it["first"] for it in items], [it["n_out"] for it in items])
    end = longs([it.get("end", -1) for it in items])
    y = np.zeros(max(int(no.sum()), 1), np.float32)
    _codec_call(f"bark_b200_resample_window ({n} items)",
                lib().bark_b200_resample_window(_p(flat), _p(nf), _p(ch), _p(sr), _p(nsr), _p(o), _p(f), _p(no), _p(end), n, _p(y)))
    return np.split(y[:int(no.sum())], np.cumsum(no)[:-1])


def _window(org, first, n_out):
    return tuple(np.ascontiguousarray(a, t) for a, t in ((org, np.int64), (first, np.int64), (n_out, np.int32)))


def codec_conv1d_window(xs, org, first, n_out, w: np.ndarray, bias: np.ndarray, stride: int = 1, elu_in: bool = False, resid=None, return_kernel: bool = False):
    """codec_conv1d over windows (bark_b200_codec_conv1d_window): item b's columns xs[b] [Cin][L_b] are global positions org[b].. of its
    signal, and its outputs first[b] .. first[b] + n_out[b] - 1 come back, [Cout][n_out[b]]; resid (stride 1) a list of [Cout][n_out[b]]."""
    w = np.ascontiguousarray(w, np.float16); Cout, Cin, k = w.shape
    x, L = _items(xs, Cin)
    o, f, no = _window(org, first, n_out)
    y = np.zeros(Cout * int(no.sum()), np.float32)
    r_flat = None if resid is None else _items(resid, Cout)[0]
    r = _codec_call(f"bark_b200_codec_conv1d_window (Cin {Cin}, Cout {Cout}, k {k}, stride {stride}, L {L.tolist()}, org {o.tolist()}, first {f.tolist()})",
                    lib().bark_b200_codec_conv1d_window(_p(x), Cin, _p(L), L.size, _p(o), _p(f), _p(no), _p(w), _p(np.ascontiguousarray(bias, np.float32)),
                                                        Cout, k, stride, int(elu_in), None if r_flat is None else _p(r_flat), _p(y)))
    out = _split(y, Cout, no.tolist())
    return (out, r) if return_kernel else out


def codec_convtr1d_window(xs, org, first, n_out, w: np.ndarray, bias: np.ndarray, stride: int):
    """codec_convtr1d over windows (bark_b200_codec_convtr1d_window): item b's frames xs[b] [Cin][L_b] are global frames org[b].., and the
    output blocks of frames first[b] .. first[b] + n_out[b] - 1 come back, [Cout][n_out[b] stride]."""
    w = np.ascontiguousarray(w, np.float16); Cin, Cout, k = w.shape
    x, L = _items(xs, Cin)
    o, f, no = _window(org, first, n_out)
    y = np.zeros(Cout * int(no.sum()) * stride, np.float32)
    _codec_call(f"bark_b200_codec_convtr1d_window (Cin {Cin}, Cout {Cout}, stride {stride}, L {L.tolist()}, org {o.tolist()}, first {f.tolist()})",
                lib().bark_b200_codec_convtr1d_window(_p(x), Cin, _p(L), L.size, _p(o), _p(f), _p(no), _p(w), _p(np.ascontiguousarray(bias, np.float32)),
                                                      Cout, stride, _p(y)))
    return _split(y, Cout, [int(t) * stride for t in no])


def codec_lstm_state(xs, wih: np.ndarray, whh: np.ndarray, bih: np.ndarray, bhh: np.ndarray, state=None, skip=None):
    """codec_lstm from the state (h, c) float32 [n][2][C] (None: zeros) (bark_b200_codec_lstm_state).  Returns (the items' outputs,
    the state after each item's last step)."""
    wih = np.ascontiguousarray(wih, np.float16); whh = np.ascontiguousarray(whh, np.float16)
    C = wih.shape[1]
    x, T = _items(xs, C)
    st = np.zeros((T.size, 2, C), np.float32) if state is None else np.array(state, np.float32).reshape(T.size, 2, C)
    s_flat = None if skip is None else _items(skip, C)[0]
    out = np.zeros(x.size, np.float32)
    _codec_call(f"bark_b200_codec_lstm_state (C {C}, T {T.tolist()})",
                lib().bark_b200_codec_lstm_state(_p(x), C, _p(T), T.size, _p(wih), _p(whh), _p(np.ascontiguousarray(bih, np.float32)),
                                                 _p(np.ascontiguousarray(bhh, np.float32)), None if s_flat is None else _p(s_flat), _p(st), _p(out)))
    return _split(out, C, T), st


def codec_rvq_decode(codes, codebooks: np.ndarray):
    """The quantizer decode (bark_b200_codec_rvq_decode) on items of codes int32 [n_q][T_b] through codebooks float32 [n_q][n_bins][hidden].
    Returns the items' latents [hidden][T_b]."""
    cb = np.ascontiguousarray(codebooks, np.float32); n_q, n_bins, hidden = cb.shape
    c, T = _items(codes, n_q, np.int32)
    x = np.zeros(hidden * int(T.sum()), np.float32)
    _codec_call(f"bark_b200_codec_rvq_decode (n_q {n_q}, T {T.tolist()})",
                lib().bark_b200_codec_rvq_decode(_p(c), n_q, _p(T), T.size, _p(cb), hidden, n_bins, _p(x)))
    return _split(x, hidden, T)


DEVICE_MATH = {"expm1f": 0, "tanhf": 1, "expf": 2, "v_expf": 3, "elu": 4, "sigmoid": 5, "round_f16": 6}


def device_math(fn: str, lo_bits: int, count: int, stride: int = 1) -> np.ndarray:
    """A device function of the codec and soft_max (bark_b200_device_math) on the floats of bit patterns lo_bits + i stride (mod 2^32),
    i < count <= 2^24: float32 [count]."""
    out = np.zeros(count, np.float32)
    _codec_call(f"bark_b200_device_math ({fn})", lib().bark_b200_device_math(DEVICE_MATH[fn], lo_bits & 0xFFFFFFFF, stride, count, _p(out)))
    return out


def fast_convert(wtype: str, W: np.ndarray):
    """Fast mode's load-time weight conversion to f16 (bark_b200_fast_convert).  W: [n_out][K] float32 for "f32", or for a quantised
    type the weight rows as the model file stores them, uint8 [n_out][K/32 * block bytes]; K % 32 == 0.  Returns (float16 [n_out][K],
    the number of results that are inf or NaN).  Raises GuardBandError when the kernel stored outside its output, RuntimeError when
    the hook failed."""
    if wtype == "f32":
        W = np.ascontiguousarray(W, np.float32)
        n_out, K = W.shape
    else:
        W = np.ascontiguousarray(W, np.uint8)
        n_out, K = W.shape[0], W.shape[1] // QUANT_BLOCK_BYTES[wtype] * 32
        assert W.shape[1] == K // 32 * QUANT_BLOCK_BYTES[wtype], (wtype, W.shape)
    out = np.zeros((n_out, K), np.float16)
    non_finite = C.c_int(0)
    r = lib().bark_b200_fast_convert(0 if wtype == "f32" else QUANT_TYPES[wtype], _p(W), n_out, K, _p(out), C.byref(non_finite))
    if r == -1:
        raise GuardBandError(f"bark_b200_fast_convert ({wtype}, {n_out}x{K}) wrote outside its output")
    if r != 1:
        raise RuntimeError(f"bark_b200_fast_convert ({wtype}, {n_out}x{K}) failed")
    return out, non_finite.value


ROW_OPS = {"layernorm": 0, "softmax": 1}
ROW_IMPLS = {"multi": 0, "decode": 1}


def parity_rows(x: np.ndarray, op: str, impl: str, g: np.ndarray | None = None, b: np.ndarray | None = None):
    """One of the parity path's row reductions on x [rows][n] float32, n <= 1024; returns (out [rows][n] float32, replays).

    op "layernorm" (eps 1e-5, gain g required, bias b optional: the f32 value before any operand rounding) or "softmax" (the
    probabilities as their consumers form them); impl "multi" (layernorm_act_kernel / softmax_row, the multi-row passes and the
    attention kernels) or "decode" (block_layernorm / softmax_exp_rcp, the persistent decode kernels).  replays = how many bracket
    decisions fell back to the sequential sum."""
    x = np.ascontiguousarray(x, np.float32)
    if x.ndim == 1:
        x = x[None]
    rows, n = x.shape
    gp = bp = None
    if g is not None:
        g = np.ascontiguousarray(g, np.float32); assert g.shape == (n,), g.shape; gp = _p(g)
    if b is not None:
        b = np.ascontiguousarray(b, np.float32); assert b.shape == (n,), b.shape; bp = _p(b)
    out = np.zeros((rows, n), np.float32)
    rep = C.c_uint(0)
    if not lib().bark_b200_parity_rows(ROW_OPS[op], ROW_IMPLS[impl], _p(x), rows, n, gp, bp, _p(out), C.byref(rep)):
        raise RuntimeError(f"bark_b200_parity_rows ({op}, {impl}, {rows} x {n}) failed")
    return out, rep.value


def _given_u(hook: str, what: str, logits, u, extra: tuple, run) -> dict:
    """What the sampler wrappers share: logits as float32 rows [rows][n], u as float64 [rows] (broadcast; None for temp 0) and the
    result dict of int32 tokens, device_tokens, flags, the extra keys and float32 eos_p.  run(logits, n, rows, u, tokens, device_tokens,
    flags, eos_p, *extra) calls the hook with pointers; its return value becomes replays, RuntimeError when it is negative."""
    l = np.ascontiguousarray(logits, np.float32)
    if l.ndim == 1:
        l = l[None]
    rows, n = l.shape
    up = None
    if u is not None:
        u = np.ascontiguousarray(np.broadcast_to(np.asarray(u, np.float64), (rows,)))
        up = _p(u)
    out = {k: np.zeros(rows, np.int32) for k in ("tokens", "device_tokens", "flags") + extra}
    out["eos_p"] = np.zeros(rows, np.float32)
    r = run(_p(l), n, rows, up, *(_p(out[k]) for k in ("tokens", "device_tokens", "flags", "eos_p") + extra))
    if r < 0:
        raise RuntimeError(f"{hook} ({rows} x {n}, {what}) failed")
    out["replays"] = r
    return out


def sample_given_u(logits: np.ndarray, temp: float, u=None, threads: int = 0):
    """The device sampler on logits [rows][n] float32 with the uniform draws u [rows] given (not used when temp == 0); threads 0 runs
    sample_rows_kernel as the library picks it, 256 or 1024 forces that instantiation.  Returns a dict: tokens (final), device_tokens
    (the kernel's, before the host replay), flags, eos_p [rows] and replays (how many rows went to the host replay)."""
    return _given_u("bark_b200_sample_given_u", f"temp {temp}, threads {threads}", logits, u, (),
                    lambda l, n, rows, up, *o: lib().bark_b200_sample_given_u(l, n, rows, temp, up, threads, *o))


def sample_filtered_given_u(logits: np.ndarray, temp: float, u=None, top_k=None, top_p=None, threads: int = 0):
    """sample_given_u with the top-k / top-p filter first (bark_b200_sample_filtered_given_u): filter_rows_kernel, then the sampler on
    its output, then the host replay of every flagged row from the raw logits.  Returns sample_given_u's dict plus kept [rows], the
    number of logits the device filter kept; flags has bit 0 for the sampler and bit 1 for the filter."""
    st = _sampling_struct(top_k, top_p)
    return _given_u("bark_b200_sample_filtered_given_u", f"temp {temp}, top_k {top_k}, top_p {top_p}, threads {threads}", logits, u, ("kept",),
                    lambda l, n, rows, up, *o: lib().bark_b200_sample_filtered_given_u(l, n, rows, temp, C.byref(st), up, threads, *o))


class Encodec:
    """One encodec_context (include/encodec.h): the 24 kHz EnCodec of a weight file, at any bandwidth its codebooks allow.
    offset: byte position of the codec section (0 for a standalone encodec.cpp file).  Mirrors encodec.cpp's examples."""

    def __init__(self, model_path: str, offset: int = 0, device: int | None = None):
        L = lib()
        if device is not None:
            L.bark_b200_set_device(device)
        self.ctx = L.encodec_load_model(os.fsencode(model_path), offset, 0)
        if not self.ctx:
            raise RuntimeError(f"encodec_load_model failed for {model_path} at offset {offset} (see stderr); no CPU fallback exists")
        self.ctx = C.c_void_p(self.ctx)
        self._bandwidth, self._sample_rate = None, None
        self._streams = []

    def close(self):
        if getattr(self, "ctx", None):
            for s in self._streams:                      # a stream must not outlive its context
                s.close()
            lib().encodec_free(self.ctx)
            self.ctx = None

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    @property
    def bandwidth(self):
        """Target bandwidth in kbps (encodec_set_target_bandwidth); None: the file's."""
        return self._bandwidth

    @bandwidth.setter
    def bandwidth(self, kbps: int):
        lib().encodec_set_target_bandwidth(self.ctx, int(kbps))
        self._bandwidth = int(kbps)

    @property
    def sample_rate(self):
        """Sample rate in Hz (encodec_set_sample_rate); it only changes n_q, as in the reference.  None: the file's."""
        return self._sample_rate

    @sample_rate.setter
    def sample_rate(self, hz: int):
        lib().encodec_set_sample_rate(self.ctx, int(hz))
        self._sample_rate = int(hz)

    @property
    def n_q(self) -> int:
        """Codebooks of the current bandwidth and sample rate, read from the codes of a minimal compress."""
        return self.compress(np.zeros(1921, np.float32)).shape[0]

    def compress(self, audio, sample_rate: int | None = None) -> np.ndarray:
        """Mono float32 samples (finite, at least 1921) -> codes [n_q][T] int32, T = ceil(n / 320).  With sample_rate, audio is mono
        [n] or [channels][n] at that rate, down-mixed and resampled to 24 kHz on the GPU first (bark_b200_encodec_compress_resampled);
        n then counts the resampled samples."""
        if sample_rate is None:
            a = np.ascontiguousarray(audio, np.float32).ravel()
            if not lib().encodec_compress_audio(self.ctx, _p(a), a.size, 1):
                raise RuntimeError("encodec_compress_audio failed (see stderr)")
            L = a.size
        else:
            a, nf, ch = _frames(audio)
            if not lib().bark_b200_encodec_compress_resampled(self.ctx, _p(a), nf, ch, int(sample_rate)):
                raise RuntimeError("bark_b200_encodec_compress_resampled failed (see stderr)")
            L = resampled_length(nf, int(sample_rate))
        n = lib().encodec_get_codes_size(self.ctx)
        T = (L + 319) // 320
        return np.ctypeslib.as_array(lib().encodec_get_codes(self.ctx), shape=(n,)).copy().reshape(n // T, T)

    def decompress(self, codes) -> np.ndarray:
        """Codes [n_q][T] (n_q of the current bandwidth) -> 320 T float32 samples."""
        c = np.ascontiguousarray(codes, np.int32)
        if not lib().encodec_decompress_audio(self.ctx, _p(c), c.size, 1):
            raise RuntimeError("encodec_decompress_audio failed (see stderr)")
        return self._audio()

    def reconstruct(self, audio, sample_rate: int | None = None) -> np.ndarray:
        """compress then decompress on the device: 320 T float32 samples (24 kHz).  sample_rate as for compress."""
        if sample_rate is None:
            a = np.ascontiguousarray(audio, np.float32).ravel()
            if not lib().encodec_reconstruct_audio(self.ctx, _p(a), a.size, 1):
                raise RuntimeError("encodec_reconstruct_audio failed (see stderr)")
        else:
            a, nf, ch = _frames(audio)
            if not lib().bark_b200_encodec_reconstruct_resampled(self.ctx, _p(a), nf, ch, int(sample_rate)):
                raise RuntimeError("bark_b200_encodec_reconstruct_resampled failed (see stderr)")
        return self._audio()

    def _audio(self):
        n = lib().encodec_get_audio_size(self.ctx)
        return np.ctypeslib.as_array(lib().encodec_get_audio(self.ctx), shape=(n,)).copy()

    # ---- batches (bark_b200_encodec_*_batch): item i equals the single call on clip i, bit for bit --------------------------------
    def compress_batch(self, clips, sample_rate=None) -> list:
        """Clips of mono float32 samples (each finite, at least 1921) -> codes [n_q][T_i] int32 per clip, in one batched call.  With
        sample_rate (one rate, or a list of one per clip), each clip is mono [n] or [channels][n] at its rate, down-mixed and resampled
        to 24 kHz on the GPU first (bark_b200_encodec_compress_batch_resampled)."""
        if sample_rate is None:
            xs = [np.ascontiguousarray(a, np.float32).ravel() for a in clips]
            self._batch("bark_b200_encodec_compress_batch", xs)
            lens = [x.size for x in xs]
        else:
            lens = self._batch_resampled("bark_b200_encodec_compress_batch_resampled", clips, sample_rate)
        out = []
        for i, n in enumerate(lens):
            c = self._item("bark_b200_encodec_batch_codes", i, np.int32)
            T = (n + 319) // 320
            out.append(c.reshape(c.size // T, T))
        return out

    def decompress_batch(self, codes) -> list:
        """Codes [n_q][T_i] per item (n_q of the current bandwidth) -> 320 T_i float32 samples per item."""
        cs = [np.ascontiguousarray(c, np.int32) for c in codes]
        self._batch("bark_b200_encodec_decompress_batch", cs)
        return [self._item("bark_b200_encodec_batch_audio", i, np.float32) for i in range(len(cs))]

    def reconstruct_batch(self, clips, sample_rate=None) -> list:
        """compress_batch then decompress_batch, the codes staying on the device: 320 T_i float32 samples per clip.  sample_rate as for
        compress_batch."""
        if sample_rate is None:
            xs = [np.ascontiguousarray(a, np.float32).ravel() for a in clips]
            self._batch("bark_b200_encodec_reconstruct_batch", xs)
        else:
            xs = self._batch_resampled("bark_b200_encodec_reconstruct_batch_resampled", clips, sample_rate)
        return [self._item("bark_b200_encodec_batch_audio", i, np.float32) for i in range(len(xs))]

    def _batch_resampled(self, fn, clips, sample_rate):
        """Runs a resampled batch call; returns the clips' resampled lengths."""
        fr = [_frames(a) for a in clips]
        n = len(fr)
        rates = [int(sample_rate)] * n if np.ndim(sample_rate) == 0 else [int(r) for r in sample_rate]
        if len(rates) != n:
            raise ValueError(f"{fn}: {n} clips but {len(rates)} sample rates")
        ptrs = (C.c_void_p * max(n, 1))(*[x.ctypes.data for x, _, _ in fr])
        frames = (C.c_int * max(n, 1))(*[nf for _, nf, _ in fr])
        chans = (C.c_int * max(n, 1))(*[ch for _, _, ch in fr])
        srs = (C.c_int * max(n, 1))(*rates)
        if not getattr(lib(), fn)(self.ctx, ptrs, frames, chans, srs, n):
            raise RuntimeError(f"{fn} failed (see stderr)")
        return [resampled_length(nf, r) for (_, nf, _), r in zip(fr, rates)]

    def _batch(self, fn, arrays):
        n = len(arrays)
        ptrs = (C.c_void_p * max(n, 1))(*[a.ctypes.data for a in arrays])
        lens = (C.c_int * max(n, 1))(*[a.size for a in arrays])
        if not getattr(lib(), fn)(self.ctx, ptrs, lens, n):
            raise RuntimeError(f"{fn} failed (see stderr)")

    def _item(self, fn, i, dtype):
        n = getattr(lib(), fn)(self.ctx, i, None, 0)
        out = np.empty(n, dtype)
        getattr(lib(), fn)(self.ctx, i, _p(out), n)
        return out

    # ---- streams (bark_b200_encodec_stream_*): their outputs joined equal the whole-clip call on their input joined --------------
    def stream(self, direction: str, sample_rate: int | None = None, channels: int | None = None) -> "EncodecStream":
        """A stream on this context: "encode" (mono 24 kHz samples in, codes out) or "decode" (codes in, samples out), at the n_q of the
        current bandwidth.  With sample_rate or channels (bark_b200_encodec_stream_open_resampled, DESIGN.md §20), an encode takes
        interleaved frames [n][channels] (or mono [n]) at sample_rate, and a decode (mono only) gives samples at sample_rate."""
        s = EncodecStream(self, direction, sample_rate, channels)
        self._streams.append(s)
        return s

    def stats(self) -> dict:
        s = lib().encodec_get_statistics(self.ctx).contents
        return {"t_load_us": s.t_load_us, "t_compute_us": s.t_compute_us}

    def reset_stats(self):
        lib().encodec_reset_statistics(self.ctx)


STREAM_DIRECTIONS = {"encode": 0, "decode": 1}


class EncodecStream:
    """A streaming EnCodec coder (bark_b200_encodec_stream_*) on an Encodec context, made by Encodec.stream.  push(x) returns the outputs
    that became final: codes [n_q][k] int32 for an encode of float32 samples, float32 samples for a decode of codes [n_q][k]; finish()
    returns the rest.  Everything returned, joined, equals compress / decompress of everything pushed."""

    def __init__(self, codec: "Encodec", direction: str, sample_rate: int | None = None, channels: int | None = None):
        self.direction = direction
        self.sample_rate = CODEC_RATE if sample_rate is None else int(sample_rate)
        self.channels = 1 if channels is None else int(channels)
        if sample_rate is None and channels is None:
            self.handle = lib().bark_b200_encodec_stream_open(codec.ctx, STREAM_DIRECTIONS[direction])
        else:
            self.handle = lib().bark_b200_encodec_stream_open_resampled(codec.ctx, STREAM_DIRECTIONS[direction], self.channels, self.sample_rate)
        if not self.handle:
            raise RuntimeError(f"bark_b200_encodec_stream_open ({direction}, {self.channels} channels at {self.sample_rate} Hz) failed (see stderr)")
        self.handle = C.c_void_p(self.handle)
        self.n_q = lib().bark_b200_encodec_stream_codebooks(self.handle)

    def close(self):
        if getattr(self, "handle", None):
            lib().bark_b200_encodec_stream_close(self.handle)
            self.handle = None

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    def _chunk(self, x):
        """x as the C call takes it: (array, count) of samples, of interleaved frames [n][channels], or of code frames"""
        if self.direction == "encode" and self.channels > 1:
            a = np.ascontiguousarray(x, np.float32)
            if a.ndim != 2 or a.shape[1] != self.channels:
                raise ValueError(f"encode stream of {self.channels} channels: frames must be [n][{self.channels}], got shape {a.shape}")
            n = a.shape[0]
        elif self.direction == "encode":
            a = np.ascontiguousarray(x, np.float32).ravel()
            n = a.size
        else:
            a = np.ascontiguousarray(x, np.int32)
            if a.ndim != 2 or a.shape[0] != self.n_q:
                raise ValueError(f"decode stream: codes must be [{self.n_q}][k], got shape {a.shape}")
            n = a.shape[1]
        return (a if n else np.zeros(1, a.dtype)), n          # an empty chunk still passes a valid pointer

    def read(self) -> np.ndarray:
        """Every final output not yet returned."""
        k = lib().bark_b200_encodec_stream_read(self.handle, None, 0)
        if self.direction == "decode":
            out = np.zeros(k, np.float32)
        else:
            out = np.zeros((self.n_q, k), np.int32)
        got = lib().bark_b200_encodec_stream_read(self.handle, _p(out), k)
        assert got == k, (got, k)
        return out

    def push(self, x) -> np.ndarray:
        a, n = self._chunk(x)
        if lib().bark_b200_encodec_stream_push(self.handle, _p(a), n) < 0:
            raise RuntimeError("bark_b200_encodec_stream_push refused (see stderr)")
        return self.read()

    def finish(self) -> np.ndarray:
        if lib().bark_b200_encodec_stream_finish(self.handle) < 0:
            raise RuntimeError("bark_b200_encodec_stream_finish refused (see stderr)")
        return self.read()


def encodec_stream_push_batch(streams, chunks) -> list:
    """Pushes chunks[i] to streams[i] (at most 32 streams of one context and direction) in one pass of the kernels
    (bark_b200_encodec_stream_push_batch); returns each stream's new final outputs, as its own push would."""
    if len(streams) != len(chunks):
        raise ValueError(f"{len(streams)} streams but {len(chunks)} chunks")
    arrs = [s._chunk(x) for s, x in zip(streams, chunks)]
    n = len(streams)
    hs = (C.c_void_p * max(n, 1))(*[s.handle.value for s in streams])
    ptrs = (C.c_void_p * max(n, 1))(*[a.ctypes.data for a, _ in arrs])
    cnt = (C.c_int * max(n, 1))(*[k for _, k in arrs])
    if lib().bark_b200_encodec_stream_push_batch(hs, ptrs, cnt, n) < 0:
        raise RuntimeError("bark_b200_encodec_stream_push_batch refused (see stderr)")
    return [s.read() for s in streams]


def encodec_stream_ready(direction: str, n: int, sample_rate: int | None = None) -> int:
    """The outputs a stream has made final after n inputs, before finish (bark_b200_encodec_stream_ready): frames after n samples for
    "encode", samples after n frames for "decode".  With sample_rate, the rule of a stream at that rate
    (bark_b200_encodec_stream_ready_resampled): frames after n frames at sample_rate, or samples at sample_rate after n frames."""
    if sample_rate is None:
        return int(lib().bark_b200_encodec_stream_ready(STREAM_DIRECTIONS[direction], int(n)))
    return int(lib().bark_b200_encodec_stream_ready_resampled(STREAM_DIRECTIONS[direction], int(sample_rate), int(n)))


def rvq_encode(latent: np.ndarray, codebooks: np.ndarray) -> np.ndarray:
    """The RVQ encode kernel on latent [hidden][T] and codebooks [n_q][n_bins][hidden] float32 (hidden % 32 == 0 and <= 128,
    n_bins <= 1024, n_q <= 32); returns codes [n_q][T] int32, bit-identical to the reference's quantizer encode."""
    lat = np.ascontiguousarray(latent, np.float32); cb = np.ascontiguousarray(codebooks, np.float32)
    hidden, T = lat.shape
    n_q, n_bins, h2 = cb.shape
    assert h2 == hidden, (lat.shape, cb.shape)
    codes = np.zeros((n_q, T), np.int32)
    if not lib().bark_b200_rvq_encode(_p(lat), T, _p(cb), hidden, n_bins, n_q, _p(codes)):
        raise RuntimeError(f"bark_b200_rvq_encode ({hidden} x {T}, {n_q} x {n_bins} codewords) failed")
    return codes


def kernel_launches() -> int:
    return int(lib().bark_b200_kernel_launches())


def profile_enable(on: bool):
    lib().bark_b200_profile_enable(int(on))


def profile_report() -> dict:
    import json
    n = lib().bark_b200_profile_report(None, 0)
    buf = C.create_string_buffer(n + 16)
    lib().bark_b200_profile_report(buf, n + 16)
    return json.loads(buf.value.decode())


def io_counters(reset: bool = False):
    a, b = C.c_ulonglong(0), C.c_ulonglong(0)
    lib().bark_b200_io_counters(C.byref(a), C.byref(b), int(reset))
    return a.value, b.value
