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
import os

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
    "bark_b200_fast_mode", "bark_b200_fast_gemm", "bark_b200_fast_attention", "bark_b200_parity_attention", "bark_b200_parity_gemm",
    "bark_b200_parity_rows", "bark_b200_sample_given_u", "bark_b200_generate_batch", "bark_b200_batch_audio", "bark_b200_batch_tokens", "bark_b200_gpt_eval_slot", "bark_b200_gpt_step_batch",
    "bark_b200_set_history_prompt", "bark_b200_generate_batch_prompted", "bark_b200_set_sampling", "bark_b200_sample_filtered_given_u",
    "bark_b200_quant_matmul",
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
    L.bark_b200_fast_attention.restype = C.c_int
    L.bark_b200_fast_attention.argtypes = [vp, vp, vp, vp, C.c_int, C.c_int, C.c_int]
    L.bark_b200_parity_attention.restype = C.c_int
    L.bark_b200_parity_attention.argtypes = [vp, vp, vp, vp] + [C.c_int] * 7
    L.bark_b200_parity_gemm.restype = C.c_int
    L.bark_b200_parity_gemm.argtypes = [vp, vp, vp] + [C.c_int] * 6 + [vp]
    L.bark_b200_quant_matmul.restype = C.c_int
    L.bark_b200_quant_matmul.argtypes = [C.c_int, vp, vp, vp] + [C.c_int] * 5 + [vp, vp, vp, vp]
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


class Bark:
    """One bark_context on one GPU.  Mirrors how examples/main/main.cpp uses bark.h."""

    def __init__(self, model_path: str, seed: int = 0, n_steps_text_encoder: int | None = None, temp=None, fine_temp=None,
                 min_eos_p=None, device: int | None = None, progress=None):
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

    def encodec_encode(self, audio, return_latent: bool = False):
        """Mono 24 kHz float32 samples (finite, at least 1921) -> codes [8][T] int32, T = ceil(n / 320), the layout encodec_decode
        takes; with return_latent also the encoder output before quantisation, [128][T] float32."""
        a = np.ascontiguousarray(audio, np.float32).ravel()
        T = (a.size + 319) // 320
        codes = np.zeros((8, max(T, 1)), np.int32); lat = np.zeros((128, max(T, 1)), np.float32)
        r = lib().bark_b200_encodec_encode(self.ctx, _p(a), a.size, _p(codes), codes.size, _p(lat), lat.size)
        if r < 0:
            raise RuntimeError("bark_b200_encodec_encode failed (see stderr)")
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


def fast_gemm(A: np.ndarray, W: np.ndarray, epilogue: str = "f32", bn: int = 0, resid: np.ndarray | None = None, return_bn: bool = False):
    """A W^T on the wgmma path through one of the fine pass's epilogues; A [M][K], W [N][K] float16, K % 64 == 0.

    Returns float32 [M][N] for "f32" and for "resid" (resid [M][N] float32 + A W^T), float16 [M][N] for "gelu16", and for "qkv16"
    (N % 6 == 0) the pair (float16 [M][2N/3], the V columns transposed: float16 [N/3][M]).  bn = 0 lets the cost model pick the tile
    width, 64 / 128 / 256 force it; with return_bn the result is (outputs, the tile width that ran)."""
    A = np.ascontiguousarray(A, np.float16); W = np.ascontiguousarray(W, np.float16)
    M, K = A.shape; N = W.shape[0]
    assert W.shape[1] == K, (A.shape, W.shape)
    if epilogue == "resid":
        out = np.array(resid, np.float32, order="C", copy=True)
        assert out.shape == (M, N), out.shape
    elif epilogue == "qkv16":
        assert N % 6 == 0, N
        out = np.zeros(M * N, np.float16)
    else:
        out = np.zeros((M, N), np.float16 if epilogue == "gelu16" else np.float32)
    r = lib().bark_b200_fast_gemm(_p(A), _p(W), _p(out), M, N, K, FAST_EPILOGUES[epilogue], bn)
    if r == -1:
        raise GuardBandError(f"bark_b200_fast_gemm ({epilogue}, {M}x{N}x{K}, bn {bn}) wrote outside its output")
    if r <= 0:
        raise RuntimeError(f"bark_b200_fast_gemm ({epilogue}, {M}x{N}x{K}, bn {bn}) failed")
    if epilogue == "qkv16":
        out = (out[:M * 2 * N // 3].reshape(M, 2 * N // 3), out[M * 2 * N // 3:].reshape(N // 3, M))
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


PARITY_EPILOGUES = {"store": 0, "resid": 1, "gelu": 2, "qkv": 3}      # EPI_* (csrc/gpt_kernels.h)


def parity_gemm(A: np.ndarray, W: np.ndarray, epilogue: str = "store", variant: int = 0, resid: np.ndarray | None = None,
                gelu_tab: np.ndarray | None = None, return_variant: bool = False):
    """Bit-exact A W^T on the parity path's tiled GEMM; A [M][K], W [N][K] both float16 or both float32, K % 32 == 0.

    Returns float32 [M][N] for "store" and for "resid" (resid [M][N] float32 + A W^T), [M][N] in the operands' dtype for "gelu"
    (GELU through gelu_tab, 65536 uint16 f16 bits), and for "qkv" (N % 3 == 0) the triple Q, K, V of float32 [M][N/3].
    variant = 0 lets the library pick the block tile, 1 (32 x 16) / 2 (32 x 32) force one; with return_variant the result is (outputs, variant)."""
    dt = np.float16 if np.asarray(A).dtype == np.float16 else np.float32
    A = np.ascontiguousarray(A, dt); W = np.ascontiguousarray(W, dt)
    M, K = A.shape; N = W.shape[0]
    assert W.shape[1] == K, (A.shape, W.shape)
    if epilogue == "resid":
        out = np.array(resid, np.float32, order="C", copy=True)
        assert out.shape == (M, N), out.shape
    else:
        out = np.zeros((M, N), dt if epilogue == "gelu" else np.float32)
    tab = None
    if epilogue == "gelu":
        tab = np.ascontiguousarray(gelu_tab, np.uint16)
        assert tab.shape == (65536,), tab.shape
    r = lib().bark_b200_parity_gemm(_p(A), _p(W), _p(out), M, N, K, 1 if dt == np.float16 else 0, PARITY_EPILOGUES[epilogue], variant,
                                    None if tab is None else _p(tab))
    if r == -1:
        raise GuardBandError(f"bark_b200_parity_gemm ({epilogue}, {M}x{N}x{K}, variant {variant}) wrote outside its output")
    if r <= 0:
        raise RuntimeError(f"bark_b200_parity_gemm ({epilogue}, {M}x{N}x{K}, variant {variant}) failed")
    if epilogue == "qkv":
        flat = out.reshape(-1)
        out = tuple(flat[i * M * (N // 3):(i + 1) * M * (N // 3)].reshape(M, N // 3) for i in range(3))
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
    if epilogue == "resid":
        out = np.array(resid, np.float32, order="C", copy=True)
        assert out.shape == (M, N), out.shape
    else:
        out = np.zeros((M, N), np.float32)
    tab = None
    if epilogue == "gelu":
        tab = np.ascontiguousarray(gelu_tab, np.uint16)
        assert tab.shape == (65536,), tab.shape
    q = np.zeros((M, K), np.int8); d = np.zeros((M, K // 32), np.float32)
    s = np.zeros((M, K // 32), np.float32) if qtype in ("q4_1", "q5_1") else None
    r = lib().bark_b200_quant_matmul(QUANT_TYPES[qtype], _p(W), _p(A), _p(out), M, N, K, PARITY_EPILOGUES[epilogue], QUANT_PATHS[path],
                                     None if tab is None else _p(tab), _p(q), _p(d), None if s is None else _p(s))
    what = f"bark_b200_quant_matmul ({qtype}, {epilogue}, {M}x{N}x{K}, {path})"
    if r == -1:
        raise GuardBandError(f"{what} wrote outside its output")
    if r != 1:
        raise RuntimeError(f"{what} failed")
    if epilogue == "qkv":
        flat = out.reshape(-1)
        out = tuple(flat[i * M * (N // 3):(i + 1) * M * (N // 3)].reshape(M, N // 3) for i in range(3))
    if not return_q8:
        return out
    return out, q, d.astype(np.float16), None if s is None else s.astype(np.float16)


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


def sample_given_u(logits: np.ndarray, temp: float, u=None, threads: int = 0):
    """The device sampler on logits [rows][n] float32 with the uniform draws u [rows] given (not used when temp == 0); threads 0 runs
    sample_rows_kernel as the library picks it, 256 or 1024 forces that instantiation.  Returns a dict: tokens (final), device_tokens
    (the kernel's, before the host replay), flags, eos_p [rows] and replays (how many rows went to the host replay)."""
    l = np.ascontiguousarray(logits, np.float32)
    if l.ndim == 1:
        l = l[None]
    rows, n = l.shape
    up = None
    if u is not None:
        u = np.ascontiguousarray(np.broadcast_to(np.asarray(u, np.float64), (rows,)))
        up = _p(u)
    out = {k: np.zeros(rows, np.int32) for k in ("tokens", "device_tokens", "flags")}
    out["eos_p"] = np.zeros(rows, np.float32)
    r = lib().bark_b200_sample_given_u(_p(l), n, rows, temp, up, threads, _p(out["tokens"]), _p(out["device_tokens"]), _p(out["flags"]),
                                       _p(out["eos_p"]))
    if r < 0:
        raise RuntimeError(f"bark_b200_sample_given_u ({rows} x {n}, temp {temp}, threads {threads}) failed")
    out["replays"] = r
    return out


def sample_filtered_given_u(logits: np.ndarray, temp: float, u=None, top_k=None, top_p=None, threads: int = 0):
    """sample_given_u with the top-k / top-p filter first (bark_b200_sample_filtered_given_u): filter_rows_kernel, then the sampler on
    its output, then the host replay of every flagged row from the raw logits.  Returns sample_given_u's dict plus kept [rows], the
    number of logits the device filter kept; flags has bit 0 for the sampler and bit 1 for the filter."""
    l = np.ascontiguousarray(logits, np.float32)
    if l.ndim == 1:
        l = l[None]
    rows, n = l.shape
    up = None
    if u is not None:
        u = np.ascontiguousarray(np.broadcast_to(np.asarray(u, np.float64), (rows,)))
        up = _p(u)
    out = {k: np.zeros(rows, np.int32) for k in ("tokens", "device_tokens", "flags", "kept")}
    out["eos_p"] = np.zeros(rows, np.float32)
    st = _sampling_struct(top_k, top_p)
    r = lib().bark_b200_sample_filtered_given_u(_p(l), n, rows, temp, C.byref(st), up, threads, _p(out["tokens"]), _p(out["device_tokens"]),
                                                _p(out["flags"]), _p(out["eos_p"]), _p(out["kept"]))
    if r < 0:
        raise RuntimeError(f"bark_b200_sample_filtered_given_u ({rows} x {n}, temp {temp}, top_k {top_k}, top_p {top_p}, threads {threads}) failed")
    out["replays"] = r
    return out


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

    def close(self):
        if getattr(self, "ctx", None):
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

    def compress(self, audio) -> np.ndarray:
        """Mono float32 samples (finite, at least 1921) -> codes [n_q][T] int32, T = ceil(n / 320)."""
        a = np.ascontiguousarray(audio, np.float32).ravel()
        if not lib().encodec_compress_audio(self.ctx, _p(a), a.size, 1):
            raise RuntimeError("encodec_compress_audio failed (see stderr)")
        n = lib().encodec_get_codes_size(self.ctx)
        T = (a.size + 319) // 320
        return np.ctypeslib.as_array(lib().encodec_get_codes(self.ctx), shape=(n,)).copy().reshape(n // T, T)

    def decompress(self, codes) -> np.ndarray:
        """Codes [n_q][T] (n_q of the current bandwidth) -> 320 T float32 samples."""
        c = np.ascontiguousarray(codes, np.int32)
        if not lib().encodec_decompress_audio(self.ctx, _p(c), c.size, 1):
            raise RuntimeError("encodec_decompress_audio failed (see stderr)")
        return self._audio()

    def reconstruct(self, audio) -> np.ndarray:
        """compress then decompress on the device: 320 T float32 samples."""
        a = np.ascontiguousarray(audio, np.float32).ravel()
        if not lib().encodec_reconstruct_audio(self.ctx, _p(a), a.size, 1):
            raise RuntimeError("encodec_reconstruct_audio failed (see stderr)")
        return self._audio()

    def _audio(self):
        n = lib().encodec_get_audio_size(self.ctx)
        return np.ctypeslib.as_array(lib().encodec_get_audio(self.ctx), shape=(n,)).copy()

    def stats(self) -> dict:
        s = lib().encodec_get_statistics(self.ctx).contents
        return {"t_load_us": s.t_load_us, "t_compute_us": s.t_compute_us}

    def reset_stats(self):
        lib().encodec_reset_statistics(self.ctx)


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
