"""TEST INFRASTRUCTURE — ctypes bindings of the two checkers under oracle/.

  Oracle : oracle/libbark_oracle.so  — our plain-C restatement (oracle/bark_oracle.c)
  Ref    : oracle/_ref/libbark_ref.so — the unmodified reference compiled by oracle/Makefile
           (exists where build() found the reference's source tree: REFERENCE_DIR below)

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs import this.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

# The C oracle uses OpenMP.  On big shared hosts (a host may report 128 logical CPUs while a container gets far fewer
# cycles) a 128-thread team that spin-waits between the hundreds of tiny parallel regions of the LSTM loop can stall
# for minutes, so cap the team and make idle threads sleep.  Must be set before libgomp initialises.
os.environ.setdefault("OMP_NUM_THREADS", str(min(16, os.cpu_count() or 1)))
os.environ.setdefault("OMP_WAIT_POLICY", "passive")

HERE = os.path.dirname(os.path.abspath(__file__))
ORACLE_SO = os.path.join(HERE, "libbark_oracle.so")
REF_SO = os.path.join(HERE, "_ref", "libbark_ref.so")
vp = C.c_void_p


def _p(a):
    return a.ctypes.data_as(vp)


def build_oracle():
    subprocess.check_call(["make", "-C", HERE, "oracle"], stdout=subprocess.DEVNULL)


# The reference's source tree (a PABannier/bark.cpp checkout with its submodules): BARK_REFERENCE_DIR overrides the default location.
REFERENCE_DIR = os.environ.get("BARK_REFERENCE_DIR") or "/root/reference"


def build_ref() -> bool:
    """Compile oracle/_ref/libbark_ref.so from REFERENCE_DIR (oracle/Makefile); False when that tree does not exist."""
    if not os.path.isdir(REFERENCE_DIR):
        return False
    subprocess.check_call(["make", "-C", HERE, "ref", "-j8", f"REF={REFERENCE_DIR}"], stdout=subprocess.DEVNULL)
    return True


def have_ref() -> bool:
    return os.path.exists(REF_SO)


class Oracle:
    def __init__(self, path: str, seed: int = 0, n_steps: int = 768, temp=0.7, fine_temp=0.5, min_eos_p=0.2):
        if not os.path.exists(ORACLE_SO):
            build_oracle()
        L = self.L = C.CDLL(ORACLE_SO)
        L.orc_load.restype = vp
        L.orc_load.argtypes = [C.c_char_p, C.c_uint32]
        L.orc_set_params.argtypes = [vp, C.c_float, C.c_float, C.c_float, C.c_int]
        L.orc_gpt_eval.argtypes = [vp, C.c_int, vp, C.c_int, C.POINTER(C.c_int), C.c_int, vp]
        L.orc_fine_eval.argtypes = [vp, vp, C.c_int, vp]
        L.orc_sample.argtypes = [vp, vp, C.c_int, C.c_float, C.POINTER(C.c_float)]
        L.orc_reseed.argtypes = [vp, C.c_uint32]
        L.orc_tokenize.argtypes = [vp, C.c_char_p, vp]
        L.orc_hparams.argtypes = [vp, C.c_int, vp]
        L.orc_semantic.argtypes = [vp, vp, vp]
        L.orc_coarse.argtypes = [vp, vp, C.c_int, vp]
        L.orc_fine.argtypes = [vp, vp, C.c_int, vp]
        L.orc_encodec_decode.argtypes = [vp, vp, C.c_int, vp]
        L.orc_generate.argtypes = [vp, C.c_char_p, vp, vp, vp, vp, vp, vp]
        L.orc_vec_dot_f16.restype = C.c_float
        L.orc_vec_dot_f16.argtypes = [C.c_int, vp, vp]
        L.orc_vec_dot_f32.restype = C.c_float
        L.orc_vec_dot_f32.argtypes = [C.c_int, vp, vp]
        L.orc_v_expf.restype = C.c_float
        L.orc_v_expf.argtypes = [C.c_float]
        self.ctx = vp(L.orc_load(os.fsencode(path), seed))
        if not self.ctx:
            raise RuntimeError(f"oracle failed to load {path}")
        L.orc_set_params(self.ctx, temp, fine_temp, min_eos_p, n_steps)

    def hparams(self, which):
        a = np.zeros(10, np.int32); self.L.orc_hparams(self.ctx, which, _p(a)); return a

    def reseed(self, seed): self.L.orc_reseed(self.ctx, seed)

    def tokenize(self, text):
        a = np.zeros(513, np.int32); self.L.orc_tokenize(self.ctx, text.encode(), _p(a)); return a

    def gpt_eval(self, which, tokens, n_past, merge_ctx):
        t = np.ascontiguousarray(tokens, np.int32)
        out = np.zeros(int(self.hparams(which)[6]), np.float32)
        np_ = C.c_int(n_past)
        assert self.L.orc_gpt_eval(self.ctx, which, _p(t), t.size, C.byref(np_), int(merge_ctx), _p(out))
        return out, np_.value

    def fine_eval(self, in_buffer, nn):
        t = np.ascontiguousarray(in_buffer, np.int32)
        out = np.zeros((1024, int(self.hparams(2)[6])), np.float32)
        assert self.L.orc_fine_eval(self.ctx, _p(t), nn, _p(out))
        return out

    def sample(self, logits, temp):
        l = np.ascontiguousarray(logits, np.float32); e = C.c_float(0)
        return self.L.orc_sample(self.ctx, _p(l), l.size, temp, C.byref(e)), e.value

    def encodec_decode(self, codes_8xT):
        c = np.ascontiguousarray(codes_8xT, np.int32); T = c.shape[1]
        out = np.zeros(320 * T, np.float32)
        n = self.L.orc_encodec_decode(self.ctx, _p(c), T, _p(out))
        return out[:n]

    def generate(self, text):
        sem = np.zeros(1024, np.int32); co = np.zeros((1024, 2), np.int32); fi = np.zeros((1024, 8), np.int32)
        au = np.zeros(320 * 1024, np.float32); ns = C.c_int(0); T = C.c_int(0)
        n = self.L.orc_generate(self.ctx, text.encode(), _p(sem), C.byref(ns), _p(co), _p(fi), C.byref(T), _p(au))
        if n < 0:
            raise RuntimeError("the clip has more than 1024 coarse frames: the reference's fine stage cannot hold it (use the stage calls)")
        return dict(semantic=sem[:ns.value].copy(), coarse=co[:T.value].copy(), fine=fi[:T.value].copy(), audio=au[:n].copy())

    # the stages of generate one at a time, on the context's RNG stream (generate calls them in this order)
    def semantic(self, prompt):
        """semantic ids of a tokenized prompt (tokenize)"""
        p = np.ascontiguousarray(prompt, np.int32); out = np.zeros(1024, np.int32)
        return out[:self.L.orc_semantic(self.ctx, _p(p), _p(out))].copy()

    def coarse(self, semantic):
        """coarse ids [T][2] (codebook ids, 0 .. 1023) of semantic ids"""
        s = np.ascontiguousarray(semantic, np.int32); out = np.zeros((2048, 2), np.int32)
        return out[:self.L.orc_coarse(self.ctx, _p(s), s.size, _p(out))].copy()

    def fine(self, coarse):
        """fine ids [T][8] of coarse ids [T][2], T <= 1024"""
        c = np.ascontiguousarray(coarse, np.int32); out = np.zeros((c.shape[0], 8), np.int32)
        self.L.orc_fine(self.ctx, _p(c), c.shape[0], _p(out))
        return out


class Ref:
    """The real reference through oracle/ref_harness.cpp."""

    def __init__(self, path: str, seed: int = 0, n_steps: int = 768, temp=0.7, fine_temp=0.5, min_eos_p=0.2):
        if not have_ref():
            raise RuntimeError(f"oracle/_ref/libbark_ref.so not built (no reference tree at {REFERENCE_DIR}; set BARK_REFERENCE_DIR)")
        L = self.L = C.CDLL(REF_SO)
        L.ref_load.restype = vp
        L.ref_load.argtypes = [C.c_char_p, C.c_uint32, C.c_int, C.c_int]
        L.ref_set_params.argtypes = [vp, C.c_float, C.c_float, C.c_float]
        L.ref_generate.argtypes = [vp, C.c_char_p, C.c_int]
        L.ref_gpt_eval.argtypes = [vp, C.c_int, vp, C.c_int, C.POINTER(C.c_int), C.c_int, C.c_int, vp]
        L.ref_fine_eval.argtypes = [vp, vp, C.c_int, C.c_int, vp]
        L.ref_sample.argtypes = [vp, vp, C.c_int, C.c_float, C.POINTER(C.c_float)]
        L.ref_reseed.argtypes = [vp, C.c_uint32]
        L.ref_tokenize.argtypes = [vp, C.c_char_p]
        L.ref_encodec_decode.argtypes = [vp, vp, C.c_int, C.c_int]
        L.ref_get_hparams.argtypes = [vp, C.c_int, vp]
        L.ref_build_info.restype = C.c_char_p
        for n in ("ref_get_prompt", "ref_get_semantic", "ref_get_coarse", "ref_get_fine", "ref_get_audio", "ref_get_stats"):
            getattr(L, n).argtypes = [vp, vp]
        for n in ("ref_n_prompt", "ref_n_semantic", "ref_n_frames", "ref_n_fine_frames", "ref_n_audio"):
            getattr(L, n).argtypes = [vp]
        for n in ("ref_run_semantic", "ref_run_coarse", "ref_run_fine"):
            getattr(L, n).argtypes = [vp, C.c_int]
        self.ctx = vp(L.ref_load(os.fsencode(path), seed, n_steps, 0))
        if not self.ctx:
            raise RuntimeError(f"reference failed to load {path}")
        L.ref_set_params(self.ctx, temp, fine_temp, min_eos_p)

    def close(self):
        """bark_free: the reference has a fixed pool of ggml contexts (64), so long test sessions must give them back"""
        if getattr(self, "ctx", None):
            self.L.ref_free.argtypes = [vp]
            self.L.ref_free(self.ctx)
            self.ctx = None

    def build_info(self): return self.L.ref_build_info().decode()

    def hparams(self, which):
        a = np.zeros(10, np.int32); self.L.ref_get_hparams(self.ctx, which, _p(a)); return a

    def reseed(self, seed): self.L.ref_reseed(self.ctx, seed)

    def tokenize(self, text):
        self.L.ref_tokenize(self.ctx, text.encode())
        a = np.zeros(513, np.int32); self.L.ref_get_prompt(self.ctx, _p(a)); return a

    def gpt_eval(self, which, tokens, n_past, merge_ctx, n_threads=4):
        t = np.ascontiguousarray(tokens, np.int32)
        out = np.zeros(int(self.hparams(which)[6]), np.float32)
        np_ = C.c_int(n_past)
        assert self.L.ref_gpt_eval(self.ctx, which, _p(t), t.size, C.byref(np_), int(merge_ctx), n_threads, _p(out))
        return out, np_.value

    def fine_eval(self, in_buffer, nn, n_threads=4):
        t = np.ascontiguousarray(in_buffer, np.int32)
        out = np.zeros((1024, int(self.hparams(2)[6])), np.float32)
        assert self.L.ref_fine_eval(self.ctx, _p(t), nn, n_threads, _p(out))
        return out

    def sample(self, logits, temp):
        l = np.ascontiguousarray(logits, np.float32); e = C.c_float(0)
        return self.L.ref_sample(self.ctx, _p(l), l.size, temp, C.byref(e)), e.value

    def encodec_decode(self, codes_8xT, n_threads=4):
        c = np.ascontiguousarray(codes_8xT, np.int32)
        n = self.L.ref_encodec_decode(self.ctx, _p(c), c.size, n_threads)
        a = np.zeros(n, np.float32); self.L.ref_get_audio(self.ctx, _p(a)); return a

    def _results(self):
        L, c = self.L, self.ctx
        ns, T, na = L.ref_n_semantic(c), L.ref_n_frames(c), L.ref_n_audio(c)
        sem = np.zeros(max(ns, 1), np.int32); co = np.zeros((max(T, 1), 2), np.int32); fi = np.zeros((max(T, 1), 8), np.int32); au = np.zeros(max(na, 1), np.float32)
        L.ref_get_semantic(c, _p(sem)); L.ref_get_coarse(c, _p(co)); L.ref_get_fine(c, _p(fi)); L.ref_get_audio(c, _p(au))
        return dict(semantic=sem[:ns], coarse=co[:T], fine=fi[:T], audio=au[:na])

    def generate(self, text, n_threads=4):
        if not self.L.ref_generate(self.ctx, text.encode(), n_threads):
            raise RuntimeError("reference bark_generate_audio failed")
        return self._results()

    def stats(self):
        a = np.zeros(14, np.int64); self.L.ref_get_stats(self.ctx, _p(a)); return a


_orc_lib = None


def _oracle_lib():
    global _orc_lib
    if _orc_lib is None:
        if not os.path.exists(ORACLE_SO):
            build_oracle()
        L = C.CDLL(ORACLE_SO)
        L.orc_sample_u.restype = C.c_int
        L.orc_sample_u.argtypes = [vp, C.c_int, C.c_float, C.c_double, C.POINTER(C.c_float)]
        L.orc_mt_seed.argtypes = [vp, C.c_uint32]
        L.orc_mt_next.restype = C.c_uint32
        L.orc_mt_next.argtypes = [vp]
        _orc_lib = L
    return _orc_lib


def sample_u(logits, temp, u):
    """gpt_sample of one logit row with the uniform draw u given (orc_sample_u): (token, probability of the last logit)."""
    l = np.ascontiguousarray(logits, np.float32); e = C.c_float(0)
    return _oracle_lib().orc_sample_u(_p(l), l.size, temp, float(u), C.byref(e)), e.value


def mt_words(seed, k):
    """The first k 32-bit outputs of std::mt19937(seed) (orc_mt_seed / orc_mt_next)."""
    L = _oracle_lib()
    st = np.zeros(625, np.uint32); L.orc_mt_seed(_p(st), seed)
    return np.array([L.orc_mt_next(_p(st)) for _ in range(k)], np.uint64)


QUANT_TYPES = {"q4_0": 2, "q4_1": 3, "q5_0": 6, "q5_1": 7, "q8_0": 8}     # enum ggml_type
QUANT_BLOCK_BYTES = {"q4_0": 18, "q4_1": 20, "q5_0": 22, "q5_1": 24, "q8_0": 34}
Q8_DTYPES = {   # block_q8_0 / block_q8_1 (ggml-common.h)
    "q8_0": np.dtype([("d", "<u2"), ("qs", "i1", 32)]),
    "q8_1": np.dtype([("d", "<u2"), ("s", "<u2"), ("qs", "i1", 32)]),
}


def vec_dot_type(qtype):
    return "q8_1" if qtype in ("q4_1", "q5_1") else "q8_0"


def _quant_lib(L):
    L.orc_quantize_row_q8_0.argtypes = L.orc_quantize_row_q8_1.argtypes = [vp, vp, C.c_int]
    L.orc_vec_dot_q.restype = C.c_float
    L.orc_vec_dot_q.argtypes = [C.c_int, C.c_int, vp, vp]
    L.orc_quant_matmul.restype = C.c_int
    L.orc_quant_matmul.argtypes = [C.c_int, vp, vp, C.c_int, C.c_int, C.c_int, vp]
    return L


def quantize_q8(x, kind):
    """the oracle's quantize_row_q8_0 / q8_1 ("q8_0" / "q8_1") of float32 rows [..][K]: a structured array [..][K/32] of Q8_DTYPES[kind]"""
    x = np.ascontiguousarray(x, np.float32)
    y = np.zeros(x.shape[:-1] + (x.shape[-1] // 32,), Q8_DTYPES[kind])
    getattr(_quant_lib(_oracle_lib()), f"orc_quantize_row_{kind}")(_p(x), _p(y), x.size)
    return y


def vec_dot_q(qtype, w_blocks, y_blocks):
    """the oracle's ggml_vec_dot_<qtype>_<q8_0|q8_1> of one weight row (uint8 file blocks) against one q8 row (quantize_q8's blocks)"""
    w = np.ascontiguousarray(w_blocks, np.uint8); y = np.ascontiguousarray(y_blocks)
    assert y.dtype == Q8_DTYPES[vec_dot_type(qtype)] and w.size == y.size * QUANT_BLOCK_BYTES[qtype], (w.shape, y.shape)
    return np.float32(_quant_lib(_oracle_lib()).orc_vec_dot_q(QUANT_TYPES[qtype], 32 * y.size, _p(w), _p(y)))


def quant_matmul(qtype, W, A):
    """out [M][N] float32: weight row o (W [N][K/32 * block bytes] uint8) against row m of A [M][K] float32 quantised, as the reference's mul_mat"""
    W = np.ascontiguousarray(W, np.uint8); A = np.ascontiguousarray(A, np.float32)
    M, K = A.shape; N = W.shape[0]
    assert W.shape[1] == K // 32 * QUANT_BLOCK_BYTES[qtype], (W.shape, A.shape)
    out = np.zeros((M, N), np.float32)
    assert _quant_lib(_oracle_lib()).orc_quant_matmul(QUANT_TYPES[qtype], _p(W), _p(A), M, N, K, _p(out))
    return out


def gelu_tables():
    """(oracle table, reference table or None): gelu evaluated at every f16 input, as f16 bits."""
    if not os.path.exists(ORACLE_SO):
        build_oracle()
    o = np.zeros(65536, np.uint16); C.CDLL(ORACLE_SO).orc_gelu_table(_p(o))
    r = None
    if have_ref():
        r = np.zeros(65536, np.uint16); C.CDLL(REF_SO).ref_gelu_table(_p(r))
    return o, r
