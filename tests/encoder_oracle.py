"""ctypes binding of tests/encoder_oracle.c (the EnCodec encoder's CPU restatement), compiled on first use into a per-user
temporary directory with the oracle's flags (oracle/Makefile: no FP contraction, OpenMP)."""
from __future__ import annotations

import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
SRC = os.path.join(HERE, "encoder_oracle.c")
DEPS = (SRC, os.path.join(ROOT, "oracle", "bark_oracle.c"), os.path.join(ROOT, "oracle", "bark_oracle.h"))
vp = C.c_void_p

os.environ.setdefault("OMP_NUM_THREADS", str(min(16, os.cpu_count() or 1)))   # as oracle/bindings.py
os.environ.setdefault("OMP_WAIT_POLICY", "passive")

_lib = None


def _p(a):
    return a.ctypes.data_as(vp)


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        h = hashlib.sha1(b"".join(open(p, "rb").read() for p in DEPS)).hexdigest()[:16]
        out_dir = os.path.join(tempfile.gettempdir(), f"bark_b200_encoder_oracle_{os.getuid()}")
        so = os.path.join(out_dir, f"libencoder_oracle_{h}.so")
        if not os.path.exists(so):
            os.makedirs(out_dir, exist_ok=True)
            tmp = f"{so}.{os.getpid()}.tmp"
            subprocess.check_call(["gcc", "-O2", "-std=gnu11", "-fPIC", "-shared", "-ffp-contract=off", "-fno-fast-math", "-w", "-fopenmp",
                                   SRC, "-o", tmp, "-lm"])
            os.replace(tmp, so)
        L = C.CDLL(so)
        L.oenc_load.restype = vp
        L.oenc_load.argtypes = [C.c_char_p]
        L.orc_encodec_encode.restype = C.c_int
        L.orc_encodec_encode.argtypes = [vp, vp, C.c_int, vp, vp]
        L.orc_rvq_encode.argtypes = [vp, C.c_int, vp, C.c_int, C.c_int, C.c_int, vp]
        L.orc_codec_conv1d.restype = C.c_int
        L.orc_codec_conv1d.argtypes = [vp, C.c_int, C.c_int, vp, vp] + [C.c_int] * 4 + [vp, vp]
        L.orc_codec_convtr1d.restype = C.c_int
        L.orc_codec_convtr1d.argtypes = [vp, C.c_int, C.c_int, vp, vp, C.c_int, C.c_int, vp]
        L.orc_codec_lstm.argtypes = [vp, C.c_int, C.c_int, vp, vp, vp, vp, vp, vp]
        L.orc_codec_rvq_decode.argtypes = [vp, C.c_int, C.c_int, vp, C.c_int, C.c_int, vp]
        L.orc_libm.argtypes = [C.c_int, vp, C.c_longlong, vp]
        _lib = L
    return _lib


class EncoderOracle:
    """The encoder and codebooks 0..7 of one weight file."""

    def __init__(self, path: str):
        self.m = vp(lib().oenc_load(os.fsencode(path)))
        if not self.m:
            raise RuntimeError(f"{path}: no EnCodec encoder in the file (or unreadable)")

    def encode(self, audio, return_latent: bool = False):
        """orc_encodec_encode: codes [8][T] int32 (and the latent [128][T] float32)."""
        a = np.ascontiguousarray(audio, np.float32).ravel()
        T = (a.size + 319) // 320
        codes = np.zeros((8, T), np.int32); lat = np.zeros((128, T), np.float32)
        r = lib().orc_encodec_encode(self.m, _p(a), a.size, _p(codes), _p(lat))
        assert r == T, (r, T)
        return (codes, lat) if return_latent else codes


def rvq_encode(latent, codebooks) -> np.ndarray:
    """orc_rvq_encode: latent [hidden][T], codebooks [n_q][n_bins][hidden] float32 -> codes [n_q][T] int32."""
    lat = np.ascontiguousarray(latent, np.float32); cb = np.ascontiguousarray(codebooks, np.float32)
    hidden, T = lat.shape
    n_q, n_bins, _ = cb.shape
    codes = np.zeros((n_q, T), np.int32)
    lib().orc_rvq_encode(_p(lat), T, _p(cb), hidden, n_bins, n_q, _p(codes))
    return codes


def _opt(a):
    return None if a is None else _p(a)


def conv1d(x, w, bias, stride: int = 1, elu_in: bool = False, resid=None) -> np.ndarray:
    """orc_codec_conv1d on one item: x [Cin][L] float32, w [Cout][Cin][k] float16, bias [Cout] -> [Cout][T]."""
    x = np.ascontiguousarray(x, np.float32); w = np.ascontiguousarray(w, np.float16); b = np.ascontiguousarray(bias, np.float32)
    Cout, Cin, k = w.shape
    assert x.shape[0] == Cin and x.shape[1] > k - stride, (x.shape, w.shape, stride)
    r = None if resid is None else np.ascontiguousarray(resid, np.float32)
    y = np.zeros(Cout * x.shape[1], np.float32)           # T <= L for every stride >= 1
    T = lib().orc_codec_conv1d(_p(x), Cin, x.shape[1], _p(w), _p(b), Cout, k, stride, int(elu_in), _opt(r), _p(y))
    return y[:Cout * T].reshape(Cout, T)


def convtr1d(x, w, bias, stride: int) -> np.ndarray:
    """orc_codec_convtr1d on one item: ELU, then the transposed conv; x [Cin][T], w [Cin][Cout][2 stride] float16 -> [Cout][T stride]."""
    x = np.ascontiguousarray(x, np.float32); w = np.ascontiguousarray(w, np.float16)
    Cin, Cout, k = w.shape
    y = np.zeros((Cout, x.shape[1] * stride), np.float32)
    L = lib().orc_codec_convtr1d(_p(x), Cin, x.shape[1], _p(w), _p(np.ascontiguousarray(bias, np.float32)), Cout, stride, _p(y))
    assert L == y.shape[1], (L, y.shape)
    return y


def lstm(x, wih, whh, bih, bhh, skip=None) -> np.ndarray:
    """orc_codec_lstm on one item: x [C][T], wih / whh [4C][C] float16, bih / bhh [4C]; skip [C][T] added when given."""
    x = np.ascontiguousarray(x, np.float32)
    C, T = x.shape
    out = np.zeros((C, T), np.float32)
    lib().orc_codec_lstm(_p(x), C, T, _p(np.ascontiguousarray(wih, np.float16)), _p(np.ascontiguousarray(whh, np.float16)),
                         _p(np.ascontiguousarray(bih, np.float32)), _p(np.ascontiguousarray(bhh, np.float32)),
                         _opt(None if skip is None else np.ascontiguousarray(skip, np.float32)), _p(out))
    return out


def rvq_decode(codes, codebooks) -> np.ndarray:
    """orc_codec_rvq_decode on one item: codes [n_q][T] int32, codebooks [n_q][n_bins][hidden] float32 -> [hidden][T]."""
    c = np.ascontiguousarray(codes, np.int32); cb = np.ascontiguousarray(codebooks, np.float32)
    n_q, n_bins, hidden = cb.shape
    x = np.zeros((hidden, c.shape[1]), np.float32)
    lib().orc_codec_rvq_decode(_p(c), n_q, c.shape[1], _p(cb), hidden, n_bins, _p(x))
    return x


LIBM = {"expm1f": 0, "tanhf": 1, "expf": 2, "v_expf": 3, "elu": 4, "sigmoid": 5, "round_f16": 6}   # bark_b200_device_math's fn


def libm(fn: str, x_bits) -> np.ndarray:
    """orc_libm: the host's function on the floats of bit patterns x_bits (uint32)."""
    x = np.ascontiguousarray(x_bits, np.uint32)
    out = np.zeros(x.size, np.float32)
    lib().orc_libm(LIBM[fn], _p(x), x.size, _p(out))
    return out


LIBM_FIXTURE = os.path.join(HERE, "golden", "libm", "glibc_2_39.npz")


def libm_fixture_mismatch() -> str | None:
    """None when this host's expm1f, tanhf and expf and the oracle's ggml_v_expf give, bit for bit and NaN for NaN, the values stored
    in tests/golden/libm/glibc_2_39.npz (tests/golden/make_golden_libm.py); else what differs."""
    g = np.load(LIBM_FIXTURE)
    x = g["x"]
    for fn in ("expm1f", "tanhf", "expf", "v_expf"):
        got, want = libm(fn, x), g[fn].view(np.float32)
        bad = np.flatnonzero((got.view(np.uint32) != want.view(np.uint32)) & ~(np.isnan(got) & np.isnan(want)))
        if bad.size:
            i = bad[0]
            return (f"the host libm is not the reference's (glibc {g['glibc']} on x86-64 with FMA): {fn} differs on {bad.size} of {x.size} "
                    f"stored inputs, first at bits {int(x[i]):#010x}: host {got[i]!r}, stored {want[i]!r}.  The oracle's waveforms would "
                    f"then not be the reference's either, and the device libm cannot be checked against this host.")
    return None


def pattern_bits(lo_bits: int, count: int, stride: int = 1) -> np.ndarray:
    """The bit patterns lo_bits + i stride (mod 2^32), i < count, as bark_b200_device_math walks them."""
    return (np.uint32(lo_bits & 0xFFFFFFFF) + np.arange(count, dtype=np.uint32) * np.uint32(stride)).astype(np.uint32)


# test signals, regenerated from seeds (tests/golden/make_golden_encoder.py stores only the reference's outputs)
def signal(kind: str, n: int, seed: int = 0) -> np.ndarray:
    t = np.arange(n, dtype=np.float64)
    if kind == "noise":
        return np.random.Generator(np.random.PCG64(seed)).uniform(-1.0, 1.0, n).astype(np.float32)
    if kind == "sine":
        return (0.5 * np.sin(2 * np.pi * 440.0 * t / 24000.0)).astype(np.float32)
    if kind == "square":
        return np.where((t // 60) % 2 == 0, 1.0, -1.0).astype(np.float32)
    if kind == "silence":
        return np.zeros(n, np.float32)
    raise ValueError(kind)


def tie_overrides(kind: str, seed: int) -> dict:
    """Codebook overrides that force exact ties in the argmax: "pairs" makes rows 2m and 2m+1 of codebook 0 identical (every code of
    codebook 0 is then odd: the last index of a maximum wins), "halves" makes row j + 512 of codebook 3 equal to row j."""
    rng = np.random.Generator(np.random.PCG64(seed))
    cb = rng.standard_normal((1024, 128), dtype=np.float32)
    if kind == "pairs":
        cb[1::2] = cb[0::2]
        return {"quantizer.vq.layers.0._codebook.embed": cb}
    if kind == "halves":
        cb[512:] = cb[:512]
        return {"quantizer.vq.layers.3._codebook.embed": cb}
    raise ValueError(kind)


# (name, signal, length, weight file): the cases whose reference outputs are stored in tests/golden/ref_pairs/encoder.npz
WEIGHTS = {"base": None, "tie_pairs": "pairs", "tie_halves": "halves"}
CASES = [
    ("noise_1921", "noise", 1921, "base"),          # the minimum: 7 frames
    ("sine_2240", "sine", 2240, "base"),            # exactly 7 frames
    ("noise_24001", "noise", 24001, "base"),        # L mod r != 0 at all four down-sampling levels: right padding everywhere
    ("square_24000", "square", 24000, "base"),
    ("silence_24000", "silence", 24000, "base"),
    ("noise_72013", "noise", 72013, "base"),        # about 3 s at an odd length
    ("noise_4800_pairs", "noise", 4800, "tie_pairs"),
    ("sine_4801_halves", "sine", 4801, "tie_halves"),
]
RECONSTRUCT = ("noise_1921", "noise_24001", "square_24000", "noise_4800_pairs")   # cases whose encodec_reconstruct_audio is stored too


def weights_path(weights_file_getter, weights_mod, which: str) -> str:
    """The tiny f16 fixture (seed 1234), or a copy with the tie overrides written next to the cached fixtures."""
    base = weights_file_getter("tiny", "f16", 1234)
    kind = WEIGHTS[which]
    if kind is None:
        return base
    path = os.path.join(os.path.dirname(base), f"tiny_f16_1234_{which}.bin")
    if not os.path.exists(path):
        weights_mod.write_weights(path + ".tmp", weights_mod.tiny(), 1234, overrides=tie_overrides(kind, 77))
        os.replace(path + ".tmp", path)
    return path
