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
