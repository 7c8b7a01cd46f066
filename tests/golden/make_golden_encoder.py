"""Regenerates tests/golden/ref_pairs/encoder.npz: what the unmodified reference (oracle/_ref/libbark_ref.so, built by oracle/Makefile
where the reference sources exist) returns from encodec_compress_audio and encodec_reconstruct_audio (encodec.cpp/encodec.cpp:860-900,
bandwidth 6 kbps, 24 kHz) for the cases of tests/encoder_oracle.py CASES.  The inputs are regenerated from seeds there; only the
reference's outputs are stored: codes [8][T] in full, reconstructed waveforms as shape / sha1 / first values (conftest.assert_pinned).

The library exports encodec.cpp's C API, so the encoder is loaded straight from the codec section of the weight file
(encodec_load_model with the section's byte offset, as bark_load_model does at bark.cpp:1149-1153).  Run where the reference exists:

    python tests/golden/make_golden_encoder.py
"""
import ctypes as C
import importlib
import os
import struct
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))
import __graft_entry__ as graft  # noqa: E402
import encoder_oracle as eo  # noqa: E402
from make_golden_ref_pairs import pin  # noqa: E402

OUT = os.path.join(HERE, "ref_pairs", "encoder.npz")
_TYPE_BYTES = {0: lambda n: 4 * n, 1: lambda n: 2 * n, 2: lambda n: n // 32 * 18}


def codec_offset(path: str) -> int:
    """Byte offset of the codec section (its magic): after the vocabulary and the three GPT sections (bark.cpp:664-1078)."""
    with open(path, "rb") as f:
        magic, n_vocab = struct.unpack("<Ii", f.read(8))
        for _ in range(n_vocab):
            (n,) = struct.unpack("<I", f.read(4)); f.seek(n, 1)
        for _ in range(3):
            f.seek(40, 1)
            (n_tensors,) = struct.unpack("<i", f.read(4))
            for _ in range(n_tensors):
                n_dims, name_len, ttype = struct.unpack("<iii", f.read(12))
                ne = struct.unpack("<%di" % n_dims, f.read(4 * n_dims))
                f.seek(name_len + _TYPE_BYTES[ttype](int(np.prod(ne))), 1)
        return f.tell()


class RefCodec:
    def __init__(self, path: str):
        orc = graft.load_oracle_bindings()
        if not orc.have_ref():
            raise SystemExit(f"{orc.REF_SO} is missing: build it first (python -c 'import __graft_entry__ as g; g.build()')")
        L = self.L = C.CDLL(orc.REF_SO)
        L.encodec_load_model.restype = C.c_void_p
        L.encodec_load_model.argtypes = [C.c_char_p, C.c_int, C.c_int]
        L.encodec_set_target_bandwidth.argtypes = [C.c_void_p, C.c_int]
        L.encodec_set_sample_rate.argtypes = [C.c_void_p, C.c_int]
        for fn in ("encodec_compress_audio", "encodec_reconstruct_audio"):
            getattr(L, fn).restype = C.c_bool
            getattr(L, fn).argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int]
        L.encodec_get_codes.restype = C.POINTER(C.c_int32)
        L.encodec_get_codes_size.restype = C.c_int
        L.encodec_get_audio.restype = C.POINTER(C.c_float)
        L.encodec_get_audio_size.restype = C.c_int
        for fn in ("encodec_get_codes", "encodec_get_codes_size", "encodec_get_audio", "encodec_get_audio_size", "encodec_free"):
            getattr(L, fn).argtypes = [C.c_void_p]
        self.ctx = L.encodec_load_model(os.fsencode(path), codec_offset(path), 0)
        assert self.ctx, path
        L.encodec_set_target_bandwidth(self.ctx, 6)      # what bark_load_model sets (bark.cpp:2207-2208 defaults)
        L.encodec_set_sample_rate(self.ctx, 24000)

    def compress(self, audio, n_threads=4):
        a = np.ascontiguousarray(audio, np.float32)
        assert self.L.encodec_compress_audio(self.ctx, a.ctypes.data, a.size, n_threads)
        n = self.L.encodec_get_codes_size(self.ctx)
        return np.ctypeslib.as_array(self.L.encodec_get_codes(self.ctx), shape=(n,)).copy().reshape(8, -1)

    def reconstruct(self, audio, n_threads=4):
        a = np.ascontiguousarray(audio, np.float32)
        assert self.L.encodec_reconstruct_audio(self.ctx, a.ctypes.data, a.size, n_threads)
        n = self.L.encodec_get_audio_size(self.ctx)
        return np.ctypeslib.as_array(self.L.encodec_get_audio(self.ctx), shape=(n,)).copy()


def main():
    graft.load_package()
    weights = importlib.import_module("bark_cpp_b200.weights")
    out = {}
    with tempfile.TemporaryDirectory() as d:
        cache = {}

        def get(config, ftype, seed):
            path = os.path.join(d, f"{config}_{ftype}_{seed}.bin")
            if not os.path.exists(path):
                weights.write_weights(path, weights.CONFIGS[config](weights.F16), seed)
            return path

        for name, kind, n, which in eo.CASES:
            path = eo.weights_path(get, weights, which)
            if path not in cache:
                cache[path] = RefCodec(path)
            ref = cache[path]
            x = eo.signal(kind, n, seed=n)
            out[name + "_codes"] = ref.compress(x)
            if name in eo.RECONSTRUCT:
                pin(out, name + "_audio", ref.reconstruct(x))
            print(name, out[name + "_codes"].shape, flush=True)
    np.savez_compressed(OUT, **out)
    print("wrote", OUT)


if __name__ == "__main__":
    main()
