"""Regenerates tests/golden/ref_pairs/encodec_bandwidths.npz: what the unmodified reference (oracle/_ref/libbark_ref.so, built by
oracle/Makefile where the reference sources exist) returns from encodec.cpp's API at bandwidths other than bark's 6 kbps, for the
cases of tests/encoder_oracle.py CASES (inputs regenerated from seeds there):
  - encodec_compress_audio codes [n_q][T] at 1, 2, 3, 12 and 24 kbps for every case, the two tie files included;
  - encodec_reconstruct_audio waveforms at 3, 12 and 24 kbps for the RECONSTRUCT cases (pinned: shape / sha1 / first values);
  - encodec_decompress_audio waveforms at 12 and 24 kbps for seeded random codes (pinned).
Run where the reference exists:

    python tests/golden/make_golden_encodec.py
"""
import ctypes as C
import importlib
import os
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_golden_encoder import RefCodec, eo, graft, pin  # noqa: E402

OUT = os.path.join(HERE, "ref_pairs", "encodec_bandwidths.npz")
COMPRESS_BW = (1, 2, 3, 12, 24)
RECONSTRUCT_BW = (3, 12, 24)
DECOMPRESS_BW = (12, 24)
DECOMPRESS_FRAMES = 83                                       # frames of the random codes


def decompress_codes(bandwidth: int, n_q: int) -> np.ndarray:
    return np.random.Generator(np.random.PCG64(500 + bandwidth)).integers(0, 1024, (n_q, DECOMPRESS_FRAMES)).astype(np.int32)


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

        def ref_for(which):
            path = eo.weights_path(get, weights, which)
            if path not in cache:
                cache[path] = RefCodec(path)
            return cache[path]

        for name, kind, n, which in eo.CASES:
            ref = ref_for(which)
            x = eo.signal(kind, n, seed=n)
            for bw in COMPRESS_BW:
                ref.L.encodec_set_target_bandwidth(ref.ctx, bw)
                a = np.ascontiguousarray(x, np.float32)
                assert ref.L.encodec_compress_audio(ref.ctx, a.ctypes.data, a.size, 4)
                size = ref.L.encodec_get_codes_size(ref.ctx)
                out[f"{name}_bw{bw}_codes"] = np.ctypeslib.as_array(ref.L.encodec_get_codes(ref.ctx), shape=(size,)).copy().reshape(-1, (n + 319) // 320)
                if name in eo.RECONSTRUCT and bw in RECONSTRUCT_BW:
                    pin(out, f"{name}_bw{bw}_audio", ref.reconstruct(x))
            print(name, flush=True)
        ref = ref_for("base")
        ref.L.encodec_decompress_audio.restype = C.c_bool
        ref.L.encodec_decompress_audio.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int]
        for bw, n_q in zip(DECOMPRESS_BW, (16, 32)):
            ref.L.encodec_set_target_bandwidth(ref.ctx, bw)
            c = decompress_codes(bw, n_q)
            assert ref.L.encodec_decompress_audio(ref.ctx, c.ctypes.data, c.size, 4)
            size = ref.L.encodec_get_audio_size(ref.ctx)
            pin(out, f"decompress_bw{bw}_audio", np.ctypeslib.as_array(ref.L.encodec_get_audio(ref.ctx), shape=(size,)).copy())
    np.savez_compressed(OUT, **out)
    print("wrote", OUT)


if __name__ == "__main__":
    main()
