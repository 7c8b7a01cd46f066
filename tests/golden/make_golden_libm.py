"""Regenerates tests/golden/libm/glibc_2_39.npz — the host libm the oracle and the reference call, on the inputs where it can go wrong.

    python tests/golden/make_golden_libm.py          (a few seconds)

Run it on a host with glibc 2.39 on x86-64 with FMA, the reference's: glibc then selects its FMA build of expf, expm1f and tanhf, and
that build is what the device restatements in csrc/common.cuh follow.  Stored, as f32 bit patterns: the inputs x, and glibc's expm1f,
tanhf and expf and the oracle's ggml_v_expf (orc_v_expf, the AVX2 ggml_v_expf restated in C) at each.  The inputs are
  - every pattern within 256 of each branch cut in CUTS, both signs;
  - ±0, ±inf, the smallest and largest subnormals and a sample of the others, quiet and signalling NaN payloads of both signs;
  - a uniform sample of 80 000 bit patterns.
tests/test_codec_oracle_ops.py checks that the host still gives these values; tests/test_codec_kernels_gpu.py compares the device
functions with the host and checks the host against this file first.
"""
import ctypes
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "libm", "glibc_2_39.npz")
FUNCTIONS = ("expm1f", "tanhf", "expf", "v_expf")

# the magnitudes (f32 bits) where a branch of expm1f, tanhf, expf, ggml_v_expf, the sigmoid or the f16 round trip changes
CUTS = [0x4195B844, 0x42B17218, 0x42B17180, 0x3EB17218, 0x3F851592, 0x33000000, 0x3E800000,   # expm1f: 27 ln2, overflow, 0.5 / 1.5 ln2, 2^-25, -0.25
        0x411C8000, 0x421C9000, 0x41797000,                                                   # expm1f's k = 23 and k = 56 cuts (near 22.5 ln2, 56.5 ln2), 15.6
        0x41B00000, 0x24000000, 0x3F800000, 0x00000000,                                       # tanhf: 22, 2^-55, 1, 0
        0x42B00000, 0x42B17217, 0x42CFF1B4, 0x7F800000,                                       # expf: 88, overflow, underflow, inf / NaN
        0x42AEAC50, 0x430517A0,                                                               # ggml_v_expf: |n| = 126, 192 (126 ln2, 192 ln2)
        0x477FF000, 0x38800000, 0x00800000,                                                   # f16: 65520, 2^-14, the f32 subnormals
        0x4202422F, 0xC27C65D9]   # the two inputs where expf differs when x log2(e) 32 is rounded before k is subtracted (glibc's FMA build fuses it)


def inputs() -> np.ndarray:
    """The fixture's inputs: sorted, distinct uint32 bit patterns."""
    rng = np.random.Generator(np.random.PCG64(239))
    parts = []
    for c in CUTS:
        for sign in (0, 0x80000000):
            parts.append((np.uint32((c | sign) - 256 & 0xFFFFFFFF) + np.arange(513, dtype=np.uint32)).astype(np.uint32))
    sub = np.concatenate([np.arange(1, 256), np.arange(0x7FFF00, 0x800000), rng.integers(1, 0x800000, 1024)]).astype(np.uint32)
    nan = np.concatenate([[0x7F800001, 0x7FA00000, 0x7FBFFFFF, 0x7FC00000, 0x7FC00001, 0x7FFFFFFF, 0x7F800100],
                          rng.integers(0x7F800001, 0x80000000, 64)]).astype(np.uint32)
    special = np.array([0, 0x7F800000], np.uint32)
    for p in (sub, nan, special):
        parts += [p, p | np.uint32(0x80000000)]
    parts.append(rng.integers(0, 1 << 32, 80000, dtype=np.uint64).astype(np.uint32))
    return np.unique(np.concatenate(parts))


def main():
    sys.path.insert(0, os.path.dirname(HERE))
    import encoder_oracle as eo
    version = ctypes.CDLL("libc.so.6").gnu_get_libc_version
    version.restype = ctypes.c_char_p
    x = inputs()
    out = {"x": x, "glibc": np.array(version().decode())}
    for fn in FUNCTIONS:
        out[fn] = eo.libm(fn, x).view(np.uint32)
    os.makedirs(os.path.dirname(OUT), exist_ok=True)
    np.savez_compressed(OUT, **out)
    print(f"{OUT}: {x.size} inputs, glibc {out['glibc']}, {os.path.getsize(OUT)} bytes")


if __name__ == "__main__":
    main()
