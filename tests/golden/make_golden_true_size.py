"""Regenerates the true-size fixtures of BASELINE.json configs[1..3] by running the UNMODIFIED reference
(oracle/_ref/libbark_ref.so, built by oracle/Makefile from the reference tree named by BARK_REFERENCE_DIR):

  small_f16_n138.npz       configs[1]: bark-small f16, THE BENCH CLIP (prompt "hello world", seed 0, n_steps_text_encoder = 138 ->
                           414 coarse steps = 7 sliding windows with prefix reuse, 207 frames, 66 240 samples)
  large_f16_n8.npz         configs[2]: bark-large dimensions (E = 1024, 24 layers, 16 heads), full depth, 8 semantic steps.  The
                           UNMODIFIED REFERENCE CANNOT LOAD THIS FILE: it is 2.24 GB and bark.cpp:1150 keeps the codec offset in an
                           `int` (the codec section starts beyond 2 GiB -> garbage header -> GGML_ASSERT in
                           encodec_load_model_weights).  This fixture therefore comes from the C oracle (oracle/bark_oracle.c,
                           pinned bit-exactly to the reference on every file the reference can load); `source` says so.
  large_f16_q4_0_n8.npz    the same bark-large file quantised to q4_0 by the reference's tool (0.66 GB, loads fine): full depth
                           E = 1024 / 24 layers / 16 heads against the unmodified reference itself
  small_f16_q4_0_n12.npz   configs[3]: bark-small, GPT weights quantised to q4_0 by the REFERENCE's bark_model_quantize, 12 steps

    python tests/golden/make_golden_true_size.py [small|large|q4]        (needs the reference build oracle/_ref)

Weight files are not committed: bark.cpp_b200/weights.py regenerates them bit-identically from (config, ftype, seed), the library's
own bark_model_quantize reproduces the reference's q4_0 file byte for byte (tests/test_quantize.py); sha1 sums are in the fixtures.
"""
import ctypes as C
import hashlib
import importlib
import os
import tempfile
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
os.environ.setdefault("BARK_B200_QUIET", "1")
import __graft_entry__ as graft  # noqa: E402

CASES = {  # name -> (config, quant, rng seed, n_steps, prompt, fixture)
    "small": ("small", "", 0, 138, "hello world", "small_f16_n138.npz"),
    "large": ("large", "", 0, 8, "hello world", "large_f16_n8.npz"),          # from the C oracle (see above)
    "large_q4": ("large", "q4_0", 0, 8, "hello world", "large_f16_q4_0_n8.npz"),
    "q4": ("small", "q4_0", 0, 12, "hello world", "small_f16_q4_0_n12.npz"),
}


def file_sha1(path):
    h = hashlib.sha1()
    with open(path, "rb") as f:
        for blk in iter(lambda: f.read(1 << 24), b""):
            h.update(blk)
    return h.hexdigest()


def main():
    graft.load_package()
    weights = importlib.import_module("bark_cpp_b200.weights")
    orc = graft.load_oracle_bindings()
    tmp = os.environ.get("BARK_B200_FIXTURES", os.path.join(tempfile.gettempdir(), f"bark_b200_fixtures_{os.getuid()}"))
    os.makedirs(tmp, exist_ok=True)
    out_dir = os.path.dirname(os.path.abspath(__file__))
    for name in (sys.argv[1:] or list(CASES)):
        config, quant, seed, n_steps, prompt, fixture = CASES[name]
        path = os.path.join(tmp, f"{config}_f16_1234.bin")
        if not os.path.exists(path):
            weights.write_weights(path, weights.CONFIGS[config](weights.F16), 1234)
        if quant:
            init = os.path.join(tmp, "tiny_f16_1234.bin")      # ggml_init first: f16 tables (examples/quantize/main.cpp:67-72); any loadable file does
            if not os.path.exists(init):
                weights.write_weights(init, weights.tiny(weights.F16), 1234)
            orc.Ref(init).close()
            R = C.CDLL(orc.REF_SO)
            R.bark_model_quantize.restype = C.c_bool
            R.bark_model_quantize.argtypes = [C.c_char_p, C.c_char_p, C.c_int]
            qpath = os.path.join(tmp, f"{config}_f16_1234_{quant}_ref.bin")
            assert quant == "q4_0" and R.bark_model_quantize(path.encode(), qpath.encode(), 2)
            path = qpath
        t0 = time.time()
        if os.path.getsize(path) >= 2 ** 31:                 # the reference's `const int offset` (bark.cpp:1150) overflows: oracle instead
            orc.build_oracle()
            r = orc.Oracle(path, seed=seed, n_steps=n_steps)
            g = r.generate(prompt)
            source, build = "oracle/bark_oracle.c (the unmodified reference cannot load files >= 2 GiB: int offset, bark.cpp:1150)", "C oracle, pinned to " + orc.Ref.__doc__.strip().split("\n")[0] if orc.Ref.__doc__ else "C oracle"
        else:
            r = orc.Ref(path, seed=seed, n_steps=n_steps)
            g = r.generate(prompt, n_threads=8)
            source, build = "oracle/_ref (unmodified reference)", r.build_info()
        np.savez_compressed(
            os.path.join(out_dir, fixture), config=config, ftype="f16", quant=quant, weight_seed=1234, seed=seed, n_steps=n_steps, prompt=prompt,
            reference_build=build, source=source, weights_sha1=file_sha1(path), prompt_ids=r.tokenize(prompt),
            semantic=g["semantic"], coarse=g["coarse"], fine=g["fine"], audio=g["audio"])
        print(name, "semantic", g["semantic"].size, "frames", g["coarse"].shape[0], "audio", g["audio"].size, f"{time.time() - t0:.1f} s", flush=True)


if __name__ == "__main__":
    main()
