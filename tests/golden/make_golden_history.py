"""Regenerates tests/golden/ref_pairs/history.npz: prompted generations (speaker history prompts) computed by
tests/history_oracle.py on the unmodified reference (oracle/_ref/libbark_ref.so), so every logit and every sample comes from the
reference's own code.  The inputs of tests/test_history_prompt.py and tests/test_history_prompt_gpu.py.  Cases, per weight file
(tiny f16 and mini f32, weight seed 1234):

  chained   the reference's own generate() ids of text A, used as the prompt for text B
  over      n_s = 300, n_c = 451, n_f = 600: the 256 / 209 / 512 history trims
  minimal   n_s = 2, n_c = 3, n_f = 0
  long      (tiny only) a 512-frame fine history under a clip long enough for two or more fine windows

Run once where the reference library exists:

    python tests/golden/make_golden_history.py
"""
import hashlib
import importlib
import os
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))
import __graft_entry__ as graft  # noqa: E402
import history_oracle as H  # noqa: E402

OUT = os.path.join(HERE, "ref_pairs", "history.npz")
FULL_AUDIO_FRAMES = 64          # waveforms up to this many frames are stored whole (for the relative tolerance), longer ones pinned

# (config, ftype, case, text, seed, n_steps); the chained case's prompt comes from generate(CHAIN_TEXT) with seed CHAIN_SEED
CHAIN_TEXT, CHAIN_SEED = "the quick brown fox", 7
CASES = [
    ("tiny", "f16", "chained", "hello world", 0, 16),
    ("tiny", "f16", "over", "hello world", 1, 16),
    ("tiny", "f16", "minimal", "the fox", 2, 16),
    ("tiny", "f16", "long", "hello world", 3, 350),
    ("mini", "f32", "chained", "hello world", 0, 12),
    ("mini", "f32", "over", "hello world", 1, 12),
    ("mini", "f32", "minimal", "the fox", 2, 12),
]


def case_prompt(orc, path, case, n_steps):
    rng = np.random.default_rng({"over": 31, "minimal": 32, "long": 33}.get(case, 0))
    if case == "chained":
        r = orc.Ref(path, seed=CHAIN_SEED, n_steps=n_steps)
        g = r.generate(CHAIN_TEXT)
        r.close()
        return H.chained_prompt(g)
    if case == "over":
        p = H.random_prompt(rng, 300, 600)
        p["coarse_prompt"] = rng.integers(0, 1024, (2, 451)).astype(np.int32)
        return p
    if case == "minimal":
        p = H.random_prompt(rng, 2, 0)
        p["coarse_prompt"] = rng.integers(0, 1024, (2, 3)).astype(np.int32)
        return p
    return H.random_prompt(rng, 100, 512)


def sha(a):
    return hashlib.sha1(np.ascontiguousarray(a).tobytes()).hexdigest()


def main():
    graft.load_package()
    weights = importlib.import_module("bark_cpp_b200.weights")
    orc = graft.load_oracle_bindings()
    if not orc.have_ref():
        sys.exit("oracle/_ref/libbark_ref.so is not built: run build() where the reference sources exist")
    d = {}
    with tempfile.TemporaryDirectory() as tmp:
        for config, ftype, case, text, seed, n_steps in CASES:
            path = os.path.join(tmp, f"{config}_{ftype}_1234.bin")
            if not os.path.exists(path):
                weights.write_weights(path, weights.CONFIGS[config](weights.F16 if ftype == "f16" else weights.F32), 1234)
            key = f"{config}_{ftype}_{case}"
            p = case_prompt(orc, path, case, n_steps)
            assert H.valid(H.as_prompt(p)), key
            r = orc.Ref(path, seed=seed, n_steps=n_steps)
            d["reference_build"] = np.array(r.build_info())
            g = H.generate(r, text, n_steps, p)
            r.close()
            T = g["fine"].shape[0]
            if case == "long":
                assert H.fine_loops(T, 512) >= 2, (T, "the long case must take two or more fine windows")
            d[key + "_weights_sha1"] = hashlib.sha1(open(path, "rb").read()).hexdigest()
            d[key + "_text"] = np.array(text); d[key + "_seed"] = np.int64(seed); d[key + "_n_steps"] = np.int64(n_steps)
            for k in ("semantic_prompt", "coarse_prompt", "fine_prompt"):
                d[f"{key}_{k}"] = np.asarray(p[k], np.int32)
            for k in ("prompt", "semantic", "coarse", "fine"):
                d[f"{key}_{k}"] = g[k]
            a = np.ascontiguousarray(g["audio"])
            d[key + "_audio_shape"] = np.array(a.shape, np.int64); d[key + "_audio_sha1"] = sha(a); d[key + "_audio_head"] = a[:64].copy()
            if T <= FULL_AUDIO_FRAMES:
                d[key + "_audio"] = a
            print(key, "semantic", g["semantic"].size, "frames", T, flush=True)
    d["cases"] = np.array([f"{c}_{f}_{k}" for c, f, k, *_ in CASES])
    np.savez_compressed(OUT, **d)
    print(OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
