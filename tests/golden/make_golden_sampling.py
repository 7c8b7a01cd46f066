"""Regenerates tests/golden/ref_pairs/sampling.npz: generations with the top-k / top-p filter (DESIGN.md §14) computed by
tests/history_oracle.py's stage loops (through tests/sampling_oracle.py's Filtered) on the unmodified reference (oracle/_ref/libbark_ref.so).  Every logit and every sample comes from the
reference's own gpt_eval and gpt_sample calls; only the mask between them is restated (tests/sampling_oracle.c).  The inputs of
tests/test_sampling_filters.py and tests/test_sampling_filters_gpu.py.  Cases (weight seed 1234), each with its settings per stage:

  k50        top_k 50 on both stages             p09      top_p 0.9 on both stages
  k5p05      top_k 5 and top_p 0.5 on both       p0       top_p 0 on both (only sorted position 0 stays)
  sem_only   top_k 50 on the semantic stage only coarse_only  top_p 0.9 on the coarse stage only
  prompted   top_k 50 and top_p 0.9 on both, under a random speaker history prompt

Run once where the reference library exists:

    python tests/golden/make_golden_sampling.py
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
import sampling_oracle as SO  # noqa: E402

OUT = os.path.join(HERE, "ref_pairs", "sampling.npz")
FULL_AUDIO_FRAMES = 64

BOTH_K50 = {"semantic": (50, None), "coarse": (50, None)}
# (config, ftype, case, text, seed, n_steps, {stage: (top_k, top_p)}, prompt seed or None)
CASES = [
    ("tiny", "f16", "k50", "hello world", 0, 16, BOTH_K50, None),
    ("tiny", "f16", "p09", "hello world", 1, 16, {"semantic": (None, 0.9), "coarse": (None, 0.9)}, None),
    ("tiny", "f16", "k5p05", "hello world", 2, 16, {"semantic": (5, 0.5), "coarse": (5, 0.5)}, None),
    ("tiny", "f16", "p0", "the fox", 3, 16, {"semantic": (None, 0.0), "coarse": (None, 0.0)}, None),
    ("tiny", "f16", "sem_only", "hello world", 4, 16, {"semantic": (50, None)}, None),
    ("tiny", "f16", "coarse_only", "hello world", 5, 16, {"coarse": (None, 0.9)}, None),
    ("tiny", "f16", "prompted", "hello world", 6, 16, {"semantic": (50, 0.9), "coarse": (50, 0.9)}, 41),
    ("mini", "f32", "k50", "hello world", 0, 12, BOTH_K50, None),
    ("mini", "f32", "p09", "hello world", 1, 12, {"semantic": (None, 0.9), "coarse": (None, 0.9)}, None),
    ("mini", "f32", "k5p05", "the fox", 2, 12, {"semantic": (5, 0.5), "coarse": (5, 0.5)}, None),
]


def settings_array(settings, stage):
    """[top_k (0: off), top_p (NaN: off)] of one stage, as stored."""
    k, p = settings.get(stage, (None, None))
    return np.array([float(k or 0), np.nan if p is None else float(p)], np.float64)


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
        for config, ftype, case, text, seed, n_steps, settings, prompt_seed in CASES:
            path = os.path.join(tmp, f"{config}_{ftype}_1234.bin")
            if not os.path.exists(path):
                weights.write_weights(path, weights.CONFIGS[config](weights.F16 if ftype == "f16" else weights.F32), 1234)
            key = f"{config}_{ftype}_{case}"
            prompt = None
            if prompt_seed is not None:
                prompt = H.random_prompt(np.random.default_rng(prompt_seed), 60, 120)
                for k in ("semantic_prompt", "coarse_prompt", "fine_prompt"):
                    d[f"{key}_{k}"] = np.asarray(prompt[k], np.int32)
            r = orc.Ref(path, seed=seed, n_steps=n_steps)
            d["reference_build"] = np.array(r.build_info())
            g = SO.generate(r, text, n_steps, prompt, settings)
            r.close()
            T = g["fine"].shape[0]
            d[key + "_weights_sha1"] = hashlib.sha1(open(path, "rb").read()).hexdigest()
            d[key + "_text"] = np.array(text); d[key + "_seed"] = np.int64(seed); d[key + "_n_steps"] = np.int64(n_steps)
            d[key + "_semantic_filter"] = settings_array(settings, "semantic"); d[key + "_coarse_filter"] = settings_array(settings, "coarse")
            d[key + "_prompted"] = np.int64(prompt is not None)
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
