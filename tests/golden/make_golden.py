"""Regenerates tests/golden/*.npz by running the UNMODIFIED reference (oracle/_ref/libbark_ref.so, built from
the reference tree by oracle/Makefile) on seeded synthetic weight files.  Run where the reference build exists:

    python tests/golden/make_golden.py

The weight files themselves are not committed: bark.cpp_b200/weights.py regenerates them bit-identically from
(config, ftype, seed).  Each fixture records the reference build string, so a reader can tell which lane
structure (AVX2, 4x8) produced the tokens (SURVEY.md App. C/E: the reference's tokens depend on its build flags).
"""
import hashlib
import importlib
import os
import tempfile
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
import __graft_entry__ as graft  # noqa: E402

CASES = [  # (config, ftype, weight seed, rng seed, n_steps_text_encoder, prompt, quant)
    ("tiny", "f16", 1234, 0, 20, "hello world", ""),
    ("mini", "f32", 1234, 0, 45, "hello world", ""),       # BASELINE config 1 shape: f32 GPT + f16 codec; 67 frames, 3 coarse windows
    ("mini", "f16", 1234, 7, 30, "The quick brown fox, 42!", ""),
    ("tiny", "f16", 1234, 0, 16, "hello world", "q4_0"),   # BASELINE config 4 shape: q4_0 GPT (the reference's own bark_model_quantize) + f16 codec
    ("mini", "f32", 1234, 3, 24, "Quantised, 7 times.", "q4_0"),
]


def sha(a):
    return hashlib.sha1(np.ascontiguousarray(a).tobytes()).hexdigest()


def main():
    graft.load_package()
    weights = importlib.import_module("bark_cpp_b200.weights")
    orc = graft.load_oracle_bindings()
    os.environ["BARK_B200_QUIET"] = "1"
    out_dir = os.path.dirname(os.path.abspath(__file__))
    tmp = os.path.join(tempfile.gettempdir(), f"bark_b200_fixtures_{os.getuid()}")
    os.makedirs(tmp, exist_ok=True)
    import ctypes as C
    for config, ftype, wseed, seed, n_steps, prompt, quant in CASES:
        path = os.path.join(tmp, f"{config}_{ftype}_{wseed}.bin")
        if not os.path.exists(path):
            weights.write_weights(path, weights.CONFIGS[config](weights.F16 if ftype == "f16" else weights.F32), wseed)
        if quant:                                            # the REFERENCE's quantizer makes the file (ggml_init first: f16 tables, examples/quantize/main.cpp:67-72)
            orc.Ref(path)
            R = C.CDLL(orc.REF_SO)
            R.bark_model_quantize.restype = C.c_bool
            R.bark_model_quantize.argtypes = [C.c_char_p, C.c_char_p, C.c_int]
            qpath = os.path.join(tmp, f"{config}_{ftype}_{wseed}_{quant}_ref.bin")
            assert quant == "q4_0" and R.bark_model_quantize(path.encode(), qpath.encode(), 2)
            path = qpath
        r = orc.Ref(path, seed=seed, n_steps=n_steps)
        prompt_ids = r.tokenize(prompt)
        # teacher-forced traces: semantic prefill + 3 decode steps, one fine pass
        toks, n_past, sem_logits = prompt_ids, 0, []
        for _ in range(4):
            lg, n_past = r.gpt_eval(0, toks, n_past, True)
            sem_logits.append(lg)
            toks = np.array([int(np.argmax(lg[:10000]))], np.int32)
        rng = np.random.default_rng(3)
        buf = rng.integers(0, 1024, (8, 1024)).astype(np.int32); buf[:, 700:] = 1024; buf[3:, :] = 1024
        fine_logits = r.fine_eval(buf, 2)
        r.reseed(seed)
        g = r.generate(prompt)
        np.savez_compressed(
            os.path.join(out_dir, f"{config}_{ftype}{'_' + quant if quant else ''}.npz"),
            config=config, ftype=ftype, quant=quant, weight_seed=wseed, seed=seed, n_steps=n_steps, prompt=prompt,
            reference_build=r.build_info(), weights_sha1=hashlib.sha1(open(path, "rb").read()).hexdigest(),
            prompt_ids=prompt_ids, semantic=g["semantic"], coarse=g["coarse"], fine=g["fine"], audio=g["audio"],
            sem_logits_head=np.stack([l[:256] for l in sem_logits]), sem_logits_sha1=np.array([sha(l) for l in sem_logits]),
            fine_logits_head=fine_logits[:8, :64].copy(), fine_logits_sha1=sha(fine_logits),
        )
        print(config, ftype, "semantic", g["semantic"].size, "frames", g["coarse"].shape[0], "audio", g["audio"].size)
    o, ref_tab = orc.gelu_tables()
    np.savez_compressed(os.path.join(out_dir, "gelu_table_f16.npz"), table=ref_tab, reference_build=orc.Ref.__doc__)
    print("gelu table sha1", sha(ref_tab))


if __name__ == "__main__":
    main()
