"""Regenerates tests/golden/ref_pairs/*.npz: what the unmodified reference (oracle/_ref/libbark_ref.so, built by oracle/Makefile
where the reference sources exist) returns for exactly the inputs of

    tests/test_oracle_vs_ref.py                                   -> ref_pairs/tiny_f16.npz   (C oracle vs reference, CPU)
    tests/test_parity_gpu.py::test_full_size_against_the_reference_itself -> ref_pairs/small_f16_n12.npz (CUDA vs reference)
    tests/test_quantize.py (the reference tool's quantised files, the reference on them) -> ref_pairs/quantized.npz
    tests/test_prefix_rows.py (the reference's from-scratch coarse evaluation)             -> ref_pairs/prefix_rows.npz
    tests/test_oracle_vs_ref.py::test_long_context_bit_exact (steps up to n_kv 1024)        -> ref_pairs/long_context.npz

so these comparisons run on machines that have no reference build.  Run once where the reference library exists:

    python tests/golden/make_golden_ref_pairs.py
"""
import hashlib
import importlib
import os
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
import __graft_entry__ as graft  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "ref_pairs")
TOKENIZER_TEXTS = ["hello world", "", "Hello, world! 123 café zz", "ÀÉÎõü ñ ç", "a" * 600, "x,y;z...", "日本語 text", "tab\there"]
CAUSAL_FIRST_COARSE_SEED = 1        # tests/test_oracle_vs_ref.py test_causal_eval_bit_exact
N_CAUSAL_STEPS = 40


def sha(a):
    return hashlib.sha1(np.ascontiguousarray(a).tobytes()).hexdigest()


def pin(d, key, a):
    """A large float array is stored as its shape, sha1 and first 64 values (tests/conftest.py assert_pinned) to keep the
    fixtures small; the comparison stays bit for bit."""
    a = np.ascontiguousarray(a)
    d[key + "_shape"] = np.array(a.shape, np.int64); d[key + "_sha1"] = sha(a); d[key + "_head"] = a.reshape(-1)[:64].copy()


def causal_traces(r):
    """Teacher-forced semantic (merged prompt) and coarse evaluations, the argmax of the reference's logits fed back."""
    rng = np.random.default_rng(CAUSAL_FIRST_COARSE_SEED)
    out = {}
    for which, first, merge in ((0, None, True), (1, np.concatenate([rng.integers(0, 10000, 256), [12050], rng.integers(10000, 12048, 37)]).astype(np.int32), False)):
        toks = r.tokenize("hello world") if first is None else first
        n_past, shas, n_pasts, heads = 0, [], [], []
        for _ in range(N_CAUSAL_STEPS):
            lg, n_past = r.gpt_eval(which, toks, n_past, merge)
            shas.append(sha(lg)); n_pasts.append(n_past); heads.append(lg[:64].copy())
            toks = np.array([int(np.argmax(lg[:10000])) if which == 0 else 10000 + int(np.argmax(lg[10000:12048]))], np.int32)
        out[f"causal{which}_sha1"] = np.array(shas); out[f"causal{which}_n_past"] = np.array(n_pasts, np.int32); out[f"causal{which}_head"] = np.stack(heads)
    return out


def tiny_pairs(orc, path):
    r = orc.Ref(path, seed=0, n_steps=16)
    d = dict(reference_build=r.build_info(), weights_sha1=hashlib.sha1(open(path, "rb").read()).hexdigest())
    d["tokenizer_texts"] = np.array(TOKENIZER_TEXTS)
    d["tokenizer_ids"] = np.stack([r.tokenize(t) for t in TOKENIZER_TEXTS])
    d.update(causal_traces(r))
    rng = np.random.default_rng(2)
    buf = rng.integers(0, 1024, (8, 1024)).astype(np.int32)
    for nn in (2, 7):
        x = buf.copy(); x[nn:, :] = 1024
        fl = r.fine_eval(x, nn)
        d[f"fine{nn}_sha1"] = sha(fl); d[f"fine{nn}_head"] = fl[:8, :64].copy()
    rng = np.random.default_rng(3)
    r.reseed(9)
    toks, eos = [], []
    for i in range(150):
        lg = (rng.standard_normal((10048, 1024)[i % 2]) * 4).astype(np.float32)
        t, e = r.sample(lg, (0.7, 0.5, 0.0)[i % 3])
        toks.append(t); eos.append(e)
    d["sampler_tokens"] = np.array(toks, np.int32); d["sampler_eos"] = np.array(eos, np.float32)
    rng = np.random.default_rng(4)
    for T in (7, 40):
        pin(d, f"encodec{T}_audio", r.encodec_decode(rng.integers(0, 1024, (8, T)).astype(np.int32)))
    r.reseed(0)
    g = r.generate("hello world")
    for k in ("semantic", "coarse", "fine"):
        d[f"generate_{k}"] = g[k]
    pin(d, "generate_audio", g["audio"])
    r.close()
    return d


def small_pairs(orc, path):
    r = orc.Ref(path, seed=0, n_steps=12)
    d = dict(reference_build=r.build_info(), weights_sha1=hashlib.sha1(open(path, "rb").read()).hexdigest())
    toks, n_past = r.tokenize("hello world"), 0
    d["prompt_ids"] = toks.copy()
    for step in range(6):
        lg, n_past = r.gpt_eval(0, toks, n_past, True, n_threads=8)
        pin(d, f"semantic_logits{step}", lg)
        d[f"semantic_argmax{step}"] = int(np.argmax(lg[:10000]))
        toks = np.array([int(np.argmax(lg[:10000]))], np.int32)
    g = r.generate("hello world", n_threads=8)
    for k in ("semantic", "coarse", "fine", "audio"):        # the waveform is small (18 frames): kept whole for the 1e-3 check
        d[k] = g[k]
    r.close()
    return d


QUANT_FTYPES = {"q4_0": 2, "q4_1": 3, "q8_0": 7, "q5_0": 8, "q5_1": 9}


def quantized(orc, weights, tmp):
    """Per (config, source ftype, type): sha1 and size of the file the reference's bark_model_quantize writes, and the reference's
    teacher-forced logits / fine pass / generation on that file (the inputs of tests/test_quantize.py)."""
    import ctypes as C
    d = {}
    for config, src_ftype in (("tiny", "f16"), ("mini", "f32")):
        src = os.path.join(tmp, f"{config}_{src_ftype}_1234.bin")
        weights.write_weights(src, weights.CONFIGS[config](weights.F16 if src_ftype == "f16" else weights.F32), 1234)
        keep = orc.Ref(src)                                   # ggml_init fills the f16 tables the quantizer relies on
        R = C.CDLL(orc.REF_SO)
        R.bark_model_quantize.restype = C.c_bool
        R.bark_model_quantize.argtypes = [C.c_char_p, C.c_char_p, C.c_int]
        for qname, ft in sorted(QUANT_FTYPES.items()):
            key = f"{config}_{src_ftype}_{qname}"
            path = os.path.join(tmp, key + ".bin")
            assert R.bark_model_quantize(src.encode(), path.encode(), ft)
            blob = open(path, "rb").read()
            d[key + "_file_sha1"] = hashlib.sha1(blob).hexdigest(); d[key + "_file_size"] = len(blob)
            r = orc.Ref(path, seed=0, n_steps=10)
            rng = np.random.default_rng(17)
            toks, pr, sem = r.tokenize("Hello, world"), 0, []
            for _ in range(4):
                lr, pr = r.gpt_eval(0, toks, pr, True)
                sem.append(sha(lr))
                toks = np.array([int(np.argmax(lr[:10000]))], np.int32)
            toks = np.concatenate([rng.integers(0, 10000, 256), [12050], rng.integers(10000, 12048, 21)]).astype(np.int32)
            pr, co = 0, []
            for _ in range(3):
                lr, pr = r.gpt_eval(1, toks, pr, False)
                co.append(sha(lr))
                toks = np.array([10000 + int(np.argmax(lr[10000:12048]))], np.int32)
            buf = rng.integers(0, 1024, (8, 1024)).astype(np.int32); buf[:, 300:] = 1024; buf[4:, :] = 1024
            d[key + "_semantic_sha1"] = np.array(sem); d[key + "_coarse_sha1"] = np.array(co); d[key + "_fine_sha1"] = sha(r.fine_eval(buf, 4))
            g = r.generate("hello world")
            for k in ("semantic", "coarse", "fine"):
                d[f"{key}_generate_{k}"] = g[k]
            pin(d, f"{key}_generate_audio", g["audio"])
            r.close()
        keep.close()
    return d


def prefix_rows(orc, weights, tmp):
    d = {}
    for ftype in ("f32", "f16"):
        path = os.path.join(tmp, f"mini_{ftype}_1234.bin")
        weights.write_weights(path, weights.CONFIGS["mini"](weights.F16 if ftype == "f16" else weights.F32), 1234)
        r = orc.Ref(path)
        rng = np.random.default_rng(21)
        full = np.concatenate([rng.integers(0, 10000, 256), [12050], rng.integers(10000, 12048, 75)]).astype(np.int32)
        scratch, _ = r.gpt_eval(1, full, 0, False)
        pin(d, f"mini_{ftype}_scratch", scratch)
        r.close()
    return d


LONG_CONTEXT_SEED = 6               # tests/test_oracle_vs_ref.py test_long_context_bit_exact
LONG_SEMANTIC_PAST = 1015           # semantic steps at n_past 1015 .. 1023: the last one sees n_kv = 1024
LONG_COARSE_PROMPT = 887            # 256 semantic ids + 1 + 630 coarse history ids: the longest coarse window prompt


def long_context(orc, path):
    """tiny f16: semantic steps at n_past 1015 .. 1023 after the merged prompt and a 758-id continuation, and coarse steps at n_past
    887 .. 902 after a whole window prompt, teacher-forced, every step's logits pinned."""
    r = orc.Ref(path)
    d = dict(reference_build=r.build_info())
    rng = np.random.default_rng(LONG_CONTEXT_SEED)
    lg, n_past = r.gpt_eval(0, r.tokenize("hello world"), 0, True)
    lg, n_past = r.gpt_eval(0, rng.integers(0, 10000, LONG_SEMANTIC_PAST - n_past).astype(np.int32), n_past, False)
    for i in range(1024 - LONG_SEMANTIC_PAST):
        lg, n_past = r.gpt_eval(0, np.array([int(np.argmax(lg[:10000]))], np.int32), n_past, False)
        pin(d, f"semantic{i}", lg)
    prompt = np.concatenate([rng.integers(0, 10000, 256), [12050], rng.integers(10000, 12048, LONG_COARSE_PROMPT - 257)]).astype(np.int32)
    lg, n_past = r.gpt_eval(1, prompt, 0, False)
    for i in range(16):
        lg, n_past = r.gpt_eval(1, np.array([10000 + int(np.argmax(lg[10000:12048]))], np.int32), n_past, False)
        pin(d, f"coarse{i}", lg)
    r.close()
    return d


def main():
    graft.load_package()
    weights = importlib.import_module("bark_cpp_b200.weights")
    orc = graft.load_oracle_bindings()
    if not orc.have_ref():
        sys.exit("oracle/_ref/libbark_ref.so is not built: run build() where the reference sources exist")
    os.makedirs(OUT, exist_ok=True)
    with tempfile.TemporaryDirectory() as tmp:
        for config, fn, name in (("tiny", tiny_pairs, "tiny_f16.npz"), ("small", small_pairs, "small_f16_n12.npz")):
            path = os.path.join(tmp, f"{config}_f16_1234.bin")
            weights.write_weights(path, weights.CONFIGS[config](weights.F16), 1234)
            np.savez_compressed(os.path.join(OUT, name), **fn(orc, path))
            print(name, os.path.getsize(os.path.join(OUT, name)), "bytes")
        path = os.path.join(tmp, "tiny_f16_1234.bin")
        np.savez_compressed(os.path.join(OUT, "long_context.npz"), **long_context(orc, path))
        print("long_context.npz", os.path.getsize(os.path.join(OUT, "long_context.npz")), "bytes")
        for fn, name in ((quantized, "quantized.npz"), (prefix_rows, "prefix_rows.npz")):
            np.savez_compressed(os.path.join(OUT, name), **fn(orc, weights, tmp))
            print(name, os.path.getsize(os.path.join(OUT, name)), "bytes")


if __name__ == "__main__":
    main()
