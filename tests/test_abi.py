"""CPU: the drop-in boundary.  The library must load without a GPU, export every symbol the two public headers
declare, keep the reference's struct layouts, and refuse (loudly, no fallback) to run without a CUDA device."""
import ctypes as C
import os
import re
import subprocess

import pytest

from conftest import ROOT, cuda_device_count


def header_symbols():
    syms = set()
    for h in ("bark.h", "bark_b200.h"):
        src = open(os.path.join(ROOT, "include", h)).read()
        syms |= set(re.findall(r"BARK_API[^;(]*?\b(bark_\w+)\s*\(", src))
    src = open(os.path.join(ROOT, "include", "ggml.h")).read()
    syms |= set(re.findall(r"\b(ggml_time_\w+|ggml_init|ggml_free)\s*\(", src))
    return syms


def test_library_exports_every_declared_symbol(pkg):
    out = subprocess.check_output(["nm", "-D", "--defined-only", pkg.LIB_PATH], text=True)
    exported = {l.split()[-1] for l in out.splitlines() if " T " in l}
    declared = header_symbols()
    assert len(declared) >= 30
    assert declared <= exported, f"declared but not exported: {sorted(declared - exported)}"
    assert declared == set(pkg.EXPORTS)
    L = pkg.lib()
    for s in declared:
        assert getattr(L, s) is not None


def test_struct_layouts_match_reference(pkg):
    # bark.h:81-141 — 23 4-byte fields, then a function pointer and a void* (8-aligned): 96 + 16 = 112 bytes on LP64
    assert C.sizeof(pkg.BarkContextParams) == 112
    assert pkg.BarkContextParams.progress_callback.offset == 96
    assert C.sizeof(pkg.BarkStatistics) == 56          # 5 x int64 + 3 x int32 (+4 padding)
    p = pkg.lib().bark_context_default_params()
    got = {n: getattr(p, n) for n, _ in pkg.BarkContextParams._fields_[:-2]}
    want = dict(verbosity=0, sliding_window_size=60, max_coarse_history=630, sample_rate=24000, target_bandwidth=6, cls_token_id=101,
                sep_token_id=102, n_steps_text_encoder=768, text_pad_token=129595, text_encoding_offset=10048, semantic_pad_token=10000,
                semantic_vocab_size=10000, semantic_infer_token=129599, coarse_infer_token=12050, coarse_semantic_pad_token=12048,
                n_coarse_codebooks=2, n_fine_codebooks=8, codebook_size=1024)      # bark.cpp:2202-2232
    for k, v in want.items():
        assert got[k] == v, k
    assert abs(got["temp"] - 0.7) < 1e-7 and abs(got["fine_temp"] - 0.5) < 1e-7 and abs(got["min_eos_p"] - 0.2) < 1e-7
    assert abs(got["semantic_rate_hz"] - 49.9) < 1e-5 and got["coarse_rate_hz"] == 75.0


def test_null_context_getters_follow_reference(pkg):
    L = pkg.lib()
    assert L.bark_get_audio_data_size(None) == 0 and L.bark_get_load_time(None) == 0 and L.bark_get_eval_time(None) == 0
    assert not L.bark_get_audio_data(None)
    assert L.bark_generate_audio(None, b"x", 1) is False
    L.bark_free(None)
    L.bark_reset_statistics(None)
    assert L.ggml_time_us() > 0


def test_load_errors_return_null(pkg, tmp_path):
    L = pkg.lib()
    p = L.bark_context_default_params()
    assert not L.bark_load_model(b"/nonexistent/ggml_weights.bin", p, 0)
    bad = tmp_path / "bad.bin"
    bad.write_bytes(b"\x00" * 64)
    assert not L.bark_load_model(str(bad).encode(), p, 0)


@pytest.mark.skipif(cuda_device_count() > 0, reason="only meaningful without a GPU")
def test_no_cpu_fallback(pkg, weights_file):
    """Without a CUDA device the product must fail, not silently compute on the host."""
    with pytest.raises(RuntimeError):
        pkg.Bark(weights_file("tiny", "f16"))


def test_reference_caller_compiles_against_our_headers(pkg, tmp_path):
    """examples/main/main.cpp-style caller: includes bark.h + ggml.h, uses the by-value params struct, links -lbark_b200."""
    src = tmp_path / "caller.cpp"
    src.write_text(r'''
#include "bark.h"
#include "ggml.h"
#include <cstdio>
static void cb(struct bark_context *, enum bark_encoding_step step, int progress, void *) { (void) step; (void) progress; }
int main(int argc, char ** argv) {
    ggml_time_init();
    const int64_t t0 = ggml_time_us();
    bark_verbosity_level verbosity = bark_verbosity_level::LOW;
    struct bark_context_params p = bark_context_default_params();
    p.verbosity = verbosity; p.progress_callback = cb; p.progress_callback_user_data = nullptr;
    struct bark_context * b = bark_load_model(argc > 1 ? argv[1] : "/nonexistent", p, 0);
    if (!b) { printf("load failed as expected in %lld us\n", (long long)(ggml_time_us() - t0)); return 3; }
    if (!bark_generate_audio(b, "hello", 4)) return 4;
    const float * a = bark_get_audio_data(b); int n = bark_get_audio_data_size(b);
    printf("%d samples %f load %lld eval %lld\n", n, a ? a[0] : 0.f, (long long) bark_get_load_time(b), (long long) bark_get_eval_time(b));
    bark_model_quantize("a", "b", GGML_FTYPE_MOSTLY_Q4_0);
    bark_free(b);
    return 0;
}
''')
    exe = tmp_path / "caller"
    libdir = os.path.dirname(pkg.LIB_PATH)
    subprocess.check_call(["g++", "-std=c++11", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe), "-L", libdir, "-lbark_b200",
                           "-Wl,-rpath," + libdir])
    r = subprocess.run([str(exe)], capture_output=True, text=True)
    assert r.returncode == 3 and "load failed as expected" in r.stdout
