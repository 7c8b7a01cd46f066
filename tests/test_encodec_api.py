"""CPU: encodec.cpp's C API (include/encodec.h) at the library boundary, and the CPU restatement of the encode at 1 to 32 codebooks
against the unmodified reference's stored codes (tests/golden/make_golden_encodec.py)."""
import os
import re
import subprocess

import numpy as np
import pytest

from conftest import GOLDEN_DIR, ROOT, cuda_device_count
import encodec_oracle as co
import encoder_oracle as eo
from encodec_oracle import codec_offset

GOLD = os.path.join(GOLDEN_DIR, "ref_pairs", "encodec_bandwidths.npz")
N_Q = {1: 1, 2: 2, 3: 4, 12: 16, 24: 32}                     # bandwidth (kbps) -> codebooks at 24 kHz


def test_library_exports_the_encodec_api(pkg):
    out = subprocess.check_output(["nm", "-D", "--defined-only", pkg.LIB_PATH], text=True)
    exported = {l.split()[-1] for l in out.splitlines() if " T " in l and l.split()[-1].startswith("encodec_")}
    declared = set(re.findall(r"ENCODEC_API[^;(]*?\b(encodec_\w+)\s*\(", open(os.path.join(ROOT, "include", "encodec.h")).read()))
    assert len(declared) == 13
    assert declared == exported == set(pkg.ENCODEC_EXPORTS)
    assert not set(pkg.ENCODEC_EXPORTS) & set(pkg.EXPORTS)


CALLER = r'''
#include "encodec.h"
#include <stdio.h>
int main(int argc, char ** argv) {
    ggml_time_init();
    struct encodec_context * e = encodec_load_model(argc > 1 ? argv[1] : "/nonexistent", 0, 0);
    if (!e) { printf("load failed as expected\n"); return 3; }
    encodec_set_target_bandwidth(e, 12);
    encodec_set_sample_rate(e, 24000);
    float x[4000] = {0};
    int32_t c[16 * 13] = {0};
    if (!encodec_compress_audio(e, x, 4000, 4)) return 4;
    if (!encodec_decompress_audio(e, c, 16 * 13, 4)) return 5;
    if (!encodec_reconstruct_audio(e, x, 4000, 4)) return 6;
    const int32_t * codes = encodec_get_codes(e); int nc = encodec_get_codes_size(e);
    const float * audio = encodec_get_audio(e); int na = encodec_get_audio_size(e);
    const struct encodec_statistics * st = encodec_get_statistics(e);
    printf("%d %d %d %f %lld %lld\n", nc, codes[0], na, audio[0], (long long) st->t_load_us, (long long) st->t_compute_us);
    encodec_reset_statistics(e);
    encodec_free(e);
    return 0;
}
'''


@pytest.mark.parametrize("lang", ["c", "c++"])
def test_c_and_cpp_callers_compile_and_link(pkg, tmp_path, lang):
    src = tmp_path / ("caller.c" if lang == "c" else "caller.cpp")
    src.write_text(CALLER)
    exe = tmp_path / "caller"
    libdir = os.path.dirname(pkg.LIB_PATH)
    cc = ["gcc", "-std=c11"] if lang == "c" else ["g++", "-std=c++11"]
    subprocess.check_call(cc + ["-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe), "-L", libdir, "-lbark_b200",
                                "-Wl,-rpath," + libdir])
    r = subprocess.run([str(exe)], capture_output=True, text=True)
    assert r.returncode == 3 and "load failed as expected" in r.stdout


def test_null_context_calls_fail_cleanly(pkg):
    L = pkg.lib()
    assert not L.encodec_load_model(None, 0, 0)
    assert not L.encodec_load_model(b"/nonexistent/ggml_weights.bin", 0, 0)
    assert not L.encodec_compress_audio(None, None, 0, 1) and not L.encodec_decompress_audio(None, None, 0, 1)
    assert not L.encodec_reconstruct_audio(None, None, 0, 1)
    assert not L.encodec_get_codes(None) and L.encodec_get_codes_size(None) == 0
    assert not L.encodec_get_audio(None) and L.encodec_get_audio_size(None) == 0 and not L.encodec_get_statistics(None)
    L.encodec_set_target_bandwidth(None, 6); L.encodec_set_sample_rate(None, 24000); L.encodec_reset_statistics(None); L.encodec_free(None)


@pytest.mark.skipif(cuda_device_count() > 0, reason="only meaningful without a GPU")
def test_no_cpu_fallback(pkg, weights_file):
    path = weights_file("tiny", "f16")
    assert not pkg.lib().encodec_load_model(os.fsencode(path), codec_offset(path), 0)
    with pytest.raises(RuntimeError):
        pkg.Encodec(path, codec_offset(path))


def test_reference_examples_compile_unchanged(pkg, tmp_path):
    orc = __import__("__graft_entry__").load_oracle_bindings()
    if not os.path.isdir(os.path.join(orc.REFERENCE_DIR, "encodec.cpp", "examples")):
        pytest.skip("no reference tree")
    subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "oracle"), "-f", "encodec_examples.mk", f"REF={orc.REFERENCE_DIR}",
                           f"OUT={tmp_path}"])
    for name in ("encodec_compress", "encodec_decompress", "encodec_main"):
        assert os.access(tmp_path / name, os.X_OK), name


def test_n_q_rule():
    assert {bw: co.n_q_for(bw) for bw in (1, 2, 3, 6, 12, 24)} == {1: 1, 2: 2, 3: 4, 6: 8, 12: 16, 24: 32}
    assert co.n_q_for(0) == 1 and co.n_q_for(-5) == 1 and co.n_q_for(25) == 33
    assert co.n_q_for(6, 48000) == 4 and co.n_q_for(6, 639) == 600 == co.n_q_for(6, 320)


@pytest.fixture(scope="module")
def oracles(weights_file, weights_mod):
    out = {}
    for w in eo.WEIGHTS:
        path = eo.weights_path(weights_file, weights_mod, w)
        out[w] = co.CodecOracle(path, codec_offset(path))
    return out


@pytest.mark.parametrize("name,kind,n,which", eo.CASES, ids=[c[0] for c in eo.CASES])
def test_oracle_codes_equal_the_reference_at_every_bandwidth(oracles, name, kind, n, which):
    gold = np.load(GOLD)
    x = eo.signal(kind, n, seed=n)
    _, lat = oracles[which].enc.encode(x, return_latent=True)
    full = eo.rvq_encode(lat, oracles[which].cb)              # 32 codebooks; fewer are its leading rows (residual quantisation)
    for bw, n_q in N_Q.items():
        ref = gold[f"{name}_bw{bw}_codes"]
        assert ref.shape == (n_q, (n + 319) // 320)
        assert np.array_equal(full[:n_q], ref), f"{name} at {bw} kbps: {int((full[:n_q] != ref).sum())} codes differ"
