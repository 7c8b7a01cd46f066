"""GPU: decode steps over the whole 1024-position context against the C oracle, bit for bit, in every staging regime and CTA split.

The semantic stage's last steps see n_kv = 1024 and coarse windows reach n_kv ~ 946; the persistent decode step changes branch past
n_kv 513 / 514 / 769 and with the CTA count (tests/decode_regimes.py restates where).  Each model runs one teacher-forced script: a
multi-row evaluation from 0 to the first band, then bands of single-token steps (decode_regimes.BANDS) joined by multi-row evaluations
on top of the filled cache, the last band ending at the last position.  The oracle runs the script once per model; the library
replays it once per CTA count (BARK_B200_DECODE_CTAS) and compares every evaluation's logits.
"""
import ctypes
import os

import numpy as np
import pytest

import decode_regimes as dr
from conftest import FIXTURE_DIR, bits
from test_parity_attention_gpu import check, ref  # noqa: F401  (the oracle-built attention reference, a fixture)

pytestmark = pytest.mark.gpu

SOURCES = {"tiny_f16": ("tiny", "f16"), "mini_f32": ("mini", "f32"), "mini_f16": ("mini", "f16"), "wide_f16": ("wide", "f16"),
           "wide_f32": ("wide", "f32"), "tiny_q4_0": ("tiny", "f16"), "wide_q4_0": ("wide", "f16")}


def device_sms() -> int:
    rt = ctypes.CDLL("libcudart.so.12")
    n = ctypes.c_int(0)
    assert rt.cudaDeviceGetAttribute(ctypes.byref(n), 16, 0) == 0              # cudaDevAttrMultiProcessorCount
    return n.value


@pytest.fixture(scope="module")
def model_path(pkg, weights_mod, weights_file):
    def get(name):
        if name == "small2_f32":                       # bark-small's width (E 768, 12 heads of 64) at 2 layers, f32
            path = os.path.join(FIXTURE_DIR, "small2_f32_1234.bin")
            if not os.path.exists(path):
                d = weights_mod.GPTDims(2, 12, 768)
                weights_mod.write_weights(path + ".tmp", weights_mod.Config("small2", d, d, d, gpt_ftype=weights_mod.F32), 1234)
                os.replace(path + ".tmp", path)
            return path
        config, ftype = SOURCES[name]
        src = weights_file(config, ftype)
        if not name.endswith("q4_0"):
            return src
        dst = os.path.join(FIXTURE_DIR, f"{config}_{ftype}_1234_q4_0.bin")
        if not os.path.exists(dst):
            assert pkg.lib().bark_model_quantize(src.encode(), (dst + ".tmp").encode(), 2)      # the library's own quantizer
            os.replace(dst + ".tmp", dst)
        return dst
    return get


def coarse_argmax(lo):
    return np.array([10000 + int(np.argmax(lo[10000:12048]))], np.int32)


@pytest.fixture(scope="module")
def script(orc, model_path):
    """model -> [(tokens, n_past, the oracle's logits)] of the model's bands, computed once"""
    cache = {}

    def get(name):
        if name not in cache:
            o = orc.Oracle(model_path(name))
            rng = np.random.default_rng(sum(map(ord, name)))
            evals, n_past, lo = [], 0, None
            for start in dr.BANDS[name][1]:
                cut = start - 1                        # the band's first step runs at n_past = cut, n_kv = start
                toks = (np.concatenate([rng.integers(0, 10000, 256), [12050], rng.integers(10000, 12048, cut - 257)]) if n_past == 0
                        else rng.integers(10000, 12048, cut - n_past)).astype(np.int32)
                for _ in range(1 + dr.BAND_STEPS):
                    before = n_past
                    lo, n_past = o.gpt_eval(1, toks, n_past, False)
                    evals.append((toks, before, lo))
                    toks = coarse_argmax(lo)
            assert n_past == dr.BLOCK_SIZE
            cache[name] = evals
        return cache[name]
    return get


def replay(b, evals, name, G, what):
    m = dr.MODELS[name]
    for toks, n_past, want in evals:
        lg, p = b.gpt_eval(1, toks, n_past, False)
        assert p == n_past + toks.size
        bad = np.flatnonzero(bits(lg) != bits(want))
        if bad.size:
            where = f"step at n_kv {p}, regimes {sorted(dr.regimes(m, G, p))}" if toks.size == 1 else f"{toks.size}-row evaluation at n_past {n_past}"
            pytest.fail(f"{what}: {where}: {bad.size} logits differ, first at {bad[0]} ({lg[bad[0]]!r} != {want[bad[0]]!r})")


def set_ctas(monkeypatch, G):
    if dr.launch_ctas(device_sms(), G) != G:
        pytest.skip(f"{G} decode CTAs do not fit this device")
    monkeypatch.setenv("BARK_B200_DECODE_CTAS", str(G))


CASES = [(name, G) for name, (ctas, _) in dr.BANDS.items() for G in ctas]


@pytest.mark.parametrize("name,G", CASES, ids=[f"{n}-{g}ctas" for n, g in CASES])
def test_teacher_forced_bands(pkg, script, model_path, monkeypatch, name, G):
    evals = script(name)
    set_ctas(monkeypatch, G)
    with pkg.Bark(model_path(name)) as b:
        replay(b, evals, name, G, f"{name}, {G} CTAs")


@pytest.mark.parametrize("name", dr.PER_OP_MODELS)
def test_per_op_path_bands(pkg, script, model_path, monkeypatch, name):
    """BARK_B200_DECODE=multi: single-token steps through the per-op kernels (attention() with one query row)"""
    evals = script(name)
    monkeypatch.setenv("BARK_B200_DECODE", "multi")
    with pkg.Bark(model_path(name)) as b:
        replay(b, evals, name, dr.launch_ctas(device_sms()), f"{name}, per-op path")


def test_last_position_then_overflow_then_generation(pkg, script, model_path, capfd):
    """The step at n_past 1023 equals the oracle's; n_past 1024 is refused with a message; the context still generates what a fresh
    one does."""
    path = model_path("tiny_f16")
    evals = script("tiny_f16")
    assert evals[-1][1] == dr.BLOCK_SIZE - 1 and evals[-1][0].size == 1
    with pkg.Bark(path, seed=4, n_steps_text_encoder=24) as b:
        replay(b, evals, "tiny_f16", dr.launch_ctas(device_sms()), "tiny_f16")
        capfd.readouterr()
        with pytest.raises(RuntimeError):
            b.gpt_eval(1, coarse_argmax(evals[-1][2]), dr.BLOCK_SIZE, False)
        assert "context overflow" in capfd.readouterr().err
        a1 = b.generate("hello world"); t1 = [b.tokens(i).copy() for i in range(3)]
    with pkg.Bark(path, seed=4, n_steps_text_encoder=24) as b:
        a0 = b.generate("hello world"); t0 = [b.tokens(i).copy() for i in range(3)]
    assert t0[0].size > 0
    for x, y in zip(t0, t1):
        assert np.array_equal(x, y)
    assert np.array_equal(bits(a0), bits(a1))


# ---- batched step --------------------------------------------------------------------------------------------------------------
BATCH_P0 = 500                                         # every slot starts from the same 500-row evaluation
BATCH_PAST = (503, 510, 600, 700, 767, 850, 950, 1016)     # then single steps to these n_past; row 1 crosses n_kv 513 / 514
BATCH_STEPS = 8                                            # row 7 ends at n_kv 1024


@pytest.mark.parametrize("name", ["tiny_f16", "wide_f16"])
def test_batched_step_ragged_long_rows(pkg, orc, model_path, name):
    """gpt_step_batch with eight slots at n_kv spread over 504 .. 1024.  Every slot's cache is the oracle's sequence S: the same
    multi-row evaluation of S[:500], then S fed one token at a time, so row r at n_past q must give the oracle's logits at q."""
    path = model_path(name)
    o = orc.Oracle(path)
    rng = np.random.default_rng(53)
    S = np.concatenate([rng.integers(0, 10000, 256), [12050], rng.integers(10000, 12048, BATCH_P0 - 257)]).astype(np.int32)
    want = {}
    lo, n = o.gpt_eval(1, S, 0, False)
    want[BATCH_P0 - 1] = lo
    S = list(S)
    for q in range(BATCH_P0, dr.BLOCK_SIZE):
        S.append(int(coarse_argmax(lo)[0]))
        lo, n = o.gpt_eval(1, np.array([S[q]], np.int32), q, False)
        want[q] = lo
    S = np.array(S, np.int32)

    def same(lg, q, what):
        bad = np.flatnonzero(bits(lg) != bits(want[q]))
        assert bad.size == 0, f"{name} {what} at n_kv {q + 1}: {bad.size} logits differ, first at {bad[0]}"

    slots = [3, 0, 6, 1, 7, 5, 2, 4]
    with pkg.Bark(path) as b:
        for r, p in enumerate(BATCH_PAST):
            lg, q = b.gpt_eval_slot(1, slots[r], S[:BATCH_P0], 0, False)
            same(lg, q - 1, f"row {r} prefill")
            while q < p:
                lg, q = b.gpt_eval_slot(1, slots[r], S[q:q + 1], q, False)
                same(lg, q - 1, f"row {r} single-slot step")
        n_past = np.array(BATCH_PAST, np.int32)
        for j in range(BATCH_STEPS):
            lg, n_past = b.gpt_step_batch(1, slots, S[n_past], n_past)
            for r in range(len(slots)):
                same(lg[r], int(n_past[r]) - 1, f"batched step {j}, row {r} (slot {slots[r]})")
        assert int(n_past.max()) == dr.BLOCK_SIZE


# ---- kernel level -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n_kv", [511, 512, 513, 767, 768, 769, 1023, 1024])
@pytest.mark.parametrize("N", [1, 2, 8])
def test_parity_attention_long_history(pkg, ref, N, n_kv):  # noqa: F811
    """bark_b200_parity_attention, both paths: N query rows on top of n_kv - N cached keys, 16 heads of 64"""
    check(pkg, ref, N, n_kv, n_kv - N, 64, 16, causal=True, seed=n_kv * 8 + N)


# ---- end to end ---------------------------------------------------------------------------------------------------------------
def test_default_length_generation(pkg, orc, model_path):
    """The default 768 semantic steps (the last one at n_kv 1024) and the 39 coarse windows they make, against the oracle's stages.
    The clip has 1154 frames: past 1024 the reference's fine stage writes out of bounds, so only its first window is defined — the
    first 512 fine frames, which later windows do not rewrite.  The waveform is the oracle codec's decoding of the library's fine ids."""
    path = model_path("tiny_f16")
    o = orc.Oracle(path, seed=0, n_steps=768)
    sem = o.semantic(o.tokenize("hello world"))
    assert sem.size == 768, "the semantic stage stopped early: choose another seed"
    co = o.coarse(sem)
    assert -(-2 * co.shape[0] // 60) == 39
    fi = o.fine(co[:1024])
    with pkg.Bark(path, seed=0, n_steps_text_encoder=768) as b:
        audio = b.generate("hello world")
        assert np.array_equal(b.tokens(0), sem)
        assert np.array_equal(b.tokens(1), co)
        got = b.tokens(2)
    assert got.shape == (co.shape[0], 8)
    assert np.array_equal(got[:, :2], co) and np.array_equal(got[:512], fi[:512])
    assert np.array_equal(bits(audio), bits(o.encodec_decode(np.ascontiguousarray(got.T))))
