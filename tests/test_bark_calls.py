"""What every bark_context entry point does with a null context, with a caller's array it may not fill, and with a context on
another device than the calling thread's current one.

Every extern "C" call on a bark_context runs through one path: a null context is reported as "<fn>: invalid bark context" and
answered with the call's failure value (bark_free and bark_reset_statistics stay silent no-ops, as the reference's are), the
context's device is made current for the call, and a CUDA failure is the call's failure value.  A call that copies results into a
caller's array copies at most `cap` elements, none for a negative cap, and returns the full size."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from conftest import ROOT, cuda_device_count

SILENT = {"bark_free", "bark_reset_statistics"}
VOID = {"bark_free", "bark_reset_statistics", "bark_b200_reseed", "bark_b200_tokenize", "bark_b200_set_tokens", "bark_b200_get_stats",
        "bark_b200_get_hparams"}
NULL = object()          # a null pointer return


def context_calls():
    """The header-declared functions whose first parameter is a bark_context"""
    names = set()
    for h in ("bark.h", "bark_b200.h"):
        src = open(os.path.join(ROOT, "include", h)).read()
        names |= set(re.findall(r"BARK_API[^;(]*?\b(bark_\w+)\s*\(\s*struct bark_context \*", src))
    return names


def null_context_table():
    """(function, arguments after the null context, failure value); the other arguments are valid"""
    i32, f32 = np.zeros(1 << 14, np.int32), np.zeros(1 << 14, np.float32)
    p, q = i32.ctypes.data, f32.ctypes.data
    n_past, eos = C.c_int(0), C.c_float(0)
    texts, seeds = (C.c_char_p * 1)(b"hello"), (C.c_uint32 * 1)(0)
    keep = (i32, f32, n_past, eos, texts, seeds)
    return keep, [
        ("bark_generate_audio", (b"hello", 1), False),
        ("bark_get_audio_data", (), NULL),
        ("bark_get_audio_data_size", (), 0),
        ("bark_get_load_time", (), 0),
        ("bark_get_eval_time", (), 0),
        ("bark_reset_statistics", (), None),
        ("bark_free", (), None),
        ("bark_b200_forward_text_encoder", (1,), False),
        ("bark_b200_forward_coarse_encoder", (1,), False),
        ("bark_b200_forward_fine_encoder", (1,), False),
        ("bark_b200_gpt_eval", (0, p, 1, C.byref(n_past), 1, q), 0),
        ("bark_b200_fine_eval", (p, 2, q), 0),
        ("bark_b200_encodec_decode", (p, 9, q, 2880), -1),
        ("bark_b200_encodec_encode", (q, 4000, p, 104, q, 1664), -1),
        ("bark_b200_encodec_encode_resampled", (q, 2000, 2, 44100, p, 104, q, 1664), -1),
        ("bark_b200_sample", (0, q, 16, 0.7, C.byref(eos)), -1),
        ("bark_b200_sample_rows", (q, 16, 2, 0.7, p, q), -1),
        ("bark_b200_reseed", (1,), None),
        ("bark_b200_tokenize", (b"hello", p), None),
        ("bark_b200_get_tokens", (0, p, 16), -1),
        ("bark_b200_set_tokens", (0, p, 16), None),
        ("bark_b200_get_stats", (None, None), None),
        ("bark_b200_get_hparams", (0, p), None),
        ("bark_b200_layernorm_fallbacks", (), 0),
        ("bark_b200_decode_timing", (p, 16), 0),
        ("bark_b200_fast_mode", (), 0),
        ("bark_b200_set_sampling", (0, None), 0),
        ("bark_b200_set_tokenizer", (0,), 0),
        ("bark_b200_text_ids", (0, b"hello", p, 16), -1),
        ("bark_b200_set_long_form", (None,), 0),
        ("bark_b200_long_chunks", (), -1),
        ("bark_b200_long_chunk_text", (0, None, 0), -1),
        ("bark_b200_long_chunk_tokens", (0, 0, p, 16), -1),
        ("bark_b200_generate_batch", (texts, seeds, 1, 1), False),
        ("bark_b200_generate_batch_prompted", (texts, seeds, None, 1, 1), False),
        ("bark_b200_set_history_prompt", (None,), 0),
        ("bark_b200_batch_audio", (0, q, 16), -1),
        ("bark_b200_batch_tokens", (0, 0, p, 16), -1),
        ("bark_b200_gpt_eval_slot", (0, 0, p, 1, C.byref(n_past), 1, q), 0),
        ("bark_b200_gpt_step_batch", (0, 1, p, p, p, q), 0),
        ("bark_b200_shard_init", (0, 1, p), 0),
        ("bark_b200_shard_connect", (p,), 0),
        ("bark_b200_shard_nvlink_bytes", (0,), 0),
    ]


def test_null_context_is_refused_the_same_way_everywhere(pkg, capfd):
    L = pkg.lib()
    keep, table = null_context_table()
    assert {fn for fn, _, _ in table} == context_calls()
    capfd.readouterr()
    for fn, args, fail in table:
        got = getattr(L, fn)(None, *args)
        err = capfd.readouterr().err
        if fail is NULL:
            assert not got, fn
        elif fn not in VOID:
            assert got == fail and type(got) is type(fail), (fn, got)
        assert err == ("" if fn in SILENT else f"{fn}: invalid bark context\n"), (fn, err)
    del keep


def test_copy_outs_without_a_context_respect_a_negative_cap(pkg):
    """bark_b200_bert_tokenize and bark_b200_split_text take no context: the same rule for cap < 0"""
    L = pkg.lib()
    vocab = [b"[UNK]", b"hello", b"world", b"."]
    v = (C.c_char_p * len(vocab))(*vocab)
    sentinel = np.full(8, 0x5A5A5A5A, np.int32)
    assert L.bark_b200_bert_tokenize(v, len(vocab), b"hello world.", sentinel.ctypes.data, -1) == 3
    assert L.bark_b200_split_text(v, len(vocab), 0, b"hello world. hello.", 48, sentinel.ctypes.data, -1) == 2
    assert (sentinel == 0x5A5A5A5A).all()


# ---- on the GPU ------------------------------------------------------------------------------------------------------------------
def noise(n, seed):
    return np.random.default_rng(seed).uniform(-0.5, 0.5, n).astype(np.float32)


def drive(b):
    """Every stage of a generation through the per-call entry points, then one evaluation and one sampled row"""
    prompt = b.tokenize("hello world")
    for stage in range(3):
        b.forward(stage)
    logits, _ = b.gpt_eval(0, prompt, 0, True)
    tok, eos, _ = b.sample_rows(logits[None, :1024], 0.7)
    return [prompt] + [b.tokens(s).copy() for s in range(3)] + [logits, tok, eos]


@pytest.mark.gpu
def test_a_context_runs_on_its_device_whatever_device_is_current(pkg, weights_file):
    """Context A on device 0, then B on device 1, loaded by one host thread, which then drives A: every call makes A's device current,
    so A computes what a context alone in its process computes."""
    if cuda_device_count() < 2:
        pytest.skip("needs two GPUs")
    path, L = weights_file("tiny", "f16"), pkg.lib()
    try:
        with pkg.Bark(path, seed=5, n_steps_text_encoder=12, device=0) as a:
            want = drive(a)
        with pkg.Bark(path, seed=5, n_steps_text_encoder=12, device=0) as a, pkg.Bark(path, seed=9, n_steps_text_encoder=12, device=1):
            got = drive(a)
    finally:
        L.bark_b200_set_device(-1)
    for w, g in zip(want, got):
        assert np.array_equal(np.asarray(w).view(np.uint8), np.asarray(g).view(np.uint8))


@pytest.mark.gpu
def test_copy_outs_respect_a_negative_cap(pkg, weights_file):
    """Every call that fills a caller's array, asked with the array set and cap = -1: it returns the size and writes nothing"""
    from encodec_oracle import codec_offset
    path, L = weights_file("tiny", "f16"), pkg.lib()
    sentinel = np.full(1 << 12, 0x5A5A5A5A, np.int32)
    s = sentinel.ctypes.data
    text = C.create_string_buffer(b"\xa5" * 64, 64)
    x = noise(4000, 1)
    with pkg.Bark(path, seed=6, n_steps_text_encoder=12) as b:
        b.generate_batch(["hello world"], [0])
        b.set_long_form("chain")
        b.generate("Hello world. The quick brown fox jumps over the lazy dog! Is it 3.5 or 4? [laughs] That was fun.")
        b.set_long_form(None)
        ctx = b.ctx
        T = (x.size + 319) // 320
        codes = b.encodec_encode(x)
        calls = [(lambda o, cap, st=st: L.bark_b200_get_tokens(ctx, st, o, cap)) for st in range(4)]
        calls += [(lambda o, cap, st=st: L.bark_b200_batch_tokens(ctx, 0, st, o, cap)) for st in range(4)]
        calls += [(lambda o, cap, st=st: L.bark_b200_long_chunk_tokens(ctx, 1, st, o, cap)) for st in range(4)]
        calls += [lambda o, cap: L.bark_b200_batch_audio(ctx, 0, o, cap),
                  lambda o, cap: L.bark_b200_text_ids(ctx, 0, b"hello world", o, cap),
                  lambda o, cap: L.bark_b200_encodec_decode(ctx, codes.ctypes.data, T, o, cap)]
        for f in calls:
            n = f(None, 0)
            assert n >= 1 and f(s, -1) == n
        n = L.bark_b200_long_chunk_text(ctx, 1, None, 0)
        assert n >= 1 and L.bark_b200_long_chunk_text(ctx, 1, text, -1) == n
        assert L.bark_b200_encodec_encode(ctx, x.ctypes.data, x.size, s, -1, s, -1) == T
        assert L.bark_b200_encodec_encode_resampled(ctx, x.ctypes.data, x.size, 1, 24000, s, -1, s, -1) == T
    with pkg.Encodec(path, codec_offset(path)) as e:
        e.bandwidth = 6
        e.compress_batch([x])
        e.reconstruct_batch([x])
        assert L.bark_b200_encodec_batch_codes(e.ctx, 0, s, -1) == 8 * T
        assert L.bark_b200_encodec_batch_audio(e.ctx, 0, s, -1) == 320 * T
    assert (sentinel == 0x5A5A5A5A).all() and text.raw == b"\xa5" * 64
