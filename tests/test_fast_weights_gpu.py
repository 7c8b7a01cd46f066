"""Fast mode for f32 and quantised files, on the GPU (tests/test_fast_weights.py states the rule and checks the constructions):
  * bark_b200_fast_convert equals the rule's f16 bits and dequant.npz, with the non-finite count, at K = 32, 768, 4096;
  * files whose fine matrices hold the same f16-exact values as an f16 file give the same fine passes and generation bit for bit
    in fast mode: the loader converts every matrix and lm_head of every type;
  * against the oracle on random (lossy) files, teacher forced as in tests/test_fast_mode.py;
  * batches, and the refusal of a fine weight outside the f16 range.
"""
import json

import numpy as np
import pytest

from test_fast_weights import DEQ, GGML_FTYPE, QTYPES, dequant, exact_pair, fixture_cases, non_finite, same_f16, to_f16

gpu = pytest.mark.gpu

# Teacher-forced fine passes, nn = 2..7, against the oracle, measured on an H100 80GB HBM3 (700 W limit), worst pass of each case:
#   f32         max |dlogit| tiny 0.0072, mini 0.0107; top-1 agreement >= 99.41 %; CDF-flip rate <= 3.3 %
#   quantised   max |dlogit| tiny 0.116-0.133, mini 0.141-0.186, wide (q4_0) 0.387; top-1 >= 95.7 % (tiny / mini), 89.8 % (wide);
#               CDF-flip rate <= 17.9 %.  The oracle's quantised passes quantise every activation row to q8 (the reference's
#               vec_dot_type) and the fast pass keeps f16 activations, so q8_0 weights agree no better than q4_0 ones.
# The bounds allow about twice the measured max |dlogit| and about twice the measured top-1 disagreement.
MAX_DLOGIT = {("tiny", "f32"): 0.015, ("mini", "f32"): 0.02, ("tiny", "quant"): 0.27, ("mini", "quant"): 0.37, ("wide", "quant"): 0.77}
MIN_TOP1 = {("tiny", "f32"): 0.988, ("mini", "f32"): 0.988, ("tiny", "quant"): 0.91, ("mini", "quant"): 0.91, ("wide", "quant"): 0.79}


@gpu
@pytest.mark.parametrize("t", QTYPES)
def test_convert_matches_the_rule(pkg, t):
    """Edge blocks (K = 32, an odd number of rows) and random rows (K = 768, 4096, odd row counts): the f16 bits of the rule, computed
    from the reference's f32 and from the restatement, and the non-finite count.  The hook checks its guard bands (GuardBandError)."""
    for name, W, K, ref in fixture_cases(t):
        if W.shape[0] % 2 == 0:
            W, ref = W[:-1], ref[:-1]
        got, nf = pkg.fast_convert(t, W)
        want = to_f16(ref)
        assert same_f16(got, want), (t, name, int((got.view(np.uint16) != want.view(np.uint16)).sum()))
        assert same_f16(got, to_f16(dequant(t, W, K))), (t, name)
        assert nf == non_finite(want), (t, name, nf, non_finite(want))


@gpu
@pytest.mark.parametrize("K", [32, 768, 4096])
def test_convert_f32(pkg, K):
    """f32: the f16 round to nearest even of the weight, with +-0, subnormals, the rounding edge of the f16 range (65519.996 -> 65504,
    65520 -> inf) and NaN / inf counted."""
    rng = np.random.default_rng(K)
    W = (rng.standard_normal((7, K)) * 0.05).astype(np.float32)
    specials = np.array([0.0, -0.0, 2.0 ** -25, 3 * 2.0 ** -26, 2.0 ** -24 * 1.5, 65504.0, np.nextafter(np.float32(65520), np.float32(0)),
                         65520.0, -65520.0, 1e30, np.inf, -np.inf, np.nan, 6e-8, -1e-9, 1.0009765625], np.float32)
    W.flat[rng.choice(W.size, specials.size, replace=False)] = specials
    got, nf = pkg.fast_convert("f32", W)
    want = to_f16(W)
    assert same_f16(got, want), int((got.view(np.uint16) != want.view(np.uint16)).sum())
    assert nf == non_finite(want) == 6


@gpu
def test_convert_rejects_bad_arguments(pkg):
    """Unsupported types (f16 included: an f16 file needs no conversion), K not a multiple of 32, empty shapes and null pointers
    return 0 without aborting; a good call still works afterwards."""
    import ctypes as C
    L = pkg.lib()
    src = np.zeros(4096, np.uint8); dst = np.zeros(4096, np.uint16); nf = C.c_int(0)
    p = lambda a: a.ctypes.data_as(C.c_void_p)                             # noqa: E731
    for wtype, n_out, K in ((1, 2, 32), (4, 2, 32), (9, 2, 32), (-1, 2, 32), (2, 2, 48), (2, 2, 0), (2, 0, 32), (0, -1, 32)):
        assert L.bark_b200_fast_convert(wtype, p(src), n_out, K, p(dst), C.byref(nf)) == 0, (wtype, n_out, K)
    assert L.bark_b200_fast_convert(2, None, 2, 32, p(dst), C.byref(nf)) == 0
    assert L.bark_b200_fast_convert(2, p(src), 2, 32, None, C.byref(nf)) == 0
    assert L.bark_b200_fast_convert(2, p(src), 2, 32, p(dst), None) == 0
    got, n = pkg.fast_convert("q8_0", DEQ["edge_q8_0"][:3])
    assert same_f16(got, to_f16(DEQ["edge_deq_q8_0"][:3])) and n == non_finite(got)


@gpu
@pytest.mark.parametrize("t", ("f32",) + QTYPES)
def test_exact_file_equals_f16_file(pkg, weights_mod, tmp_path, monkeypatch, t):
    """A file whose fine matrices are of type t but hold the f16 file's f16-exact values (tests/test_fast_weights.py exact_pair)
    runs the same fast fine passes bit for bit, for every codebook's lm_head, and a whole generation gives the same ids and waveform:
    every converted matrix lands where the fine passes read it."""
    f16, path = exact_pair(pkg, weights_mod, "mini", t, str(tmp_path))
    monkeypatch.setenv("BARK_B200_MODE", "fast")
    buf = np.random.default_rng(11).integers(0, 1024, (8, 1024)).astype(np.int32)
    out = {}
    for name, p in (("f16", f16), (t, path)):
        with pkg.Bark(p, seed=0, n_steps_text_encoder=16) as b:
            assert b.fast_mode, name
            logits = [b.fine_eval(buf, nn) for nn in range(1, 8)]
            audio = b.generate("hello world")
            out[name] = (logits, audio, [b.tokens(s) for s in range(3)])
    (l16, a16, k16), (lt, at, kt) = out["f16"], out[t]
    for nn, (x, y) in enumerate(zip(l16, lt), start=1):
        assert np.array_equal(x.view(np.uint32), y.view(np.uint32)), (t, nn, int((x != y).sum()))
    for s in range(3):
        assert np.array_equal(k16[s], kt[s]), (t, s)
    assert k16[2].size > 0 and np.array_equal(a16.view(np.uint32), at.view(np.uint32))


TF_CASES = [(c, t) for c in ("tiny", "mini") for t in ("f32",) + QTYPES] + [("wide", "q4_0")]


def lossy_file(pkg, weights_file, tmp_path, config, t):
    if t == "f32":
        return weights_file(config, "f32")
    path = str(tmp_path / f"{config}_{t}.bin")
    assert pkg.lib().bark_model_quantize(weights_file(config, "f16").encode(), path.encode(), GGML_FTYPE[t])
    return path


@gpu
@pytest.mark.parametrize("config,t", TF_CASES)
def test_fast_fine_passes_teacher_forced_by_type(pkg, orc, weights_file, tmp_path, monkeypatch, config, t):
    """tests/test_fast_mode.py's teacher-forced procedure on random f32 and quantised files: every fast pass sees the oracle's
    inputs; max |dlogit|, top-1 agreement and the CDF-flip rate per pass are printed and bounded; a pass repeated is bit-identical; the
    semantic and coarse ids of a whole generation equal the oracle's (those stages run the parity path)."""
    path = lossy_file(pkg, weights_file, tmp_path, config, t)
    o = orc.Oracle(path, seed=0, n_steps=16)
    ref = o.generate("hello world")
    T = ref["fine"].shape[0]
    buf = np.full((8, 1024), 1024, np.int32)
    buf[:, :T] = ref["fine"].T
    monkeypatch.setenv("BARK_B200_MODE", "fast")
    report = {}
    with pkg.Bark(path, seed=0, n_steps_text_encoder=16) as b:
        assert b.fast_mode
        for nn in range(2, 8):
            lf = b.fine_eval(buf, nn)
            lo = o.fine_eval(buf, nn)
            d = float(np.abs(lf - lo).max())
            top1 = float((lf[:, :1024].argmax(1) == lo[:, :1024].argmax(1)).mean())
            b.reseed(5); tf, _, _ = b.sample_rows(lf[:, :1024].copy(), 0.5)
            b.reseed(5); to, _, _ = b.sample_rows(lo[:, :1024].copy(), 0.5)
            report[nn] = dict(max_dlogit=round(d, 5), top1=round(top1, 4), cdf_flip_rate=round(float((tf != to).mean()), 5))
        again = b.fine_eval(buf, 7)
        assert np.array_equal(again.view(np.uint32), lf.view(np.uint32)), "a repeated pass differs"
        b.reseed(0)
        audio = b.generate("hello world")
        assert np.array_equal(b.tokens(0), ref["semantic"]) and np.array_equal(b.tokens(1), ref["coarse"])
        report["generate"] = dict(fine_ids_equal=round(float((b.tokens(2) == ref["fine"]).mean()), 4), frames=int(T),
                                  wav_rel=round(float(np.abs(audio - ref["audio"]).max() / np.abs(ref["audio"]).max()), 4))
    print("fast-mode agreement", config, t, json.dumps(report))
    key = config, "f32" if t == "f32" else "quant"
    for nn in range(2, 8):
        assert report[nn]["max_dlogit"] < MAX_DLOGIT[key] and report[nn]["top1"] >= MIN_TOP1[key], report


@gpu
def test_batch_q4_0_fast_items_equal_single_runs(pkg, weights_file, tmp_path, monkeypatch):
    """generate_batch in fast mode on a q4_0 file: each item equals its own single fast run (ids and waveform)."""
    path = lossy_file(pkg, weights_file, tmp_path, "mini", "q4_0")
    monkeypatch.setenv("BARK_B200_MODE", "fast")
    texts, seeds = ["hello world", "the quick brown fox"], [0, 3]
    with pkg.Bark(path, seed=0, n_steps_text_encoder=16) as b:
        assert b.fast_mode
        audios = b.generate_batch(texts, seeds)
        batch = [[b.batch_tokens(i, s) for s in range(3)] for i in range(2)]
    for i, (text, seed) in enumerate(zip(texts, seeds)):
        with pkg.Bark(path, seed=seed, n_steps_text_encoder=16) as b:
            a = b.generate(text)
            for s in range(3):
                assert np.array_equal(batch[i][s], b.tokens(s)), (i, s)
            assert np.array_equal(audios[i].view(np.uint32), a.view(np.uint32)), i


@gpu
def test_weight_outside_f16_range_refuses_fast_mode(pkg, weights_mod, tmp_path, monkeypatch, capfd):
    """An f32 file with one fine weight of 1e5 loads in fast mode, reports fast_mode False with a message naming the tensor, and
    computes exactly what the parity path computes."""
    cfg = weights_mod.tiny(weights_mod.F32)
    w = (np.random.default_rng(2).standard_normal((4 * 128, 128)) * 0.02).astype(np.float32)
    w[17, 5] = 1e5
    path = weights_mod.write_weights(str(tmp_path / "big.bin"), cfg, overrides={"fine/model/h1/mlp/c_fc/w": w})
    buf = np.random.default_rng(4).integers(0, 1024, (8, 1024)).astype(np.int32)
    runs = {}
    for mode in ("fast", "parity"):
        monkeypatch.setenv("BARK_B200_MODE", mode)
        capfd.readouterr()
        with pkg.Bark(path, seed=0, n_steps_text_encoder=12) as b:
            err = capfd.readouterr().err
            assert not b.fast_mode
            if mode == "fast":
                assert "model/h1/mlp/c_fc/w" in err and "parity path" in err, err
            runs[mode] = (b.fine_eval(buf, 3), b.generate("hello world"), b.tokens(2))
    (lf, af, kf), (lp, ap, kp) = runs["fast"], runs["parity"]
    assert np.array_equal(lf.view(np.uint32), lp.view(np.uint32))
    assert np.array_equal(kf, kp) and np.array_equal(af.view(np.uint32), ap.view(np.uint32))
