"""Batched EnCodec on the GPU (bark_b200_encodec_*_batch, Encodec.compress_batch / decompress_batch / reconstruct_batch): item i of a
batch equals the single call on clip i on the same context, bit for bit, whatever the other items, their count and i's place, and
the reference's stored outputs where they exist (tests/golden/ref_pairs/encodec_bandwidths.npz)."""
import ctypes as C
import os
import threading

import numpy as np
import pytest

from conftest import GOLDEN_DIR, assert_pinned
import encoder_oracle as eo
from encodec_oracle import codec_offset

pytestmark = pytest.mark.gpu
GOLD = os.path.join(GOLDEN_DIR, "ref_pairs", "encodec_bandwidths.npz")
N_Q = {1: 1, 2: 2, 6: 8, 24: 32}
LENGTHS = (1921, 1922, 2240, 24000, 24001, 240000, 720000)
MAX_ITEMS, MAX_FRAMES = 32, 24000          # one launch's items and frames (include/bark_b200.h)


@pytest.fixture(scope="module")
def codecs(pkg, weights_file, weights_mod):
    out = {}
    for w in eo.WEIGHTS:
        path = eo.weights_path(weights_file, weights_mod, w)
        out[w] = pkg.Encodec(path, codec_offset(path))
    yield out
    for e in out.values():
        e.close()


@pytest.fixture(scope="module")
def ragged():
    return [eo.signal(("noise", "sine", "square")[i % 3], n, seed=300 + i) for i, n in enumerate(LENGTHS)]


def same_codes(got, want, what):
    assert len(got) == len(want), what
    for i, (g, w) in enumerate(zip(got, want)):
        assert g.shape == w.shape and np.array_equal(g, w), f"{what}: item {i}: {int((g != w).sum()) if g.shape == w.shape else g.shape} differ"


def same_audio(got, want, what):
    assert len(got) == len(want), what
    for i, (g, w) in enumerate(zip(got, want)):
        assert g.shape == w.shape and np.array_equal(g.view(np.uint32), w.view(np.uint32)), f"{what}: item {i} differs"


@pytest.mark.parametrize("bw", sorted(N_Q))
def test_compress_batch_equals_single_calls(codecs, ragged, bw):
    e = codecs["base"]
    e.bandwidth = bw
    single = [e.compress(x) for x in ragged]
    assert all(c.shape[0] == N_Q[bw] for c in single)
    same_codes(e.compress_batch(ragged), single, f"{bw} kbps")
    same_codes(e.compress_batch(ragged[::-1]), single[::-1], f"{bw} kbps reversed")
    dup = [ragged[3], ragged[0], ragged[3], ragged[3]]
    same_codes(e.compress_batch(dup), [single[3], single[0], single[3], single[3]], f"{bw} kbps duplicated")
    loud = [x * np.float32(40) for x in ragged[2:5]]
    mixed = [loud[0], np.zeros(24000, np.float32), loud[1], loud[2]]
    same_codes(e.compress_batch(mixed), [e.compress(x) for x in mixed], f"{bw} kbps zeros beside loud clips")
    e.bandwidth = 24


def test_stored_cases_batched_per_model_file(codecs):
    gold = np.load(GOLD)
    for which in eo.WEIGHTS:
        cases = [c for c in eo.CASES if c[3] == which]
        xs = [eo.signal(kind, n, seed=n) for _, kind, n, _ in cases]
        e = codecs[which]
        for bw in (1, 2, 3, 12, 24):
            e.bandwidth = bw
            got = e.compress_batch(xs)
            for (name, *_), c in zip(cases, got):
                ref = gold[f"{name}_bw{bw}_codes"]
                assert c.shape == ref.shape and np.array_equal(c, ref), f"{name} at {bw} kbps"
            same_codes(got, [e.compress(x) for x in xs], f"{which} at {bw} kbps")
        stored = [(name, x) for (name, *_), x in zip(cases, xs) if name in eo.RECONSTRUCT]
        for bw in (3, 12, 24):
            e.bandwidth = bw
            for (name, _), a in zip(stored, e.reconstruct_batch([x for _, x in stored] + xs)):
                assert_pinned(a, gold, f"{name}_bw{bw}_audio", f"{name} batched reconstruction at {bw} kbps")
        e.bandwidth = 24


def test_decompress_batch_of_ragged_codes(codecs):
    import make_golden_encodec as mg
    gold = np.load(GOLD)
    e = codecs["base"]
    rng = np.random.default_rng(7)
    for bw, n_q in ((6, 8), (24, 32)):
        e.bandwidth = bw
        codes = [rng.integers(0, 1024, (n_q, T)).astype(np.int32) for T in (7, 8, 31, 75, 750, 2250, 9)]
        same_audio(e.decompress_batch(codes), [e.decompress(c) for c in codes], f"{bw} kbps")
    for bw, n_q in zip(mg.DECOMPRESS_BW, (16, 32)):
        e.bandwidth = bw
        c = mg.decompress_codes(bw, n_q)
        got = e.decompress_batch([c[:, :40], c, c[:, 40:]])
        assert_pinned(got[1], gold, f"decompress_bw{bw}_audio", f"batched decompress at {bw} kbps")
        same_audio([got[0], got[2]], [e.decompress(c[:, :40]), e.decompress(np.ascontiguousarray(c[:, 40:]))], f"{bw} kbps slices")
    e.bandwidth = 24


def test_reconstruct_batch_equals_single_and_decompress_of_compress(codecs, ragged):
    e = codecs["base"]
    for bw in (6, 24):
        e.bandwidth = bw
        got = e.reconstruct_batch(ragged)
        same_audio(got, [e.reconstruct(x) for x in ragged], f"{bw} kbps")
        same_audio(got, e.decompress_batch(e.compress_batch(ragged)), f"{bw} kbps decompress of compress")
    e.bandwidth = 24


def test_batches_over_the_item_cap_and_the_frame_budget(codecs):
    e = codecs["base"]
    e.bandwidth = 6
    many = [eo.signal("noise", 1921 + 331 * i, seed=900 + i) for i in range(MAX_ITEMS * 2 + 5)]          # three launches by count
    same_codes(e.compress_batch(many), [e.compress(x) for x in many], "over the item cap")
    same_codes(e.compress_batch(many), [c for i in range(0, len(many), 7) for c in e.compress_batch(many[i:i + 7])], "small batches")
    same_audio(e.reconstruct_batch(many), [e.reconstruct(x) for x in many], "reconstruct over the item cap")
    long = [eo.signal("noise", 320 * MAX_FRAMES // 3 + 17 * i, seed=950 + i) for i in range(4)]          # about 8000 frames each
    long.insert(2, eo.signal("sine", 320 * (MAX_FRAMES + 100), seed=5))          # longer than a launch: launches of 2, 1 and 2 items
    want = [e.compress(x) for x in long]
    same_codes(e.compress_batch(long), want, "over the frame budget")
    same_audio(e.decompress_batch(want), [e.decompress(c) for c in want], "decompress over the frame budget")
    e.bandwidth = 24


def test_refusals_leave_results_and_context_alone(pkg, codecs, capfd):
    L, e = pkg.lib(), codecs["base"]
    e.bandwidth = 12
    xs = [eo.signal("noise", n, seed=n) for n in (4000, 9999, 1921)]
    single_codes, single_audio = e.compress(xs[0]), e.reconstruct(xs[1])
    codes = e.compress_batch(xs)
    audio = e.decompress_batch(codes)
    n_q = codes[0].shape[0]

    def arrays(items):
        return (C.c_void_p * len(items))(*[a.ctypes.data for a in items]), (C.c_int * len(items))(*[a.size for a in items])
    ptrs, lens = arrays(xs)
    assert not L.bark_b200_encodec_compress_batch(e.ctx, ptrs, lens, 0)
    assert not L.bark_b200_encodec_compress_batch(e.ctx, ptrs, lens, -1)
    big = xs * 400
    bp, bl = arrays(big)
    assert not L.bark_b200_encodec_compress_batch(e.ctx, bp, bl, 1025)
    assert not L.bark_b200_encodec_compress_batch(e.ctx, None, lens, 3)
    assert not L.bark_b200_encodec_reconstruct_batch(e.ctx, ptrs, None, 3)
    assert not L.bark_b200_encodec_decompress_batch(e.ctx, None, lens, 3)
    nulls = (C.c_void_p * 3)(ptrs[0], None, ptrs[2])
    assert not L.bark_b200_encodec_compress_batch(e.ctx, nulls, lens, 3)
    assert not L.bark_b200_encodec_compress_batch(None, ptrs, lens, 3)
    capfd.readouterr()
    bad_audio = [
        (2, [xs[0], xs[1], np.zeros(1920, np.float32)]),                                    # short
        (1, [xs[0], np.where(np.arange(9999) == 77, np.nan, 0.1).astype(np.float32)]),     # NaN
        (3, [xs[2], xs[0], xs[1], np.where(np.arange(4000) == 3999, np.inf, 0.1).astype(np.float32)]),
    ]
    for k, bad in bad_audio:
        for f in (e.compress_batch, e.reconstruct_batch):
            with pytest.raises(RuntimeError):
                f(bad)
            assert f"item {k}:" in capfd.readouterr().err
    with pytest.raises(RuntimeError):                                                  # a batch of one names its item too
        e.compress_batch([np.zeros(1920, np.float32)])
    assert "bark_b200_encodec_compress_batch: item 0:" in capfd.readouterr().err
    outside = [c.copy() for c in codes]
    outside[1][3, 5] = 1024
    bad_codes = [(1, outside), (1, [codes[0], codes[1][:, :6]]), (2, [codes[0], codes[1], np.full((n_q, 9), -1, np.int32)])]
    for k, bad in bad_codes:
        with pytest.raises(RuntimeError):
            e.decompress_batch(bad)
        assert f"bark_b200_encodec_decompress_batch: item {k}:" in capfd.readouterr().err
    cp, cl = arrays([c.ravel() for c in codes])
    cl[1] -= 1                                                                          # n_codes % n_q != 0
    assert not L.bark_b200_encodec_decompress_batch(e.ctx, cp, cl, 3)
    assert "item 1:" in capfd.readouterr().err
    for i, c in enumerate(codes):
        got = np.empty(c.size, np.int32)
        assert L.bark_b200_encodec_batch_codes(e.ctx, i, got.ctypes.data, got.size) == c.size and np.array_equal(got, c.ravel())
        a = np.empty(audio[i].size, np.float32)
        assert L.bark_b200_encodec_batch_audio(e.ctx, i, a.ctypes.data, a.size) == audio[i].size
        assert np.array_equal(a.view(np.uint32), audio[i].view(np.uint32))
    assert L.bark_b200_encodec_batch_codes(e.ctx, 3, None, 0) == -1 and L.bark_b200_encodec_batch_audio(e.ctx, -1, None, 0) == -1
    assert L.bark_b200_encodec_batch_codes(None, 0, None, 0) == -1
    n = L.encodec_get_codes_size(e.ctx)                                                 # the single-call getters: the last single calls'
    assert np.array_equal(np.ctypeslib.as_array(L.encodec_get_codes(e.ctx), shape=(n,)), single_codes.ravel())
    n = L.encodec_get_audio_size(e.ctx)
    assert np.array_equal(np.ctypeslib.as_array(L.encodec_get_audio(e.ctx), shape=(n,)).view(np.uint32), single_audio.view(np.uint32))
    same_codes(e.compress_batch(xs), codes, "after the refusals")
    e.bandwidth = 24


def test_two_contexts_batching_on_two_threads(pkg, codecs, weights_file):
    """Batches of different sizes on two contexts at once (the recurrence's launch shape differs between them)."""
    path = weights_file("tiny", "f16", 1234)
    xs = [eo.signal("noise", 4000 + 1321 * i, seed=70 + i) for i in range(MAX_ITEMS)]
    sizes = (MAX_ITEMS, 5)
    e = codecs["base"]
    e.bandwidth = 24
    want = {k: (e.compress_batch(xs[:n]), e.reconstruct_batch(xs[:n])) for k, n in enumerate(sizes)}
    got, errors = {}, []

    def work(k):
        try:
            with pkg.Encodec(path, codec_offset(path)) as mine:
                for _ in range(3):
                    got[k] = (mine.compress_batch(xs[:sizes[k]]), mine.reconstruct_batch(xs[:sizes[k]]))
        except Exception as exc:      # noqa: BLE001  (reported below)
            errors.append(exc)
    ts = [threading.Thread(target=work, args=(k,)) for k in range(2)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    assert not errors, errors
    for k in range(2):
        same_codes(got[k][0], want[k][0], f"thread {k}")
        same_audio(got[k][1], want[k][1], f"thread {k}")
