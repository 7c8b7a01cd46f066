"""Resampling on the GPU (bark_b200_resample and the resampled EnCodec calls, DESIGN.md §16): bit-identical to the rule's CPU
restatement (tests/resample_oracle.py) at every rate pair and channel count, within the bound of torchaudio's stored outputs
(tests/golden/resample/torchaudio.npz), and each resampled EnCodec call equal to its mono 24 kHz counterpart on the restated clip."""
import ctypes as C
import functools
import os

import numpy as np
import pytest

from conftest import GOLDEN_DIR
import encoder_oracle as eo
from encodec_oracle import codec_offset
import resample_oracle as ro

pytestmark = pytest.mark.gpu
GOLD = os.path.join(GOLDEN_DIR, "resample", "torchaudio.npz")
FIXTURE_PAIRS = [(sr, 24000) for sr in (8000, 11025, 16000, 22050, 32000, 44100, 44056, 48000, 96000)] + [(24000, 44100), (24000, 48000)]
EXTRA_PAIRS = [(383999, 24000), (24000, 383999), (4000, 24000)]
KINDS = ("silent", "full", "zeros", "subnormal", "noise")


@functools.lru_cache(maxsize=None)
def table(sr, nsr):
    return ro.sparse_taps(sr, nsr)


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def planar(x):
    """interleaved [n][C] (or mono [n]) -> the [C][n] layout the Python calls take"""
    return x if x.ndim == 1 else np.ascontiguousarray(x.T)


@pytest.fixture(scope="module")
def codec(pkg, weights_file, weights_mod):
    path = eo.weights_path(weights_file, weights_mod, "base")
    with pkg.Encodec(path, codec_offset(path)) as e:
        yield e


@pytest.fixture(scope="module")
def bark(pkg, weights_file, weights_mod):
    with pkg.Bark(eo.weights_path(weights_file, weights_mod, "base"), seed=0, n_steps_text_encoder=12) as b:
        yield b


@pytest.mark.parametrize("sr,nsr", FIXTURE_PAIRS + EXTRA_PAIRS)
def test_resample_bit_identical_to_the_rule(pkg, sr, nsr):
    t = table(sr, nsr)
    for ch in (1, 2, 3, 8):
        for kind in KINDS:
            n = {"noise": sr // 4 + 7, "full": 1921}.get(kind, 333)
            x = ro.clip(kind, n, ch, seed=ch * 31 + len(kind))
            got, want = pkg.resample(planar(x), sr, nsr), ro.resample(x, sr, nsr, t)
            assert got.size == want.size == ro.out_len(n, sr, nsr)
            assert np.array_equal(bits(got), bits(want)), f"{kind}, {ch} channels: {int((bits(got) != bits(want)).sum())} differ"
    for n in (1, 2, 3):
        x = ro.clip("noise", n, 2, seed=n)
        assert np.array_equal(bits(pkg.resample(planar(x), sr, nsr)), bits(ro.resample(x, sr, nsr, t))), n


@pytest.mark.parametrize("sr,nsr", FIXTURE_PAIRS)
def test_resample_within_the_bound_of_torchaudio(pkg, sr, nsr):
    gold, t, k = np.load(GOLD), table(sr, nsr), f"{sr}_{nsr}"
    for n in (1, 2, 3, 1920, 1921, 10 * sr):
        x = ro.clip("noise", n, seed=n)
        y = pkg.resample(x, sr, nsr)
        assert np.array_equal(bits(y), bits(ro.resample(x, sr, nsr, t))), n
        b = ro.bound(x, sr, nsr, y, t)
        if n == 10 * sr:
            idx = gold[f"{k}_n{n}_idx"]
            assert y.size == int(gold[f"{k}_n{n}_len"])
            y, b = y[idx], b[idx]
        ref = gold[f"{k}_n{n}"]
        assert y.size == ref.size and (np.abs(y.astype(np.float64) - ref) <= b).all(), n


def test_identity_calls_equal_their_counterparts(pkg, codec, bark):
    x = eo.signal("noise", 24001, seed=5)
    assert np.array_equal(bits(pkg.resample(x, 24000, 24000)), bits(x))
    for bw in (6, 24):
        codec.bandwidth = bw
        assert np.array_equal(codec.compress(x, sample_rate=24000), codec.compress(x))
        assert np.array_equal(bits(codec.reconstruct(x, sample_rate=24000)), bits(codec.reconstruct(x)))
        xs = [x, eo.signal("sine", 1921), eo.signal("square", 4800)]
        for a, b in zip(codec.compress_batch(xs, sample_rate=24000), codec.compress_batch(xs)):
            assert np.array_equal(a, b)
        for a, b in zip(codec.reconstruct_batch(xs, sample_rate=[24000] * 3), codec.reconstruct_batch(xs)):
            assert np.array_equal(bits(a), bits(b))
    codec.bandwidth = 24
    c1, l1 = bark.encodec_encode(x, return_latent=True, sample_rate=24000)
    c0, l0 = bark.encodec_encode(x, return_latent=True)
    assert np.array_equal(c1, c0) and np.array_equal(bits(l1), bits(l0))


CLIPS = [(44100, 2, 44100 // 2 + 11), (48000, 1, 48000), (16000, 6, 4000), (22050, 8, 3000), (383999, 1, 40000), (4000, 3, 700)]


@pytest.mark.parametrize("bw", [6, 24])
def test_resampled_calls_equal_their_counterparts_on_the_restated_clip(codec, bark, bw):
    codec.bandwidth = bw
    for sr, ch, n in CLIPS:
        x = ro.clip("noise", n, ch, seed=sr + ch)
        u = ro.resample(x, sr, 24000, table(sr, 24000))
        assert np.array_equal(codec.compress(planar(x), sample_rate=sr), codec.compress(u)), (sr, ch)
        assert np.array_equal(bits(codec.reconstruct(planar(x), sample_rate=sr)), bits(codec.reconstruct(u))), (sr, ch)
        if bw == 6:                          # the bark context's codec runs 8 codebooks (6 kbps)
            c1, l1 = bark.encodec_encode(planar(x), return_latent=True, sample_rate=sr)
            c0, l0 = bark.encodec_encode(u, return_latent=True)
            assert np.array_equal(c1, c0) and np.array_equal(bits(l1), bits(l0)), (sr, ch)
    codec.bandwidth = 24


def test_batches_of_mixed_formats_equal_their_single_calls(codec):
    codec.bandwidth = 6
    rates = (44100, 48000, 16000, 24000, 24000, 11025, 96000, 32000)
    items = []
    for i in range(70):                                  # three launches by count
        sr, ch = rates[i % len(rates)], 1 + i % 4
        items.append((ro.clip("noise", sr // 10 + 97 * i, ch, seed=400 + i), sr))
    xs, srs = [planar(x) for x, _ in items], [sr for _, sr in items]
    want = [codec.compress(x, sample_rate=sr) for x, sr in zip(xs, srs)]
    got = codec.compress_batch(xs, sample_rate=srs)
    assert all(np.array_equal(a, b) for a, b in zip(got, want))
    rec = codec.reconstruct_batch(xs[:9], sample_rate=srs[:9])
    assert all(np.array_equal(bits(a), bits(codec.reconstruct(x, sample_rate=sr))) for a, x, sr in zip(rec, xs[:9], srs[:9]))
    # over the frame budget: about 8000 frames each, and one item longer than a launch
    long = [(ro.clip("noise", 48000 * 107 + 13 * i, 2, seed=i), 48000) for i in range(3)]
    long.insert(1, (ro.clip("noise", 44100 * 330, 1, seed=9), 44100))
    xs, srs = [planar(x) for x, _ in long], [sr for _, sr in long]
    got = codec.compress_batch(xs, sample_rate=srs)
    assert all(np.array_equal(a, codec.compress(x, sample_rate=sr)) for a, x, sr in zip(got, xs, srs))
    codec.bandwidth = 24


def test_refusals_name_the_item_and_change_nothing(pkg, codec, capfd):
    L = pkg.lib()
    codec.bandwidth = 12
    ok = [planar(ro.clip("noise", 9000, 2, seed=1)), planar(ro.clip("noise", 3841, 1, seed=2))]
    codes = codec.compress_batch(ok, sample_rate=[44100, 48000])          # 3841 frames at 48 kHz: L = 1921, accepted
    assert codes[1].shape[1] == 7
    single = codec.compress(ok[0], sample_rate=44100)
    capfd.readouterr()
    bad = [
        (1, [ok[0], np.zeros(3840, np.float32)], [44100, 48000], "1920"),        # L = 1920
        (2, [ok[0], ok[1], np.zeros((9, 4000), np.float32)], [44100, 48000, 48000], "9 channels"),
        (0, [ok[0]], [3999], "sample rate 3999"),
        (1, [ok[0], ok[1]], [44100, 384001], "sample rate 384001"),
        (1, [ok[0], np.where(np.arange(5000) == 77, np.nan, 0.1).astype(np.float32)], [44100, 16000], "sample 77"),
        (1, [ok[0], np.full((2, 5000), 2.0 ** 65, np.float32)], [44100, 16000], "sample 0"),
    ]
    for k, xs, srs, what in bad:
        for f in (codec.compress_batch, codec.reconstruct_batch):
            with pytest.raises(RuntimeError):
                f(xs, sample_rate=srs)
            err = capfd.readouterr().err
            assert f"item {k}:" in err and what in err, err
    with pytest.raises(RuntimeError):
        codec.compress(np.zeros(3840, np.float32), sample_rate=48000)
    assert "1920" in capfd.readouterr().err
    with pytest.raises(ValueError):
        codec.compress_batch(ok, sample_rate=[44100])
    ptrs = (C.c_void_p * 2)(*[np.ascontiguousarray(x.T).ctypes.data for x in ok])
    ints = (C.c_int * 2)(9000, 3841)
    assert not L.bark_b200_encodec_compress_batch_resampled(codec.ctx, ptrs, ints, None, ints, 2)
    assert not L.bark_b200_encodec_compress_batch_resampled(codec.ctx, ptrs, ints, ints, None, 2)
    assert not L.bark_b200_encodec_compress_resampled(codec.ctx, None, 100, 1, 24000)
    for args in ((3841, 0, 24000, 24000), (3841, 1, 24000, 3999), (0, 1, 24000, 24000)):
        assert L.bark_b200_resample(ok[1].ctypes.data, *args, None, 0) == -1
    x = ro.clip("noise", 100, 1)
    assert L.bark_b200_resample(x.ctypes.data, 100, 1, 24000, 48000, None, 0) == 200
    out = np.zeros(199, np.float32)
    assert L.bark_b200_resample(x.ctypes.data, 100, 1, 24000, 48000, out.ctypes.data, 199) == -1
    capfd.readouterr()
    for i, c in enumerate(codes):                                       # the last successful batch is still there
        got = np.empty(c.size, np.int32)
        assert L.bark_b200_encodec_batch_codes(codec.ctx, i, got.ctypes.data, got.size) == c.size and np.array_equal(got, c.ravel())
    n = L.encodec_get_codes_size(codec.ctx)
    assert np.array_equal(np.ctypeslib.as_array(L.encodec_get_codes(codec.ctx), shape=(n,)), single.ravel())
    assert codec.compress_batch(ok, sample_rate=[44100, 48000])[0].shape == codes[0].shape
    codec.bandwidth = 24
