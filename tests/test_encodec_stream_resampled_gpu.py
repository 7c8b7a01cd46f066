"""Resampled EnCodec streams on the GPU (bark_b200_encodec_stream_open_resampled, Encodec.stream(..., sample_rate=, channels=), DESIGN.md
§20): everything a stream returns, joined, equals the whole-clip call on everything it was pushed, bit for bit, whatever the chunks and the
other streams of a batch: bark_b200_encodec_compress_resampled for an encode, bark_b200_resample of encodec_decompress_audio for a decode.
Outputs come back exactly when the readiness rule says they are final.  The window hook equals slices of bark_b200_resample."""
import ctypes as C

import numpy as np
import pytest

import encoder_oracle as eo
from encodec_oracle import codec_offset
import resample_oracle as ro

pytestmark = pytest.mark.gpu
N_Q = {1: 1, 6: 8, 24: 32}                 # kbps -> codebooks (1 kbps: one codebook, as 1.5 kbps gives upstream)
ENCODE_RATES = (8000, 16000, 22050, 44100, 48000, 96000, 383999)


@pytest.fixture(scope="module")
def codec(pkg, weights_file, weights_mod):
    path = eo.weights_path(weights_file, weights_mod, "base")
    e = pkg.Encodec(path, codec_offset(path))
    yield e
    e.close()


def rates(sr, nsr=24000):
    o, q, w, _ = ro.rates(sr, nsr)
    return (1, 1, 0) if sr == nsr else (o, q, w)


def planar(x):
    return x if x.ndim == 1 else np.ascontiguousarray(x.T)


def same_bits(a, b):
    return a.shape == b.shape and np.array_equal(np.ascontiguousarray(a, np.float32).view(np.uint32), np.ascontiguousarray(b, np.float32).view(np.uint32))


def sizes(schedule, n, seed=0):
    """Chunk sizes summing to n: one push, pushes of k frames, one frame each, or random sizes with zeros among them."""
    if schedule == "one":
        return [n]
    if schedule == "ones":
        return [1] * n
    if schedule == "random":
        rng = np.random.default_rng(seed)
        out = []
        while sum(out) < n:
            k = int(rng.choice([0, 1, int(rng.integers(2, 700)), int(rng.integers(700, 9000))]))
            out.append(min(k, n - sum(out)))
        return out[:1] + [0] + out[1:]
    k = int(schedule)
    return [k] * (n // k) + ([n % k] if n % k else [])


def encode_stream(pkg, e, x, sr, chunks):
    """Codes of the frames x ([n] or [n][C]) through an encode stream at sr in the given chunk sizes; checks the frame count after every
    push against the rule."""
    ch = 1 if x.ndim == 1 else x.shape[1]
    with e.stream("encode", sample_rate=sr, channels=ch) as s:
        got, pushed, frames = [], 0, 0
        for k in chunks:
            c = s.push(x[pushed:pushed + k])
            pushed += k
            frames += c.shape[1]
            assert c.shape[0] == s.n_q and frames == pkg.encodec_stream_ready("encode", pushed, sample_rate=sr), (pushed, frames)
            got.append(c)
        got.append(s.finish())
    return np.concatenate(got, axis=1)


def decode_stream(pkg, e, codes, sr, chunks):
    with e.stream("decode", sample_rate=sr) as s:
        got, pushed, samples = [], 0, 0
        for k in chunks:
            a = s.push(codes[:, pushed:pushed + k])
            pushed += k
            samples += a.size
            assert samples == pkg.encodec_stream_ready("decode", pushed, sample_rate=sr), (pushed, samples)
            got.append(a)
        got.append(s.finish())
    return np.concatenate(got)


def clip_frames(sr):
    """a clip past two of sr's blocks and about 0.3 s long"""
    o, _, w = rates(sr)
    return max(int(0.3 * sr), 2 * o + w + 5) + 17


# ---- 1. encode equality -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bw", sorted(N_Q))
@pytest.mark.parametrize("ch", (1, 2, 8))
@pytest.mark.parametrize("sr", ENCODE_RATES)
def test_encode_equals_compress_resampled(pkg, codec, sr, ch, bw):
    codec.bandwidth = bw
    n = clip_frames(sr)
    x = ro.clip("noise", n, ch, seed=sr + ch)
    want = codec.compress(planar(x), sample_rate=sr)
    L = pkg.resampled_length(n, sr)
    assert want.shape == (N_Q[bw], (L + 319) // 320)
    for schedule in ("one", "random"):
        got = encode_stream(pkg, codec, x, sr, sizes(schedule, n, seed=sr + bw))
        assert got.shape == want.shape and np.array_equal(got, want), schedule


@pytest.mark.parametrize("sr", ENCODE_RATES)
def test_encode_in_pushes_of_o_and_one_frame(pkg, codec, sr):
    """pushes of o - 1, o and o + 1 frames (o: the input frames of one block of q outputs), and one frame at a time, on short clips"""
    codec.bandwidth = 6
    o, _, w = rates(sr)
    n = clip_frames(sr) if o > 16 else pkg.resampled_length(2600, 24000, sr)   # L about 2600 when a block is a few frames
    x = ro.clip("noise", n, 2, seed=sr)
    want = codec.compress(planar(x), sample_rate=sr)
    schedules = [str(k) for k in (o - 1, o, o + 1) if k > 0] + (["ones"] if sr in (8000, 44100, 48000) else [])
    for schedule in schedules:
        got = encode_stream(pkg, codec, x, sr, sizes(schedule, n))
        assert got.shape == want.shape and np.array_equal(got, want), schedule


def test_ready_frames_do_not_change_with_later_samples(pkg, codec):
    """Two clips share their first n frames: the frames a stream reported final after n are those of both whole-clip compresses, and
    the next frame is not final (some continuation changes it)."""
    codec.bandwidth = 24
    rng = np.random.default_rng(5)
    changed = trials = 0
    for sr in (44100, 48000, 16000):
        for trial in range(4):
            n = int(rng.integers(rates(sr)[0] + 4493, 4 * sr)) if trial else ro.out_len(2240, 24000, sr) + 40
            head = ro.clip("noise", n, 2, seed=trial)
            a_x = np.concatenate([head, ro.clip("noise", sr // 5, 2, seed=50 + trial)])
            b_x = np.concatenate([head, np.float32(3) * ro.clip("noise", sr // 5, 2, seed=80 + trial)])
            with codec.stream("encode", sample_rate=sr, channels=2) as s:
                part = s.push(head)
            r = pkg.encodec_stream_ready("encode", n, sample_rate=sr)
            assert part.shape[1] == r > 0
            a, b = codec.compress(planar(a_x), sample_rate=sr), codec.compress(planar(b_x), sample_rate=sr)
            assert np.array_equal(a[:, :r], part) and np.array_equal(b[:, :r], part), (sr, n)
            changed += not np.array_equal(a[:, r], b[:, r])
            trials += 1
    assert changed >= trials - 2, f"the frame after the ready ones was final in {trials - changed} of {trials} trials"


# ---- 2. decode equality -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("T", (7, 8, 150, 750))
@pytest.mark.parametrize("sr", (16000, 44100, 48000))
def test_decode_equals_resample_of_decompress(pkg, codec, sr, T):
    codec.bandwidth = 6
    codes = np.random.default_rng(T + sr).integers(0, 1024, (8, T)).astype(np.int32)
    want = pkg.resample(codec.decompress(codes), 24000, sr)
    assert want.size == ro.out_len(320 * T, 24000, sr)
    for schedule in ("ones", "random"):
        got = decode_stream(pkg, codec, codes, sr, sizes(schedule, T, seed=T) if schedule == "random" else [1] * T)
        assert same_bits(got, want), schedule


def test_encode_stream_feeds_decode_stream(pkg, codec):
    """48 kHz stereo in, 48 kHz out, one code frame (640 source frames) per push"""
    codec.bandwidth = 6
    x = ro.clip("noise", 48000, 2, seed=9)
    enc, dec = codec.stream("encode", sample_rate=48000, channels=2), codec.stream("decode", sample_rate=48000)
    out = []
    for i in range(0, x.shape[0], 640):
        c = enc.push(x[i:i + 640])
        if c.shape[1]:
            out.append(dec.push(c))
    out.append(dec.push(enc.finish()))
    out.append(dec.finish())
    enc.close(), dec.close()
    want = pkg.resample(codec.reconstruct(planar(x), sample_rate=48000), 24000, 48000)
    assert same_bits(np.concatenate(out), want)


def test_mono_24k_through_open_resampled_is_the_plain_stream(pkg, codec):
    codec.bandwidth = 24
    x = eo.signal("noise", 9000, seed=3)
    chunks = sizes("random", x.size, seed=3)
    with codec.stream("encode") as a, codec.stream("encode", sample_rate=24000, channels=1) as b:
        assert not a.channels > 1 and b.sample_rate == 24000
        pushed = 0
        for k in chunks:
            ca, cb = a.push(x[pushed:pushed + k]), b.push(x[pushed:pushed + k])
            pushed += k
            assert np.array_equal(ca, cb) and pkg.encodec_stream_ready("encode", pushed, sample_rate=24000) == pkg.encodec_stream_ready("encode", pushed)
        assert np.array_equal(a.finish(), b.finish())
    codes = codec.compress(x)
    with codec.stream("decode") as a, codec.stream("decode", sample_rate=24000) as b:
        for t in range(codes.shape[1]):
            assert same_bits(a.push(codes[:, t:t + 1]), b.push(codes[:, t:t + 1]))
        assert a.finish().size == b.finish().size == 0


# ---- 3. batches -------------------------------------------------------------------------------------------------------------------
def test_32_streams_of_mixed_formats(pkg, codec):
    codec.bandwidth = 6
    fmts = [(48000, 2), (44100, 2), (24000, 1), (16000, 1), (22050, 8), (96000, 3), (8000, 1), (24000, 2)] * 4
    xs = [ro.clip("noise", int(sr * 0.4) + 37 * i, ch, seed=i) for i, (sr, ch) in enumerate(fmts)]
    streams = [codec.stream("encode") if (sr, ch) == (24000, 1) and i // 8 % 2 else codec.stream("encode", sample_rate=sr, channels=ch)
               for i, (sr, ch) in enumerate(fmts)]
    got = [[] for _ in fmts]
    pos = [0] * len(fmts)
    rng = np.random.default_rng(32)
    step = 0
    while any(p < x.shape[0] for p, x in zip(pos, xs)):
        ks = [min(int(rng.integers(0, 3000)), x.shape[0] - p) for p, x in zip(pos, xs)]
        chunks = [x[p:p + k] for x, p, k in zip(xs, pos, ks)]
        if step % 3 == 2:                                            # single pushes between the batches
            outs = [s.push(c) for s, c in zip(streams, chunks)]
        else:
            sel = list(range(len(fmts))) if step % 3 == 0 else list(range(step % 5, len(fmts), 3))
            outs = [np.zeros((8, 0), np.int32)] * len(fmts)
            for i, o in zip(sel, pkg.encodec_stream_push_batch([streams[i] for i in sel], [chunks[i] for i in sel])):
                outs[i] = o
            ks = [k if i in sel else 0 for i, k in enumerate(ks)]
        for i, (o, k) in enumerate(zip(outs, ks)):
            got[i].append(o)
            pos[i] += k
            sr, ch = fmts[i]
            assert sum(g.shape[1] for g in got[i]) == pkg.encodec_stream_ready("encode", pos[i], sample_rate=sr), (i, pos[i])
        step += 1
    for i, (s, x, (sr, ch)) in enumerate(zip(streams, xs, fmts)):
        got[i].append(s.finish())
        s.close()
        assert np.array_equal(np.concatenate(got[i], axis=1), codec.compress(planar(x), sample_rate=sr)), (i, sr, ch)
    # decode streams of three rates and plain ones in one batch
    codes = [np.random.default_rng(i).integers(0, 1024, (8, 40 + i)).astype(np.int32) for i in range(32)]
    drates = [(16000, 44100, 48000, None)[i % 4] for i in range(32)]
    ds = [codec.stream("decode") if r is None else codec.stream("decode", sample_rate=r) for r in drates]
    dout = [[] for _ in ds]
    for t in range(0, 72, 9):
        for i, o in enumerate(pkg.encodec_stream_push_batch(ds, [c[:, t:t + 9] for c in codes])):
            dout[i].append(o)
    for i, (s, c, r) in enumerate(zip(ds, codes, drates)):
        dout[i].append(s.finish())
        s.close()
        want = codec.decompress(c)
        assert same_bits(np.concatenate(dout[i]), want if r is None else pkg.resample(want, 24000, r)), (i, r)


# ---- 4. refusals ------------------------------------------------------------------------------------------------------------------
def test_refusals_leave_the_streams_unchanged(pkg, codec, capfd):
    L = pkg.lib()
    codec.bandwidth = 6
    for direction, ch, sr, what in ((0, 0, 48000, "0 channels"), (0, 9, 48000, "9 channels"), (0, 2, 3999, "sample rate 3999"),
                                    (1, 1, 384001, "sample rate 384001"), (1, 2, 48000, "channels 1"), (2, 1, 48000, "unknown direction")):
        assert not L.bark_b200_encodec_stream_open_resampled(codec.ctx, direction, ch, sr)
        assert what in capfd.readouterr().err, what
    assert not L.bark_b200_encodec_stream_open_resampled(None, 0, 1, 48000)
    x = ro.clip("noise", 3841, 2, seed=1)
    y = ro.clip("noise", 9000, 1, seed=2)
    with codec.stream("encode", sample_rate=48000, channels=2) as s, codec.stream("encode", sample_rate=44100) as t:
        assert s.push(x[:2000]).shape[1] == 0
        bad = [np.where(np.arange(200)[:, None] == 77, np.nan, 0.1).astype(np.float32) * np.ones((1, 2), np.float32),
               np.full((5, 2), 2.0 ** 65, np.float32), np.full((5, 2), np.inf, np.float32)]
        for b in bad:
            with pytest.raises(RuntimeError):
                s.push(b)
            with pytest.raises(RuntimeError):                          # a batch with one bad stream changes neither
                pkg.encodec_stream_push_batch([t, s], [y[:100], b])
            assert "not finite or exceeds 2^64" in capfd.readouterr().err
        # n * channels >= 2^31 is refused before a sample is read
        h = (C.c_void_p * 1)(s.handle.value)
        buf = np.zeros(16, np.float32)
        assert L.bark_b200_encodec_stream_push(s.handle, buf.ctypes.data, 1 << 30) == -1
        assert "2^31" in capfd.readouterr().err
        assert L.bark_b200_encodec_stream_push_batch(h, (C.c_void_p * 1)(buf.ctypes.data), (C.c_int * 1)(-1), 1) == -1
        capfd.readouterr()
        assert s.push(x[2000:3840]).shape[1] == 0
        with pytest.raises(RuntimeError):                              # 3840 frames at 48 kHz resample to 1920 samples
            s.finish()
        assert "1920 samples" in capfd.readouterr().err
        got = [s.push(x[3840:]), s.finish()]                           # 3841 to 1921
        assert np.array_equal(np.concatenate(got, axis=1), codec.compress(planar(x), sample_rate=48000))
        with pytest.raises(RuntimeError):
            s.push(x[:10])
        got = [t.push(y[:100]), t.push(y[100:]), t.finish()]
        assert np.array_equal(np.concatenate(got, axis=1), codec.compress(y, sample_rate=44100))
    with codec.stream("decode", sample_rate=44100) as d:
        codes = np.random.default_rng(1).integers(0, 1024, (8, 7)).astype(np.int32)
        assert d.push(codes[:, :6]).size == 0
        with pytest.raises(RuntimeError):
            d.finish()
        bad = codes.copy()
        bad[3, 0] = 1024
        with pytest.raises(RuntimeError):
            d.push(bad[:, :1])
        capfd.readouterr()
        got = [d.push(codes[:, 6:]), d.finish()]
        assert same_bits(np.concatenate(got), pkg.resample(codec.decompress(codes), 24000, 44100))
    with codec.stream("encode", sample_rate=48000, channels=2) as s:
        with pytest.raises(ValueError):
            s.push(np.zeros((10, 3), np.float32))


# ---- 5. a long stream -------------------------------------------------------------------------------------------------------------
def test_ten_minutes_of_44k1_stereo_in_20ms_chunks(pkg, codec):
    codec.bandwidth = 6
    n = 600 * 44100
    x = np.random.Generator(np.random.PCG64(600)).uniform(-1, 1, (n, 2)).astype(np.float32)
    got, frames = [], 0
    with codec.stream("encode", sample_rate=44100, channels=2) as s:
        for i in range(0, n, 882):
            c = s.push(x[i:i + 882])
            frames += c.shape[1]
            got.append(c)
        assert frames == pkg.encodec_stream_ready("encode", n, sample_rate=44100)
        got.append(s.finish())
    assert np.array_equal(np.concatenate(got, axis=1), codec.compress(planar(x), sample_rate=44100))


# ---- 6. the window hook -----------------------------------------------------------------------------------------------------------
def window(x, sr, nsr, first, n_out, at_end):
    """the window item of outputs first .. first + n_out - 1 of x's resampling: the frames their blocks read over the full support,
    and the signal's end where the window reaches it"""
    o, q, w = rates(sr, nsr)
    n = x.shape[0]
    lo = max(0, first // q * o - w)
    hi = (first + n_out - 1) // q * o + o + w - 1
    it = dict(sr=sr, new_sr=nsr, org=lo, first=first, n_out=n_out, frames=x[lo:min(hi, n - 1) + 1])
    if at_end:
        it["end"] = n
    else:
        assert hi < n
    return it


def test_window_hook_equals_slices_of_resample(pkg):
    cases = [(48000, 24000, 2), (44100, 24000, 1), (24000, 48000, 1), (383999, 24000, 3), (16000, 24000, 8), (24000, 24000, 2), (4000, 384000, 1)]
    items, want = [], []
    for i, (sr, nsr, ch) in enumerate(cases):
        n = max(sr // 3, 2 * rates(sr, nsr)[0] + 100)
        x = ro.clip("noise", n, ch, seed=i)
        y = pkg.resample(planar(x), sr, nsr)
        L = y.size
        o, q, w = rates(sr, nsr)
        mid = L // 2 - (L // 2) % q
        last_safe = ((n - o - w) // o) * q                           # outputs from here on read past the last frame
        for first, n_out, at_end in ((0, min(300, last_safe), False), (mid, min(777, last_safe - mid), False), (L - 500, 500, True),
                                     (0, L, True), (3, q + 5, False)):
            if n_out < 1 or (not at_end and first + n_out > last_safe):
                continue
            items.append(window(x, sr, nsr, first, n_out, at_end))
            want.append(y[first:first + n_out])
    for k in range(0, len(items), 32):                                 # every item of a launch its own format
        got = pkg.resample_window(items[k:k + 32])
        for g, wv, it in zip(got, want[k:k + 32], items[k:k + 32]):
            assert same_bits(g, wv), (it["sr"], it["new_sr"], it["first"], it["n_out"])
    # each item alone too, and a window one frame short is refused
    for it, wv in zip(items[::5], want[::5]):
        assert same_bits(pkg.resample_window([it])[0], wv)
    it = dict(items[1])
    it["frames"] = it["frames"][:-1]
    with pytest.raises(RuntimeError):
        pkg.resample_window([it])
