"""Streaming EnCodec on the GPU (bark_b200_encodec_stream_*, Encodec.stream): everything a stream returns, joined, equals the whole-clip
call on everything it was pushed, bit for bit, whatever the chunks, the other streams of a batch and the other calls on the context; outputs
come back exactly when the readiness rule (DESIGN.md §19) says they are final.  The window and state hooks equal slices of the whole-signal
kernels."""
import ctypes as C
import os
import threading

import numpy as np
import pytest

from conftest import GOLDEN_DIR
import encoder_oracle as eo
from encodec_oracle import codec_offset

pytestmark = pytest.mark.gpu
GOLD = os.path.join(GOLDEN_DIR, "ref_pairs", "encodec_bandwidths.npz")
N_Q = {1: 1, 6: 8, 24: 32}                 # kbps -> codebooks (1 kbps: one codebook, as 1.5 kbps gives upstream)
LENGTHS = (1921, 2239, 2240, 2241, 24000, 24001, 240000)
SCHEDULES = ("one", "319", "320", "321", "ones", "random")


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
def second(pkg, weights_file, weights_mod):
    path = eo.weights_path(weights_file, weights_mod, "base")
    e = pkg.Encodec(path, codec_offset(path))
    yield e
    e.close()


def clip(n, seed=0):
    return eo.signal(("noise", "sine", "square")[seed % 3], n, seed=1000 + seed)


def sizes(schedule, n, seed=0):
    """Chunk sizes summing to n."""
    if schedule == "one":
        return [n]
    if schedule == "ones":
        return [1] * n
    if schedule == "random":
        rng = np.random.default_rng(seed)
        out = []
        while sum(out) < n:
            k = int(rng.choice([0, 1, int(rng.integers(2, 700)), int(rng.integers(700, 4000))]))
            out.append(min(k, n - sum(out)))
        return out[:1] + [0] + out[1:]
    k = int(schedule)
    return [k] * (n // k) + ([n % k] if n % k else [])


def ready(pkg, direction, n):
    return pkg.encodec_stream_ready(direction, n)


def encode_stream(pkg, e, x, chunks):
    """Codes of x through an encode stream pushed in the given chunk sizes; checks the frames after every push against the rule."""
    with e.stream("encode") as s:
        got, pushed, frames = [], 0, 0
        for k in chunks:
            c = s.push(x[pushed:pushed + k])
            pushed += k
            frames += c.shape[1]
            assert c.shape[0] == s.n_q and frames == ready(pkg, "encode", pushed), (pushed, frames)
            got.append(c)
        got.append(s.finish())
    return np.concatenate(got, axis=1)


def decode_stream(pkg, e, codes, chunks):
    with e.stream("decode") as s:
        got, pushed, samples = [], 0, 0
        for k in chunks:
            a = s.push(codes[:, pushed:pushed + k])
            pushed += k
            samples += a.size
            assert samples == ready(pkg, "decode", pushed), (pushed, samples)
            got.append(a)
        tail = s.finish()
        assert tail.size == 0
    return np.concatenate(got)


def same_bits(a, b):
    return a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))


# ---- 1. encode equality ---------------------------------------------------------------------------------------------------------
_whole = {}


def whole(e, bw, n, seed=0):
    key = (id(e), bw, n, seed)
    if key not in _whole:
        e.bandwidth = bw
        _whole[key] = e.compress(clip(n, seed))
    return _whole[key]


@pytest.mark.parametrize("bw", sorted(N_Q))
@pytest.mark.parametrize("n", LENGTHS)
@pytest.mark.parametrize("schedule", SCHEDULES)
def test_encode_equals_compress(pkg, codecs, bw, n, schedule):
    if schedule == "ones" and (n > 2241 or bw != 24):
        pytest.skip("one sample per push: the short clips at 24 kbps")
    e = codecs["base"]
    want = whole(e, bw, n)
    e.bandwidth = bw
    got = encode_stream(pkg, e, clip(n), sizes(schedule, n, seed=n + bw))
    assert got.shape == want.shape == (N_Q[bw], (n + 319) // 320) and np.array_equal(got, want), f"{int((got != want).sum()) if got.shape == want.shape else got.shape} codes differ"


def test_encode_equals_stored_reference(pkg, codecs):
    gold = np.load(GOLD)
    for name, kind, n, which in eo.CASES:
        x = eo.signal(kind, n, seed=n)
        e = codecs[which]
        for bw in (1, 2, 3, 12, 24):
            e.bandwidth = bw
            ref = gold[f"{name}_bw{bw}_codes"]
            got = encode_stream(pkg, e, x, sizes("321", n))
            assert got.shape == ref.shape and np.array_equal(got, ref), f"{name} at {bw} kbps"


# ---- 2. readiness ---------------------------------------------------------------------------------------------------------------
def test_ready_rule(pkg):
    for n in list(range(0, 3000)) + [10 ** 6 + 7, 2 ** 40 + 1]:
        assert ready(pkg, "encode", n) == (n // 320 if n >= 2240 else 0), n
    for t in list(range(0, 40)) + [2 ** 40]:
        assert ready(pkg, "decode", t) == (320 * t if t >= 7 else 0), t
    assert pkg.lib().bark_b200_encodec_stream_ready(2, 5) == -1 and pkg.lib().bark_b200_encodec_stream_ready(0, -1) == -1


def test_ready_frames_do_not_depend_on_later_samples(pkg, codecs):
    """For random n, two clips that share their first n samples agree on the first ready(n) frames of the whole-clip compress, and the
    next frame is not final: some continuation changes it."""
    e = codecs["base"]
    e.bandwidth = 24
    rng = np.random.default_rng(11)
    changed = 0
    for trial in range(12):
        n = int(rng.integers(2240, 40000)) if trial else 2240
        head = clip(n, trial)
        a = e.compress(np.concatenate([head, clip(3000, 50 + trial)]))
        b = e.compress(np.concatenate([head, np.float32(3) * clip(3000, 80 + trial)]))
        r = ready(pkg, "encode", n)
        assert np.array_equal(a[:, :r], b[:, :r]), n
        changed += not np.array_equal(a[:, r], b[:, r])
    assert changed >= 10, f"the frame after the ready ones was final in {12 - changed} of 12 trials"


# ---- 3. decode equality ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("T", (7, 8, 150, 750))
@pytest.mark.parametrize("schedule", ("ones", "seven_then_ones", "random"))
def test_decode_equals_decompress(pkg, codecs, T, schedule):
    e = codecs["base"]
    rng = np.random.default_rng(T)
    for bw in (6, 24):
        e.bandwidth = bw
        codes = rng.integers(0, 1024, (N_Q[bw], T)).astype(np.int32)
        chunks = {"ones": [1] * T, "seven_then_ones": [7] + [1] * (T - 7), "random": sizes("random", T, seed=T)}[schedule]
        got = decode_stream(pkg, e, codes, chunks)
        assert same_bits(got, e.decompress(codes)), f"{bw} kbps"


def test_decode_finish_refuses_short(pkg, codecs, capfd):
    e = codecs["base"]
    e.bandwidth = 6
    codes = np.random.default_rng(3).integers(0, 1024, (8, 7)).astype(np.int32)
    with e.stream("decode") as s:
        assert s.push(codes[:, :6]).size == 0
        with pytest.raises(RuntimeError):
            s.finish()
        assert "need at least 7 frames" in capfd.readouterr().err
        got = s.push(codes[:, 6:])
        assert s.finish().size == 0
    assert same_bits(got, e.decompress(codes))


def test_encode_finish_refuses_short(pkg, codecs, capfd):
    e = codecs["base"]
    e.bandwidth = 6
    x = clip(1921)
    with e.stream("encode") as s:
        assert s.push(x[:1920]).shape == (8, 0)
        with pytest.raises(RuntimeError):
            s.finish()
        assert "need at least 1921 samples" in capfd.readouterr().err
        assert s.push(x[1920:]).shape == (8, 0)
        got = s.finish()
    assert np.array_equal(got, e.compress(x))


def test_first_frames_on_a_fresh_context(pkg, weights_file, weights_mod):
    """The k = 7 convolutions release 7 frames at once when a stream reaches them, more than a small push brings in: on a context whose
    scratch no whole-clip call has grown, a batch of streams at 32 codebooks still equals the whole clips."""
    path = eo.weights_path(weights_file, weights_mod, "base")
    with pkg.Encodec(path, codec_offset(path)) as e:
        e.bandwidth = 24
        xs = [clip(2600, i) for i in range(32)]
        enc = [e.stream("encode") for _ in xs]
        dec = [e.stream("decode") for _ in xs]
        got, wav = [[] for _ in xs], [[] for _ in xs]
        for p in range(0, 2600, 320):
            for i, (c, s) in enumerate(zip(pkg.encodec_stream_push_batch(enc, [x[p:p + 320] for x in xs]), dec)):
                got[i].append(c)
            for i, a in enumerate(pkg.encodec_stream_push_batch(dec, [c[-1] for c in got])):
                wav[i].append(a)
        for i, s in enumerate(enc):
            got[i].append(s.finish())
            wav[i].append(dec[i].push(got[i][-1]))
            wav[i].append(dec[i].finish())
            s.close(); dec[i].close()
        for i, x in enumerate(xs):
            want = e.compress(x)
            assert np.array_equal(np.concatenate(got[i], axis=1), want), i
            assert same_bits(np.concatenate(wav[i]), e.decompress(want)), i


# ---- 4. round trip --------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bw", (6, 24))
def test_round_trip_equals_reconstruct(pkg, codecs, bw):
    e = codecs["base"]
    e.bandwidth = bw
    x = clip(24001, 2)
    out = []
    with e.stream("encode") as enc, e.stream("decode") as dec:
        for i in range(0, x.size, 320):
            out.append(dec.push(enc.push(x[i:i + 320])))
        out.append(dec.push(enc.finish()))
        out.append(dec.finish())
    assert same_bits(np.concatenate(out), e.reconstruct(x))


# ---- 5. batches -----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("count", (1, 2, 5, 32))
def test_encode_batches_equal_single_streams(pkg, codecs, count):
    e = codecs["base"]
    e.bandwidth = 6
    rng = np.random.default_rng(count)
    xs = [clip(int(rng.integers(1921, 30000)), i) for i in range(count)]
    streams = [e.stream("encode") for _ in range(count)]
    got, pos = [[] for _ in range(count)], [0] * count
    for rnd in range(40):
        k = [int(rng.choice([0, 1, 319, 320, int(rng.integers(0, 3000))])) for _ in range(count)]
        k = [min(a, x.size - p) for a, x, p in zip(k, xs, pos)]
        if rnd % 3 == 2:                                  # streams moving between batches and single pushes
            for i in range(count):
                got[i].append(streams[i].push(xs[i][pos[i]:pos[i] + k[i]]))
        else:
            order = rng.permutation(count)
            outs = pkg.encodec_stream_push_batch([streams[i] for i in order], [xs[i][pos[i]:pos[i] + k[i]] for i in order])
            for i, o in zip(order, outs):
                got[i].append(o)
        pos = [p + a for p, a in zip(pos, k)]
    for i in range(count):
        got[i].append(streams[i].push(xs[i][pos[i]:]))
        got[i].append(streams[i].finish())
        streams[i].close()
        c = np.concatenate(got[i], axis=1)
        assert np.array_equal(c, e.compress(xs[i])), f"stream {i}"


@pytest.mark.parametrize("count", (3, 32))
def test_decode_batches_equal_single_streams(pkg, codecs, count):
    e = codecs["base"]
    e.bandwidth = 24
    rng = np.random.default_rng(100 + count)
    cs = [rng.integers(0, 1024, (32, int(rng.integers(7, 60)))).astype(np.int32) for _ in range(count)]
    streams = [e.stream("decode") for _ in range(count)]
    got, pos = [[] for _ in range(count)], [0] * count
    for rnd in range(12):
        k = [min(int(rng.integers(0, 9)), c.shape[1] - p) for c, p in zip(cs, pos)]
        outs = pkg.encodec_stream_push_batch(streams, [c[:, p:p + a] for c, p, a in zip(cs, pos, k)])
        for i, o in enumerate(outs):
            got[i].append(o)
        pos = [p + a for p, a in zip(pos, k)]
    outs = pkg.encodec_stream_push_batch(streams, [c[:, p:] for c, p in zip(cs, pos)])
    for i in range(count):
        got[i].append(outs[i])
        got[i].append(streams[i].finish())
        streams[i].close()
        assert same_bits(np.concatenate(got[i]), e.decompress(cs[i])), f"stream {i}"


# ---- 6. isolation ---------------------------------------------------------------------------------------------------------------
def codes_of(pkg, e):
    n = pkg.lib().encodec_get_codes_size(e.ctx)
    return np.ctypeslib.as_array(pkg.lib().encodec_get_codes(e.ctx), shape=(n,)).copy() if n else np.zeros(0, np.int32)


def test_other_calls_between_pushes(pkg, codecs):
    e = codecs["base"]
    e.bandwidth = 6
    x, y = clip(50000, 4), clip(30000, 5)
    want_x, want_y, codes_y = e.compress(x), e.compress(y), None
    wave = e.decompress(want_y)
    codes_y = codes_of(pkg, e)
    e.compress(y)
    codes_y = codes_of(pkg, e)
    stats = e.stats()
    a, b = e.stream("encode"), e.stream("encode")
    dec = e.stream("decode")
    got_a, got_b, got_d = [], [], []
    for i, p in enumerate(range(0, 50000, 1234)):
        got_a.append(a.push(x[p:p + 1234]))
        if p < 30000:
            got_b.append(b.push(y[p:p + 1234]))
        got_d.append(dec.push(want_y[:, 3 * i:3 * i + 3]))
        assert codes_of(pkg, e).tobytes() == codes_y.tobytes() and e.stats() == stats
        if i % 10 == 3:                                   # whole-clip, batch and resampled calls on the same context
            assert np.array_equal(e.compress(y), want_y)
            e.compress_batch([x[:5000], y[:7000]])
            e.compress(np.stack([x[:9000], y[:9000]]), sample_rate=48000)
            e.decompress_batch([want_x[:, :9]])
            codes_y = codes_of(pkg, e)
            stats = e.stats()
    got_a.append(a.finish()); got_b.append(b.push(np.zeros(0, np.float32))); got_b.append(b.finish())
    got_d.append(dec.push(want_y[:, 3 * (i + 1):])); got_d.append(dec.finish())
    for s in (a, b, dec):
        s.close()
    assert np.array_equal(np.concatenate(got_a, axis=1), want_x)
    assert np.array_equal(np.concatenate(got_b, axis=1), want_y)
    assert same_bits(np.concatenate(got_d), wave)
    assert same_bits(e.decompress(want_y), wave)


def test_bandwidth_fixed_at_open(pkg, codecs):
    e = codecs["base"]
    e.bandwidth = 6
    x = clip(24000, 6)
    want = e.compress(x)
    with e.stream("encode") as s, e.stream("decode") as d:
        out, wav = [s.push(x[:10000])], [d.push(want[:, :20])]
        e.bandwidth = 24
        out += [s.push(x[10000:]), s.finish()]
        wav += [d.push(want[:, 20:]), d.finish()]
        assert s.n_q == 8
    assert np.array_equal(np.concatenate(out, axis=1), want)
    e.bandwidth = 6
    assert same_bits(np.concatenate(wav), e.decompress(want))


def test_two_contexts_on_two_threads(pkg, codecs, second):
    xs = [clip(40000, 7), clip(40000, 8)]
    results, errors = [None, None], []

    def run(i, e):
        try:
            results[i] = encode_stream(pkg, e, xs[i], sizes("random", xs[i].size, seed=i))
        except Exception as exc:                          # reported below
            errors.append(exc)

    codecs["base"].bandwidth = second.bandwidth = 24
    th = [threading.Thread(target=run, args=(i, e)) for i, e in enumerate((codecs["base"], second))]
    for t in th:
        t.start()
    for t in th:
        t.join()
    assert not errors, errors
    for i in range(2):
        assert np.array_equal(results[i], codecs["base"].compress(xs[i])), i


# ---- 7. refusals ----------------------------------------------------------------------------------------------------------------
def test_refusals_leave_streams_unchanged(pkg, codecs, second, capfd):
    L = pkg.lib()
    e = codecs["base"]
    e.bandwidth = 6
    x = clip(30000, 9)
    codes = e.compress(x)
    enc, dec = e.stream("encode"), e.stream("decode")
    out, wav = [enc.push(x[:5000])], [dec.push(codes[:, :10])]

    def refused(call, text):
        assert call() == -1
        assert text in capfd.readouterr().err

    bad = x[5000:6000].copy(); bad[17] = np.nan
    refused(lambda: L.bark_b200_encodec_stream_push(enc.handle, bad.ctypes.data, bad.size), "not finite")
    bad[17] = np.inf
    refused(lambda: L.bark_b200_encodec_stream_push(enc.handle, bad.ctypes.data, bad.size), "not finite")
    for v in (-1, 1024):
        c = np.ascontiguousarray(codes[:, 10:14]); c[3, 2] = v
        refused(lambda: L.bark_b200_encodec_stream_push(dec.handle, c.ctypes.data, 4), "outside the codebooks")
    refused(lambda: L.bark_b200_encodec_stream_push(enc.handle, None, 5), "null input")
    refused(lambda: L.bark_b200_encodec_stream_push(enc.handle, x.ctypes.data, -1), "negative count")
    refused(lambda: L.bark_b200_encodec_stream_push(None, x.ctypes.data, 1), "null stream")
    refused(lambda: L.bark_b200_encodec_stream_push_batch(None, None, None, 1), "null")
    refused(lambda: L.bark_b200_encodec_stream_finish(None), "null stream")
    assert L.bark_b200_encodec_stream_open(None, 0) is None and "null context" in capfd.readouterr().err
    assert L.bark_b200_encodec_stream_open(e.ctx, 2) is None and "unknown direction" in capfd.readouterr().err
    assert L.bark_b200_encodec_stream_read(None, None, 0) == -1

    def batch(streams, chunks, count=None):
        hs = (C.c_void_p * len(streams))(*[s.handle.value for s in streams])
        ps = (C.c_void_p * len(streams))(*[c.ctypes.data for c in chunks])
        ns = (C.c_int * len(streams))(*[c.size if s.direction == "encode" else c.shape[1] for s, c in zip(streams, chunks)])
        return L.bark_b200_encodec_stream_push_batch(hs, ps, ns, len(streams) if count is None else count)

    other = second.stream("encode")
    refused(lambda: batch([enc, other], [x[5000:5100], x[:10]]), "another context or direction")
    refused(lambda: batch([enc, dec], [x[5000:5100], np.ascontiguousarray(codes[:, 10:11])]), "another context or direction")
    refused(lambda: batch([enc, enc], [x[5000:5100], x[5100:5200]]), "stream 1 is stream 0 again")
    many = [e.stream("encode") for _ in range(33)]
    refused(lambda: batch([enc] + many[:32], [x[5000:5100]] * 33), "33 streams")
    refused(lambda: batch([enc], [x[5000:5100]], count=0), "0 streams")
    for s in many:
        s.close()
    other.close()
    done = e.stream("encode")
    done.push(x[:2000]); done.finish()
    refused(lambda: L.bark_b200_encodec_stream_push(done.handle, x.ctypes.data, 10), "finished")
    refused(lambda: L.bark_b200_encodec_stream_finish(done.handle), "finished")
    done.close()
    out += [enc.push(x[5000:]), enc.finish()]
    wav += [dec.push(codes[:, 10:]), dec.finish()]
    enc.close(); dec.close()
    assert np.array_equal(np.concatenate(out, axis=1), codes)
    assert same_bits(np.concatenate(wav), e.decompress(codes))


# ---- 8. long streams ------------------------------------------------------------------------------------------------------------
def test_ten_minutes_in_one_second_chunks(pkg, codecs):
    e = codecs["base"]
    e.bandwidth = 6
    x = clip(600 * 24000, 10)
    want = e.compress(x)
    got = encode_stream(pkg, e, x, [24000] * 600)
    assert np.array_equal(got, want)
    wav = decode_stream(pkg, e, want, [75] * 600)
    assert same_bits(wav, e.decompress(want))


# ---- 9. kernel hooks ------------------------------------------------------------------------------------------------------------
def rand_conv(rng, cout, cin, k):
    return (rng.standard_normal((cout, cin, k)) * (1.0 / np.sqrt(cin * k))).astype(np.float16), rng.standard_normal(cout).astype(np.float32) * 0.1


# (Cin, Cout, k, stride): the short, lane and stream kernels at stride 1 and every strided instantiation
CONVS = [(1, 32, 7, 1), (32, 16, 3, 1), (64, 64, 7, 1), (512, 128, 7, 1), (32, 64, 4, 2), (64, 128, 8, 4), (128, 256, 10, 5), (256, 512, 16, 8)]


@pytest.mark.parametrize("cin,cout,k,stride", CONVS, ids=[f"cin{c[0]}_k{c[2]}_s{c[3]}" for c in CONVS])
def test_conv_window_hook(pkg, cin, cout, k, stride):
    rng = np.random.default_rng(cin * k + stride)
    w, b = rand_conv(rng, cout, cin, k)
    xs = [rng.standard_normal((cin, L)).astype(np.float32) for L in (300, 97, 1001)]
    whole = pkg.codec_conv1d(xs, w, b, stride=stride, elu_in=True)
    for firsts in ([0, 0, 0], [1, 5, 37], [3, 11, 120]):
        org, wins, n_out = [], [], []
        for x, y, f in zip(xs, whole, firsts):
            o = max(0, f * stride - (k - stride))         # the columns a stream keeps for output f on
            org.append(o); wins.append(x[:, o:]); n_out.append(y.shape[1] - f)
        got = pkg.codec_conv1d_window(wins, org, firsts, n_out, w, b, stride=stride, elu_in=True)
        for i, (g, y, f) in enumerate(zip(got, whole, firsts)):
            assert same_bits(g, np.ascontiguousarray(y[:, f:])), (firsts, i)
    # a window that does not hold the columns its outputs read is refused
    with pytest.raises(RuntimeError):
        pkg.codec_conv1d_window([xs[0][:, 20:]], [20], [20 // stride], [3], w, b, stride=stride)


@pytest.mark.parametrize("cin,stride", ((512, 8), (256, 5), (128, 4), (64, 2)))
def test_convtr_window_hook(pkg, cin, stride):
    rng = np.random.default_rng(cin)
    w = (rng.standard_normal((cin, cin // 2, 2 * stride)) / np.sqrt(cin)).astype(np.float16)
    b = rng.standard_normal(cin // 2).astype(np.float32) * 0.1
    xs = [rng.standard_normal((cin, T)).astype(np.float32) for T in (40, 7, 100)]
    whole = pkg.codec_convtr1d(xs, w, b, stride)
    for firsts in ([0, 0, 0], [1, 6, 50], [39, 3, 99]):
        org = [max(0, f - 1) for f in firsts]
        got = pkg.codec_convtr1d_window([x[:, o:] for x, o in zip(xs, org)], org, firsts, [x.shape[1] - f for x, f in zip(xs, firsts)], w, b, stride)
        for i, (g, y, f) in enumerate(zip(got, whole, firsts)):
            assert same_bits(g, np.ascontiguousarray(y[:, f * stride:])), (firsts, i)


@pytest.mark.parametrize("items", (1, 3))
def test_lstm_state_hook(pkg, items):
    rng = np.random.default_rng(items)
    C_ = 512
    wih, whh = [(rng.standard_normal((4 * C_, C_)) / np.sqrt(C_)).astype(np.float16) for _ in range(2)]
    bih, bhh = [rng.standard_normal(4 * C_).astype(np.float32) * 0.1 for _ in range(2)]
    xs = [rng.standard_normal((C_, T)).astype(np.float32) for T in (60, 1, 33)[:items]]
    skip = [rng.standard_normal(x.shape).astype(np.float32) for x in xs]
    whole = pkg.codec_lstm(xs, wih, whh, bih, bhh, skip=skip)
    for cut in (1, 17, 32):
        cuts = [min(cut, x.shape[1] - 1) if x.shape[1] > 1 else 0 for x in xs]
        live = [i for i, c in enumerate(cuts) if c > 0]
        state = np.zeros((items, 2, C_), np.float32)
        head, st = pkg.codec_lstm_state([xs[i][:, :cuts[i]] for i in live], wih, whh, bih, bhh, skip=[skip[i][:, :cuts[i]] for i in live])
        state[live] = st
        tail, st2 = pkg.codec_lstm_state([x[:, c:] for x, c in zip(xs, cuts)], wih, whh, bih, bhh, state=state, skip=[s[:, c:] for s, c in zip(skip, cuts)])
        for i in range(items):
            parts = ([head[live.index(i)]] if i in live else []) + [tail[i]]
            assert same_bits(np.ascontiguousarray(np.concatenate(parts, axis=1)), whole[i]), (cut, i)
        _, st_whole = pkg.codec_lstm_state(xs, wih, whh, bih, bhh, skip=skip)
        assert same_bits(st2, st_whole)
