"""encodec.cpp's C API on the GPU (include/encodec.h, bark_cpp_b200.Encodec) against the unmodified reference's stored outputs at
1 to 32 codebooks (tests/golden/ref_pairs/encodec_bandwidths.npz), the CPU restatement (tests/encodec_oracle.py) and the bark context's
6 kbps codec: bit for bit."""
import os
import subprocess
import threading
import wave

import numpy as np
import pytest

from conftest import GOLDEN_DIR, ROOT, assert_pinned
import encodec_oracle as co
import encoder_oracle as eo
from encodec_oracle import codec_offset

pytestmark = pytest.mark.gpu
GOLD = os.path.join(GOLDEN_DIR, "ref_pairs", "encodec_bandwidths.npz")
N_Q = {1: 1, 2: 2, 3: 4, 12: 16, 24: 32}


@pytest.fixture(scope="module")
def gold():
    return np.load(GOLD)


@pytest.fixture(scope="module")
def codecs(pkg, weights_file, weights_mod):
    out = {}
    for w in eo.WEIGHTS:
        path = eo.weights_path(weights_file, weights_mod, w)
        out[w] = pkg.Encodec(path, codec_offset(path))
    yield out
    for e in out.values():
        e.close()


@pytest.mark.parametrize("name,kind,n,which", eo.CASES, ids=[c[0] for c in eo.CASES])
def test_compress_equals_the_reference_at_every_bandwidth(codecs, gold, name, kind, n, which):
    e = codecs[which]
    x = eo.signal(kind, n, seed=n)
    for bw, n_q in N_Q.items():
        e.bandwidth = bw
        codes, ref = e.compress(x), gold[f"{name}_bw{bw}_codes"]
        assert codes.shape == ref.shape == (n_q, (n + 319) // 320)
        assert np.array_equal(codes, ref), f"{name} at {bw} kbps: {int((codes != ref).sum())} codes differ"
    e.bandwidth = 24


@pytest.mark.parametrize("name", eo.RECONSTRUCT)
def test_reconstruct_equals_the_reference_and_decompress_of_compress(codecs, gold, name):
    _, kind, n, which = next(c for c in eo.CASES if c[0] == name)
    e = codecs[which]
    x = eo.signal(kind, n, seed=n)
    for bw in (3, 12, 24):
        e.bandwidth = bw
        audio = e.reconstruct(x)
        assert_pinned(audio, gold, f"{name}_bw{bw}_audio", f"{name} reconstruction at {bw} kbps")
        assert np.array_equal(audio.view(np.uint32), e.decompress(e.compress(x)).view(np.uint32))
    e.bandwidth = 24


def test_decompress_equals_the_reference(codecs, gold):
    import make_golden_encodec as mg
    e = codecs["base"]
    for bw, n_q in zip(mg.DECOMPRESS_BW, (16, 32)):
        e.bandwidth = bw
        assert_pinned(e.decompress(mg.decompress_codes(bw, n_q)), gold, f"decompress_bw{bw}_audio", f"decompress at {bw} kbps")
    e.bandwidth = 24


def test_6_kbps_equals_the_bark_context(pkg, codecs, weights_file):
    e = codecs["base"]
    with pkg.Bark(weights_file("tiny", "f16", 1234), seed=0, n_steps_text_encoder=12) as b:
        for i, n in enumerate((1921, 24001, 100003)):
            x = eo.signal(("noise", "sine", "square")[i], n, seed=40 + i)
            e.bandwidth = 6
            codes = e.compress(x)
            assert np.array_equal(codes, b.encodec_encode(x))
            assert np.array_equal(e.decompress(codes).view(np.uint32), b.encodec_decode(codes).view(np.uint32))
            e.bandwidth = 24
            assert np.array_equal(e.compress(x)[:8], codes)        # residual quantisation: 6 kbps is the first 8 rows of 24 kbps


def test_codes_equal_the_oracle_on_a_length_sweep(codecs, weights_file, weights_mod):
    path = eo.weights_path(weights_file, weights_mod, "base")
    oracle = co.CodecOracle(path, codec_offset(path))
    e = codecs["base"]
    e.bandwidth = 24
    for i, n in enumerate((1921, 2241, 5119, 33333, 240000, 720000)):
        x = eo.signal(("noise", "sine", "square")[i % 3], n, seed=200 + i)
        codes = e.compress(x)
        want = oracle.encode(x, 32)
        assert np.array_equal(codes, want), f"n={n}: {int((codes != want).sum())} codes differ; first at {np.argwhere(codes != want)[:1].tolist()}"


# ---- the RVQ encode kernel at 9..32 codebooks ------------------------------------------------------------------------------------
def _check_rvq(pkg, lat, cb):
    got, want = pkg.rvq_encode(lat, cb), eo.rvq_encode(lat, cb)
    assert np.array_equal(got, want), f"{int((got != want).sum())} codes differ; first at {np.argwhere(got != want)[:1].tolist()}"
    return got


def _case(rng, n_q, T, hidden=128, n_bins=1024):
    return rng.standard_normal((hidden, T), dtype=np.float32) * np.float32(2), rng.standard_normal((n_q, n_bins, hidden), dtype=np.float32)


@pytest.mark.parametrize("n_q", [9, 16, 23, 32])
def test_rvq_encode_random_rows(pkg, n_q):
    for T in (1, 9, 300):
        _check_rvq(pkg, *_case(np.random.default_rng(n_q * 100 + T), n_q, T))


def test_rvq_encode_edge_rows_at_32_codebooks(pkg):
    rng = np.random.default_rng(21)
    lat, cb = _case(rng, 32, 40)
    cb[9, -1] = cb[9, 0]; cb[20, 700] = cb[20, 0]; cb[31, 1023] = cb[31, 5]      # exact ties across slices
    lat[:, 0] = cb[0, 0]; lat[:, 1] = cb[0, 17]                                  # residuals equal to a codeword
    lat[:, 2] = 0.0; lat[:, 3] = -0.0; lat[:, 4] = np.float32(1e-41) * rng.choice([-1, 1], 128)
    cb[12, 3] = 0.0; cb[13, 9] = -0.0; cb[14, :10] = np.float32(3e-42)
    lat[:, 5] = np.float32(3e19); lat[:, 6] = np.float32(-2e19) * rng.choice([-1, 1], 128)
    cb[10, 10] = np.float32(3e19); cb[10, 20] = np.float32(-3e19)
    _check_rvq(pkg, lat, cb)
    for hidden, n_bins in ((32, 1), (32, 5), (64, 33), (96, 1000)):
        _check_rvq(pkg, *_case(rng, 12, 17, hidden, n_bins))


@pytest.mark.parametrize("where", [0, 63, 64, 127, 128, 511, 512, 1023])
def test_rvq_encode_nan_at_slice_boundaries(pkg, where):
    rng = np.random.default_rng(30 + where)
    lat, cb = _case(rng, 12, 9)
    cb[0, where, 5] = np.nan
    cb[9, where, 0] = np.nan
    cb[11, (where + 128) % 1024, 1] = np.nan
    lat[:, 4] = np.nan
    _check_rvq(pkg, lat, cb)


# ---- loading, the n_q rule, refusals, threads, coexistence ---------------------------------------------------------------------
def test_standalone_codec_file_equals_the_bark_file_section(pkg, codecs, weights_file, tmp_path):
    path = weights_file("tiny", "f16", 1234)
    off = codec_offset(path)
    solo = tmp_path / "encodec.bin"
    solo.write_bytes(open(path, "rb").read()[off:])
    x = eo.signal("noise", 24001, seed=3)
    with pkg.Encodec(str(solo)) as e:
        assert np.array_equal(e.compress(x), codecs["base"].compress(x))
        assert np.array_equal(e.reconstruct(x).view(np.uint32), codecs["base"].reconstruct(x).view(np.uint32))


def test_bandwidth_and_sample_rate_rule(pkg, codecs):
    e = codecs["base"]
    x = eo.signal("noise", 4000, seed=1)
    for sr in (24000, 16000, 32000, 44100, 48000):
        e.sample_rate = sr
        for bw in (-3, 0, 1, 2, 3, 4, 6, 8, 12, 16, 24, 25, 40):
            e.bandwidth = bw
            n_q = co.n_q_for(bw, sr)
            if n_q > 32:
                with pytest.raises(RuntimeError):
                    e.compress(x)
                continue
            codes = e.compress(x)
            assert codes.shape == (n_q, 13), (sr, bw)
            assert e.decompress(codes).size == 320 * 13
    e.sample_rate, e.bandwidth = 24000, 24


def test_refusals_leave_the_context_usable(pkg, codecs, weights_file, weights_mod, tmp_path):
    L, e = pkg.lib(), codecs["base"]
    x = eo.signal("noise", 4000, seed=2)
    e.bandwidth = 12
    good_codes, good_audio = e.compress(x), e.reconstruct(x)
    bad_calls = [
        lambda: e.decompress(good_codes.ravel()[:-1]),                            # n_codes % n_q != 0
        lambda: e.decompress(np.where(np.arange(good_codes.size) == 7, 1024, good_codes.ravel())),
        lambda: e.decompress(np.full(16 * 13, -1, np.int32)),
        lambda: e.decompress(good_codes[:, :6]),                                  # fewer than 7 frames
        lambda: e.compress(np.zeros(1920, np.float32)), lambda: e.reconstruct(np.zeros(1920, np.float32)),
        lambda: e.compress(np.where(np.arange(4000) == 9, np.nan, 0.1).astype(np.float32)),
        lambda: e.reconstruct(np.where(np.arange(4000) == 3999, np.inf, 0.1).astype(np.float32)),
    ]
    for bad in bad_calls:
        with pytest.raises(RuntimeError):
            bad()
    assert not L.encodec_compress_audio(e.ctx, None, 4000, 1) and not L.encodec_decompress_audio(e.ctx, None, 16, 1)
    for bw, sr in ((25, 24000), (6, 319), (6, 0), (6, -24000)):                   # too many codebooks; sr < hop
        e.bandwidth, e.sample_rate = bw, sr
        with pytest.raises(RuntimeError):
            e.compress(x)
        with pytest.raises(RuntimeError):
            e.decompress(good_codes)
    e.bandwidth, e.sample_rate = 12, 24000
    assert np.array_equal(e.compress(x), good_codes)
    assert np.array_equal(e.reconstruct(x).view(np.uint32), good_audio.view(np.uint32))
    e.bandwidth = 24
    path = str(tmp_path / "no_encoder.bin")
    weights_mod.write_weights(path, weights_mod.tiny(), 1234, with_encoder=False)
    with pkg.Encodec(path, codec_offset(path)) as ne:
        for f in (ne.compress, ne.reconstruct):
            with pytest.raises(RuntimeError):
                f(x)
        assert ne.decompress(np.zeros((32, 9), np.int32)).size == 320 * 9
    assert not L.encodec_load_model(os.fsencode(path), 5, 0)                       # not a codec section
    s = e.stats()
    assert s["t_load_us"] > 0 and s["t_compute_us"] > 0
    e.reset_stats()
    assert e.stats() == {"t_load_us": 0, "t_compute_us": 0}


def test_two_contexts_on_two_threads(pkg, codecs, weights_file):
    path = weights_file("tiny", "f16", 1234)
    xs = [eo.signal("noise", 48000 + 777 * i, seed=60 + i) for i in range(4)]
    e = codecs["base"]
    e.bandwidth = 24
    want = [(e.compress(x), e.reconstruct(x)) for x in xs]
    got, errors = {}, []

    def work(k):
        try:
            with pkg.Encodec(path, codec_offset(path)) as mine:
                for _ in range(2):
                    got[k] = [(mine.compress(x), mine.reconstruct(x)) for x in xs]
        except Exception as exc:      # noqa: BLE001  (reported below)
            errors.append(exc)
    ts = [threading.Thread(target=work, args=(k,)) for k in range(2)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    assert not errors, errors
    for k in range(2):
        for (c, a), (wc, wa) in zip(got[k], want):
            assert np.array_equal(c, wc) and np.array_equal(a.view(np.uint32), wa.view(np.uint32))


def test_an_encodec_context_leaves_a_bark_context_alone(pkg, weights_file):
    path = weights_file("tiny", "f16", 1234)

    def gen(b):
        audio = b.generate("hello world")
        return [b.tokens(s).copy() for s in (0, 1, 2)], audio
    with pkg.Bark(path, seed=0, n_steps_text_encoder=12) as fresh:
        ids_f, audio_f = gen(fresh)
    with pkg.Bark(path, seed=0, n_steps_text_encoder=12) as b:
        with pkg.Encodec(path, codec_offset(path)) as e:
            e.reconstruct(eo.signal("noise", 24001, seed=4))
            ids, audio = gen(b)
            e.compress(eo.signal("sine", 9600))
            assert np.array_equal(b.tokens(2), ids[2])
    for x, y in zip(ids, ids_f):
        assert np.array_equal(x, y)
    assert np.array_equal(audio.view(np.uint32), audio_f.view(np.uint32))


def _write_wav(path, x):
    with wave.open(str(path), "wb") as w:
        w.setnchannels(1); w.setsampwidth(2); w.setframerate(24000)
        w.writeframes((np.clip(x, -1, 1) * 32767).astype("<i2").tobytes())


def _read_f32_wav(path):
    b = open(path, "rb").read()
    i = 12
    while b[i:i + 4] != b"data":
        i += 8 + int.from_bytes(b[i + 4:i + 8], "little")
    n = int.from_bytes(b[i + 4:i + 8], "little")
    return np.frombuffer(b[i + 8:i + 8 + n], "<f4")


def test_reference_examples_agree_with_the_python_api(pkg, weights_file, tmp_path):
    ref_dir = os.path.join(ROOT, "oracle", "_ref")
    exes = {k: os.path.join(ref_dir, f"encodec_{k}") for k in ("compress", "decompress", "main")}
    if not all(os.path.exists(p) for p in exes.values()):
        pytest.skip("encodec.cpp's examples were not built (no reference tree at build time)")
    path = weights_file("tiny", "f16", 1234)
    solo = tmp_path / "encodec.bin"
    solo.write_bytes(open(path, "rb").read()[codec_offset(path):])
    x = eo.signal("sine", 24000 * 2 + 17, seed=0) * np.float32(0.8)
    wav, ecdc, out_wav, main_wav = tmp_path / "in.wav", tmp_path / "in.ecdc", tmp_path / "out.wav", tmp_path / "main.wav"
    _write_wav(wav, x)
    env = dict(os.environ, LD_LIBRARY_PATH=os.path.dirname(pkg.LIB_PATH))
    run = lambda exe, *a: subprocess.run([exe, "-m", str(solo), *a], capture_output=True, text=True, env=env, cwd=tmp_path, timeout=600)  # noqa: E731
    r = run(exes["compress"], "-i", str(wav), "-o", str(ecdc)); assert r.returncode == 0, r.stderr
    r = run(exes["decompress"], "-i", str(ecdc), "-o", str(out_wav)); assert r.returncode == 0, r.stderr
    r = run(exes["main"], "-i", str(wav), "-o", str(main_wav)); assert r.returncode == 0, r.stderr
    with wave.open(str(wav)) as w:                    # what the examples read: the 16-bit samples as float
        xin = np.frombuffer(w.readframes(w.getnframes()), "<i2").astype(np.float32) / np.float32(32768)
    with pkg.Encodec(str(solo)) as e:
        e.bandwidth = 12
        codes, audio = e.compress(xin), e.reconstruct(xin)
        assert np.array_equal(e.decompress(codes).view(np.uint32), audio.view(np.uint32))
    for f in (out_wav, main_wav):                    # both trim to the input length and write 32-bit float wav files
        got = _read_f32_wav(f)
        assert np.array_equal(got.view(np.uint32), audio[:xin.size].view(np.uint32)), f.name
    assert ecdc.stat().st_size > 0
