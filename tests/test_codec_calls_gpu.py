"""What every EnCodec entry point prints and returns when it refuses a call, and what the device does for a valid one.

The ten encodec_context calls (encodec_compress_audio / decompress / reconstruct and the bark_b200_encodec_* batch and resampled
calls) and the three bark_context hooks (bark_b200_encodec_encode[_resampled], bark_b200_encodec_decode): each refusal's whole
stderr line and return value, and for a fixed set of valid calls the kernel launches and the host-to-device and device-to-host bytes."""
import ctypes as C

import numpy as np
import pytest

import encoder_oracle as eo
from encodec_oracle import codec_offset

pytestmark = pytest.mark.gpu

ENCODER_MISSING = "the model file has no EnCodec encoder tensors (encoder.*)"
SHORT = "need at least 1921 samples (7 frames), got 1920"
FEW_FRAMES = "need at least 7 frames (reflect padding of the k=7 convolutions), got 6"
OUTSIDE = "code 1024 (codebook 3, frame 5) is outside the codebooks (1024 bins)"
RESAMPLED_SHORT = "3840 frames at 48000 Hz resample to 1920 samples at 24000 Hz (1921 to 2^31 - 1: at least 7 frames)"
NAN_FRAME = "sample 77 (frame 38, channel 1) is not finite or exceeds 2^64 in magnitude (nan)"

# Kernel launches of the valid calls below, recorded on an H100 with the tiny f16 fixture
LAUNCHES = {"compress": 23, "decompress": 23, "reconstruct": 46, "bark_encode": 23, "batch70": 69, "batch_long": 69, "resampled": 26}
TABLE_BYTES = 8716          # the resampled batch's rate tables, uploaded on the first run only


def ptrs(arrays):
    return (C.c_void_p * len(arrays))(*[None if a is None else a.ctypes.data for a in arrays])


def ints(vals):
    return (C.c_int * len(vals))(*vals)


def noise(n, seed=0):
    return eo.signal("noise", n, seed=seed)


def with_nan(n, at):
    return np.where(np.arange(n) == at, np.nan, 0.1).astype(np.float32)


@pytest.fixture(scope="module")
def paths(weights_file, weights_mod, tmp_path_factory):
    base = eo.weights_path(weights_file, weights_mod, "base")
    bare = str(tmp_path_factory.mktemp("codec_calls") / "no_encoder.bin")
    weights_mod.write_weights(bare, weights_mod.tiny(), 1234, with_encoder=False)
    return base, bare


@pytest.fixture(scope="module")
def codec(pkg, paths):
    with pkg.Encodec(paths[0], codec_offset(paths[0])) as e:
        e.bandwidth = 6
        yield e


@pytest.fixture(scope="module")
def bark(pkg, paths):
    with pkg.Bark(paths[0], seed=0, n_steps_text_encoder=12) as b:
        yield b


def check(L, capfd, cases):
    """cases: (function, args, expected return, expected stderr line or None for silence)"""
    capfd.readouterr()
    for fn, args, ret, line in cases:
        got = getattr(L, fn)(*args)
        err = capfd.readouterr().err
        assert got == ret, (fn, line, got)
        assert err == ("" if line is None else line + "\n"), (fn, err)


def test_encodec_context_refusals(pkg, codec, capfd):
    L, e = pkg.lib(), codec.ctx
    x, short, nan, ninf = noise(4000), np.zeros(1920, np.float32), with_nan(4000, 5), np.full(4000, -np.inf, np.float32)
    codes = np.zeros((8, 9), np.int32)
    outside = codes.copy(); outside[3, 5] = 1024
    few = np.zeros((8, 6), np.int32)
    keep = (x, short, nan, ninf, codes, outside, few)
    cases = []
    for fn in ("encodec_compress_audio", "encodec_reconstruct_audio"):
        cases += [
            (fn, (None, x.ctypes.data, x.size, 1), False, f"{fn}: null context"),
            (fn, (e, None, x.size, 1), False, f"{fn}: null input audio"),
            (fn, (e, short.ctypes.data, short.size, 1), False, f"codec_encode: {SHORT}"),
            (fn, (e, nan.ctypes.data, nan.size, 1), False, "codec_encode: sample 5 is not finite (nan)"),
            (fn, (e, ninf.ctypes.data, ninf.size, 1), False, "codec_encode: sample 0 is not finite (-inf)"),
        ]
    fn = "encodec_decompress_audio"
    cases += [
        (fn, (None, codes.ctypes.data, codes.size, 1), False, f"{fn}: null context"),
        (fn, (e, None, codes.size, 1), False, f"{fn}: null codes"),
        (fn, (e, codes.ctypes.data, codes.size - 3, 1), False, f"{fn}: 69 codes are not a whole number of frames of 8 codebooks"),
        (fn, (e, codes.ctypes.data, -8, 1), False, f"{fn}: -8 codes are not a whole number of frames of 8 codebooks"),
        (fn, (e, few.ctypes.data, few.size, 1), False, f"codec_decode: {FEW_FRAMES}"),
        (fn, (e, outside.ctypes.data, outside.size, 1), False, f"codec_decode: {OUTSIDE}"),
    ]
    check(L, capfd, cases)

    # the rules of the bandwidth: the context's sample rate and bandwidth, checked before the inputs' contents
    single = {"encodec_compress_audio": (x.ctypes.data, x.size, 1), "encodec_reconstruct_audio": (x.ctypes.data, x.size, 1),
              "encodec_decompress_audio": (codes.ctypes.data, codes.size, 1)}
    codec.sample_rate = 319
    check(L, capfd, [(fn, (e,) + a, False, f"{fn}: sample rate 319 is below the hop length 320 (frame rate 0)") for fn, a in single.items()])
    codec.sample_rate = 24000
    codec.bandwidth = 48
    check(L, capfd, [(fn, (e,) + a, False, f"{fn}: bandwidth 48 kbps at 24000 Hz needs 64 codebooks; the file has 32")
                     for fn, a in single.items()])
    codec.bandwidth = 6
    del keep


def test_batch_refusals(pkg, codec, capfd):
    L, e = pkg.lib(), codec.ctx
    xs = [noise(4000, 1), noise(2500, 2), noise(1921, 3)]
    cs = [np.zeros((8, T), np.int32) for T in (7, 9, 12)]
    cs_outside = [c.copy() for c in cs]; cs_outside[1][3, 5] = 1024
    cs_few = [cs[0], np.zeros((8, 6), np.int32), cs[2]]
    keep = (xs, cs, cs_outside, cs_few)
    lens, clens = ints([x.size for x in xs]), ints([c.size for c in cs])
    cases = []
    for fn in ("bark_b200_encodec_compress_batch", "bark_b200_encodec_reconstruct_batch"):
        bad_short, bad_nan = xs[:2] + [np.zeros(1920, np.float32)], [xs[0], with_nan(9999, 77)]
        keep += (bad_short, bad_nan)
        cases += [
            (fn, (None, ptrs(xs), lens, 3), False, f"{fn}: null context"),
            (fn, (e, ptrs(xs), lens, 0), False, f"{fn}: 0 items (1 to 1024 per batch)"),
            (fn, (e, ptrs(xs), lens, 1025), False, f"{fn}: 1025 items (1 to 1024 per batch)"),
            (fn, (e, None, lens, 3), False, f"{fn}: null item array"),
            (fn, (e, ptrs(xs), None, 3), False, f"{fn}: null length array"),
            (fn, (e, ptrs([xs[0], None, xs[2]]), lens, 3), False, f"{fn}: item 1 is null"),
            (fn, (e, ptrs(bad_short), ints([4000, 2500, 1920]), 3), False, f"{fn}: item 2: {SHORT}"),
            (fn, (e, ptrs(bad_nan), ints([4000, 9999]), 2), False, f"{fn}: item 1: sample 77 is not finite (nan)"),
            (fn, (e, ptrs(bad_short[2:]), ints([1920]), 1), False, f"{fn}: item 0: {SHORT}"),
        ]
    fn = "bark_b200_encodec_decompress_batch"
    cases += [
        (fn, (None, ptrs(cs), clens, 3), False, f"{fn}: null context"),
        (fn, (e, ptrs(cs), clens, -1), False, f"{fn}: -1 items (1 to 1024 per batch)"),
        (fn, (e, None, clens, 3), False, f"{fn}: null item array"),
        (fn, (e, ptrs(cs), None, 3), False, f"{fn}: null length array"),
        (fn, (e, ptrs([cs[0], cs[1], None]), clens, 3), False, f"{fn}: item 2 is null"),
        (fn, (e, ptrs(cs), ints([56, 71, 96]), 3), False, f"{fn}: item 1: 71 codes are not a whole number of frames of 8 codebooks"),
        (fn, (e, ptrs(cs_few), ints([c.size for c in cs_few]), 3), False, f"{fn}: item 1: {FEW_FRAMES}"),
        (fn, (e, ptrs(cs_outside), clens, 3), False, f"{fn}: item 1: {OUTSIDE}"),
    ]
    check(L, capfd, cases)
    codec.sample_rate = 319
    check(L, capfd, [(fn, (e, ptrs(a), ints([v.size for v in a]), 3), False, f"{fn}: sample rate 319 is below the hop length 320 (frame rate 0)")
                     for fn, a in (("bark_b200_encodec_compress_batch", xs), ("bark_b200_encodec_reconstruct_batch", xs),
                                   ("bark_b200_encodec_decompress_batch", cs))])
    codec.sample_rate = 24000
    del keep


def test_resampled_refusals(pkg, codec, capfd):
    L, e = pkg.lib(), codec.ctx
    x = noise(9000, 4)
    stereo_nan = with_nan(5000, 77)                 # 2500 interleaved stereo frames
    keep = (x, stereo_nan)
    bad_formats = [                                 # (frames, channels, rate, line without the caller)
        (3840, 1, 48000, RESAMPLED_SHORT),
        (400, 9, 24000, "9 channels (1 to 8)"),
        (0, 1, 24000, "0 frames of 1 channels (1 frame to 2^31 - 1 samples)"),
        (4000, 1, 3999, "sample rate 3999 Hz (4000 to 384000)"),
        (4000, 1, 384001, "sample rate 384001 Hz (4000 to 384000)"),
    ]
    cases = []
    for fn in ("bark_b200_encodec_compress_resampled", "bark_b200_encodec_reconstruct_resampled"):
        cases += [(fn, (None, x.ctypes.data, 4500, 2, 44100), False, f"{fn}: null context"),
                  (fn, (e, None, 4500, 2, 44100), False, f"{fn}: null input audio"),
                  (fn, (e, stereo_nan.ctypes.data, 2500, 2, 16000), False, f"codec_encode: {NAN_FRAME}")]
        cases += [(fn, (e, x.ctypes.data, n, ch, sr), False, f"codec_encode: {what}") for n, ch, sr, what in bad_formats]
    for fn in ("bark_b200_encodec_compress_batch_resampled", "bark_b200_encodec_reconstruct_batch_resampled"):
        two = ptrs([x, x])
        cases += [
            (fn, (None, two, ints([4500, 4500]), ints([2, 2]), ints([44100, 44100]), 2), False, f"{fn}: null context"),
            (fn, (e, two, ints([4500, 4500]), ints([2, 2]), ints([44100, 44100]), 0), False, f"{fn}: 0 items (1 to 1024 per batch)"),
            (fn, (e, None, ints([4500, 4500]), ints([2, 2]), ints([44100, 44100]), 2), False, f"{fn}: null item array"),
            (fn, (e, two, None, ints([2, 2]), ints([44100, 44100]), 2), False, f"{fn}: null length array"),
            (fn, (e, ptrs([x, None]), ints([4500, 4500]), ints([2, 2]), ints([44100, 44100]), 2), False, f"{fn}: item 1 is null"),
            (fn, (e, two, ints([4500, 4500]), None, ints([44100, 44100]), 2), False, f"{fn}: null channel array"),
            (fn, (e, two, ints([4500, 4500]), ints([2, 2]), None, 2), False, f"{fn}: null sample rate array"),
            (fn, (e, ptrs([x, stereo_nan]), ints([4500, 2500]), ints([2, 2]), ints([44100, 16000]), 2), False, f"{fn}: item 1: {NAN_FRAME}"),
        ]
        cases += [(fn, (e, two, ints([4500, n]), ints([2, ch]), ints([44100, sr]), 2), False, f"{fn}: item 1: {what}")
                  for n, ch, sr, what in bad_formats]
    check(L, capfd, cases)
    codec.bandwidth = 48
    line = "bandwidth 48 kbps at 24000 Hz needs 64 codebooks; the file has 32"
    check(L, capfd, [("bark_b200_encodec_compress_resampled", (e, x.ctypes.data, 4500, 2, 44100), False, f"bark_b200_encodec_compress_resampled: {line}"),
                     ("bark_b200_encodec_reconstruct_batch_resampled", (e, ptrs([x]), ints([4500]), ints([2]), ints([44100]), 1), False,
                      f"bark_b200_encodec_reconstruct_batch_resampled: {line}")])
    codec.bandwidth = 6
    del keep


def test_bark_context_hook_refusals(pkg, bark, capfd):
    L, b = pkg.lib(), bark.ctx
    x, short, inf = noise(4000, 5), np.zeros(1920, np.float32), np.where(np.arange(4000) == 7, np.inf, 0.1).astype(np.float32)
    stereo_nan = with_nan(5000, 77)
    codes = np.zeros((8, 9), np.int32)
    outside = codes.copy(); outside[3, 5] = 1024
    few = np.zeros((8, 6), np.int32)
    keep = (x, short, inf, stereo_nan, codes, outside, few)
    out, lat = np.zeros(8 * 13, np.int32), np.zeros(128 * 13, np.float32)
    o = (out.ctypes.data, out.size, lat.ctypes.data, lat.size)
    fn = "bark_b200_encodec_encode"
    cases = [
        (fn, (None, x.ctypes.data, x.size) + o, -1, f"{fn}: invalid bark context"),
        (fn, (b, None, x.size) + o, -1, f"{fn}: null audio"),
        (fn, (b, short.ctypes.data, short.size) + o, -1, f"codec_encode: {SHORT}"),
        (fn, (b, inf.ctypes.data, inf.size) + o, -1, "codec_encode: sample 7 is not finite (inf)"),
    ]
    fn = "bark_b200_encodec_encode_resampled"
    cases += [
        (fn, (None, x.ctypes.data, 2000, 2, 44100) + o, -1, f"{fn}: invalid bark context"),
        (fn, (b, None, 2000, 2, 44100) + o, -1, f"{fn}: null audio"),
        (fn, (b, x.ctypes.data, 3840, 1, 48000) + o, -1, f"codec_encode: {RESAMPLED_SHORT}"),
        (fn, (b, x.ctypes.data, 400, 9, 24000) + o, -1, "codec_encode: 9 channels (1 to 8)"),
        (fn, (b, x.ctypes.data, 4000, 1, 3999) + o, -1, "codec_encode: sample rate 3999 Hz (4000 to 384000)"),
        (fn, (b, stereo_nan.ctypes.data, 2500, 2, 16000) + o, -1, f"codec_encode: {NAN_FRAME}"),
    ]
    fn = "bark_b200_encodec_decode"
    wav = np.zeros(320 * 9, np.float32)
    cases += [
        (fn, (None, codes.ctypes.data, 9, wav.ctypes.data, wav.size), -1, f"{fn}: invalid bark context"),
        (fn, (b, None, 9, wav.ctypes.data, wav.size), -1, None),
        (fn, (b, few.ctypes.data, 6, wav.ctypes.data, wav.size), -1, f"codec_decode: {FEW_FRAMES}"),
        (fn, (b, outside.ctypes.data, 9, wav.ctypes.data, wav.size), -1, f"codec_decode: {OUTSIDE}"),
    ]
    check(L, capfd, cases)
    del keep


def test_files_without_encoder_tensors(pkg, paths, capfd):
    L, bare = pkg.lib(), paths[1]
    x, codes = noise(4000, 6), np.zeros((8, 9), np.int32)
    frames, chans, rates = ints([2000]), ints([2]), ints([44100])
    with pkg.Encodec(bare, codec_offset(bare)) as ne, pkg.Bark(bare, seed=0, n_steps_text_encoder=12) as nb:
        ne.bandwidth = 6
        e = ne.ctx
        one = ptrs([x])
        cases = [
            ("encodec_compress_audio", (e, x.ctypes.data, x.size, 1), False, f"codec_encode: {ENCODER_MISSING}"),
            ("encodec_reconstruct_audio", (e, x.ctypes.data, x.size, 1), False, f"codec_encode: {ENCODER_MISSING}"),
            ("bark_b200_encodec_compress_batch", (e, one, ints([x.size]), 1), False, f"bark_b200_encodec_compress_batch: {ENCODER_MISSING}"),
            ("bark_b200_encodec_reconstruct_batch", (e, one, ints([x.size]), 1), False, f"bark_b200_encodec_reconstruct_batch: {ENCODER_MISSING}"),
            ("bark_b200_encodec_compress_resampled", (e, x.ctypes.data, 2000, 2, 44100), False, f"codec_encode: {ENCODER_MISSING}"),
            ("bark_b200_encodec_reconstruct_resampled", (e, x.ctypes.data, 2000, 2, 44100), False, f"codec_encode: {ENCODER_MISSING}"),
            ("bark_b200_encodec_compress_batch_resampled", (e, one, frames, chans, rates, 1), False,
             f"bark_b200_encodec_compress_batch_resampled: {ENCODER_MISSING}"),
            ("bark_b200_encodec_reconstruct_batch_resampled", (e, one, frames, chans, rates, 1), False,
             f"bark_b200_encodec_reconstruct_batch_resampled: {ENCODER_MISSING}"),
            ("bark_b200_encodec_encode", (nb.ctx, x.ctypes.data, x.size, None, 0, None, 0), -1, f"codec_encode: {ENCODER_MISSING}"),
            ("bark_b200_encodec_encode_resampled", (nb.ctx, x.ctypes.data, 2000, 2, 44100, None, 0, None, 0), -1, f"codec_encode: {ENCODER_MISSING}"),
            # the decoder needs no encoder
            ("encodec_decompress_audio", (e, codes.ctypes.data, codes.size, 1), True, None),
        ]
        check(L, capfd, cases)
        assert nb.encodec_decode(codes).size == 320 * 9


# ---- device work of valid calls ----------------------------------------------------------------------------------------------------
def measure(pkg, f):
    """(kernel launches, H2D bytes, D2H bytes) of f()"""
    pkg.io_counters(reset=True)
    k0 = pkg.kernel_launches()
    f()
    h2d, d2h = pkg.io_counters(reset=True)
    return pkg.kernel_launches() - k0, h2d, d2h


def frames_of(n):
    return (n + 319) // 320


def test_device_work_of_valid_calls(pkg, codec, bark, paths):
    e, n_q = codec, 8
    x = noise(24001, 7)
    T = frames_of(x.size)
    codes = e.compress(x)
    got = {}

    got["compress"] = measure(pkg, lambda: e.compress(x))
    assert got["compress"][1:] == (4 * x.size, 4 * n_q * T)
    got["decompress"] = measure(pkg, lambda: e.decompress(codes))
    assert got["decompress"][1:] == (4 * n_q * T, 4 * 320 * T)
    got["reconstruct"] = measure(pkg, lambda: e.reconstruct(x))
    assert got["reconstruct"][1:] == (4 * x.size, 4 * 320 * T)
    got["bark_encode"] = measure(pkg, lambda: bark.encodec_encode(x, return_latent=True))
    assert got["bark_encode"][1:] == (4 * x.size, 4 * (8 + 128) * T)

    many = [noise(1921 + 331 * i, 900 + i) for i in range(70)]                # three launches by count
    got["batch70"] = measure(pkg, lambda: e.compress_batch(many))
    assert got["batch70"][1:] == (4 * sum(v.size for v in many), 4 * n_q * sum(frames_of(v.size) for v in many))
    long = [noise(320 * 8000 + 17 * i, 950 + i) for i in range(2)]
    long.insert(1, eo.signal("sine", 320 * (24000 + 100), seed=5))           # longer than a launch: launches of 1, 1 and 1 item
    got["batch_long"] = measure(pkg, lambda: e.compress_batch(long))
    assert got["batch_long"][1:] == (4 * sum(v.size for v in long), 4 * n_q * sum(frames_of(v.size) for v in long))

    import resample_oracle as ro
    clips = [(ro.clip("noise", 4410 * 3, 2, seed=11), 44100), (ro.clip("noise", 16000, 1, seed=12), 16000),
             (ro.clip("noise", 4800 * 2, 1, seed=13), 48000)]
    xs, srs = [x if x.ndim == 1 else np.ascontiguousarray(x.T) for x, _ in clips], [sr for _, sr in clips]
    inputs = 4 * sum(c.size for c, _ in clips)
    outputs = 4 * n_q * sum(frames_of(pkg.resampled_length(c.shape[0], sr)) for c, sr in clips)
    with pkg.Encodec(paths[0], codec_offset(paths[0])) as fresh:             # an empty table cache
        fresh.bandwidth = 6
        first = measure(pkg, lambda: fresh.compress_batch(xs, sample_rate=srs))
        second = measure(pkg, lambda: fresh.compress_batch(xs, sample_rate=srs))
    assert first[0] == second[0] and first[2] == second[2] == outputs
    assert second[1] == inputs and first[1] > inputs
    got["resampled"] = second
    assert {k: v[0] for k, v in got.items()} == LAUNCHES
    assert first[1] - inputs == TABLE_BYTES
