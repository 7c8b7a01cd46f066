"""EnCodec encoding on the GPU (bark_b200_encodec_encode, bark_b200_rvq_encode) against the unmodified reference's stored outputs
(tests/golden/ref_pairs/encoder.npz) and the CPU restatement (tests/encoder_oracle.c): bit for bit."""
import ctypes as C
import os

import numpy as np
import pytest

from conftest import GOLDEN_DIR, assert_pinned
import encoder_oracle as eo

pytestmark = pytest.mark.gpu
GOLD = os.path.join(GOLDEN_DIR, "ref_pairs", "encoder.npz")
SWEEP = [1921, 1922, 2239, 2241, 3200, 5119, 9601, 16001, 33333, 48000, 100003, 240000]   # 240000 = 10 s


@pytest.fixture(scope="module")
def gold():
    return np.load(GOLD)


@pytest.fixture(scope="module")
def ctxs(pkg, weights_file, weights_mod):
    out = {w: pkg.Bark(eo.weights_path(weights_file, weights_mod, w), seed=0, n_steps_text_encoder=12) for w in eo.WEIGHTS}
    yield out
    for b in out.values():
        b.close()


@pytest.mark.parametrize("name,kind,n,which", eo.CASES, ids=[c[0] for c in eo.CASES])
def test_codes_equal_the_reference(ctxs, gold, name, kind, n, which):
    codes = ctxs[which].encodec_encode(eo.signal(kind, n, seed=n))
    ref = gold[name + "_codes"]
    assert codes.shape == ref.shape
    assert np.array_equal(codes, ref), f"{name}: {int((codes != ref).sum())} codes differ; first at {np.argwhere(codes != ref)[:1].tolist()}"


@pytest.mark.parametrize("name", eo.RECONSTRUCT)
def test_decode_of_encode_equals_the_reference_reconstruction(ctxs, gold, name):
    _, kind, n, which = next(c for c in eo.CASES if c[0] == name)
    b = ctxs[which]
    assert_pinned(b.encodec_decode(b.encodec_encode(eo.signal(kind, n, seed=n))), gold, name + "_audio", f"{name} reconstruction")


def test_codes_and_latent_equal_the_oracle_on_a_length_sweep(ctxs, weights_file, weights_mod):
    oracle = eo.EncoderOracle(eo.weights_path(weights_file, weights_mod, "base"))
    for i, n in enumerate(SWEEP):
        x = eo.signal(("noise", "sine", "square")[i % 3], n, seed=100 + i)
        if i % 3 == 0:
            x *= np.float32(0.25 * (1 + i % 4))
        codes, lat = ctxs["base"].encodec_encode(x, return_latent=True)
        o_codes, o_lat = oracle.encode(x, return_latent=True)
        assert np.array_equal(lat.view(np.uint32), o_lat.view(np.uint32)), f"n={n}: latent differs at {np.argwhere(lat != o_lat)[:1].tolist()}"
        assert np.array_equal(codes, o_codes), f"n={n}: codes differ at {np.argwhere(codes != o_codes)[:1].tolist()}"


def test_encoding_twice_gives_identical_codes(ctxs):
    x = eo.signal("noise", 48001, seed=9)
    a, la = ctxs["base"].encodec_encode(x, return_latent=True)
    b, lb = ctxs["base"].encodec_encode(x, return_latent=True)
    assert np.array_equal(a, b) and np.array_equal(la.view(np.uint32), lb.view(np.uint32))


# ---- the RVQ encode kernel on built rows --------------------------------------------------------------------------------------
def _rvq_case(rng, n_q, T, hidden=128, n_bins=1024):
    cb = rng.standard_normal((n_q, n_bins, hidden), dtype=np.float32)
    lat = rng.standard_normal((hidden, T), dtype=np.float32) * np.float32(2)
    return lat, cb


def _check_rvq(pkg, lat, cb):
    got = pkg.rvq_encode(lat, cb)
    want = eo.rvq_encode(lat, cb)
    assert np.array_equal(got, want), f"{int((got != want).sum())} codes differ; first at {np.argwhere(got != want)[:1].tolist()}"
    return got


@pytest.mark.parametrize("n_q", range(1, 9))
@pytest.mark.parametrize("T", [1, 7, 1000])
def test_rvq_encode_random_rows(pkg, n_q, T):
    _check_rvq(pkg, *_rvq_case(np.random.default_rng(n_q * 1000 + T), n_q, T))


def test_rvq_encode_small_shapes(pkg):
    rng = np.random.default_rng(3)
    for hidden, n_bins in ((32, 1), (32, 5), (64, 33), (96, 1000)):
        _check_rvq(pkg, *_rvq_case(rng, 3, 17, hidden, n_bins))


def test_rvq_encode_exact_ties_and_codeword_residuals(pkg):
    rng = np.random.default_rng(11)
    lat, cb = _rvq_case(rng, 4, 40)
    cb[0, -1] = cb[0, 0]                       # first and last codeword tie
    cb[1, 700] = cb[1, 0]                      # the first codeword ties a middle one
    cb[2, 1023] = cb[2, 5]                     # the last ties a middle one
    lat[:, 0] = cb[0, 0]                       # residual equal to the tied first / last codeword
    lat[:, 1] = cb[0, 17]                      # residual equal to a codeword: distance exactly representable
    lat[:, 2] = cb[0, 1023]
    got = _check_rvq(pkg, lat, cb)
    assert got[0, 0] == 1023 and got[0, 2] == 1023 and got[0, 1] == 17


def test_rvq_encode_zeros_and_subnormals(pkg):
    rng = np.random.default_rng(12)
    lat, cb = _rvq_case(rng, 8, 8)
    lat[:, 0] = 0.0
    lat[:, 1] = -0.0
    lat[:, 2] = np.float32(1e-41) * rng.choice([-1, 1], 128)
    lat[:, 3] = np.float32(1.2e-38)
    cb[0, 3] = 0.0
    cb[1, 9] = -0.0
    cb[2, :10] = np.float32(3e-42)
    _check_rvq(pkg, lat, cb)


def test_rvq_encode_overflowing_dots(pkg):
    rng = np.random.default_rng(13)
    lat, cb = _rvq_case(rng, 8, 12)
    lat[:, 0] = np.float32(3e19)               # s overflows to inf: every distance -inf
    lat[:, 1] = np.float32(-2e19) * rng.choice([-1, 1], 128)
    cb[0, 10] = np.float32(3e19)               # dot and norm overflow for this codeword
    cb[0, 20] = np.float32(-3e19)
    lat[:, 2] = np.float32(1e18)
    _check_rvq(pkg, lat, cb)


@pytest.mark.parametrize("where", [0, 511, 1023])
def test_rvq_encode_nan_in_a_row(pkg, where):
    rng = np.random.default_rng(14 + where)
    lat, cb = _rvq_case(rng, 3, 9)
    cb[0, where, 5] = np.nan                   # distance of codeword `where` is NaN in every frame of codebook 0
    cb[1, where, 0] = np.nan
    lat[:, 4] = np.nan                         # a whole NaN frame
    _check_rvq(pkg, lat, cb)


# ---- refusals and the generation state ----------------------------------------------------------------------------------------
def _gen(b):
    audio = b.generate("hello world")
    return [b.tokens(s) for s in (0, 1, 2)], audio


def test_refusals_leave_the_context_usable(pkg, weights_file, weights_mod, ctxs, tmp_path):
    L = pkg.lib()
    b = ctxs["base"]
    for bad in (np.zeros(1920, np.float32), np.where(np.arange(4000) == 3999, np.nan, 0.1).astype(np.float32),
                np.where(np.arange(4000) == 7, np.inf, 0.1).astype(np.float32), np.full(4000, -np.inf, np.float32)):
        with pytest.raises(RuntimeError):
            b.encodec_encode(bad)
    x = np.zeros(4000, np.float32)
    assert L.bark_b200_encodec_encode(b.ctx, None, 4000, None, 0, None, 0) == -1
    assert L.bark_b200_encodec_encode(None, x.ctypes.data_as(C.c_void_p), 4000, None, 0, None, 0) == -1
    after = _gen(b)
    with pkg.Bark(weights_file("tiny", "f16", 1234), seed=0, n_steps_text_encoder=12) as fresh:
        _same(after, _gen(fresh))
    path = str(tmp_path / "no_encoder.bin")                  # without the encoder draws the decoder's seeded weights differ too
    weights_mod.write_weights(path, weights_mod.tiny(), 1234, with_encoder=False)
    with pkg.Bark(path, seed=0, n_steps_text_encoder=12) as ne:
        with pytest.raises(RuntimeError):
            ne.encodec_encode(eo.signal("noise", 4000))
        after = _gen(ne)
    with pkg.Bark(path, seed=0, n_steps_text_encoder=12) as fresh:
        _same(after, _gen(fresh))


def _same(a, b):
    for x, y in zip(a[0], b[0]):
        assert np.array_equal(x, y)
    assert np.array_equal(a[1].view(np.uint32), b[1].view(np.uint32))


def test_generation_after_an_encode_matches_a_fresh_context(pkg, weights_file):
    path = weights_file("tiny", "f16", 1234)
    with pkg.Bark(path, seed=0, n_steps_text_encoder=12) as fresh:
        ids_f, audio_f = _gen(fresh)
    with pkg.Bark(path, seed=0, n_steps_text_encoder=12) as b:
        codes = b.encodec_encode(eo.signal("noise", 24001, seed=1))
        assert codes.shape == (8, 76)
        ids, audio = _gen(b)
        before = b.tokens(2).copy(), audio.copy()
        b.encodec_encode(eo.signal("sine", 9600))     # and an encode after a generation leaves its results in place
        assert np.array_equal(b.tokens(2), before[0])
        n = pkg.lib().bark_get_audio_data_size(b.ctx)
        assert np.array_equal(np.ctypeslib.as_array(pkg.lib().bark_get_audio_data(b.ctx), shape=(n,)), before[1])
    _same((ids, audio), (ids_f, audio_f))
