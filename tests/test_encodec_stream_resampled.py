"""CPU: the readiness rule of resampled EnCodec streams (bark_b200_encodec_stream_ready_resampled, DESIGN.md §20) against a brute force
over torchaudio's kernel support.  torchaudio's resampling kernel for sr -> new_sr is [q][2w + o] (tests/resample_oracle.py's rates), and
output k q + j reads the frames k o - w .. k o + o + w - 1; an output is final once every frame it reads has arrived.  The rule needs no
device."""
import numpy as np
import pytest

import resample_oracle as ro

ENCODE, DECODE = 0, 1
HOP, MIN_FRAMES = 320, 7
FIXTURE_RATES = (8000, 11025, 16000, 22050, 32000, 44100, 44056, 48000, 96000)     # the 11 fixture pairs: these -> 24 kHz, 24 kHz -> 44.1 / 48
RATES = sorted(set(FIXTURE_RATES + (44100, 48000, 4000, 383999, 384000, 24000)))


def support(sr, new_sr):
    """(o, q, w, width): torchaudio's kernel is q phases of width = 2w + o taps, phase j of block k starting at frame k o - w."""
    o, q, w, _ = ro.rates(sr, new_sr)
    if sr == new_sr:
        return 1, 1, 0, 1
    return o, q, w, 2 * w + o


def brute_final(n, sr, new_sr):
    """Outputs whose every read frame lies below n: blocks k with k o - w + width - 1 <= n - 1, found by bisection over k (the last read
    frame grows with k), so it holds for n near 2^40 too.  Each block holds q outputs."""
    o, q, w, width = support(sr, new_sr)
    last = lambda k: k * o - w + width - 1                      # noqa: E731
    lo, hi = 0, n // o + 2                                      # blocks [0, lo) final, [hi, ...) not
    while lo < hi:
        mid = (lo + hi) // 2
        if last(mid) <= n - 1:
            lo = mid + 1
        else:
            hi = mid
    assert lo == 0 or last(lo - 1) <= n - 1
    assert last(lo) > n - 1
    return q * lo


def codec_frames(n24):
    return n24 // HOP if n24 >= MIN_FRAMES * HOP else 0


def want(direction, sr, n):
    if direction == ENCODE:
        return codec_frames(brute_final(n, sr, 24000))
    return brute_final(n * HOP if n >= MIN_FRAMES else 0, 24000, sr)


def ready(pkg, direction, sr, n):
    return int(pkg.lib().bark_b200_encodec_stream_ready_resampled(direction, sr, n))


def first_ready(pkg, direction, sr):
    """the least n with outputs (bisection over the library's rule, checked by the brute force below)"""
    lo, hi = 0, 1
    while ready(pkg, direction, sr, hi) == 0:
        hi *= 2
    while lo < hi:
        mid = (lo + hi) // 2
        if ready(pkg, direction, sr, mid) > 0:
            hi = mid
        else:
            lo = mid + 1
    return lo


@pytest.mark.parametrize("direction", [ENCODE, DECODE])
@pytest.mark.parametrize("sr", RATES)
def test_ready_equals_the_brute_force_up_to_a_few_blocks_past_first_readiness(pkg, direction, sr):
    n0 = first_ready(pkg, direction, sr)
    assert ready(pkg, direction, sr, n0 - 1) == 0 and want(direction, sr, n0 - 1) == 0 and want(direction, sr, n0) > 0
    if direction == ENCODE:
        o, q, _, _ = support(sr, 24000)
        span = 3 * max(o, -(-HOP * o // q))                      # three blocks, and at least three code frames
    else:
        o, q, _, _ = support(24000, sr)
        span = 3 * max(1, -(-o // HOP))
    for n in range(0, n0 + span + 1):
        assert ready(pkg, direction, sr, n) == want(direction, sr, n), (direction, sr, n)


@pytest.mark.parametrize("direction", [ENCODE, DECODE])
@pytest.mark.parametrize("sr", RATES)
def test_ready_near_2_to_the_40(pkg, direction, sr):
    o, q, w, _ = support(sr, 24000) if direction == ENCODE else support(24000, sr)
    rng = np.random.default_rng(sr + direction)
    if direction == ENCODE:
        k = (1 << 40) // o
        ns = [k * o + w + d for d in (-HOP * o - 1, -2, -1, 0, 1, 2, o - 1, o)] + [int(v) for v in rng.integers((1 << 40) - 10 ** 6, (1 << 40) + 10 ** 6, 50)]
    else:
        base = (1 << 40) // HOP
        ns = [base + d for d in range(-3, 4)] + [int(v) for v in rng.integers(base - 10 ** 6, base + 10 ** 6, 50)]
        k = ((1 << 40) - w) // o                                 # n with 320 n - w crossing a block boundary of the 24 kHz samples
        ns += [(k * o + w) // HOP + d for d in (-1, 0, 1)]
    for n in ns:
        assert ready(pkg, direction, sr, n) == want(direction, sr, n), (direction, sr, n)


def test_identity_rates_and_the_stated_examples(pkg):
    for n in list(range(0, 3000)) + [1 << 40, (1 << 40) + 319]:
        assert ready(pkg, ENCODE, 24000, n) == pkg.encodec_stream_ready("encode", n)
    for n in list(range(0, 20)) + [1 << 40]:
        assert ready(pkg, DECODE, 24000, n) == pkg.encodec_stream_ready("decode", n)
    assert support(48000, 24000)[::2] == (2, 13) and support(44100, 24000)[::2] == (147, 12)
    assert ready(pkg, ENCODE, 48000, 4492) == 0 and ready(pkg, ENCODE, 48000, 4493) == 7
    assert pkg.encodec_stream_ready("encode", 4493, sample_rate=48000) == 7
    assert pkg.encodec_stream_ready("decode", 7, sample_rate=48000) == want(DECODE, 48000, 7)


def test_ready_refuses_what_the_streams_refuse(pkg):
    for direction, sr, n in ((2, 48000, 5), (-1, 48000, 5), (ENCODE, 3999, 5), (ENCODE, 384001, 5), (DECODE, 0, 5), (ENCODE, 48000, -1), (DECODE, 48000, -1)):
        assert ready(pkg, direction, sr, n) == -1, (direction, sr, n)
    assert ready(pkg, ENCODE, 4000, 0) == 0 and ready(pkg, DECODE, 384000, 0) == 0
