"""CPU: the resampling rule's restatement (tests/resample_oracle.py) against torchaudio's outputs stored in tests/golden/resample/torchaudio.npz
(tests/golden/make_golden_resample.py): the f32 taps bit for bit, the outputs within 2^-23 sum|h x| + 2^-24 |y| of torchaudio's
float64 resample, the lengths equal, and the down-mix against torch.mean."""
import functools
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN_DIR
import resample_oracle as ro

GOLD = os.path.join(GOLDEN_DIR, "resample", "torchaudio.npz")
PAIRS = [(sr, 24000) for sr in (8000, 11025, 16000, 22050, 32000, 44100, 44056, 48000, 96000)] + [(24000, 44100), (24000, 48000)]
SHORT = (1, 2, 3, 1920, 1921)


@functools.lru_cache(maxsize=None)
def table(sr, nsr):
    return ro.sparse_taps(sr, nsr)


@pytest.fixture(scope="module")
def gold():
    return np.load(GOLD)


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


@pytest.mark.parametrize("sr,nsr", PAIRS)
def test_taps_bit_identical_to_torchaudio(gold, sr, nsr):
    first, count, taps = table(sr, nsr)
    k = f"{sr}_{nsr}"
    assert np.array_equal(first, gold[f"{k}_first"]) and np.array_equal(count, gold[f"{k}_count"])
    assert np.array_equal(bits(taps), bits(gold[f"{k}_taps"]))


@pytest.mark.parametrize("sr,nsr", [p for p in PAIRS if ro.rates(*p)[1] * (2 * ro.rates(*p)[2] + ro.rates(*p)[0]) <= 60000])
def test_dense_taps_are_zero_outside_the_sparse_span(sr, nsr):
    dense = ro.dense_taps(sr, nsr)
    first, count, taps = table(sr, nsr)
    offs = np.concatenate([[0], np.cumsum(count)])
    for j, row in enumerate(dense):
        lo, hi = first[j], first[j] + count[j]
        assert not row[:lo].any() and not row[hi:].any(), f"phase {j}"
        assert np.array_equal(bits(row[lo:hi]), bits(taps[offs[j]:offs[j + 1]])), f"phase {j}"


@pytest.mark.parametrize("sr,nsr", PAIRS)
def test_outputs_within_the_bound_of_torchaudio(gold, sr, nsr):
    t = table(sr, nsr)
    k = f"{sr}_{nsr}"
    for n in SHORT + (10 * sr,):
        x = ro.clip("noise", n, seed=n)
        y = ro.resample(x, sr, nsr, t)
        assert y.size == ro.out_len(n, sr, nsr)
        b = ro.bound(x, sr, nsr, y, t)
        if n in SHORT:
            ref = gold[f"{k}_n{n}"]
            assert y.size == ref.size, n
        else:
            assert y.size == int(gold[f"{k}_n{n}_len"])
            idx = gold[f"{k}_n{n}_idx"]
            ref, y, b = gold[f"{k}_n{n}"], y[idx], b[idx]
        err = np.abs(y.astype(np.float64) - ref)
        assert (err <= b).all(), f"n={n}: worst {float((err / b).max()):.3f} of the bound"


def test_lengths_match_torchaudio_rule():
    for sr, nsr in PAIRS + [(383999, 24000), (24000, 383999), (4000, 24000), (384000, 4000)]:
        o, q, _, _ = ro.rates(sr, nsr)
        for n in (1, 2, 3, 1919, 1920, 1921, 3840, 3841, 441000, 2 ** 31 - 1):
            assert ro.out_len(n, sr, nsr) == int(np.ceil(np.float64(q * n) / o)) or q * n >= 2 ** 53, (sr, nsr, n)


@pytest.mark.parametrize("C", [2, 6, 8])
def test_downmix_against_torch_mean(C):
    for kind in ("noise", "full", "subnormal", "zeros"):
        x = ro.clip(kind, 4099, C, seed=C)
        u = ro.downmix(x)
        m = torch.mean(torch.from_numpy(x), dim=1).numpy()
        if C <= 2:
            assert np.array_equal(bits(u), bits(m)) or kind == "zeros" and np.array_equal(u, m), kind
        else:       # torch sums in another order: each of the C - 1 roundings is at most half an ulp of its partial sum
            tol = (C - 1) * 2.0 ** -24 * np.abs(x.astype(np.float64)).sum(axis=1) / C + np.spacing(np.abs(m))
            assert (np.abs(u.astype(np.float64) - m) <= tol).all(), kind


def test_equal_rates_are_the_downmix_and_48k_to_24k_of_3840_frames_is_1920():
    x = ro.clip("noise", 1000, 2, seed=3)
    assert np.array_equal(bits(ro.resample(x, 24000, 24000)), bits(ro.downmix(x)))
    assert ro.out_len(3840, 48000, 24000) == 1920 and ro.out_len(3841, 48000, 24000) == 1921
