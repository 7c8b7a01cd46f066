"""The EnCodec encoder's CPU restatement (tests/encoder_oracle.c) against the unmodified reference's stored encodec_compress_audio
codes and encodec_reconstruct_audio waveforms (tests/golden/make_golden_encoder.py), and static guards on the encoder kernels."""
import os

import numpy as np
import pytest

from conftest import GOLDEN_DIR, assert_pinned
import encoder_oracle as eo
from test_decode_resources import res_usage

GOLD = os.path.join(GOLDEN_DIR, "ref_pairs", "encoder.npz")


@pytest.fixture(scope="module")
def gold():
    return np.load(GOLD)


@pytest.fixture(scope="module")
def enc_oracles(weights_file, weights_mod):
    return {w: eo.EncoderOracle(eo.weights_path(weights_file, weights_mod, w)) for w in eo.WEIGHTS}


@pytest.mark.parametrize("name,kind,n,which", eo.CASES, ids=[c[0] for c in eo.CASES])
def test_oracle_codes_equal_the_reference(enc_oracles, gold, name, kind, n, which):
    codes = enc_oracles[which].encode(eo.signal(kind, n, seed=n))
    ref = gold[name + "_codes"]
    assert codes.shape == ref.shape == (8, (n + 319) // 320)
    assert np.array_equal(codes, ref), f"{name}: {int((codes != ref).sum())} codes differ; first at {np.argwhere(codes != ref)[:1].tolist()}"


@pytest.mark.parametrize("name", eo.RECONSTRUCT)
def test_oracle_reconstruction_equals_the_reference(orc, weights_file, weights_mod, enc_oracles, gold, name):
    _, kind, n, which = next(c for c in eo.CASES if c[0] == name)
    path = eo.weights_path(weights_file, weights_mod, which)
    codes = enc_oracles[which].encode(eo.signal(kind, n, seed=n))
    audio = orc.Oracle(path).encodec_decode(codes)          # encodec_reconstruct_audio = the decoder on the encoder's codes
    assert_pinned(audio, gold, name + "_audio", f"{name} reconstruction")


def test_tied_codewords_resolve_to_the_last_index(enc_oracles, gold):
    # codebook 0 with rows 2m and 2m+1 identical: the argmax keeps the last index of a maximum, so every code is odd
    codes = enc_oracles["tie_pairs"].encode(eo.signal("noise", 6400, seed=5))
    assert (codes[0] % 2 == 1).all(), codes[0]
    assert (gold["noise_4800_pairs_codes"][0] % 2 == 1).all()
    # codebook 3 with row j + 512 equal to row j: every code of codebook 3 is in the upper half
    codes = enc_oracles["tie_halves"].encode(eo.signal("noise", 6400, seed=6))
    assert (codes[3] >= 512).all(), codes[3]
    assert (gold["sine_4801_halves_codes"][3] >= 512).all()


def test_encoder_kernels_have_no_stack_frame():
    table = res_usage()
    want = ["conv1d_short_kernel", "rvq_encode_kernel", "rvq_norms_kernel"] + \
           [f"conv1d_stream_kernelILi{k}ELi{s}E" for k, s in ((4, 2), (8, 4), (10, 5), (16, 8), (7, 1))]
    for frag in want:
        hits = {k: v for k, v in table.items() if frag in k}
        assert len(hits) == 1, f"expected one kernel matching {frag}, found {sorted(hits)}"
        (name, r), = hits.items()
        assert r["stack"] == 0, f"{name}: {r['stack']} bytes of stack"
