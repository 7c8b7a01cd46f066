"""CPU: the oracle's EnCodec ops one at a time (tests/encoder_oracle.c orc_codec_*) and the host libm under them (orc_libm), the
references of tests/test_codec_kernels_gpu.py.

Chained in the order of the reference's decoder (decoder.h) and encoder (encoder.h) on the tiny fixture's codec tensors, they must
reproduce orc_encodec_decode and the latent of orc_encodec_encode bit for bit.  Those two pipelines are pinned to the reference's stored
outputs (tests/test_encodec_api.py, tests/test_encoder.py), so every wrapper is tied to the reference through them.  The host libm
must give the values of tests/golden/libm/glibc_2_39.npz, the reference's glibc 2.39 (tests/golden/make_golden_libm.py)."""
from __future__ import annotations

import numpy as np
import pytest

from conftest import bits
import encodec_oracle as ec
import encoder_oracle as eo

RATIOS = (8, 5, 4, 2)


@pytest.fixture(scope="module")
def tiny(weights_file):
    path = weights_file("tiny", "f16", 1234)
    return path, ec.codec_tensors(path, ec.codec_offset(path))


def _conv(t, name):
    return t[name + ".conv.conv.weight"], t[name + ".conv.conv.bias"]


def _lstm(t, prefix, layer, x, skip=None):
    g = lambda n: t[f"{prefix}.lstm.{n}_l{layer}"]
    return eo.lstm(x, g("weight_ih"), g("weight_hh"), g("bias_ih"), g("bias_hh"), skip)


def decode_chain(t, codes):
    """encodec_forward_quantizer_decode + encodec_forward_decoder (decoder.h:43-113) out of the one-op wrappers."""
    cb = np.stack([t[f"quantizer.vq.layers.{q}._codebook.embed"] for q in range(codes.shape[0])])
    x = eo.rvq_decode(codes, cb)
    y = eo.conv1d(x, *_conv(t, "decoder.model.0"))
    h = _lstm(t, "decoder.model.1", 0, y)
    y = _lstm(t, "decoder.model.1", 1, h, skip=y)
    for b, r in enumerate(RATIOS):
        i = 3 + 3 * b                                        # decoder.model.{3, 6, 9, 12}: transposed conv; {4, 7, 10, 13}: resblock
        u = eo.convtr1d(y, t[f"decoder.model.{i}.convtr.convtr.weight"], t[f"decoder.model.{i}.convtr.convtr.bias"], r)
        sc = eo.conv1d(u, *_conv(t, f"decoder.model.{i + 1}.shortcut"))
        r1 = eo.conv1d(u, *_conv(t, f"decoder.model.{i + 1}.block.1"), elu_in=True)
        y = eo.conv1d(r1, *_conv(t, f"decoder.model.{i + 1}.block.3"), elu_in=True, resid=sc)
    return eo.conv1d(y, *_conv(t, "decoder.model.15"), elu_in=True)[0]


def encode_chain(t, audio):
    """encodec_forward_encoder (encoder.h:39-109) out of the one-op wrappers: the latent [128][T]."""
    y = eo.conv1d(audio[None, :], *_conv(t, "encoder.model.0"))
    for b, r in enumerate(reversed(RATIOS)):
        i = 1 + 3 * b                                        # encoder.model.{1, 4, 7, 10}: resblock; {3, 6, 9, 12}: down-sampling conv
        sc = eo.conv1d(y, *_conv(t, f"encoder.model.{i}.shortcut"))
        r1 = eo.conv1d(y, *_conv(t, f"encoder.model.{i}.block.1"), elu_in=True)
        y = eo.conv1d(r1, *_conv(t, f"encoder.model.{i}.block.3"), elu_in=True, resid=sc)
        y = eo.conv1d(y, *_conv(t, f"encoder.model.{i + 2}"), stride=r, elu_in=True)
    h = _lstm(t, "encoder.model.13", 0, y)
    y = _lstm(t, "encoder.model.13", 1, h, skip=y)
    return eo.conv1d(y, *_conv(t, "encoder.model.15"), elu_in=True)


@pytest.mark.parametrize("T", [7, 16, 33])
def test_decoder_chain_equals_orc_encodec_decode(orc, tiny, T):
    path, t = tiny
    rng = np.random.Generator(np.random.PCG64(T))
    codes = rng.integers(0, 1024, (8, T), dtype=np.int32)
    want = orc.Oracle(path).encodec_decode(codes)
    got = decode_chain(t, codes)
    assert np.array_equal(bits(got), bits(want)), f"T={T}: the chained wrappers differ from orc_encodec_decode"


@pytest.mark.parametrize("n", [1921, 4801])
def test_encoder_chain_equals_orc_encodec_encode(tiny, n):
    path, t = tiny
    audio = eo.signal("noise", n, seed=n)
    _, want = eo.EncoderOracle(path).encode(audio, return_latent=True)
    got = encode_chain(t, audio)
    assert np.array_equal(bits(got), bits(want)), f"n={n}: the chained wrappers differ from orc_encodec_encode's latent"


def test_host_libm_equals_glibc_2_39():
    problem = eo.libm_fixture_mismatch()
    assert problem is None, problem
