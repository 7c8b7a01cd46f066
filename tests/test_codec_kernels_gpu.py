"""GPU: the EnCodec kernels one launcher at a time (bark_b200_codec_*) against the oracle's single ops (tests/encoder_oracle.c orc_codec_*,
pinned by tests/test_codec_oracle_ops.py), bit for bit, and the device libm under them (bark_b200_device_math) against the host's.

Every call is a batch of items of their own lengths, concatenated item by item; item b must equal the oracle on item b alone.  The
hooks lay the weights out with the loader's own routines, make every padding element and every scratch buffer NaN and check guard bands
around every output (a store outside raises GuardBandError).  The shapes are the ones where the kernels can go wrong: each kernel
instantiation at the smallest and largest contraction it takes, the K % 32 leftovers, tile tails (TT = 32 / 128 for the stride-1
convolutions, TF = 16 for the transposed one, TT = 8 / 16 for the strided one, 8 for the LSTM input projection, 128 for the RVQ decode),
every L mod stride of the strided convolution, odd channel chunks, ragged LSTM batches, and every (Cin, Cout, k, stride) of the 24 kHz
model's decoder and encoder.  test_every_instantiation_ran, last in the file, fails when an instantiation has no case.

BARK_B200_LIBM_EXHAUSTIVE=1 makes the libm test walk all 2^32 bit patterns of each function instead of every 256th."""
from __future__ import annotations

import hashlib
import importlib
import os

import numpy as np
import pytest

import __graft_entry__ as graft
from conftest import bits
import encodec_oracle as ec
import encoder_oracle as eo
from make_golden_libm import CUTS          # tests/golden (on the path through encodec_oracle)

pytestmark = pytest.mark.gpu

# every kernel the launchers can run (codec_kernels.h): conv ids as the hook returns them, the transposed conv's NG, the LSTM recurrence
LANE = {(1, 1), (1, 2), (3, 1), (3, 2), (3, 3), (7, 1), (7, 4)}
STREAM = {(4, 2), (8, 4), (10, 5), (16, 8), (7, 1)}
ALL_KERNELS = ({("conv", 1)} | {("conv", 1000 + 10 * kw + ng) for kw, ng in LANE} | {("conv", 10000 + 100 * kw + s) for kw, s in STREAM}
               | {("convtr", 1), ("convtr", 2), ("lstm", 1), ("lstm", 2), ("rvq_decode", 1)})
SEEN: set = set()


def _rng(*key):
    return np.random.Generator(np.random.PCG64(int(hashlib.sha1(repr(key).encode()).hexdigest()[:15], 16)))


def _same(got, want, what):
    got = np.asarray(got, np.float32); want = np.asarray(want, np.float32)
    assert got.shape == want.shape, f"{what}: shape {got.shape} != {want.shape}"
    bad = np.flatnonzero(bits(got).ravel() != bits(want).ravel())
    assert bad.size == 0, (f"{what}: {bad.size} of {got.size} values differ from the oracle; first at flat index {bad[0]}: "
                           f"{got.ravel()[bad[0]]!r} != {want.ravel()[bad[0]]!r}")


def _conv_case(pkg, Cin, Cout, k, stride, Ls, elu_in=False, resid=False, seed=0, what=""):
    """conv1d on items of lengths Ls against orc_codec_conv1d per item; returns the kernel id."""
    rng = _rng("conv", Cin, Cout, k, stride, seed)
    w = (rng.standard_normal((Cout, Cin, k)) / np.sqrt(Cin * k)).astype(np.float16)
    b = rng.standard_normal(Cout).astype(np.float32)
    xs = [rng.standard_normal((Cin, L)).astype(np.float32) for L in Ls]
    rs = [rng.standard_normal((Cout, L)).astype(np.float32) for L in Ls] if resid else None
    got, kid = pkg.codec_conv1d(xs, w, b, stride, elu_in, rs, return_kernel=True)
    SEEN.add(("conv", kid))
    for i, x in enumerate(xs):
        _same(got[i], eo.conv1d(x, w, b, stride, elu_in, None if rs is None else rs[i]), f"{what} conv Cin {Cin} Cout {Cout} k {k} s {stride} item {i} of {Ls}")
    return kid


def _extra(L, k, stride):
    """get_extra_padding_for_conv_1d (ops.cpp:10-16) in float32, as the reference evaluates it: the right reflection's length."""
    f32 = np.float32
    n_frames = (f32(L) - f32(k) + f32(k - stride)) / f32(stride) + f32(1)
    ideal = int((np.ceil(n_frames) - f32(1)) * f32(stride) + (f32(k) - f32(k - stride)))
    return int(f32(ideal) - f32(L))


def _min_len(k, stride):
    """The shortest item strided_conv_1d takes: both reflections (k - stride on the left, the extra padding on the right) inside it."""
    L = 1
    while not (k - stride < L and _extra(L, k, stride) <= L - 1):
        L += 1
    return L


# ---------------------------------------------------------------------------------------------------------------------------------
# stride-1 convolutions: conv1d_short_kernel (K < 32) and conv1d_lane_kernel<KW, NG>
# ---------------------------------------------------------------------------------------------------------------------------------
SHORT_LENGTHS = [7, 8, 127, 128, 129, 256, 257]                   # around TT = 128


@pytest.mark.parametrize("Cin,k", [(1, 7), (16, 1), (2, 7), (4, 7), (10, 3), (31, 1)])
@pytest.mark.parametrize("Cout,elu_in,resid", [(1, False, False), (2, True, False), (3, False, True), (64, True, True)])
def test_short_conv(pkg, Cin, k, Cout, elu_in, resid):
    assert _conv_case(pkg, Cin, Cout, k, 1, SHORT_LENGTHS, elu_in, resid) == 1


def _lane_bounds():
    """(Cin, k, NG) at the smallest and largest Cin each conv1d_lane_kernel<k, NG> takes (K = Cin k >= 32, launcher's NG rule)."""
    out = []
    for kw, ng in sorted(LANE):
        def ng_of(cin):
            groups = ((cin * kw) // 32 + 7) // 8
            if cin * kw < 32:
                return None
            caps = {1: (1, 2), 3: (1, 2, 3), 7: (1, 4)}[kw]
            return next((c for c in caps if groups <= c), None)
        cins = [c for c in range(1, 1200) if ng_of(c) == ng]
        out += [(cins[0], kw, ng), (cins[-1], kw, ng)]
    return out


LANE_LENGTHS = [7, 31, 32, 33, 63, 64, 65, 1000]                  # around TT = 32


@pytest.mark.parametrize("Cin,k,ng", _lane_bounds() + [(33, 1, 1), (48, 3, 1)])
def test_lane_conv(pkg, Cin, k, ng):
    Cout = 33 if Cin * k < 600 else 16                            # an odd channel count where the oracle is cheap
    for i, (elu_in, resid) in enumerate([(False, True), (True, False)]):
        kid = _conv_case(pkg, Cin, Cout, k, 1, [k] + LANE_LENGTHS, elu_in, resid, seed=i)   # L = k: the shortest reflection
        assert kid == 1000 + 10 * k + ng, (Cin, k, kid)


# ---------------------------------------------------------------------------------------------------------------------------------
# strided convolutions: conv1d_stream_kernel<KW, STRIDE>
# ---------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("Cin,Cout,k,stride", [(32, 64, 4, 2), (64, 128, 8, 4), (128, 256, 10, 5), (256, 512, 16, 8), (512, 128, 7, 1),
                                               (32, 33, 4, 2), (256, 33, 16, 8), (160, 33, 7, 1)])
def test_stream_conv(pkg, Cin, Cout, k, stride):
    TT = 8 if stride >= 8 else 16
    L0 = _min_len(k, stride)
    # every L mod stride, at Tout around TT (one full tile and a one-frame tail), and the shortest item accepted
    Ls = [L0] + [stride * TT + r for r in range(stride)] + [stride * (TT + 1) + 1]
    kid = _conv_case(pkg, Cin, Cout, k, stride, Ls, elu_in=True)
    assert kid == 10000 + 100 * k + stride
    assert any(pkg.conv1d_out_len(L, k, stride) > TT for L in Ls)
    # one item too short for its left reflection (k - stride past position 0), refused with nothing launched.  Above stride 1 the hook
    # passes it to the launcher and its right reflection would fit, so the launcher's own left-reflection check is what refuses it
    # (it used to read out of bounds there)
    L = L0 - 1
    assert k - stride >= L and (stride == 1 or _extra(L, k, stride) <= L - 1)
    with pytest.raises(RuntimeError):
        pkg.codec_conv1d([np.zeros((Cin, L), np.float32)], np.zeros((Cout, Cin, k), np.float16), np.zeros(Cout, np.float32), stride)


def test_conv_refusals(pkg):
    z = lambda *s: np.zeros(s, np.float32)
    with pytest.raises(RuntimeError):                              # (k, stride) without an instantiation
        pkg.codec_conv1d([z(32, 40)], np.zeros((8, 32, 6), np.float16), z(8), 3)
    with pytest.raises(RuntimeError):                              # a residual on a strided conv
        pkg.codec_conv1d([z(32, 40)], np.zeros((8, 32, 4), np.float16), z(8), 2, resid=[z(8, 20)])
    with pytest.raises(RuntimeError):                              # k = 1 beyond the lane kernel's two chain groups
        pkg.codec_conv1d([z(544, 40)], np.zeros((8, 544, 1), np.float16), z(8), 1)
    with pytest.raises(RuntimeError):                              # 33 items
        pkg.codec_conv1d([z(32, 8)] * 33, np.zeros((8, 32, 1), np.float16), z(8), 1)


# ---------------------------------------------------------------------------------------------------------------------------------
# transposed convolution: convtr1d_lane_kernel<NG>
# ---------------------------------------------------------------------------------------------------------------------------------
CONVTR_LENGTHS = [7, 15, 16, 17, 33]                               # around TF = 16


@pytest.mark.parametrize("Cin,Cout,stride,ng", [(512, 256, 8, 2), (256, 128, 5, 1), (128, 64, 4, 1), (64, 32, 2, 1),
                                                (32, 17, 2, 1), (288, 33, 5, 2), (256, 7, 8, 1), (480, 2, 4, 2)])
def test_convtr(pkg, Cin, Cout, stride, ng):
    rng = _rng("convtr", Cin, Cout, stride)
    w = (rng.standard_normal((Cin, Cout, 2 * stride)) / np.sqrt(Cin)).astype(np.float16)
    b = rng.standard_normal(Cout).astype(np.float32)
    xs = [rng.standard_normal((Cin, T)).astype(np.float32) for T in CONVTR_LENGTHS]
    got, r = pkg.codec_convtr1d(xs, w, b, stride, return_kernel=True)
    assert r == ng
    SEEN.add(("convtr", r))
    for i, x in enumerate(xs):
        _same(got[i], eo.convtr1d(x, w, b, stride), f"convtr Cin {Cin} Cout {Cout} s {stride} item {i}")


@pytest.mark.parametrize("Cin", [48, 544])
def test_convtr_refusals(pkg, Cin):
    with pytest.raises(RuntimeError):                              # Cin % 32 != 0, or more than two chain groups
        pkg.codec_convtr1d([np.zeros((Cin, 8), np.float32)], np.zeros((Cin, 4, 4), np.float16), np.zeros(4, np.float32), 2)


# ---------------------------------------------------------------------------------------------------------------------------------
# LSTM: lstm_inproj_lane_kernel, then lstm_recur_one_kernel (one item) or lstm_recur_kernel (several)
# ---------------------------------------------------------------------------------------------------------------------------------
_LSTM_W: dict = {}


def _lstm_weights(C):
    if C not in _LSTM_W:
        rng = _rng("lstm", C)
        s = 1.5 / np.sqrt(C)                                       # gates well inside and outside the sigmoid's linear range
        _LSTM_W[C] = ((rng.standard_normal((4 * C, C)) * s).astype(np.float16), (rng.standard_normal((4 * C, C)) * s).astype(np.float16),
                      rng.standard_normal(4 * C).astype(np.float32), rng.standard_normal(4 * C).astype(np.float32))
    return _LSTM_W[C]


def _lstm_case(pkg, C, Ts, skip):
    W = _lstm_weights(C)
    rng = _rng("lstm_x", C, tuple(Ts), skip)
    xs = [(2 * rng.standard_normal((C, T))).astype(np.float32) for T in Ts]
    ss = [rng.standard_normal((C, T)).astype(np.float32) for T in Ts] if skip else None
    got, r = pkg.codec_lstm(xs, *W, skip=ss, return_kernel=True)
    assert r == (1 if len(Ts) == 1 else 2)
    SEEN.add(("lstm", r))
    for i, x in enumerate(xs):
        _same(got[i], eo.lstm(x, *W, None if ss is None else ss[i]), f"LSTM C {C} item {i} of lengths {Ts}")


@pytest.mark.parametrize("C", [32, 128, 512])
@pytest.mark.parametrize("T", [1, 2, 7, 8, 9, 100])
def test_lstm_one_item(pkg, C, T):
    _lstm_case(pkg, C, [T], skip=T % 2 == 0)


RAGGED_32 = [1 + (37 * b) % 100 for b in range(31)] + [100]


@pytest.mark.parametrize("C", [32, 128, 512])
@pytest.mark.parametrize("Ts", [[1, 100], [100, 1], [1, 2, 7, 8, 9, 100, 3], RAGGED_32], ids=["n2", "n2_rev", "n7", "n32"])
@pytest.mark.parametrize("skip", [False, True])
def test_lstm_batched(pkg, C, Ts, skip):
    if C == 512 and len(Ts) == 32:
        Ts = [1 + t % 24 for t in Ts]                              # the oracle's cost; T = 1 still beside the longest
    _lstm_case(pkg, C, Ts, skip)


def test_lstm_refusals(pkg):
    z = np.zeros(4 * 544, np.float32)
    with pytest.raises(RuntimeError):                              # wider than 512
        pkg.codec_lstm([np.zeros((544, 4), np.float32)], np.zeros((4 * 544, 544), np.float16), np.zeros((4 * 544, 544), np.float16), z, z)
    W = _lstm_weights(32)
    with pytest.raises(RuntimeError):                              # 33 items
        pkg.codec_lstm([np.zeros((32, 2), np.float32)] * 33, *W)


# ---------------------------------------------------------------------------------------------------------------------------------
# RVQ decode: rvq_decode_kernel
# ---------------------------------------------------------------------------------------------------------------------------------
def _order_codebooks(n_q, n_bins=1024, hidden=128):
    """Codebook q % 3 == 0 large (about 1e6), 1 tiny (about 1e-3), 2 the exact negative of codebook q - 2, with the codes of q - 2 repeated
    at q.  (B + s) - B and (-B + s) + B both lose s wherever ulp(B) > |s|, so up to n_q = 3 the two orders give the same sums; from
    n_q = 4 on, the next large codebook meets a different partial sum in each order, and the sums depend on the order."""
    rng = _rng("rvq", n_bins, hidden)
    big = (rng.standard_normal((n_bins, hidden)) * 1e6).astype(np.float32)
    small = (rng.standard_normal((n_bins, hidden)) * 1e-3).astype(np.float32)
    return np.stack([(big, small, -big)[q % 3] for q in range(n_q)])


@pytest.mark.parametrize("n_q", range(1, 33))
def test_rvq_decode(pkg, n_q):
    cb = _order_codebooks(n_q)
    rng = _rng("codes", n_q)
    Ts = [1, 127, 128, 129]                                        # around the 128-frame tile
    codes = []
    for T in Ts:
        c = rng.integers(0, 1024, (n_q, T), dtype=np.int32)
        c[:, 0] = 0; c[:, -1] = 1023
        for q in range(2, n_q, 3):
            c[q] = c[q - 2]
        codes.append(c)
    got = pkg.codec_rvq_decode(codes, cb)
    SEEN.add(("rvq_decode", 1))
    for i, c in enumerate(codes):
        _same(got[i], eo.rvq_decode(c, cb), f"RVQ decode n_q {n_q} item {i}")


def test_rvq_decode_refuses_codes_out_of_range(pkg):
    cb = _order_codebooks(2)
    for bad in (-1, 1024):
        c = np.zeros((2, 4), np.int32); c[1, 2] = bad
        with pytest.raises(RuntimeError):
            pkg.codec_rvq_decode([c], cb)


# ---------------------------------------------------------------------------------------------------------------------------------
# ragged batches of 1, 2, 3 and 32 items, tile tails in different places
# ---------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [1, 2, 3, 32])
@pytest.mark.parametrize("Cin,Cout,k,stride", [(16, 32, 1, 1), (256, 128, 3, 1), (128, 512, 7, 1), (32, 64, 4, 2), (256, 512, 16, 8)])
def test_conv_ragged(pkg, n, Cin, Cout, k, stride):
    L0 = max(k, _min_len(k, stride))
    Ls = [L0 + (29 * b + 3 * n) % (40 if Cin * k > 1000 else 140) for b in range(n)]
    _conv_case(pkg, Cin, Cout, k, stride, Ls, elu_in=True, resid=stride == 1, seed=n, what="ragged")


@pytest.mark.parametrize("n", [1, 2, 3, 32])
def test_convtr_ragged(pkg, n):
    rng = _rng("convtr_ragged", n)
    w = (rng.standard_normal((64, 32, 4)) / 8).astype(np.float16)
    b = rng.standard_normal(32).astype(np.float32)
    xs = [rng.standard_normal((64, 1 + (13 * i + n) % 40)).astype(np.float32) for i in range(n)]
    got = pkg.codec_convtr1d(xs, w, b, 2)
    for i, x in enumerate(xs):
        _same(got[i], eo.convtr1d(x, w, b, 2), f"ragged convtr item {i} of {n}")


# ---------------------------------------------------------------------------------------------------------------------------------
# every layer of the 24 kHz model, as the fixture's codec section lays it out (the loader's shapes)
# ---------------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def codec_layers(weights_file):
    path = weights_file("tiny", "f16", 1234)
    return ec.codec_tensors(path, ec.codec_offset(path))


DEC_RATIOS, ENC_RATIOS = (8, 5, 4, 2), (2, 4, 5, 8)


def _model_conv_layers():
    """(name, Cin, Cout, k, stride) of every conv of the 24 kHz decoder and encoder, the shapes the weight writer gives the codec section
    and the loader checks (bark.cpp_b200/weights.py _write_codec), read without writing a file."""
    graft.load_package()                                           # bark_cpp_b200, without its library
    W = importlib.import_module("bark_cpp_b200.weights")

    class Shapes:
        def __init__(self):
            self.shape = {}
        def i32(self, *a):
            pass
        def normal(self, shape, *a):
            return shape
        def tensor(self, name, shape, t):
            self.shape[name] = shape

    rec = Shapes()
    W._write_codec(rec, W.F16, True)
    out = []
    for key, shape in rec.shape.items():
        if not key.endswith(".conv.conv.weight"):
            continue
        name = key[:-len(".conv.conv.weight")]
        Cout, Cin, k = shape
        parts = name.split(".")
        stride = ENC_RATIOS[int(parts[2]) // 3 - 1] if parts[0] == "encoder" and len(parts) == 3 and parts[2] not in ("0", "15") else 1
        out.append((name, Cin, Cout, k, stride))
    return out


@pytest.mark.parametrize("name,Cin,Cout,k,stride", [pytest.param(*c, id=f"{c[0]}-Cin{c[1]}-Cout{c[2]}-k{c[3]}-s{c[4]}")
                                                    for c in _model_conv_layers()])
def test_model_conv_layer(pkg, codec_layers, name, Cin, Cout, k, stride):
    w = codec_layers[name + ".conv.conv.weight"]; b = codec_layers[name + ".conv.conv.bias"]
    assert w.shape == (Cout, Cin, k), (name, w.shape)
    rng = _rng("layer", name)
    L0 = max(k, _min_len(k, stride))
    Ls = [L0, L0 + 17, 3 * L0 + 5] if Cin * k * Cout < 1e6 else [L0, 40]
    xs = [rng.standard_normal((Cin, L)).astype(np.float32) for L in Ls]
    elu_in = name.endswith(("block.1", "block.3")) or name.endswith(".15") or stride > 1
    got, kid = pkg.codec_conv1d(xs, w, b, stride, elu_in, return_kernel=True)
    SEEN.add(("conv", kid))
    for i, x in enumerate(xs):
        _same(got[i], eo.conv1d(x, w, b, stride, elu_in), f"{name} (Cin {Cin} Cout {Cout} k {k} stride {stride}) item {i}")


@pytest.mark.parametrize("b", range(4), ids=[f"decoder.model.{3 * b + 3}-Cin{512 >> b}-Cout{256 >> b}-k{2 * r}-s{r}" for b, r in enumerate(DEC_RATIOS)])
def test_model_convtr_layer(pkg, codec_layers, b):
    name = f"decoder.model.{3 * b + 3}.convtr.convtr"
    w = codec_layers[name + ".weight"]; bias = codec_layers[name + ".bias"]
    assert w.shape == (512 >> b, 256 >> b, 2 * DEC_RATIOS[b]), (name, w.shape)
    rng = _rng("layer", name)
    xs = [rng.standard_normal((w.shape[0], T)).astype(np.float32) for T in (7, 17)]
    got = pkg.codec_convtr1d(xs, w, bias, DEC_RATIOS[b])
    for i, x in enumerate(xs):
        _same(got[i], eo.convtr1d(x, w, bias, DEC_RATIOS[b]), f"{name} (Cin {w.shape[0]} Cout {w.shape[1]} stride {DEC_RATIOS[b]}) item {i}")


@pytest.mark.parametrize("prefix", ["decoder.model.1", "encoder.model.13"])
def test_model_lstm_layers(pkg, codec_layers, prefix):
    rng = _rng("layer", prefix)
    xs = [rng.standard_normal((512, T)).astype(np.float32) for T in (9, 3)]
    for l in range(2):
        W = [codec_layers[f"{prefix}.lstm.{n}_l{l}"] for n in ("weight_ih", "weight_hh", "bias_ih", "bias_hh")]
        got = pkg.codec_lstm(xs, *W, skip=xs if l else None)
        for i, x in enumerate(xs):
            _same(got[i], eo.lstm(x, *W, x if l else None), f"{prefix} layer {l} item {i}")


# ---------------------------------------------------------------------------------------------------------------------------------
# the device libm against the host's, NaN for NaN
# ---------------------------------------------------------------------------------------------------------------------------------
FUNCTIONS = ["expm1f", "tanhf", "expf", "v_expf", "elu", "sigmoid", "round_f16"]
CHUNK = 1 << 24


@pytest.fixture(scope="module")
def host_libm():
    """The device is compared with this host's libm, so the host must be the reference's first (tests/golden/libm/glibc_2_39.npz)."""
    problem = eo.libm_fixture_mismatch()
    assert problem is None, problem


def _compare(pkg, fn, lo, count, stride):
    got = pkg.device_math(fn, lo, count, stride)
    x = eo.pattern_bits(lo, count, stride)
    want = eo.libm(fn, x)
    both_nan = np.isnan(got) & np.isnan(want)
    bad = np.flatnonzero((bits(got) != bits(want)) & ~both_nan)
    if bad.size:
        i = bad[0]
        pytest.fail(f"{fn}: {bad.size} of {count} device results differ from the host libm; first at x = {x[i:i + 1].view(np.float32)[0]!r} "
                    f"(bits {int(x[i]):#010x}): device {got[i]!r}, host {want[i]!r}")
    return count


@pytest.mark.parametrize("fn", FUNCTIONS)
def test_device_libm(pkg, host_libm, fn):
    n = 0
    if os.environ.get("BARK_B200_LIBM_EXHAUSTIVE") == "1":
        for lo in range(0, 1 << 32, CHUNK):
            n += _compare(pkg, fn, lo, CHUNK, 1)
        assert n == 1 << 32
        return
    n += _compare(pkg, fn, 0x5A, CHUNK, 256)                       # every 256th bit pattern
    for c in CUTS:                                                 # the branch cuts of tests/golden/make_golden_libm.py
        for sign in (0, 0x80000000):
            n += _compare(pkg, fn, (sign | c) - (1 << 16), 1 << 17, 1)   # within 2^16 patterns of each cut, both signs
    assert n > CHUNK


# ---------------------------------------------------------------------------------------------------------------------------------
def test_every_instantiation_ran(request):
    """Last in the file: every kernel instantiation the launchers can pick ran in one of the cases above."""
    if not SEEN or request.config.option.keyword:
        pytest.skip("the kernel cases did not all run in this session (run the whole file)")
    missing = ALL_KERNELS - SEEN
    assert not missing, f"kernel instantiations without a case: {sorted(missing)}"
    assert SEEN <= ALL_KERNELS, f"kernels that ran but are not in the list: {sorted(SEEN - ALL_KERNELS)}"
