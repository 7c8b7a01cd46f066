"""CPU restatement of the library's resampling rule (DESIGN.md §16): torchaudio.functional.resample with its defaults (sinc_interp_hann,
lowpass_filter_width 6, rolloff 0.99), taps in double rounded to f32, a sequential double sum over each phase's nonzero taps, and the
channel down-mix of upstream EnCodec's convert_audio.  The GPU's bark_b200_resample must equal it bit for bit."""
import math

import numpy as np

WIDTH, ROLLOFF = 6, 0.99


def rates(sr: int, new_sr: int):
    """(o, q, w, base): sr / g, new_sr / g with g = gcd, the half width w and the cut-off base, as torchaudio derives them."""
    g = math.gcd(sr, new_sr)
    o, q = sr // g, new_sr // g
    base = min(o, q) * ROLLOFF
    return o, q, math.ceil(WIDTH * o / base), base


def out_len(n: int, sr: int, new_sr: int) -> int:
    """L = ceil(q n / o): samples of the resampled clip (n at sr itself when the rates are equal)."""
    o, q, _, _ = rates(sr, new_sr)
    return -(-q * n // o)


def tap(j: int, m: int, o: int, q: int, w: int, base: float) -> float:
    """h[j][m] in double, in torchaudio's expression order, with the C library's sin and cos (the math module)."""
    t = ((-j) / q + (m - w) / o) * base
    t = min(max(t, -WIDTH), WIDTH)
    c = math.cos(t * math.pi / WIDTH / 2)
    win = c * c
    t *= math.pi
    s = 1.0 if t == 0 else math.sin(t) / t
    return s * (win * (base / o))


def dense_taps(sr: int, new_sr: int) -> np.ndarray:
    """Every tap, [q][2w + o] f32 (the whole torchaudio kernel): only for small q (2w + o)."""
    o, q, w, base = rates(sr, new_sr)
    return np.array([[tap(j, m, o, q, w, base) for m in range(2 * w + o)] for j in range(q)], np.float64).astype(np.float32)


def sparse_taps(sr: int, new_sr: int):
    """(first [q], count [q], taps) of each phase's nonzero f32 taps: the candidates |t| < W plus one index on each side (every tap
    outside is the clamped sinc(±6 pi) cos^2(±pi/2), ±0 in f32), trimmed of their ±0 ends.  taps is phase after phase, count[j] values
    from m = first[j]."""
    o, q, w, base = rates(sr, new_sr)
    first, count, taps = np.zeros(q, np.int64), np.zeros(q, np.int64), []
    hi_m = 2 * w + o - 1
    for j in range(q):
        centre = w + o * j / q
        lo = max(0, math.floor(centre - WIDTH * o / base) - 1)
        hi = min(hi_m, math.ceil(centre + WIDTH * o / base) + 1)
        v = [np.float32(tap(j, m, o, q, w, base)) for m in range(lo, hi + 1)]
        a, b = 0, len(v)
        while a < b and v[a] == 0:
            a += 1
        while b > a and v[b - 1] == 0:
            b -= 1
        first[j], count[j] = lo + a, b - a
        taps.extend(v[a:b])
    return first, count, np.array(taps, np.float32)


def downmix(x: np.ndarray) -> np.ndarray:
    """u[i] = (x[i][0] + ... + x[i][C-1]) / C for interleaved [n][C] f32 frames: a sequential f32 sum, then one division."""
    x = np.asarray(x, np.float32)
    if x.ndim == 1:
        return x.copy()
    s = x[:, 0].copy()
    for c in range(1, x.shape[1]):
        s = s + x[:, c]
    return s if x.shape[1] == 1 else s / np.float32(x.shape[1])


def resample(x: np.ndarray, sr: int, new_sr: int, table=None) -> np.ndarray:
    """The rule on interleaved frames x ([n] mono or [n][C]): the down-mix, then y[k q + j] = (float) sum_m u[k o + m - w] h[j][m]
    over phase j's nonzero taps, a double accumulator from 0 in increasing m, zeros outside [0, n).  Equal rates: the down-mix."""
    u = downmix(x)
    if sr == new_sr:
        return u
    o, q, w, _ = rates(sr, new_sr)
    first, count, taps = table if table is not None else sparse_taps(sr, new_sr)
    n = u.size
    L = out_len(n, sr, new_sr)
    ud = u.astype(np.float64)
    offs = np.concatenate([[0], np.cumsum(count)])
    i = np.arange(L, dtype=np.int64)
    k, j = i // q, i % q
    start, cnt, off = k * o + first[j] - w, count[j], offs[j]
    acc = np.zeros(L, np.float64)
    # tap c of every output at once; a phase shorter than c adds u * 0 = ±0, which leaves the sum alone (it is never -0)
    for c in range(int(count.max())):
        h = np.where(c < cnt, taps[np.minimum(off + c, taps.size - 1)], np.float32(0)).astype(np.float64)
        idx = start + c
        acc += np.where((idx >= 0) & (idx < n), ud[np.clip(idx, 0, max(n - 1, 0))], 0.0) * h
    return acc.astype(np.float32)


def bound(x: np.ndarray, sr: int, new_sr: int, y: np.ndarray, table=None) -> np.ndarray:
    """2^-23 sum |h x| + 2^-24 |y| per output: how far a correctly rounded result of the rule may sit from torchaudio's float64 one."""
    u = np.abs(downmix(x))
    first, count, taps = table if table is not None else sparse_taps(sr, new_sr)
    return resample(u, sr, new_sr, (first, count, np.abs(taps))).astype(np.float64) * 2.0 ** -23 * (1 + 2.0 ** -20) + np.abs(y.astype(np.float64)) * 2.0 ** -24


def clip(kind: str, n: int, channels: int = 1, seed: int = 0) -> np.ndarray:
    """Test clips, interleaved [n][channels] f32 (1-D for one channel), regenerated from seeds."""
    rng = np.random.Generator(np.random.PCG64(seed))
    if kind == "noise":
        x = rng.standard_normal((n, channels)).astype(np.float32)
    elif kind == "silent":
        x = np.zeros((n, channels), np.float32)
    elif kind == "full":
        x = np.where(rng.random((n, channels)) < 0.5, -1.0, 1.0).astype(np.float32)
    elif kind == "zeros":                         # +0 and -0
        x = np.where(rng.random((n, channels)) < 0.5, -0.0, 0.0).astype(np.float32)
    elif kind == "subnormal":
        x = (rng.integers(-(1 << 23) + 1, 1 << 23, (n, channels)).astype(np.float64) * 2.0 ** -149).astype(np.float32)
    else:
        raise ValueError(kind)
    return x[:, 0].copy() if channels == 1 else x
