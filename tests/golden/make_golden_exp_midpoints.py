"""Regenerates tests/golden/sampler/exp_midpoints.npz — float32 exponent arguments x < 0 whose glibc exp(x) (double) lies within 2^-50
(relative) of a float rounding boundary, the midpoint between two adjacent floats.

    python tests/golden/make_golden_exp_midpoints.py          (about 15 seconds on one core)

The sampler (csrc/sampling.cu) rounds CUDA's double exp of l - max to float, where the reference rounds glibc's.  The two doubles can
round to different floats only next to such a midpoint, so the kernel flags a row when y * (1 -+ 2^-50) round differently.  Every x
here makes that bracket fire; tests/test_sampler_orders.py and tests/test_sampler_gpu.py build sampler rows from them.

Scanned: every float x in [-104, -2^-26] (below -103.98 the float exp is 0; above -2^-26 it rounds to 1 by a wide margin).  numpy's
float64 exp prefilters with a 2^-46 window, glibc's exp (Python's math.exp) decides.  Stored: x (float32), glibc's exp(x) (float64),
and its signed distance to the nearest midpoint in units of the double's ulp.
"""
import math
import os

import numpy as np

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "sampler", "exp_midpoints.npz")
LO_BITS = int(np.float32(-2.0 ** -26).view(np.uint32))       # negative floats: bits grow with the magnitude
HI_BITS = int(np.float32(-104.0).view(np.uint32))


def midpoint_distance(y):
    """y float64 [k] > 0 -> signed distance (float64, exact) from y to the nearest rounding boundary of float32."""
    f = y.astype(np.float32)
    lo = (f.astype(np.float64) + np.nextafter(f, np.float32(-np.inf)).astype(np.float64)) / 2
    hi = (f.astype(np.float64) + np.nextafter(f, np.float32(np.inf)).astype(np.float64)) / 2
    return np.where(np.abs(y - lo) < np.abs(y - hi), y - lo, y - hi)


def main():
    xs = []
    chunk = 1 << 22
    for start in range(LO_BITS, HI_BITS + 1, chunk):
        b = np.arange(start, min(start + chunk, HI_BITS + 1), dtype=np.uint64).astype(np.uint32)
        x = b.view(np.float32)
        y = np.exp(x.astype(np.float64))
        near = np.abs(midpoint_distance(y)) <= y * 2.0 ** -46
        xs.extend(x[near].tolist())
    keep, ys, dist = [], [], []
    for x in xs:
        y = math.exp(float(np.float32(x)))
        d = float(midpoint_distance(np.array([y]))[0])
        if abs(d) <= y * 2.0 ** -50:
            keep.append(x); ys.append(y); dist.append(d / math.ulp(y))
    np.savez(OUT, x=np.array(keep, np.float32), exp=np.array(ys, np.float64), ulps=np.array(dist, np.float64),
             scanned=np.array([LO_BITS, HI_BITS], np.uint32))
    print(f"{len(xs)} prefiltered, {len(keep)} within 2^-50 of a midpoint -> {OUT}")


if __name__ == "__main__":
    main()
