"""Writes tests/golden/resample/torchaudio.npz from torchaudio (run where torchaudio is installed; no test imports it):
  - <sr>_<new_sr>_first / _count / _taps: torchaudio's float64 sinc_interp_hann kernel (width 6, rolloff 0.99) rounded to f32, each
    phase's span from its first to its last nonzero tap, phase after phase (the generator checks that every other tap is ±0);
  - <sr>_<new_sr>_n<n>: torchaudio.functional.resample of the float64 noise clip resample_oracle.clip("noise", n, seed=n), whole, for
    the short lengths; for 10 s, the outputs at _n<n>_idx (a stride of 401 plus both ends), the total length in _n<n>_len.
    python tests/golden/make_golden_resample.py"""
import math
import os
import sys

import numpy as np
import torch
import torchaudio
import torchaudio.functional as F
from torchaudio.functional.functional import _get_sinc_resample_kernel

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import resample_oracle as ro  # noqa: E402

PAIRS = [(sr, 24000) for sr in (8000, 11025, 16000, 22050, 32000, 44100, 44056, 48000, 96000)] + [(24000, 44100), (24000, 48000)]
SHORT = (1, 2, 3, 1920, 1921)


def main():
    out = {"torchaudio_version": np.array(torchaudio.__version__)}
    for sr, nsr in PAIRS:
        key = f"{sr}_{nsr}"
        g = math.gcd(sr, nsr)
        k, _ = _get_sinc_resample_kernel(sr, nsr, g, ro.WIDTH, ro.ROLLOFF, "sinc_interp_hann", None, "cpu", torch.float64)
        k = k[:, 0, :].numpy().astype(np.float32)
        first, count, taps = [], [], []
        for row in k:
            nz = np.flatnonzero(row)
            first.append(nz[0]); count.append(nz[-1] - nz[0] + 1)
            taps.append(row[nz[0]:nz[-1] + 1])
            rest = np.concatenate([row[:nz[0]], row[nz[-1] + 1:]])
            assert not rest.any()
        out[f"{key}_first"] = np.array(first, np.int32)
        out[f"{key}_count"] = np.array(count, np.int32)
        out[f"{key}_taps"] = np.concatenate(taps)
        for n in SHORT + (10 * sr,):
            y = F.resample(torch.from_numpy(ro.clip("noise", n, seed=n).astype(np.float64)), sr, nsr).numpy()
            assert y.size == ro.out_len(n, sr, nsr)
            if n in SHORT:
                out[f"{key}_n{n}"] = y
            else:
                idx = np.unique(np.concatenate([np.arange(0, y.size, 401), np.arange(512), np.arange(y.size - 512, y.size)]))
                out[f"{key}_n{n}_idx"] = idx.astype(np.int32)
                out[f"{key}_n{n}"] = y[idx]
                out[f"{key}_n{n}_len"] = np.array(y.size)
    np.savez_compressed(os.path.join(os.path.dirname(os.path.abspath(__file__)), "resample", "torchaudio.npz"), **out)


if __name__ == "__main__":
    main()
