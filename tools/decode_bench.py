#!/usr/bin/env python
"""Average device time of the production decode-step kernel (no stamps) under different exchange knobs, on an H100.

usage: python tools/decode_bench.py [--n-past 300,900] poll_ns[/q:att:x1:ff:x2:scores] [...]
One context per setting: BARK_B200_POLL_NS = poll_ns and, where given, BARK_B200_HEADSTART = the head starts (ns) after the slash.
60 single-token steps of the coarse model of the bark-small f16 bench file per context length, timed with the library's CUDA-event profiler
(bark_b200_profile_report).  Writes $BARK_TOOLS_OUT/decode_bench.json.
"""
import json
import os
import tempfile
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.environ.get("BARK_TOOLS_OUT", os.path.join(tempfile.gettempdir(), "bark_tools"))   # results stay out of the tree
os.makedirs(OUT, exist_ok=True)
sys.path.insert(0, ROOT)
os.environ.setdefault("BARK_B200_QUIET", "1")
import bench  # noqa: E402
import __graft_entry__ as graft  # noqa: E402


def main():
    pkg = graft.load_package()
    path = bench.weights_path()
    args = sys.argv[1:]
    pasts = [300, 900]
    if args and args[0] == "--n-past":
        pasts = [int(v) for v in args[1].split(",")]; args = args[2:]
    out = []
    rng = np.random.default_rng(0)
    for item in args or ["40"]:
        poll, _, headstart = item.partition("/")
        os.environ["BARK_B200_POLL_NS"] = poll
        if headstart: os.environ["BARK_B200_HEADSTART"] = headstart
        else: os.environ.pop("BARK_B200_HEADSTART", None)
        with pkg.Bark(path) as b:
            for n_past in pasts:
                toks = rng.integers(10000, 12048, n_past).astype(np.int32)
                _, p = b.gpt_eval(1, toks, 0, False)
                for _ in range(5):
                    _, p = b.gpt_eval(1, np.array([10001], np.int32), p, False)
                pkg.profile_enable(True)
                for _ in range(60):
                    _, p = b.gpt_eval(1, np.array([10001], np.int32), p, False)
                rep = pkg.profile_report()
                pkg.profile_enable(False)
                v = rep["gpt_decode_step_kernel"]
                us = v["ms"] * 1e3 / v["launches"]
                out.append(dict(poll_ns=int(poll), headstart=headstart or "default", n_kv_start=n_past + 6, us_per_token=round(us, 2), launches=v["launches"]))
                print(f"poll {poll:>5s} headstart {headstart or 'default'}  n_kv {n_past + 6:4d}..{p:4d}: {us:7.2f} us per decode step", flush=True)
    os.makedirs(OUT, exist_ok=True)
    json.dump(out, open(os.path.join(OUT, "decode_bench.json"), "w"), indent=1)


if __name__ == "__main__":
    main()
