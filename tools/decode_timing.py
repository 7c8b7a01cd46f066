#!/usr/bin/env python
"""Per-phase globaltimer stamps of the persistent decode kernel (BARK_B200_DECODE_TIMING=1), on an H100.

usage: python tools/decode_timing.py [--sweep tid:poll_ns,...] [n_past ...]   (coarse model, bark-small f16 bench file;
       tid = stamping thread (lane 0 of a warp), poll_ns = back-off between polls of the tagged exchange words)
Prints, per n_past: the time between consecutive stamps on CTA 0 (median over layers) and, at layer 5, the spread over CTAs
of each stamp.  The raw [256][32] dump is saved to $BARK_TOOLS_OUT/decode_timing_<n_kv>.npy.  Stamp ids: decode_kernels.cu tstamp().
"""
import ctypes as C
import os
import tempfile
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.environ.get("BARK_TOOLS_OUT", os.path.join(tempfile.gettempdir(), "bark_tools"))   # results stay out of the tree
os.makedirs(OUT, exist_ok=True)
sys.path.insert(0, ROOT)
os.environ["BARK_B200_DECODE_TIMING"] = "1"
os.environ.setdefault("BARK_B200_QUIET", "1")
import bench  # noqa: E402
import __graft_entry__ as graft  # noqa: E402

NAMES = {0: "layer start", 1: "LN1 mean", 2: "LN1 done", 3: "QKV rows ready (mbarrier)", 4: "QKV rows done", 6: "K prefetched",
         7: "q arrived", 8: "scores done", 9: "V prefetched + v_new", 10: "scores arrived", 11: "max", 12: "exp", 13: "sum", 14: "x2 arrived", 15: "PV partials",
         16: "P3 done", 17: "att arrived", 18: "c_proj rows ready", 19: "c_proj rows done", 21: "x arrived", 22: "LN2 mean", 23: "LN2 done",
         24: "fc rows ready", 25: "fc rows done", 27: "fc block sync", 28: "ff arrived", 29: "proj rows ready", 30: "proj rows done"}


SUMMARY = []


# exchange -> (stamp after which the stamping warp has published its outputs, stamp at which the consumer holds the whole vector)
EXCHANGES = (("q", 4, 7), ("scores", 8, 10), ("att", 16, 17), ("x1", 19, 21), ("ff", 25, 28), ("x2", 30, 14))


def exchange_table(cta, base, n_kv):
    """Layer 5, over the CTAs that stamp both ends: when the last producer published, when the consumers held the vector, and the gap
    between the last publish and the last consumer (the cost of the exchange itself); the producers' spread is what precedes it.
    The stamping warp must produce in every phase (BARK_B200_DECODE_TIMING_TID=480: warp 15 owns rows of all four row phases)."""
    print(f"   exchange table, layer 5, n_kv {n_kv} (us from the first CTA's layer start)")
    print("   exchange  first publish  last publish  consumer median  consumer last   gap (last publish -> last consumer)")
    for name, prod, cons in EXCHANGES:
        pv, cv = cta[:, prod], cta[:, cons]
        pv, cv = (pv[pv != 0] - base) / 1e3, (cv[cv != 0] - base) / 1e3
        if not len(pv) or not len(cv):
            continue
        print(f"   {name:<8s}  {pv.min():13.2f}  {pv.max():12.2f}  {np.median(cv):15.2f}  {cv.max():13.2f}   {cv.max() - pv.max():6.2f}")
        SUMMARY.append(dict(exchange=name, n_kv=n_kv, first_publish=round(float(pv.min()), 3), last_publish=round(float(pv.max()), 3),
                            consumer_median=round(float(np.median(cv)), 3), consumer_last=round(float(cv.max()), 3), gap=round(float(cv.max() - pv.max()), 3)))


def measure(pkg, path, pasts, tid, poll):
    os.environ["BARK_B200_DECODE_TIMING_TID"] = str(tid)
    os.environ["BARK_B200_POLL_NS"] = str(poll)
    rng = np.random.default_rng(0)
    with pkg.Bark(path) as b:
        L = int(b.hparams(1)[0])
        for n_past in pasts:
            toks = rng.integers(10000, 12048, n_past).astype(np.int32)
            _, p = b.gpt_eval(1, toks, 0, False)
            for _ in range(int(os.environ.get("WARM_STEPS", "48"))):   # warm, then keep the last step's stamps
                _, p = b.gpt_eval(1, np.array([10001], np.int32), p, False)
            t = np.zeros(256 * 32, np.uint64)
            pkg.lib().bark_b200_decode_timing(b.ctx, t.ctypes.data_as(C.c_void_p), t.size)
            t = t.reshape(256, 32).astype(np.int64)
            tag = f"tid{tid}_poll{poll}"
            np.save(os.path.join(OUT, f"decode_timing_{p}_{tag}.npy"), t)
            lay = t[:L + 1]
            SUMMARY.append(dict(tid=tid, poll_ns=poll, n_kv=int(p), us_per_layer=float((lay[L, 0] - lay[0, 0]) / 1e3 / L)))
            print(f"== [{tag}] n_kv {p}: {(lay[L, 0] - lay[0, 0]) / 1e3:.1f} us for {L} layers on CTA 0 ({(lay[L, 0] - lay[0, 0]) / 1e3 / L:.2f} us per layer)")
            used = sorted((i for i in range(32) if lay[1, i] != 0), key=lambda i: (i == 14, i))     # stamp 14 closes the layer
            for a, c in zip(used[:-1], used[1:]):
                d = (lay[:L, c] - lay[:L, a]) / 1e3
                print(f"   -> {c:2d} {NAMES[c]:<28s} median {np.median(d):6.2f} us   min {d.min():6.2f}   max {d.max():6.2f}")
            d = (lay[1:L + 1, 0] - lay[:L, used[-1]]) / 1e3
            print(f"   ->  0 {'x arrived (next layer)':<28s} median {np.median(d):6.2f} us   min {d.min():6.2f}   max {d.max():6.2f}")
            # finer stamps (tstamp2): rows 32 + layer = the four row phases (8 slots each), rows 48 + layer = LN1 / LN2 (16 slots each)
            for row0, groups, names in ((32, ((0, "QKV"), (8, "c_proj"), (16, "fc"), (24, "proj")), {0: "entry", 1: "sched loaded, loop start", 2: "pair row_dot done", 3: "pair emitted", 4: "single row_dot done", 5: "single emitted"}),
                                        (48, ((0, "LN1"), (16, "LN2")), {0: "entry", 1: "warp sums done", 2: "barrier 1 passed", 3: "tree done", 5: "variance warp sums done", 6: "barrier 2 passed", 7: "scale known", 8: "act written", 9: "final barrier passed"})):
                sub = t[row0:row0 + L]
                for g0, gname in groups:
                    idx = [i for i in sorted(names) if sub[1, g0 + i] != 0]
                    if not idx: continue
                    print(f"   [{gname}] stamps relative to entry (median over layers, us): " + "  ".join(f"{names[i]}={np.median((sub[1:L, g0 + i] - sub[1:L, g0 + idx[0]]) / 1e3):.2f}" for i in idx))
            cta = t[64:64 + 132]                             # rows of CTAs beyond the grid stay zero
            base = cta[:, 0][cta[:, 0] != 0].min()
            for c in used:
                col = cta[:, c]; col = col[col != 0]
                v = (col - base) / 1e3
                print(f"   layer5 stamp {c:2d} over {len(v):3d} CTAs: min {v.min():7.2f}  median {np.median(v):7.2f}  max {v.max():7.2f} us   {NAMES[c]}")
            exchange_table(cta, base, int(p))


def main():
    pkg = graft.load_package()
    path = bench.weights_path()
    args = sys.argv[1:]
    sweep = [(int(os.environ.get("BARK_B200_DECODE_TIMING_TID", "0")), int(os.environ.get("BARK_B200_POLL_NS", "40")))]
    if args and args[0] == "--sweep":                        # --sweep tid:poll,tid:poll,...   one context per setting
        sweep = [tuple(int(v) for v in item.split(":")) for item in args[1].split(",")]
        args = args[2:]
    pasts = [int(a) for a in args] or [300, 900]
    os.makedirs(OUT, exist_ok=True)
    for item in sweep:
        measure(pkg, path, pasts, *item)
    import json
    json.dump(SUMMARY, open(os.path.join(OUT, "decode_sweep.json"), "w"), indent=1)


if __name__ == "__main__":
    main()
