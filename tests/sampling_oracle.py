"""ctypes binding of tests/sampling_oracle.c (the top-k / top-p filter restated in C, DESIGN.md §14), compiled on first use into a
per-user temporary directory with the oracle's flags (oracle/Makefile: no FP contraction)."""
from __future__ import annotations

import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

import history_oracle as H

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "sampling_oracle.c")
vp = C.c_void_p

_lib = None


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        h = hashlib.sha1(open(SRC, "rb").read()).hexdigest()[:16]
        out_dir = os.path.join(tempfile.gettempdir(), f"bark_b200_sampling_oracle_{os.getuid()}")
        so = os.path.join(out_dir, f"libsampling_oracle_{h}.so")
        if not os.path.exists(so):
            os.makedirs(out_dir, exist_ok=True)
            tmp = f"{so}.{os.getpid()}.tmp"
            subprocess.check_call(["gcc", "-O2", "-std=gnu11", "-fPIC", "-shared", "-ffp-contract=off", "-fno-fast-math", "-w", SRC, "-o", tmp, "-lm"])
            os.replace(tmp, so)
        L = C.CDLL(so)
        L.orc_filter_row.restype = C.c_int
        L.orc_filter_row.argtypes = [vp, C.c_int, C.c_int, C.c_int, C.c_float, vp]
        _lib = L
    return _lib


def filter_row(logits, top_k=None, top_p=None):
    """orc_filter_row on one row: (filtered float32 row, kept mask as bool, number kept).  top_k None / 0 and top_p None: off."""
    row = np.array(logits, np.float32).reshape(-1)
    mask = np.zeros(row.size, np.uint8)
    kept = lib().orc_filter_row(row.ctypes.data_as(vp), row.size, int(top_k or 0), int(top_p is not None),
                                float(top_p) if top_p is not None else 1.0, mask.ctypes.data_as(vp))
    return row, mask.astype(bool), kept


def stored_settings(G, key):
    """{stage: (top_k or None, top_p or None)} of a case of ref_pairs/sampling.npz (make_golden_sampling.settings_array)."""
    out = {}
    for stage in ("semantic", "coarse"):
        k, p = G[f"{key}_{stage}_filter"]
        out[stage] = (int(k) or None, None if np.isnan(p) else float(p))
    return out


def make_filter(top_k=None, top_p=None):
    """The filter as Filtered takes it (logits -> filtered logits), or None when both are off."""
    if not top_k and top_p is None:
        return None
    return lambda lg: filter_row(lg, top_k, top_p)[0]


class Filtered:
    """A backend of tests/history_oracle.py (oracle.bindings.Ref or Oracle) whose sample() filters the row first when the evaluation
    before it was a stage with a filter: gpt_eval(0, ...) the semantic stage, gpt_eval(1, ...) the coarse stage; fine_eval has none.
    history_oracle's loops evaluate and then sample the row the reference samples (all n_out_vocab logits / the codebook window), so
    every gpt_eval and sample call is still the backend's own and only the mask between them is restated.
    filters: {"semantic": f, "coarse": f}, each f from make_filter (a missing or None entry: that stage unfiltered)."""

    def __init__(self, backend, filters):
        self.b = backend
        self.filters = {0: filters.get("semantic"), 1: filters.get("coarse")}
        self.stage = None

    def gpt_eval(self, which, *a, **k):
        self.stage = which
        return self.b.gpt_eval(which, *a, **k)

    def fine_eval(self, *a, **k):
        self.stage = None
        return self.b.fine_eval(*a, **k)

    def sample(self, logits, temp):
        f = self.filters.get(self.stage)
        return self.b.sample(logits if f is None else f(logits), temp)

    def __getattr__(self, name):                  # tokenize, encodec_decode, ...: the backend's own
        return getattr(self.b, name)


def generate(b, text, n_steps, prompt=None, settings=None):
    """history_oracle.generate on backend b with {stage: (top_k, top_p)} settings applied between evaluation and sampling."""
    filters = {st: make_filter(*kp) for st, kp in (settings or {}).items()}
    return H.generate(Filtered(b, filters), text, n_steps, prompt)
