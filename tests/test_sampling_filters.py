"""CPU: the top-k / top-p filter of the semantic and coarse stages (DESIGN.md §14).  Its C restatement (tests/sampling_oracle.c),
through the restated stage loops (tests/history_oracle.py, filtered by sampling_oracle.Filtered) on the C oracle, against the
unmodified reference's filtered generations stored in tests/golden/ref_pairs/sampling.npz (tests/golden/make_golden_sampling.py), bit for bit; its top-k against torch.topk;
its top-p against upstream Bark's literal numpy code; and the edge rows the rule spells out."""
import hashlib
import os

import numpy as np
import pytest
import torch
from scipy.special import softmax

import sampling_oracle as SO
from conftest import GOLDEN_DIR, assert_pinned, bits

G = np.load(os.path.join(GOLDEN_DIR, "ref_pairs", "sampling.npz"))
CASES = [str(c) for c in G["cases"]]
NEG_INF = np.float32(-np.inf)


def stored_prompt(key):
    if not int(G[key + "_prompted"]):
        return None
    return {k: G[f"{key}_{k}"] for k in ("semantic_prompt", "coarse_prompt", "fine_prompt")}


def test_stored_cases_cover_the_settings():
    s = {key: SO.stored_settings(G, key) for key in CASES}
    assert s["tiny_f16_k50"]["semantic"] == (50, None) and s["tiny_f16_p09"]["coarse"] == (None, 0.9)
    assert s["tiny_f16_k5p05"]["semantic"] == (5, 0.5) and s["tiny_f16_p0"]["semantic"] == (None, 0.0)
    assert s["tiny_f16_sem_only"]["coarse"] == (None, None) and s["tiny_f16_coarse_only"]["semantic"] == (None, None)
    assert stored_prompt("tiny_f16_prompted") is not None
    assert any(k.startswith("mini_f32") for k in CASES)
    for key in CASES:                                          # a filter changes the ids: the cases are not unfiltered runs
        assert G[key + "_semantic"].size > 0


@pytest.mark.parametrize("key", CASES)
def test_restatement_on_the_oracle_equals_the_reference(orc, weights_file, key):
    config, ftype, _ = key.split("_", 2)
    path = weights_file(config, ftype)
    assert hashlib.sha1(open(path, "rb").read()).hexdigest() == str(G[key + "_weights_sha1"]), "weight generator is not reproducible"
    n_steps = int(G[key + "_n_steps"])
    got = SO.generate(orc.Oracle(path, seed=int(G[key + "_seed"]), n_steps=n_steps), str(G[key + "_text"]), n_steps, stored_prompt(key),
                      SO.stored_settings(G, key))
    for k in ("prompt", "semantic", "coarse", "fine"):
        assert np.array_equal(got[k], G[f"{key}_{k}"]), f"{key}: {k} ids differ from the reference's"
    assert_pinned(got["audio"], G, key + "_audio", f"{key} waveform")
    if key + "_audio" in G.files:
        assert np.array_equal(bits(got["audio"]), bits(G[key + "_audio"]))


def test_filters_change_the_ids(orc, weights_file):
    """The stored k50 case is not what the same seed gives unfiltered (the fixtures exercise the filter)."""
    key = "tiny_f16_k50"
    n_steps = int(G[key + "_n_steps"])
    plain = orc.Oracle(weights_file("tiny", "f16"), seed=int(G[key + "_seed"]), n_steps=n_steps).generate(str(G[key + "_text"]))
    assert not (np.array_equal(plain["semantic"], G[key + "_semantic"]) and np.array_equal(plain["coarse"], G[key + "_coarse"]))


def random_rows(seed):
    rng = np.random.default_rng(seed)
    rows = []
    for n in (2, 7, 1024, 10048):
        rows.append((rng.standard_normal(n) * rng.uniform(0.5, 8)).astype(np.float32))
        rows.append(rng.integers(-4, 5, n).astype(np.float32))                       # many ties
    return rows


@pytest.mark.parametrize("k", [1, 2, 5, 50, 1023, 1024, 5000, 20000])
def test_top_k_is_torch_topk(k):
    for x in random_rows(k):
        got, mask, kept = SO.filter_row(x, top_k=k)
        t = torch.from_numpy(x.copy())
        v = torch.topk(t, min(k, t.numel()))[0][-1]
        t[t < v] = -float("inf")
        assert np.array_equal(bits(got), bits(t.numpy())), (k, x.size)
        assert kept == int(mask.sum()) == int((x >= v.item()).sum())


def upstream_top_p(x, top_p):
    """Upstream Bark's top-p code (generate_text_semantic), with the stable sort the rule fixes for ties."""
    x = x.copy()
    sorted_indices = np.argsort(x, kind="stable")[::-1]
    sorted_logits = x[sorted_indices]
    cumulative_probs = np.cumsum(softmax(sorted_logits))
    sorted_indices_to_remove = cumulative_probs > top_p
    sorted_indices_to_remove[1:] = sorted_indices_to_remove[:-1].copy()
    sorted_indices_to_remove[0] = False
    x[sorted_indices[sorted_indices_to_remove]] = -np.inf
    return x, cumulative_probs


@pytest.mark.parametrize("top_p", [0.05, 0.5, 0.9, 0.99])
def test_top_p_is_upstream_away_from_the_cut(top_p):
    """Upstream's softmax and cumsum round differently from the reference's, so rows whose cut lies within rounding of top_p are
    skipped; every other row must give the same mask."""
    compared = 0
    for x in random_rows(int(top_p * 100)):
        want, c = upstream_top_p(x, top_p)
        if np.abs(c.astype(np.float64) - top_p).min() < 1e-5 * x.size:
            continue
        got, _, _ = SO.filter_row(x, top_p=top_p)
        assert np.array_equal(bits(got), bits(want)), (top_p, x.size)
        compared += 1
    assert compared >= 4


def test_ties_go_by_descending_index():
    x = np.array([1, 3, 3, 0, 3, -1], np.float32)
    _, mask, kept = SO.filter_row(x, top_p=0.0)                  # only sorted position 0: of the tied maxima, the highest index
    assert kept == 1 and mask.tolist() == [0, 0, 0, 0, 1, 0]
    _, mask, _ = SO.filter_row(x, top_k=2)                        # every tie of the 2nd value stays
    assert mask.tolist() == [0, 1, 1, 0, 1, 0]
    p = softmax(x.astype(np.float64))                             # cut after two of the three tied maxima
    _, mask, kept = SO.filter_row(x, top_p=float(np.float32(p[1] * 1.5)))
    assert kept == 2 and mask.tolist() == [0, 0, 1, 0, 1, 0]


def test_signed_zeros_are_equal():
    x = np.array([0.0, -0.0, 0.0, -0.0], np.float32)
    _, mask, _ = SO.filter_row(x, top_p=0.0)
    assert mask.tolist() == [0, 0, 0, 1]                          # -0 at the highest index comes first
    got, mask, _ = SO.filter_row(x, top_p=0.3)                    # c_0 = 0.25 <= 0.3 < c_1: two stay
    assert mask.tolist() == [0, 0, 1, 1] and np.signbit(got[3])


def test_top_p_bounds_and_k_limits():
    rng = np.random.default_rng(3)
    x = rng.standard_normal(1024).astype(np.float32)
    for top_p in (0.0, 1.0):
        got, mask, kept = SO.filter_row(x, top_p=top_p)
        want, _ = upstream_top_p(x, top_p)
        if top_p == 0.0:
            assert kept == 1 and mask[int(np.argmax(x))]
        assert np.array_equal(bits(got), bits(want))
    for k in (1024, 1025, 100000):
        got, _, kept = SO.filter_row(x, top_k=k)
        assert kept == 1024 and np.array_equal(bits(got), bits(x))
    got, mask, kept = SO.filter_row(x, top_k=1)
    assert kept == 1 and mask[int(np.argmax(x))] and (got[~mask] == NEG_INF).all()


def test_both_filters_compose():
    """top-k applies to what top-p left: k beyond the top-p set removes nothing more."""
    rng = np.random.default_rng(4)
    x = (rng.standard_normal(10048) * 3).astype(np.float32)
    _, mp, kp = SO.filter_row(x, top_p=0.5)
    _, mb, kb = SO.filter_row(x, top_k=kp + 10, top_p=0.5)
    assert kb == kp and np.array_equal(mb, mp)
    _, mb, kb = SO.filter_row(x, top_k=3, top_p=0.5)
    assert kb == min(3, kp) and not (mb & ~mp).any()
