"""CPU: speaker history prompts.  The restatement of prompted generation (tests/history_oracle.py) on the C oracle against the
unmodified reference's prompted generations stored in tests/golden/ref_pairs/history.npz (tests/golden/make_golden_history.py), bit
for bit; the restatement without a prompt against the oracle's own generate(); and the voice-file loader of the Python package."""
import hashlib
import os

import numpy as np
import pytest

import history_oracle as H
from conftest import GOLDEN_DIR, assert_pinned, bits

G = np.load(os.path.join(GOLDEN_DIR, "ref_pairs", "history.npz"))
CASES = [str(c) for c in G["cases"]]


def stored_prompt(key):
    return {k: G[f"{key}_{k}"] for k in ("semantic_prompt", "coarse_prompt", "fine_prompt")}


def check_case(got, key):
    for k in ("prompt", "semantic", "coarse", "fine"):
        assert np.array_equal(got[k], G[f"{key}_{k}"]), f"{key}: {k} ids differ from the reference's"
    assert_pinned(got["audio"], G, key + "_audio", f"{key} waveform")
    if key + "_audio" in G.files:
        assert np.array_equal(bits(got["audio"]), bits(G[key + "_audio"]))


def test_stored_cases_cover_the_limits():
    over = H.as_prompt(stored_prompt("tiny_f16_over"))
    sh, ch = H.coarse_history(over)
    assert over[0].size > 256 and over[2].shape[1] > 512                        # semantic and fine histories trimmed to 256 / 512
    assert sh.size == H.MAX_SEMANTIC_HISTORY == 209 and ch.size < 2 * over[1].shape[1]
    minimal = H.as_prompt(stored_prompt("tiny_f16_minimal"))
    assert (minimal[0].size, minimal[1].shape[1], minimal[2].shape[1]) == (2, 3, 0)
    assert H.coarse_history(minimal)[1].size == 1                               # 3 flat ids, minus the two of the time alignment
    assert H.fine_loops(G["tiny_f16_long_fine"].shape[0], min(G["tiny_f16_long_fine_prompt"].shape[1], 512)) >= 2
    for key in CASES:
        assert H.valid(H.as_prompt(stored_prompt(key))), key


@pytest.mark.parametrize("key", CASES)
def test_restatement_on_the_oracle_equals_the_reference(orc, weights_file, key):
    config, ftype, _ = key.split("_", 2)
    path = weights_file(config, ftype)
    assert hashlib.sha1(open(path, "rb").read()).hexdigest() == str(G[key + "_weights_sha1"]), "weight generator is not reproducible"
    n_steps = int(G[key + "_n_steps"])
    o = orc.Oracle(path, seed=int(G[key + "_seed"]), n_steps=n_steps)
    check_case(H.generate(o, str(G[key + "_text"]), n_steps, stored_prompt(key)), key)


@pytest.mark.parametrize("config,ftype,n_steps", [("tiny", "f16", 16), ("mini", "f32", 12)])
def test_restatement_without_prompt_is_generate(orc, weights_file, config, ftype, n_steps):
    path = weights_file(config, ftype)
    want = orc.Oracle(path, seed=4, n_steps=n_steps).generate("hello world")
    got = H.generate(orc.Oracle(path, seed=4, n_steps=n_steps), "hello world", n_steps)
    for k in ("semantic", "coarse", "fine"):
        assert np.array_equal(got[k], want[k]), k
    assert np.array_equal(bits(got["audio"]), bits(want["audio"]))


def test_chained_prompt_is_the_first_generation(orc, weights_file):
    """The chained case's prompt is exactly what the oracle generates for the first text (upstream's voice-file layout)."""
    from golden.make_golden_history import CHAIN_SEED, CHAIN_TEXT
    p = stored_prompt("tiny_f16_chained")
    g = orc.Oracle(weights_file("tiny", "f16"), seed=CHAIN_SEED, n_steps=int(G["tiny_f16_chained_n_steps"])).generate(CHAIN_TEXT)
    want = H.chained_prompt(g)
    for k in p:
        assert np.array_equal(p[k], want[k]), k


def test_load_history_prompt_reads_a_voice_file(pkg, tmp_path):
    rng = np.random.default_rng(5)
    p = H.random_prompt(rng, 40, 17)
    path = tmp_path / "voice.npz"
    np.savez(path, **{k: v.astype(np.int64) for k, v in p.items()})
    got = pkg.load_history_prompt(str(path))
    for k in p:
        assert got[k].dtype == np.int32 and got[k].flags.c_contiguous and np.array_equal(got[k], p[k]), k
    same = pkg.load_history_prompt({k: np.asfortranarray(v) for k, v in p.items()})
    assert all(np.array_equal(same[k], p[k]) and same[k].flags.c_contiguous for k in p)
    empty_fine = dict(p, fine_prompt=np.zeros((8, 0), np.int64))
    assert pkg.load_history_prompt(empty_fine)["fine_prompt"].shape == (8, 0)


@pytest.mark.parametrize("change", [
    {"semantic_prompt": None}, {"coarse_prompt": None}, {"fine_prompt": None},
    {"semantic_prompt": np.zeros((2, 20), np.int32)}, {"semantic_prompt": np.int32(5)},
    {"coarse_prompt": np.zeros(60, np.int32)}, {"coarse_prompt": np.zeros((3, 30), np.int32)},
    {"fine_prompt": np.zeros((2, 30), np.int32)}, {"fine_prompt": np.zeros((8, 30, 1), np.int32)},
    {"coarse_prompt": np.zeros((2, 30), np.float32)},
])
def test_load_history_prompt_rejects_bad_shapes(pkg, change):
    p = H.random_prompt(np.random.default_rng(6), 20, 30)
    for k, v in change.items():
        if v is None:
            del p[k]
        else:
            p[k] = v
    with pytest.raises(ValueError):
        pkg.load_history_prompt(p)
