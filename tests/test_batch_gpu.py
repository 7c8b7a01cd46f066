"""Batched generation (bark_b200_generate_batch): up to 8 prompts per context, their semantic and coarse decode steps evaluated
together.  Every item must be bit-identical to its own single run.

The free-running checks cannot choose which rows meet in one step, so the batched step is also checked teacher-forced through the
slot hooks: rows whose n_kv sit on both sides of the % 8 (soft_max tail) and % 32 (P.V leftovers) cuts in the same step, slots used
in a permuted order, every row against the oracle following that row's own sequence.
"""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from conftest import FIXTURE_DIR, GOLDEN_DIR, ROOT, bits

QUANT_IDS = {"q4_0": 2, "q8_0": 7}                  # GGML_FTYPE_MOSTLY_*
CONFIGS = [("tiny", "f16", None), ("mini", "f32", None), ("mini", "f16", None), ("tiny", "f16", "q4_0"), ("tiny", "f16", "q8_0")]
TEXTS = ["hello world", "the quick brown fox", "Hello, world! 123", "brown fox the", "world hello the quick", "fox", "quick quick world",
         "the world"]


def model_path(pkg, weights_file, config, ftype, quant):
    src = weights_file(config, ftype)
    if not quant:
        return src
    dst = os.path.join(FIXTURE_DIR, f"{config}_{ftype}_1234_{quant}.bin")
    if not os.path.exists(dst):
        assert pkg.lib().bark_model_quantize(src.encode(), (dst + ".tmp").encode(), QUANT_IDS[quant])      # as tests/test_quantize.py
        os.replace(dst + ".tmp", dst)
    return dst


def ids(cfg):
    return "-".join(c for c in cfg if c)


# ---- 1. teacher-forced batched step ------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("cfg", CONFIGS, ids=ids)
def test_teacher_forced_batched_step_bit_exact(pkg, orc, weights_file, cfg):
    path = model_path(pkg, weights_file, *cfg)
    rng = np.random.default_rng(41)
    slots = [3, 0, 6, 1, 7, 5, 2, 4]                                      # row r uses slot slots[r]
    with pkg.Bark(path) as b:
        # coarse: prompts of 256 + 1 + {1, 5, 31, 32, 37, 63, 64, 90} ids -> n_kv crosses % 8 and % 32 in different rows of one step
        oracles = [orc.Oracle(path) for _ in slots]
        n_past, toks = [], []
        for r, extra in enumerate((1, 5, 31, 32, 37, 63, 64, 90)):
            prompt = np.concatenate([rng.integers(0, 10000, 256), [12050], rng.integers(10000, 12048, extra)]).astype(np.int32)
            lg, p = b.gpt_eval_slot(1, slots[r], prompt, 0, False)
            lo, po = oracles[r].gpt_eval(1, prompt, 0, False)
            assert p == po and np.array_equal(bits(lg), bits(lo)), f"coarse prefill of row {r}"
            n_past.append(p); toks.append(10000 + int(np.argmax(lo[10000:12048])))
        for step in range(45):
            lg, n_past = b.gpt_step_batch(1, slots, toks, n_past)
            for r in range(len(slots)):
                lo, po = oracles[r].gpt_eval(1, np.array([toks[r]], np.int32), int(n_past[r]) - 1, False)
                assert po == n_past[r]
                assert np.array_equal(bits(lg[r]), bits(lo)), \
                    f"coarse step {step}, row {r} (slot {slots[r]}, n_kv {po}): {int((lg[r] != lo).sum())} logits differ, max {np.abs(lg[r] - lo).max():.3e}"
                toks[r] = 10000 + int(np.argmax(lo[10000:12048]))
        # semantic: merged prompts, then each slot advanced by a different number of single-slot steps, so its rows are ragged too
        oracles = [orc.Oracle(path) for _ in slots]
        n_past, toks = [], []
        for r in range(len(slots)):
            prompt = oracles[r].tokenize(TEXTS[r])
            lg, p = b.gpt_eval_slot(0, slots[r], prompt, 0, True)
            lo, po = oracles[r].gpt_eval(0, prompt, 0, True)
            assert p == po and np.array_equal(bits(lg), bits(lo)), f"semantic prefill of row {r}"
            for _ in range(5 * r):
                t = np.array([int(np.argmax(lo[:10000]))], np.int32)
                lg, p = b.gpt_eval_slot(0, slots[r], t, p, False)
                lo, po = oracles[r].gpt_eval(0, t, po, False)
                assert np.array_equal(bits(lg), bits(lo)), f"semantic single-slot step of row {r}"
            n_past.append(p); toks.append(int(np.argmax(lo[:10000])))
        for step in range(40):
            lg, n_past = b.gpt_step_batch(0, slots, toks, n_past)
            for r in range(len(slots)):
                lo, _ = oracles[r].gpt_eval(0, np.array([toks[r]], np.int32), int(n_past[r]) - 1, False)
                assert np.array_equal(bits(lg[r]), bits(lo)), f"semantic step {step}, row {r} (n_kv {n_past[r]}): {int((lg[r] != lo).sum())} logits differ"
                toks[r] = int(np.argmax(lo[:10000]))


# ---- 2. free-running batch == single runs ------------------------------------------------------------------------------------
N_STEPS = 60
SEEDS = [11, 12, 13, 14, 15, 16, 17, 18]


def semantic_lengths(b, items):
    """Semantic ids of each (text, seed) alone, semantic stage only (cheap enough to scan min_eos_p)."""
    out = []
    for text, seed in items:
        b.tokenize(text); b.reseed(seed); b.forward(0)
        out.append(len(b.tokens(0)))
    return out


def ragged_items(pkg, path):
    """Eight (text, seed) items, the seventh repeating the second, and a min_eos_p under which their semantic lengths differ: several
    stop early, at different steps, and at least one runs to N_STEPS (the precondition of the free-running checks)."""
    items = [(TEXTS[i], SEEDS[i]) for i in range(8)]
    items[6] = items[1]
    for eos in np.geomspace(1e-6, 2e-3, 24):
        with pkg.Bark(path, seed=0, n_steps_text_encoder=N_STEPS, min_eos_p=float(eos)) as b:
            lens = semantic_lengths(b, items)
        if len({n for n in lens if n < N_STEPS}) >= 2 and N_STEPS in lens:
            return items, float(eos), lens
    pytest.fail("no min_eos_p gives ragged semantic lengths: extend the scan")


def singles(pkg, path, items, eos):
    """Each item alone: a context with that seed, one generate."""
    res = []
    with pkg.Bark(path, seed=0, n_steps_text_encoder=N_STEPS, min_eos_p=eos) as b:
        for text, seed in items:
            b.reseed(seed)                                               # the state of a fresh context with this seed
            audio = b.generate(text)
            res.append(([b.tokens(s).copy() for s in range(4)], audio))
    return res


def check_batch(b, items, ref, what):
    audios = b.generate_batch([t for t, _ in items], [s for _, s in items])
    assert len(audios) == len(items)
    for i, (toks, audio) in enumerate(ref):
        for s in range(4):
            got = b.batch_tokens(i, s)
            assert got.shape == toks[s].shape and np.array_equal(got, toks[s]), f"{what}: item {i} stage {s} differs from its single run"
        assert audios[i].shape == audio.shape and np.array_equal(bits(audios[i]), bits(audio)), f"{what}: item {i} waveform differs"


def run_free(pkg, path):
    items, eos, lens = ragged_items(pkg, path)
    ref = singles(pkg, path, items, eos)
    assert [len(r[0][0]) for r in ref] == lens
    with pkg.Bark(path, seed=0, n_steps_text_encoder=N_STEPS, min_eos_p=eos) as b:
        check_batch(b, items[:3], ref[:3], "B=3")
        order = [5, 1, 7, 0, 6, 3, 2, 4]                                 # other positions, other partners, the repeated item twice
        check_batch(b, [items[i] for i in order], [ref[i] for i in order], "B=8")
    return lens


@pytest.mark.gpu
@pytest.mark.parametrize("cfg", CONFIGS, ids=ids)
def test_free_running_batch_equals_single_runs(pkg, weights_file, cfg):
    run_free(pkg, model_path(pkg, weights_file, *cfg))


# ---- 3. the bench clip inside a batch ------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_bench_clip_inside_a_batch_matches_the_reference(pkg, weights_file):
    g = np.load(os.path.join(GOLDEN_DIR, "small_f16_n138.npz"))
    path = weights_file("small", "f16", int(g["weight_seed"]))
    texts = ["the quick brown fox", str(g["prompt"]), "world", "hello the fox"]
    seeds = [5, int(g["seed"]), 6, 7]
    with pkg.Bark(path, seed=0, n_steps_text_encoder=int(g["n_steps"])) as b:
        audios = b.generate_batch(texts, seeds)
        assert np.array_equal(b.batch_tokens(1, 3), g["prompt_ids"])
        for stage, key in ((0, "semantic"), (1, "coarse"), (2, "fine")):
            got = b.batch_tokens(1, stage)
            assert got.shape == g[key].shape and np.array_equal(got, g[key]), f"{key} ids differ from the reference's"
        assert audios[1].shape == g["audio"].shape
        assert float(np.abs(audios[1] - g["audio"]).max() / np.abs(g["audio"]).max()) < 1e-3


# ---- 4. host replays inside batched steps ------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_forced_host_replays_inside_a_batch(pkg, weights_file, monkeypatch):
    path = weights_file("tiny", "f16")
    monkeypatch.setenv("BARK_B200_SAMPLE_FLAG_EVERY", "5")
    run_free(pkg, path)


# ---- 5. fast mode ------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("config", ["tiny", "mini"])
def test_fast_mode_batch_equals_single_fast_runs(pkg, weights_file, monkeypatch, config):
    monkeypatch.setenv("BARK_B200_MODE", "fast")
    path = weights_file(config, "f16")
    items = [(TEXTS[i], SEEDS[i]) for i in range(4)]
    ref = singles(pkg, path, items, 0.2)
    with pkg.Bark(path, seed=0, n_steps_text_encoder=N_STEPS) as b:
        assert b.fast_mode
        check_batch(b, items, ref, "fast mode")


# ---- 6. the context's own state ----------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_batch_leaves_the_context_state_alone(pkg, weights_file):
    path = weights_file("mini", "f16")
    with pkg.Bark(path, seed=3, n_steps_text_encoder=40) as b:
        a1 = b.generate("hello world"); t1 = [b.tokens(s).copy() for s in range(4)]
        a2 = b.generate("the quick brown fox"); t2 = [b.tokens(s).copy() for s in range(4)]
    with pkg.Bark(path, seed=3, n_steps_text_encoder=40) as b:
        b.generate("hello world")
        b.generate_batch(["fox", "world the"], [1, 2])
        for s in range(4):
            assert np.array_equal(b.tokens(s), t1[s])
        L = pkg.lib()
        n = L.bark_get_audio_data_size(b.ctx)
        assert np.array_equal(bits(np.ctypeslib.as_array(L.bark_get_audio_data(b.ctx), shape=(n,))), bits(a1))
        a = b.generate("the quick brown fox")
        for s in range(4):
            assert np.array_equal(b.tokens(s), t2[s])
        assert np.array_equal(bits(a), bits(a2))


# ---- 7. arguments ------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_batch_arguments_are_checked(pkg, weights_file):
    import ctypes as C
    L = pkg.lib()
    with pkg.Bark(weights_file("tiny", "f16"), n_steps_text_encoder=12) as b:
        texts = (C.c_char_p * 9)(*([b"hello"] * 9))
        seeds = (C.c_uint32 * 9)(*range(9))
        assert L.bark_b200_generate_batch(b.ctx, texts, seeds, 0, 1) is False
        assert L.bark_b200_generate_batch(b.ctx, texts, seeds, 9, 1) is False
        assert L.bark_b200_generate_batch(b.ctx, None, seeds, 2, 1) is False
        assert L.bark_b200_generate_batch(b.ctx, texts, None, 2, 1) is False
        holed = (C.c_char_p * 2)(b"hello", None)
        assert L.bark_b200_generate_batch(b.ctx, holed, seeds, 2, 1) is False
        assert L.bark_b200_generate_batch(None, texts, seeds, 2, 1) is False
        assert L.bark_b200_batch_audio(b.ctx, 0, None, 0) == -1                  # no batch yet
        b.generate_batch(["hello", "world"], [1, 2])
        assert L.bark_b200_batch_audio(b.ctx, 1, None, 0) > 0
        for i in (-1, 2, 8):
            assert L.bark_b200_batch_audio(b.ctx, i, None, 0) == -1
            assert L.bark_b200_batch_tokens(b.ctx, i, 0, None, 0) == -1
        assert L.bark_b200_batch_tokens(b.ctx, 0, 4, None, 0) == -1
        kept = [b.batch_tokens(i, 0).copy() for i in range(2)]
        assert L.bark_b200_generate_batch(b.ctx, texts, seeds, 9, 1) is False                 # a refused batch keeps the last results
        with pytest.raises(RuntimeError):
            b.generate_batch(["hello"], [1, 2])                                               # more seeds than prompts
        assert all(np.array_equal(b.batch_tokens(i, 0), kept[i]) for i in range(2))
        with pytest.raises(RuntimeError):
            b.gpt_step_batch(1, [0, 0], [10001, 10002], [300, 300])             # one slot twice
        with pytest.raises(RuntimeError):
            b.gpt_eval_slot(1, 8, [10001], 0, False)                             # no slot 8


@pytest.mark.gpu
def test_failed_batch_changes_nothing(pkg, weights_file):
    """min_eos_p = 0 stops every item at its first semantic sample, so the coarse stage has nothing to generate and the batch fails
    after the semantic stage ran: the statistics and the (absent) results must be as before."""
    with pkg.Bark(weights_file("tiny", "f16"), n_steps_text_encoder=12, min_eos_p=0.0) as b:
        before, per_model = b.stats()
        with pytest.raises(RuntimeError):
            b.generate_batch(["hello", "world"], [1, 2])
        after, per_model_after = b.stats()
        assert bytes(before) == bytes(after) and np.array_equal(per_model, per_model_after)
        assert pkg.lib().bark_b200_batch_audio(b.ctx, 0, None, 0) == -1


@pytest.mark.gpu
def test_sharded_context_refuses_a_batch_one_rank(pkg, weights_file):
    """A context whose fine stage is sharded (here a world of one rank: shard_init + shard_connect with its own handle) refuses."""
    with pkg.Bark(weights_file("tiny", "f16"), n_steps_text_encoder=12) as b:
        h = b.shard_init(0, 1)
        b.shard_connect(h)
        with pytest.raises(RuntimeError):
            b.generate_batch(["hello", "world"], [1, 2])


def _sharded_rank(rank, path, handles_out, handles_in, result):
    import sys
    sys.path.insert(0, ROOT)
    import __graft_entry__ as graft
    pkg = graft.load_package()
    try:
        with pkg.Bark(path, n_steps_text_encoder=12, device=rank) as b:
            handles_out.put((rank, b.shard_init(rank, 2)))
            b.shard_connect(handles_in.get(timeout=120))
            try:
                b.generate_batch(["hello", "world"], [1, 2])
                result.put((rank, "accepted"))
            except RuntimeError:
                result.put((rank, "refused"))
    except Exception as e:                                                  # surfaces in the asserting process
        result.put((rank, repr(e)))


@pytest.mark.gpu
def test_sharded_context_refuses_a_batch_two_gpus(pkg, weights_file):
    """The same with two ranks on two GPUs, one process each (CUDA IPC handles cannot be opened in the process that made them)."""
    import multiprocessing as mp
    from conftest import cuda_device_count
    if cuda_device_count() < 2:
        pytest.skip("needs two GPUs")
    path = weights_file("tiny", "f16")
    ctx = mp.get_context("spawn")
    out, result = ctx.Queue(), ctx.Queue()
    ins = [ctx.Queue() for _ in range(2)]
    procs = [ctx.Process(target=_sharded_rank, args=(r, path, out, ins[r], result)) for r in range(2)]
    for p in procs:
        p.start()
    got = dict(out.get(timeout=300) for _ in procs)
    for q in ins:
        q.put(got[0] + got[1])
    res = dict(result.get(timeout=300) for _ in procs)
    for p in procs:
        p.join(120)
    assert res == {0: "refused", 1: "refused"}, res


# ---- 8. resources (CPU) ------------------------------------------------------------------------------------------------------
def test_batched_step_kernels_do_not_spill():
    lib = os.path.join(ROOT, "bark.cpp_b200", "libbark_b200.so")
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(lib) or not os.path.exists(cuobjdump):
        pytest.skip("library or cuobjdump not available")
    out = subprocess.run([cuobjdump, "-res-usage", lib], capture_output=True, text=True, check=True).stdout
    table = {m.group(1): int(m.group(2)) for m in re.finditer(r"Function (\S+):\s*\n\s*REG:\d+ STACK:(\d+)", out)}
    for frag, count in (("attn_scores_batch_kernel", 4), ("attn_softmax_batch_kernel", 1), ("attn_pv_batch_kernel", 1),
                        ("embed_causal_kernel", 1), ("embed_causal_q_kernel", 1)):
        hits = {k: v for k, v in table.items() if frag in k}
        assert len(hits) == count, f"{frag}: {sorted(hits)}"
        for name, stack in hits.items():
            assert stack == 0, f"{name}: {stack} bytes of stack"
