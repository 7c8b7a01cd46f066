"""GPU: what the stage loops report besides their ids.  The progress callback's (step, percent) sequence of a single generate and the
sample counts of the statistics and of each model, derived from the ids the run produced; a batch calls no progress callback, reports
the sum of its items' single-run counts and leaves the models' counters as they were.  The semantic stage runs ahead of its stop test
in chunks of 64 steps, so the cases include stops inside a chunk (the surplus steps must not be counted) and runs to the step limit."""
import numpy as np
import pytest

import history_oracle as H

pytestmark = pytest.mark.gpu

SEMANTIC, COARSE, FINE = 0, 1, 2


def recorder():
    calls = []
    return calls, lambda ctx, step, percent, user: calls.append((step, percent))


def fine_loops(n_frames, n_prompt_fine):
    """Passes of run_fine's outer loop: 1024-frame windows, advanced by 512, behind at most 512 prompt frames."""
    length = max(min(n_prompt_fine, 512) + n_frames, 1024)
    return max(0, -(-(length - 1024) // 512)) + 1


def expected(n_steps, n_semantic, n_coarse, n_prompt_fine=0):
    """(progress calls, (semantic, coarse, fine) sample counts) of one generate that produced these ids.  A semantic stop is a
    sample that is evaluated and counted but not kept."""
    n_eval = n_semantic + (n_semantic < n_steps)
    loops = fine_loops(n_coarse // 2, n_prompt_fine)
    calls = [(SEMANTIC, 100 * k // n_steps) for k in range(1, n_eval + 1)]
    calls += [(COARSE, 100 * (s + 1) // n_coarse) for s in range(n_coarse)]
    calls += [(FINE, 100 * (n * 6 + c) // (loops * 6)) for n in range(loops) for c in range(1, 7)]
    return calls, (n_eval, n_coarse, 1024 * 6 * loops)


def generate(pkg, path, seed, n_steps, text, min_eos_p=None, prompt=None, sampling=None):
    """One generate on a fresh context: its ids, progress calls, statistics and per-model counters."""
    calls, cb = recorder()
    with pkg.Bark(path, seed=seed, n_steps_text_encoder=n_steps, min_eos_p=min_eos_p, progress=cb) as b:
        for stage, (k, p) in (sampling or {}).items():
            b.set_sampling(stage, top_k=k, top_p=p)
        b.generate(text, history_prompt=prompt)
        sem, coarse = b.tokens(0).copy(), b.tokens(1).copy()
        stats, per_model = b.stats()
    return sem, coarse, calls, stats, per_model


def check_single(pkg, path, seed, n_steps, text, **kw):
    sem, coarse, calls, stats, per_model = generate(pkg, path, seed, n_steps, text, **kw)
    prompt = kw.get("prompt")
    n_prompt_fine = prompt["fine_prompt"].shape[1] if prompt is not None else 0
    want_calls, counts = expected(n_steps, sem.size, coarse.size, n_prompt_fine)
    assert calls == want_calls
    assert (stats.n_sample_semantic, stats.n_sample_coarse, stats.n_sample_fine) == counts
    assert tuple(per_model[:, 2]) == counts                      # rows: semantic, coarse, fine; columns: predict us, sample us, samples
    return sem.size, counts


@pytest.mark.parametrize("config,ftype,seed,n_steps,min_eos_p,ids", [
    ("tiny", "f16", 0, 150, 7.0e-6, (1, 62)),                    # stops inside the first 64-step chunk (39 ids)
    ("tiny", "f16", 1, 150, 1.2e-5, (64, 126)),                  # stops inside the second (85 ids)
    ("tiny", "f16", 0, 70, None, (70, 70)),                      # runs to the limit, past one chunk
    ("mini", "f16", 0, 30, None, (30, 30)),
])
def test_single_run_progress_and_sample_counts(pkg, weights_file, config, ftype, seed, n_steps, min_eos_p, ids):
    n_semantic, _ = check_single(pkg, weights_file(config, ftype), seed, n_steps, "hello world", min_eos_p=min_eos_p)
    assert ids[0] <= n_semantic <= ids[1], f"{n_semantic} semantic ids: adjust min_eos_p so the case keeps what it is named for"


def test_history_prompted_run_progress_and_sample_counts(pkg, weights_file):
    prompt = H.random_prompt(np.random.default_rng(46), 120, 40)
    check_single(pkg, weights_file("tiny", "f16"), 3, 24, "hello world", prompt=prompt)


def test_filtered_run_progress_and_sample_counts(pkg, weights_file):
    sampling = {"semantic": (30, None), "coarse": (5, 0.9)}
    check_single(pkg, weights_file("mini", "f16"), 4, 30, "the quick brown fox", sampling=sampling)


def test_batch_counts_are_the_sum_of_its_items_and_call_no_progress(pkg, weights_file):
    path = weights_file("tiny", "f16")
    n_steps, eos = 150, 1.2e-5                                       # seed 1 stops after 85 ids; seeds 0 and 2 keep more than 30
    items = [("hello world", 0), ("hello world", 1), ("hello world", 2)]
    singles = [check_single(pkg, path, seed, n_steps, text, min_eos_p=eos) for text, seed in items]
    assert any(n < n_steps for n, _ in singles), "no item stops early: adjust min_eos_p"
    calls, cb = recorder()
    with pkg.Bark(path, seed=0, n_steps_text_encoder=n_steps, min_eos_p=eos, progress=cb) as b:
        b.generate("hello world")                                    # counters of the context's own run, which the batch must keep
        _, per_model = b.stats()
        del calls[:]
        b.generate_batch([t for t, _ in items], [s for _, s in items])
        stats, per_model_after = b.stats()
    assert calls == []
    assert np.array_equal(per_model, per_model_after)
    assert (stats.n_sample_semantic, stats.n_sample_coarse, stats.n_sample_fine) == tuple(np.sum([c for _, c in singles], axis=0))
