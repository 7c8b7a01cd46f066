"""GPU: the per-op (parity-mode) forward passes against each other and against the oracle.

Every per-op pass runs the same layer loop and output head; what differs is where its K / V rows go (the causal cache, the fine
model's scratch, the batch slots, the row-sharded buffers) and, for quantised weights, the context's q8 activation scratch.  Two
quantised contexts driven from one host thread, their calls interleaved, must each give the oracle's logits; on an f16 model the
causal passes, the batched step and the sharded fine stage must give what the unsharded single run gives.
"""
import numpy as np
import pytest

from conftest import bits

TEXTS = ["hello world", "the quick brown fox", "Hello, world! 123"]


def quantised(pkg, weights_file, tmp_path, qtype, ftype):
    path = str(tmp_path / f"tiny_{qtype}.bin")
    assert pkg.lib().bark_model_quantize(weights_file("tiny", "f16").encode(), path.encode(), ftype)
    return path


@pytest.mark.gpu
def test_interleaved_quantised_contexts(pkg, orc, weights_file, tmp_path):
    """a q4_0 and a q4_1 context (q4_1 also fills the block sums) on one thread: semantic passes, batched coarse steps and fine
    passes alternate between them, and every call equals the oracle bit for bit (a batched row: the oracle's run of its own sequence)"""
    slots = [2, 0, 5]
    rng = np.random.default_rng(11)
    paths = {"q4_0": quantised(pkg, weights_file, tmp_path, "q4_0", 2), "q4_1": quantised(pkg, weights_file, tmp_path, "q4_1", 3)}
    with pkg.Bark(paths["q4_0"]) as b0, pkg.Bark(paths["q4_1"]) as b1:
        runs = []
        for name, b in (("q4_0", b0), ("q4_1", b1)):
            o = orc.Oracle(paths[name], seed=0, n_steps=8)
            runs.append({"name": name, "b": b, "o": o, "rows": [orc.Oracle(paths[name]) for _ in slots], "toks": o.tokenize("Hello, world"), "pg": 0, "po": 0})
        for step in range(4):                                                       # semantic: merged prefill, then single rows
            for r in runs:
                lg, r["pg"] = r["b"].gpt_eval(0, r["toks"], r["pg"], step == 0)
                lo, r["po"] = r["o"].gpt_eval(0, r["toks"], r["po"], step == 0)
                assert r["pg"] == r["po"] and np.array_equal(bits(lg), bits(lo)), f"{r['name']} semantic step {step}"
                r["toks"] = np.array([int(np.argmax(lo[:10000]))], np.int32)
        for r in runs:                                                              # coarse: one prefill per slot, interleaved contexts
            r["np"], r["bt"] = [], []
            for i, slot in enumerate(slots):
                prompt = np.concatenate([rng.integers(0, 10000, 256), [12050], rng.integers(10000, 12048, 3 + 9 * i)]).astype(np.int32)
                lg, p = r["b"].gpt_eval_slot(1, slot, prompt, 0, False)
                lo, po = r["rows"][i].gpt_eval(1, prompt, 0, False)
                assert p == po and np.array_equal(bits(lg), bits(lo)), f"{r['name']} coarse prefill of row {i}"
                r["np"].append(p); r["bt"].append(10000 + int(np.argmax(lo[10000:12048])))
        for step in range(4):
            for r in runs:
                lg, r["np"] = r["b"].gpt_step_batch(1, slots, r["bt"], r["np"])
                for i in range(len(slots)):
                    lo, _ = r["rows"][i].gpt_eval(1, np.array([r["bt"][i]], np.int32), int(r["np"][i]) - 1, False)
                    assert np.array_equal(bits(lg[i]), bits(lo)), f"{r['name']} batched coarse step {step}, row {i}"
                    r["bt"][i] = 10000 + int(np.argmax(lo[10000:12048]))
        buf = rng.integers(0, 1024, (8, 1024)).astype(np.int32); buf[4:, :] = 1024
        for nn in (2, 3):
            for r in runs:
                assert np.array_equal(bits(r["b"].fine_eval(buf, nn)), bits(r["o"].fine_eval(buf, nn))), f"{r['name']} fine pass {nn}"


def semantic_run(b, prompts, n_steps):
    """each prompt's merged prefill, then n_steps greedy single-row steps on the model's own cache: the logits of every call"""
    out = []
    for prompt in prompts:
        lg, p = b.gpt_eval(0, prompt, 0, True)
        seq = [lg]
        for _ in range(n_steps):
            lg, p = b.gpt_eval(0, np.array([int(np.argmax(lg[:10000]))], np.int32), p, False)
            seq.append(lg)
        out.append(seq)
    return out


@pytest.mark.gpu
def test_per_op_paths_agree(pkg, weights_file, monkeypatch):
    """f16: the causal prefill and single-row steps on the per-op kernels (BARK_B200_DECODE=multi), the same sequences as rows of
    batched steps in shuffled slots, and a world-of-one sharded fine stage give the logits, ids and waveform of the single run"""
    path = weights_file("mini", "f16")
    n_steps = 6
    with pkg.Bark(path, seed=3, n_steps_text_encoder=40) as b:
        want_audio = b.generate("hello world"); want_ids = [b.tokens(i).copy() for i in range(3)]
        prompts = [b.tokenize(t).copy() for t in TEXTS]
        want = semantic_run(b, prompts, n_steps)
    assert want_ids[2].shape[0] > 0

    monkeypatch.setenv("BARK_B200_DECODE", "multi")
    with pkg.Bark(path, seed=3, n_steps_text_encoder=40) as b:
        audio = b.generate("hello world")
        assert all(np.array_equal(b.tokens(s), want_ids[s]) for s in range(3)), "per-op decode: ids"
        assert np.array_equal(bits(audio), bits(want_audio)), "per-op decode: waveform"
        have = semantic_run(b, prompts, n_steps)
        for i in range(len(prompts)):
            for k in range(n_steps + 1):
                assert np.array_equal(bits(have[i][k]), bits(want[i][k])), f"per-op decode, prompt {i}, call {k}"
    monkeypatch.delenv("BARK_B200_DECODE")

    slots = [6, 1, 4]
    with pkg.Bark(path, seed=3, n_steps_text_encoder=40) as b:
        n_past, toks = [], []
        for i, prompt in enumerate(prompts):
            lg, p = b.gpt_eval_slot(0, slots[i], prompt, 0, True)
            assert np.array_equal(bits(lg), bits(want[i][0])), f"slot prefill of prompt {i}"
            n_past.append(p); toks.append(int(np.argmax(lg[:10000])))
        for k in range(1, n_steps + 1):
            lg, n_past = b.gpt_step_batch(0, slots, toks, n_past)
            for i in range(len(prompts)):
                assert np.array_equal(bits(lg[i]), bits(want[i][k])), f"batched step {k}, prompt {i} (slot {slots[i]})"
                toks[i] = int(np.argmax(lg[i][:10000]))

    with pkg.Bark(path, seed=3, n_steps_text_encoder=40) as b:
        b.shard_connect(b.shard_init(0, 1))
        audio = b.generate("hello world")
        assert all(np.array_equal(b.tokens(s), want_ids[s]) for s in range(3)), "sharded fine stage: ids"
        assert np.array_equal(bits(audio), bits(want_audio)), "sharded fine stage: waveform"
