"""TEST INFRASTRUCTURE — a plain restatement of prompted generation (speaker history prompts, DESIGN.md §12) on the per-call
interface that oracle.bindings.Ref (the unmodified reference) and oracle.bindings.Oracle (the C oracle) both expose: tokenize,
gpt_eval, fine_eval, sample, encodec_decode.

It replays the reference's stage loops (bark.cpp:1645-1701, 1745-1863, 1961-2059): one RNG stream consumed semantic -> coarse ->
fine, every coarse window prefilled from n_past = 0, every fine row sampled in row order.  A history prompt only changes which ids
go into those calls, by upstream Bark's rules:

  semantic  prompt positions [256, 512) are the last 256 ids of S, right-padded with semantic_pad_token
  coarse    Sh = S[-n_sh:] before the semantic ids, Ch = (C flattened)[-n_ch:] minus its last two ids before the coarse ids
  fine      the last min(n_f, 512) frames of F before the coarse frames; windows of 1024 frames advance by 512

With prompt=None every call is the reference's own, so generate() equals the backend's generate() (the first self-check).
The float arithmetic (stc, floorf / roundf / ceilf) is done in float32, as the C code does it.
"""
from __future__ import annotations

import math

import numpy as np

F32 = np.float32
SEMANTIC_VOCAB, SEMANTIC_PAD, SEMANTIC_INFER = 10000, 10000, 129599
CODEBOOK, N_COARSE, N_FINE = 1024, 2, 8
COARSE_SEMANTIC_PAD, COARSE_INFER = 12048, 12050
MAX_COARSE_HISTORY, WINDOW = 630, 60
STC = F32(F32(75.0) / F32(49.9)) * F32(N_COARSE)                  # coarse_rate_hz / semantic_rate_hz * n_coarse_codebooks
MAX_SEMANTIC_HISTORY = int(math.floor(F32(MAX_COARSE_HISTORY) / STC))


def roundf(x) -> int:
    x = float(x)
    return int(math.copysign(math.floor(abs(x) + 0.5), x))


def as_prompt(p):
    """(S [n_s], C [2][n_c], F [8][n_f]) as int32 arrays, or None; accepts the keys of an upstream voice file."""
    if p is None:
        return None
    if isinstance(p, dict) or hasattr(p, "files"):
        p = (p["semantic_prompt"], p["coarse_prompt"], p["fine_prompt"])
    S, C, F = (np.asarray(a, np.int32) for a in p)
    return S.reshape(-1), C.reshape(N_COARSE, -1), F.reshape(N_FINE, -1)


def valid(p) -> bool:
    """The validation rules of bark_b200_set_history_prompt, for the default rates (29 n_s < 20 n_c < 31 n_s)."""
    S, C, F = p
    n_s, n_c = S.size, C.shape[1]
    return (n_s >= 1 and n_c >= 1 and ((S >= 0) & (S < SEMANTIC_VOCAB)).all() and ((C >= 0) & (C < CODEBOOK)).all()
            and ((F >= 0) & (F < CODEBOOK)).all() and 29 * n_s < 20 * n_c < 31 * n_s)


def prompt_ids(b, text, prompt=None):
    """The 513-id semantic prompt."""
    t = np.array(b.tokenize(text), np.int32)
    if prompt is not None:
        hist = prompt[0][-256:]
        t[256:512] = SEMANTIC_PAD
        t[256:256 + hist.size] = hist
    return t


def semantic(b, prompt513, n_steps, temp=0.7, min_eos_p=0.2):
    inp, n_past, out = np.asarray(prompt513, np.int32), 0, []
    for _ in range(n_steps):
        lg, n_past = b.gpt_eval(0, inp, n_past, True)
        t, e = b.sample(lg, temp)                                  # all n_out_vocab logits (quirk D.1)
        if t == SEMANTIC_VOCAB or F32(e) >= F32(min_eos_p):
            break
        out.append(t)
        inp = np.array([t], np.int32)
    return np.array(out, np.int32)


def coarse_history(prompt):
    """(Sh, Ch): the semantic and flat coarse ids the coarse stage puts before its own."""
    if prompt is None:
        return np.zeros(0, np.int32), np.zeros(0, np.int32)
    S, C, _ = prompt
    n_s, n_c = S.size, C.shape[1]
    flat = (C + (SEMANTIC_VOCAB + CODEBOOK * np.arange(N_COARSE, dtype=np.int32))[:, None]).T.reshape(-1)   # c0[0], c1[0], c0[1], ...
    n_sh = min(MAX_SEMANTIC_HISTORY, n_s - n_s % 2, int(math.floor(F32(2 * n_c) / STC)))
    assert n_sh >= 1
    n_ch = roundf(F32(n_sh) * STC)
    return S[-n_sh:], flat[-n_ch:][:-2]


def coarse(b, sem, prompt=None, temp=0.7):
    """Coarse codes [T][2] of the generated frames."""
    Sh, Ch = coarse_history(prompt)
    sem_in = np.concatenate([Sh, np.asarray(sem, np.int32)])
    out = list(Ch)
    n_steps = int(math.floor(F32(len(sem)) * STC / F32(N_COARSE)) * N_COARSE)
    step = 0
    for _ in range(int(math.ceil(n_steps / WINDOW))):
        idx = Sh.size + roundf(F32(step) / STC)
        x = list(sem_in[max(0, idx - MAX_SEMANTIC_HISTORY):][:256])
        x += [COARSE_SEMANTIC_PAD] * (256 - len(x)) + [COARSE_INFER] + out[-MAX_COARSE_HISTORY:]
        inp, n_past = np.array(x, np.int32), 0
        for _ in range(WINDOW):
            if step >= n_steps:
                break
            lg, n_past = b.gpt_eval(1, inp, n_past, False)
            lo = SEMANTIC_VOCAB + (step % N_COARSE) * CODEBOOK
            t = b.sample(lg[lo:lo + CODEBOOK], temp)[0] + lo
            out.append(t)
            inp = np.array([t], np.int32)
            step += 1
    gen = np.array(out[Ch.size:], np.int32).reshape(-1, N_COARSE)
    return gen - (SEMANTIC_VOCAB + CODEBOOK * np.arange(N_COARSE, dtype=np.int32))


def fine_loops(T, H):
    return max(0, -(-(T - (1024 - H)) // 512)) + 1


def fine(b, coarse_Tx2, prompt=None, fine_temp=0.5):
    """Fine codes [T][8] of the generated frames."""
    co = np.asarray(coarse_Tx2, np.int32).reshape(-1, N_COARSE)
    T = co.shape[0]
    F = prompt[2] if prompt is not None else np.zeros((N_FINE, 0), np.int32)
    H = min(F.shape[1], 512)
    n = max(H + T, 1024)
    arr = np.full((n, N_FINE), CODEBOOK, np.int32)
    if H:
        arr[:H] = F[:, -H:].T
    arr[H:H + T, :N_COARSE] = co
    for loop in range(fine_loops(T, H)):
        start, fill = min(loop * 512, n - 1024), min(H + loop * 512, n - 512)
        rel = fill - start
        buf = np.ascontiguousarray(arr[start:start + 1024].T)
        for nn in range(N_COARSE, N_FINE):
            lg = b.fine_eval(buf, nn)
            s = np.array([b.sample(lg[i, :CODEBOOK], fine_temp)[0] for i in range(1024)], np.int32)
            buf[nn, rel:] = s[rel:]
        arr[fill:fill + 1024 - rel, N_COARSE:] = buf[N_COARSE:, rel:].T
    return arr[H:H + T].copy()


def generate(b, text, n_steps, prompt=None, temp=0.7, fine_temp=0.5, min_eos_p=0.2):
    """The whole prompted generation on backend b (its RNG as it stands); returns prompt, semantic, coarse, fine and audio."""
    prompt = as_prompt(prompt)
    p = prompt_ids(b, text, prompt)
    s = semantic(b, p, n_steps, temp, min_eos_p)
    c = coarse(b, s, prompt, temp)
    f = fine(b, c, prompt, fine_temp)
    return dict(prompt=p, semantic=s, coarse=c, fine=f, audio=b.encodec_decode(np.ascontiguousarray(f.T)))


def chained_prompt(g):
    """A finished generation's ids as the next one's prompt (upstream's voice-file layout)."""
    return dict(semantic_prompt=g["semantic"], coarse_prompt=np.ascontiguousarray(g["coarse"].T),
                fine_prompt=np.ascontiguousarray(g["fine"].T))


def coarse_lengths(n_s):
    """The coarse frame counts that align with n_s semantic ids (29 n_s < 20 n_c < 31 n_s); empty for some n_s (3, 5, 7, 9, ...)."""
    return range((29 * n_s) // 20 + 1, -(-31 * n_s // 20))


def random_prompt(rng, n_s, n_f):
    """A valid prompt with n_s semantic ids, an aligned coarse length and n_f fine frames."""
    lengths = coarse_lengths(n_s)
    assert len(lengths), f"no coarse length aligns with {n_s} semantic ids"
    n_c = int(rng.integers(lengths.start, lengths.stop))
    assert 29 * n_s < 20 * n_c < 31 * n_s
    return dict(semantic_prompt=rng.integers(0, SEMANTIC_VOCAB, n_s).astype(np.int32),
                coarse_prompt=rng.integers(0, CODEBOOK, (N_COARSE, n_c)).astype(np.int32),
                fine_prompt=rng.integers(0, CODEBOOK, (N_FINE, n_f)).astype(np.int32))
