"""FAST MODE (BARK_B200_MODE=fast): wgmma GEMM + flash-style attention for the fine model's 1024-row passes (csrc/fast_kernels.cu).

Tensor cores cannot replay the reference's 32 IEEE FMA chains, so this path is validated the way SURVEY.md §7 step 6 prescribes:
  * the two kernels against a float32 numpy evaluation of the same f16 operands (tolerances below),
  * teacher-forced fine passes against the oracle: max |dlogit|, top-1 agreement and the CDF-flip rate (same uniforms, same inputs),
  * a whole generation: semantic / coarse ids stay bit-identical (those stages run the parity kernels), fine ids may differ.
The parity path stays the contract (tests/test_parity_gpu.py); numbers measured here are printed for DESIGN.md / profiles.
"""
import json

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

GEMM_RTOL, GEMM_ATOL = 2e-3, 2e-2          # f16 operands, f32 accumulation in a different order than numpy's
ATT_ATOL = 6e-3                            # probabilities are rounded to f16 before P.V; outputs are O(0.1)
MAX_DLOGIT = 0.08                          # fine logits are O(1-5); f16 activations between layers
MIN_TOP1 = 0.97


@pytest.mark.parametrize("M,N,K", [(1024, 3072, 768), (1024, 2304, 768), (1024, 768, 768), (1024, 768, 3072), (1024, 1056, 768), (257, 2304, 768), (128, 64, 64), (100, 96, 128), (1024, 1024, 4096)])
def test_umma_gemm_matches_numpy(pkg, M, N, K):
    rng = np.random.default_rng(M * 7 + N * 3 + K)
    A = (rng.standard_normal((M, K)) * 0.5).astype(np.float16)
    W = (rng.standard_normal((N, K)) * 0.5).astype(np.float16)
    C = pkg.fast_gemm(A, W)
    ref = A.astype(np.float32) @ W.astype(np.float32).T
    assert np.isfinite(C).all()
    err = np.abs(C - ref)
    assert np.allclose(C, ref, rtol=GEMM_RTOL, atol=GEMM_ATOL), f"max err {err.max():.4f} at {np.unravel_index(err.argmax(), err.shape)}, ref {ref.flat[err.argmax()]:.4f}"


def attention_ref(q, k, v, H):
    n, E = q.shape
    D = E // H
    out = np.zeros((n, E), np.float32)
    for h in range(H):
        s = (q[:, h * D:(h + 1) * D].astype(np.float32) @ k[:, h * D:(h + 1) * D].astype(np.float32).T) / np.sqrt(D)
        p = np.exp(s - s.max(1, keepdims=True))
        p /= p.sum(1, keepdims=True)
        out[:, h * D:(h + 1) * D] = p @ v[:, h * D:(h + 1) * D].astype(np.float32)
    return out


@pytest.mark.parametrize("n,E,H", [(256, 128, 2), (384, 128, 2), (1024, 768, 12), (512, 1024, 16)])
def test_flash_attention_matches_numpy(pkg, n, E, H):
    rng = np.random.default_rng(n + E)
    q, k, v = ((rng.standard_normal((n, E)) * s).astype(np.float16) for s in (1.5, 1.5, 1.0))
    out = pkg.fast_attention(q, k, v, H).astype(np.float32)
    ref = attention_ref(q, k, v, H)
    assert np.isfinite(out).all()
    err = np.abs(out - ref)
    assert err.max() < ATT_ATOL, f"max err {err.max():.5f} (ref magnitude {np.abs(ref).max():.3f}) at {np.unravel_index(err.argmax(), err.shape)}"


@pytest.mark.parametrize("config", ["tiny", "mini"])
def test_fast_fine_passes_teacher_forced(pkg, orc, weights_file, monkeypatch, config):
    path = weights_file(config, "f16")
    o = orc.Oracle(path, seed=0, n_steps=16)
    ref = o.generate("hello world")
    T = ref["fine"].shape[0]
    buf = np.full((8, 1024), 1024, np.int32)
    buf[:, :T] = ref["fine"].T                                   # the oracle's own codes: every pass sees the reference's inputs
    monkeypatch.setenv("BARK_B200_MODE", "fast")
    report = {}
    with pkg.Bark(path, seed=0, n_steps_text_encoder=16) as b:
        assert b.fast_mode
        for nn in range(2, 8):
            lf = b.fine_eval(buf, nn)
            lo = o.fine_eval(buf, nn)
            d = float(np.abs(lf - lo).max())
            top1 = float((lf[:, :1024].argmax(1) == lo[:, :1024].argmax(1)).mean())
            b.reseed(5); tf, _, _ = b.sample_rows(lf[:, :1024].copy(), 0.5)
            b.reseed(5); to, _, _ = b.sample_rows(lo[:, :1024].copy(), 0.5)
            report[nn] = dict(max_dlogit=round(d, 5), top1=round(top1, 4), cdf_flip_rate=round(float((tf != to).mean()), 5))
            assert d < MAX_DLOGIT and top1 >= MIN_TOP1, report
        b.reseed(0)                                               # back to the load-time RNG state: the stream the oracle's generate consumed
        audio = b.generate("hello world")
        assert np.array_equal(b.tokens(0), ref["semantic"]) and np.array_equal(b.tokens(1), ref["coarse"])      # parity stages untouched
        fine = b.tokens(2)
        report["generate"] = dict(fine_ids_equal=round(float((fine == ref["fine"]).mean()), 4), frames=int(T),
                                  wav_rel=round(float(np.abs(audio - ref["audio"]).max() / np.abs(ref["audio"]).max()), 4))
    print("fast-mode agreement", config, json.dumps(report))
