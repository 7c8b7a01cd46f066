"""CPU: the decode step's regime thresholds (tests/decode_regimes.py) and the coverage of tests/test_long_context_gpu.py's bands."""
import pytest

import decode_regimes as dr

M = dr.MODELS


def test_constants_read_from_the_kernel():
    assert dr.K_THREADS == 512 and dr.K_WARPS == 16
    assert dr.K_HALF_SLOT_BYTES == 6144 and dr.K_MAX_TASKS == 8 and dr.CAP_TASKS == 16
    assert dr.SPLIT_SCORE_CTAS == 64


def test_cta_count():
    assert dr.launch_ctas(132) == 128                          # H100 SXM
    assert dr.launch_ctas(114) == 114                          # H100 PCIe
    assert dr.launch_ctas(132, 97) == 97 and dr.launch_ctas(132, 64) == 64
    assert dr.launch_ctas(132, 63) == 128 and dr.launch_ctas(132, 129) == 128      # outside [64, n_sm]: ignored
    assert dr.launch_ctas(114, 128) == 114


def test_split_boundaries():
    assert dr.layout(M["wide_f16"], 128).split and not dr.layout(M["wide_f16"], 127).split          # 64 soft_max + 64 score CTAs
    assert dr.layout(M["wide_f16"], dr.launch_ctas(114)).score_cta0 == 0                             # bark-large on a 114-SM card
    assert dr.layout(M["tiny_f16"], 72).split and not dr.layout(M["tiny_f16"], 71).split            # 8 soft_max tiles
    assert dr.layout(M["small2_f32"], 112).split and not dr.layout(M["small2_f32"], 111).split
    with pytest.raises(ValueError):
        dr.layout(M["wide_f16"], 63)


def first_beyond(name, G):
    lay = dr.layout(M[name], G)
    return lay.first(lambda n: lay.beyond_cap(n).any())


def first_v_global(name, G):
    lay = dr.layout(M[name], G)
    return lay.first(lambda n: not lay.vs_ok(n).all())


def test_bark_large_f16_keys_beyond_the_tail_from_514():
    lay = dr.layout(M["wide_f16"], 128)
    assert set(lay.cap.ravel()) == {8}                     # (6144 - 4096) / 256: behind two fc rows of 2048 bytes
    assert lay.nw == 1024
    assert first_beyond("wide_f16", 128) == 514            # 16 * n_past > 8 * 1024
    assert not lay.beyond_cap(513).any() and lay.beyond_cap(514).any()


def test_v_from_global_thresholds():
    assert first_v_global("small2_f32", 128) == 769        # bark-small f32: one 3072-byte c_proj row + 24 V steps
    assert first_v_global("wide_f32", 128) == 513          # bark-large f32: one 4096-byte row + 16 V steps
    assert first_v_global("wide_f16", 128) is None         # bark-large f16: one 2048-byte row + 32 steps = exactly 6144 at n_kv 1024
    lay = dr.layout(M["wide_f16"], 128)
    assert int((lay.voff + 32 * 128).max()) == dr.K_HALF_SLOT_BYTES


def test_unsplit_grids_take_every_score_task_from_global():
    for name, G in (("wide_f16", 127), ("tiny_f16", 71), ("wide_f16", 64)):
        lay = dr.layout(M[name], G)
        assert lay.score_cta0 == 0 and not lay.cap.any() and lay.beyond_cap(2).any()


def test_regime_labels():
    assert dr.regimes(M["wide_f16"], 128, 1024) == {"split", "K staged + beyond cap", "V staged", "no tail", "last position"}
    assert dr.regimes(M["wide_f32"], 128, 513) == {"split", "K staged only", "V from global", "n_kv % 8 tail"}
    assert dr.regimes(M["tiny_f16"], 71, 520) == {"unsplit", "K from global only", "V staged", "n_kv % 32 tail"}


def test_bands_reach_every_regime_of_each_weight_type():
    """The coverage map: for each weight type of the GPU table, every regime its models can take (any CTA count from 64 to 128, any
    n_kv) is taken by at least one band.  A retuned staging slot moves the thresholds; then the bands must move with them."""
    can, did = dr.reachable(), dr.reached()
    assert set(can) == set(did) == {"f16", "f32", "q4_0"}
    for wt in sorted(can):
        print(wt, "reached:", ", ".join(sorted(did[wt])))
        assert can[wt] <= did[wt], f"{wt}: no band reaches {sorted(can[wt] - did[wt])}"
    assert "V from global" in did["f32"] and "K staged + beyond cap" in did["f16"]


def test_band_steps_cross_the_thresholds():
    for name, ctas, kv in (("wide_f16", 128, 514), ("wide_f32", 128, 513), ("small2_f32", 128, 769)):
        G, starts = dr.BANDS[name]
        assert ctas in G and any(s < kv <= s + dr.BAND_STEPS - 1 for s in starts), name
    for name, (_, starts) in dr.BANDS.items():
        assert max(starts) + dr.BAND_STEPS - 1 == dr.BLOCK_SIZE, f"{name}: no band ends at the last position"
