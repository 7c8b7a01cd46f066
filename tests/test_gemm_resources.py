"""Static guard on the parity path's tiled GEMM (no GPU needed): every f16 block-tile instantiation of lane_gemm_tiled_kernel keeps
its accumulators and operand words in registers (no stack frame) within the register budget its occupancy needs:
65536 / (threads per CTA x CTAs per SM)."""
import re

from test_decode_resources import res_usage


def test_f16_gemm_tiles_fit_their_register_budget():
    table = res_usage()
    hits = {k: v for k, v in table.items() if "lane_gemm_tiled_kernelI6__half" in k}
    found = set()
    for name, r in hits.items():
        wm, wo, ot, minb = (int(x) for x in re.search(r"TileCfgILi(\d+)ELi(\d+)ELi(\d+)ELi(\d+)E", name).groups())
        found.add((wm, wo, ot, minb))
        budget = 65536 // (32 * wm * wo * minb)
        assert r["reg"] <= budget and r["stack"] == 0, f"{name}: {r}, budget {budget} registers"
    assert found == {(4, 2, 8, 2), (4, 4, 8, 1)}, sorted(found)


def test_f32_gemm_tile_stack_is_bounded():
    # f32 operand words are twice as wide: the 32 x 16 tile's 128 registers hold 64 accumulators and 64 operand registers, so a few
    # values live on the stack; 16 bytes (24 before the branch-free inner loop) is the bound
    table = res_usage()
    hits = {k: v for k, v in table.items() if "lane_gemm_tiled_kernelIf" in k}
    assert len(hits) == 1, sorted(hits)
    (name, r), = hits.items()
    assert "TileCfgILi4ELi2ELi8ELi2E" in name, name
    assert r["reg"] <= 128 and r["stack"] <= 16, f"{name}: {r}"
