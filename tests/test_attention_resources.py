"""Static guard on the parity path's multi-row attention kernel (no GPU needed): every head-size instantiation keeps its query row
and 32 lane chains in registers, so a stack frame would mean spills inside the scores loop."""
from test_decode_resources import res_usage


def test_attention_kernel_has_no_stack_frame():
    table = res_usage()
    hits = {k: v for k, v in table.items() if "attn_fused_kernel" in k}
    assert sorted(k.split("attn_fused_kernel")[1][:5] for k in hits) == ["ILi1E", "ILi2E", "ILi3E", "ILi4E"], sorted(hits)
    for name, r in hits.items():
        assert r["reg"] <= 255 and r["stack"] == 0, f"{name}: {r}"
