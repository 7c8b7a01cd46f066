"""Static guard on the persistent decode step (no GPU needed): the production instantiations must not spill.

Round 2's largest single gain came from finding that the "prefetched" K / V registers of this 128-register kernel were stack slots —
every LDG followed by an STL of its own result, i.e. every load waited for its data (DESIGN.md §4.1).
`cuobjdump -res-usage` of the built library is cheap to check, so a change that brings spills back fails here instead of on the GPU clock.
"""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "bark.cpp_b200", "libbark_b200.so")
CUOBJDUMP = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"


def res_usage():
    if not os.path.exists(LIB) or not os.path.exists(CUOBJDUMP):
        pytest.skip("library or cuobjdump not available")
    out = subprocess.run([CUOBJDUMP, "-res-usage", LIB], capture_output=True, text=True, check=True).stdout
    table = {}
    for m in re.finditer(r"Function (\S+):\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:(\d+)", out):
        table[m.group(1)] = dict(reg=int(m.group(2)), stack=int(m.group(3)), shared=int(m.group(4)))
    return table


def test_production_decode_step_has_no_stack_frame():
    table = res_usage()
    # bark-small / bark-large: 64-wide heads (DSTEPS = 2), f16 or f32 weights, stamps compiled out (TM = false)
    want = {"f16": "gpt_decode_step_kernelI6__halfLi2ELb0E", "f32": "gpt_decode_step_kernelIfLi2ELb0E"}
    for label, frag in want.items():
        hits = {k: v for k, v in table.items() if frag in k}
        assert len(hits) == 1, f"{label}: expected one instantiation matching {frag}, found {sorted(hits)}"
        (name, r), = hits.items()
        assert r["reg"] <= 128, f"{name}: {r}"            # 512 threads per CTA: 65536 / 512
        assert r["stack"] == 0, f"{name}: {r['stack']} bytes of stack — spills are back on the token's critical path (check LDG -> STL pairs in the SASS)"


def test_q4_decode_step_stack_is_bounded():
    table = res_usage()
    hits = {k: v for k, v in table.items() if "gpt_decode_step_kernel" in k and "Q4ELi2ELb0E" in k}
    assert len(hits) == 1, sorted(hits)
    (name, r), = hits.items()
    assert r["reg"] <= 128 and r["stack"] <= 96, f"{name}: {r}"      # 24 bytes at the end of round 2 (192 before the attention rework)
