"""Regenerates tests/golden/small_f32_n12.npz — BASELINE.json configs[0] at its true size: bark-small dimensions, f32 GPT + f16 codec,
one prompt, seed 0, the UNMODIFIED reference (oracle/_ref/libbark_ref.so) at -t 4, n_steps_text_encoder = 12 (a 15 s CPU run).

    python tests/golden/make_golden_small.py          (needs the reference build oracle/_ref)

The 1.6 GB weight file is not committed: bark.cpp_b200/weights.py regenerates it bit-identically from (config, ftype, seed); its sha1
is stored in the fixture.
"""
import hashlib
import importlib
import os
import tempfile
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
os.environ.setdefault("BARK_B200_QUIET", "1")
import __graft_entry__ as graft  # noqa: E402


def main():
    graft.load_package()
    weights = importlib.import_module("bark_cpp_b200.weights")
    orc = graft.load_oracle_bindings()
    tmp = os.environ.get("BARK_B200_FIXTURES", os.path.join(tempfile.gettempdir(), f"bark_b200_fixtures_{os.getuid()}"))
    os.makedirs(tmp, exist_ok=True)
    path = os.path.join(tmp, "small_f32_1234.bin")
    if not os.path.exists(path):
        weights.write_weights(path, weights.small(weights.F32), 1234)
    h = hashlib.sha1()
    with open(path, "rb") as f:
        for blk in iter(lambda: f.read(1 << 24), b""):
            h.update(blk)
    prompt = "hello world"
    r = orc.Ref(path, seed=0, n_steps=12)
    out = r.generate(prompt, n_threads=4)
    np.savez_compressed(
        os.path.join(os.path.dirname(os.path.abspath(__file__)), "small_f32_n12.npz"),
        config="small", ftype="f32", quant="", weight_seed=1234, seed=0, n_steps=12, prompt=prompt, reference_build=r.build_info(),
        weights_sha1=h.hexdigest(), prompt_ids=r.tokenize(prompt), semantic=out["semantic"], coarse=out["coarse"], fine=out["fine"], audio=out["audio"],
        note="BASELINE configs[0]: bark-small dimensions, f32 GPT + f16 codec, 1 prompt, seed 0, reference at -t 4; n_steps_text_encoder=12 keeps the CPU run short")
    print("semantic", out["semantic"].size, "frames", out["coarse"].shape[0], "audio", out["audio"].size)


if __name__ == "__main__":
    main()
