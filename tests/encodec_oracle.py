"""The EnCodec encode at any number of codebooks on the CPU restatement: the latent of tests/encoder_oracle.c's orc_encodec_encode,
quantised by its orc_rvq_encode over the weight file's codebooks 0..n_q-1 (encodec_forward_quantizer_encode, quantizer.h:20-76).
Also the reference's n_q rule (encodec.cpp/utils.h:22-30 as encodec.cpp:650-651 calls it)."""
from __future__ import annotations

import math
import os
import struct
import sys

import numpy as np

import encoder_oracle as eo

sys.path.insert(0, os.path.join(eo.HERE, "golden"))
from make_golden_encoder import codec_offset  # noqa: E402,F401  (byte offset of a bark file's codec section)

HOP = 320


def n_q_for(bandwidth: int, sample_rate: int = 24000, n_bins: int = 1024) -> int:
    """get_num_quantizers_for_bandwidth in float32 arithmetic; sample_rate >= HOP."""
    f32 = np.float32
    frame_rate = int(math.ceil(sample_rate // HOP))
    bw_per_q = f32(int(f32(np.log2(f32(n_bins))) * f32(frame_rate)))
    return int(max(f32(1), np.floor(f32(bandwidth) * f32(1000) / bw_per_q)))


def codec_tensors(path: str, offset: int) -> dict:
    """Every tensor of the codec section at byte `offset`, by name: float32 or float16 arrays in the file's shape, outermost dimension
    first (ggml's ne reversed)."""
    out = {}
    with open(path, "rb") as f:
        f.seek(offset + 4 + 9 * 4)                               # magic, 9 hyper-parameters (encodec.cpp:156-165)
        while True:
            head = f.read(12)
            if len(head) < 12:
                break
            n_dims, name_len, ttype = struct.unpack("<iii", head)
            ne = struct.unpack("<%di" % n_dims, f.read(4 * n_dims))
            name = f.read(name_len).decode()
            dt = np.float32 if ttype == 0 else np.float16
            n = int(np.prod(ne))
            out[name] = np.frombuffer(f.read(n * np.dtype(dt).itemsize), dt).reshape(ne[::-1])
    return out


def codebooks(path: str, offset: int) -> np.ndarray:
    """Every quantizer.vq.layers.<q>._codebook.embed of the codec section at byte `offset`: [n_q][n_bins][hidden] float32."""
    t = codec_tensors(path, offset)
    cb = {int(k.split(".")[3]): v for k, v in t.items() if k.startswith("quantizer.vq.layers.")}
    return np.stack([cb[q] for q in range(len(cb))])


class CodecOracle:
    """Encoder of one weight file with all its codebooks."""

    def __init__(self, path: str, offset: int):
        self.enc = eo.EncoderOracle(path)
        self.cb = codebooks(path, offset)

    def encode(self, audio, n_q: int) -> np.ndarray:
        _, lat = self.enc.encode(audio, return_latent=True)
        return eo.rvq_encode(lat, self.cb[:n_q])
