"""Oracle of SGF-metadata (human SL) nets, layered on the numpy oracle (oracle/kg_nn_oracle.py), which stays the reference of every
other net.  TEST INFRASTRUCTURE ONLY.

A metadata net is an ordinary net plus the SGF-metadata encoder between the initial matmul and the first block (desc.cpp:1571-1617,
1729-1746): 192 metadata inputs -> mul1 + bias1, act1 -> mul2 + bias2, act2 -> mul3, whose output the reference adds to the initial
convolution as a per-image bias, like the global inputs' matmul (eigenbackend.cpp:1839-1857, 1927-1932).  This module parses the
encoder, hands the rest of the file to the plain oracle, and evaluates the encoder's output e [n, trunk] as extra global inputs
whose initial-matmul rows are the identity: g @ W + e @ I.  transformToReduceActivations scales mul3 by the trunk tip's factors
(desc.cpp:1924-1926); those identity rows take the same factors, so the oracle's own transform covers it.
"""
from __future__ import annotations

import copy
import gzip

import numpy as np

import kg_nn_oracle as orc

NUM_META = 192


class MetaEncoder:
    def __init__(self, r: "orc._Reader", version: int):
        self.name = r.tok()
        n = r.int()
        if n != NUM_META:
            raise ValueError(f"{self.name}: number of in channels ({n}) did not match expected ({NUM_META})")
        self.mul1, self.bias1, self.act1 = orc.MatMul.parse(r), orc.MatBias.parse(r), orc._parse_act(r, version)
        self.mul2, self.bias2, self.act2 = orc.MatMul.parse(r), orc.MatBias.parse(r), orc._parse_act(r, version)
        self.mul3 = orc.MatMul.parse(r)

    def apply(self, meta: np.ndarray, dt=np.float32) -> np.ndarray:
        """eigenbackend.cpp:1839-1857 (mask of the PyTorch model's feature 86: already folded into mul1 by the exporter)."""
        x = orc.act_fn(np.asarray(np.asarray(meta, dt) @ self.mul1.w + self.bias1.w, dt), self.act1, dt)
        x = orc.act_fn(np.asarray(np.asarray(x, dt) @ self.mul2.w + self.bias2.w, dt), self.act2, dt)
        return np.asarray(np.asarray(x, dt) @ self.mul3.w, dt)


class MetaModel:
    """`base`: the oracle's Model with the encoder folded into its initial matmul (takes [global | encoder output]);
    `encoder`: the encoder with its raw (untransformed) mul3."""

    def __init__(self, base: "orc.Model", encoder: MetaEncoder, span=(0, 0)):
        self.base, self.encoder = base, encoder
        self.span = span   # the encoder's bytes in the file


def parse_meta_model(data: bytes, binary: bool, apply_transform: bool = True) -> MetaModel:
    r = orc._Reader(data, binary)
    r.tok()
    version = r.int()
    if version < 15:
        raise ValueError("SGF-metadata encoders need model version >= 15")
    r.int(); r.int()
    if version >= 13:
        for _ in range(7):
            r.float()
    tok = r.tok()
    flag_end = r.p
    if tok != "1":
        raise ValueError(f"not an SGF-metadata net (metaEncoderVersion {tok})")
    r.int()
    for _ in range(6):
        r.int()
    r.tok()  # trunk
    for _ in range(6):
        r.int()
    for _ in range(6):
        r.int()
    orc.Conv.parse(r)
    orc.MatMul.parse(r)
    start = r.p
    enc = MetaEncoder(r, version)
    end = r.p
    # the same file without its encoder, metaEncoderVersion 0
    plain = data[:flag_end - 1] + b"0" + data[flag_end:start] + data[end:]
    base = orc.parse_model(plain, binary, apply_transform=False)
    if enc.mul3.cout != base.trunk_c:
        raise ValueError(f"trunk: {enc.name} sgfMetadataEncoder.mul3.outChannels ({enc.mul3.cout}) != trunkNumChannels ({base.trunk_c})")
    g = base.initial_matmul
    base.initial_matmul = orc.MatMul(g.name, g.cin + base.trunk_c, g.cout,
                                     np.concatenate([g.w, np.eye(base.trunk_c, dtype=np.float32)], axis=0))
    base.num_input_global = g.cin + base.trunk_c
    if apply_transform:
        base.transform_to_reduce_activations()
    return MetaModel(base, enc, (start, end))


def load_meta_model(path: str, apply_transform: bool = True) -> MetaModel:
    raw = open(path, "rb").read()
    if path.endswith(".gz"):
        raw = gzip.decompress(raw)
    base = path[:-3] if path.endswith(".gz") else path
    return parse_meta_model(raw, not base.endswith(".txt"), apply_transform)


def get_output(m: MetaModel, spatial, glob, meta, symmetries=None, policy_optimism=None, dtype=np.float32) -> dict:
    """orc.get_output of a metadata net; meta [n, 192] as SGFMetadata::fillMetadataRow writes it."""
    e = m.encoder.apply(meta, dtype)
    return orc.get_output(m.base, spatial, np.concatenate([np.asarray(glob, dtype), e], axis=1), symmetries, policy_optimism, dtype)


def without_encoder(m: MetaModel) -> "orc.Model":
    """The twin net without an encoder (same trunk and heads)."""
    b = copy.deepcopy(m.base)
    g = b.initial_matmul
    cin = g.cin - b.trunk_c
    b.initial_matmul = orc.MatMul(g.name, cin, g.cout, g.w[:cin].copy())
    b.num_input_global = cin
    return b


def bin_to_text(data: bytes) -> bytes:
    """The text form of a binary metadata net (desc.cpp:40-90 reads both): every '@BIN@' block written as decimal floats that read
    back to the same fp32 values."""
    blocks = []
    orig = orc._Reader.floats

    def recording(self, n, name):
        at = self.d.find(b"@", self.p)
        out = orig(self, n, name)
        blocks.append((self.d is data, at, self.p, out))
        return out

    orc._Reader.floats = recording
    try:
        m = parse_meta_model(data, True, apply_transform=False)
    finally:
        orc._Reader.floats = orig
    start, end = m.span
    # the encoder's blocks from the first reader, every other one from the plain file's (offsets past the encoder shifted back)
    spans = [(a, b, v) for own, a, b, v in blocks if own and start <= a < end]
    spans += [(a, b, v) if a < start else (a + end - start, b + end - start, v) for own, a, b, v in blocks if not own]
    spans.sort(key=lambda t: t[0])
    out, p = [], 0
    for a, b, v in spans:
        out += [data[p:a], " ".join(str(x) for x in v).encode()]
        p = b
    return b"".join(out + [data[p:]])
