"""Synthetic KataGo model files (random weights, real architecture).

There is no network on the build or GPU boxes, so the b18c384nbt / b28c512nbt weights the reference's test scripts
download (cpp/runsearchtests.sh:5-23) are unavailable; this writes correctly-shaped nets in the reference's own
`.bin` model format (SURVEY.md Appendix A; cpp/neuralnet/desc.cpp:40-90 and the parse order listed there), so the
very same file loads in libkgb200, in the numpy oracle and in the reference's C++ loader.  Architectures follow
python/katago/train/modelconfigs.py (:605-641 b18c384nbt, :876-922 b28c512nbt, :142-166 b6c96) as exported by
python/export_model_pytorch.py (version 15: mish activations, 2 policy channels, 6 score-value channels).

Random weights are fine for throughput and parity work and useless for playing strength.
"""
from __future__ import annotations

import gzip
import io
from typing import List, Optional

import numpy as np

CONFIGS = {
    # name: (trunk, mid, gpool, blocks, p1, g1, v1, v2)  blocks: 'r' regular, 'g' regular+gpool, 'n' nested, 'N' nested+gpool
    "b18c384nbt": dict(trunk=384, mid=192, gpool=64, blocks="nnNnnNnnNnnNnnNnnn", p1=48, g1=48, v1=96, v2=128),
    "b28c512nbt": dict(trunk=512, mid=256, gpool=64, blocks="nnNnnNnnNnnNnnNnnNnnNnnNnnNn", p1=64, g1=64, v1=128, v2=144),
    "b6c96": dict(trunk=96, mid=96, gpool=32, blocks="rrgrgr", p1=32, g1=32, v1=32, v2=64),
    "b10c128": dict(trunk=128, mid=128, gpool=32, blocks="rrrrgrrgrr", p1=32, g1=32, v1=32, v2=80),
    # small shapes for unit tests
    "tiny_nbt": dict(trunk=64, mid=32, gpool=16, blocks="nNn", p1=16, g1=16, v1=24, v2=32),
    "tiny_reg": dict(trunk=48, mid=48, gpool=16, blocks="rgr", p1=8, g1=8, v1=12, v2=16),
    "mid_nbt": dict(trunk=128, mid=64, gpool=32, blocks="nNnN", p1=32, g1=32, v1=48, v2=64),
}


class _Writer:
    def __init__(self, version: int = 15):
        self.buf = io.BytesIO()
        self.version = version

    def line(self, *toks):
        self.buf.write((" ".join(str(t) for t in toks) + "\n").encode("ascii"))

    def floats(self, arr: np.ndarray):
        a = np.ascontiguousarray(arr, dtype="<f4")
        self.buf.write(b"@BIN@")
        self.buf.write(a.tobytes())
        self.buf.write(b"\n")


def _conv(w: _Writer, rng, name, k, cin, cout, gain=1.0):
    w.line(name)
    w.line(k, k, cin, cout, 1, 1)
    std = gain * np.sqrt(2.0 / (k * k * cin))
    w.floats(rng.standard_normal((k, k, cin, cout)) * std)


def _bn(w: _Writer, rng, name, c):
    w.line(name)
    w.line(c, "0.0001", 1, 1)
    w.floats(rng.standard_normal(c) * 0.1)             # mean
    w.floats(rng.uniform(0.5, 1.5, c))                  # variance
    w.floats(rng.uniform(0.6, 1.4, c))                  # scale (some |s|<1, some >1: exercises the load-time folding)
    w.floats(rng.standard_normal(c) * 0.1)             # bias


def _act(w: _Writer, name, act):
    w.line(name)
    if w.version >= 11:  # desc.cpp:382-403: older nets have implicit relu
        w.line(act)


def _matmul(w: _Writer, rng, name, cin, cout, gain=1.0):
    w.line(name)
    w.line(cin, cout)
    w.floats(rng.standard_normal((cin, cout)) * gain * np.sqrt(1.0 / cin))


def _matbias(w: _Writer, rng, name, c):
    w.line(name)
    w.line(c)
    w.floats(rng.standard_normal(c) * 0.1)


def _ordinary(w, rng, name, c, act):
    w.line("ordinary_block")
    w.line(name)
    _bn(w, rng, name + ".norm1", c); _act(w, name + ".act1", act)
    _conv(w, rng, name + ".conv1", 3, c, c)
    _bn(w, rng, name + ".norm2", c); _act(w, name + ".act2", act)
    _conv(w, rng, name + ".conv2", 3, c, c, gain=0.4)


def _gpool(w, rng, name, c, cg, act):
    w.line("gpool_block")
    w.line(name)
    creg = c - cg
    _bn(w, rng, name + ".norm1", c); _act(w, name + ".act1", act)
    _conv(w, rng, name + ".conv1r", 3, c, creg)
    _conv(w, rng, name + ".conv1g", 3, c, cg)
    _bn(w, rng, name + ".normg", cg); _act(w, name + ".actg", act)
    _matmul(w, rng, name + ".linear_g", 3 * cg, creg, gain=0.5)
    _bn(w, rng, name + ".norm2", creg); _act(w, name + ".act2", act)
    _conv(w, rng, name + ".conv2", 3, creg, c, gain=0.4)


def _nested(w, rng, name, c, cmid, cg: Optional[int], act, ninner=2):
    w.line("nested_bottleneck_block")
    w.line(name)
    w.line(ninner)
    _bn(w, rng, name + ".normp", c); _act(w, name + ".actp", act)
    _conv(w, rng, name + ".convp", 1, c, cmid)
    for i in range(ninner):
        if cg is not None and i == 0:
            _gpool(w, rng, f"{name}.blockstack.{i}", cmid, cg, act)
        else:
            _ordinary(w, rng, f"{name}.blockstack.{i}", cmid, act)
    _bn(w, rng, name + ".normq", cmid); _act(w, name + ".actq", act)
    _conv(w, rng, name + ".convq", 1, cmid, c, gain=0.4)


def model_bytes(config: str, seed: int = 0, name: Optional[str] = None, activation: str = "ACTIVATION_MISH",
                version: int = 15, num_input_channels: int = 22, num_global: int = 19, meta_channels: int = 0,
                meta_out_gain: float = 1.0) -> bytes:
    """meta_channels > 0 adds an SGF-metadata encoder of that internal width (metaEncoderVersion 1, as the reference's
    `-meta` configs export it: desc.cpp:1571-1617, export_model_pytorch.py write_metadata_encoder), drawn from its own generator so
    that the trunk and heads equal those of the net without it; meta_out_gain scales its last layer (0: an encoder that adds nothing)."""
    cfg = CONFIGS[config]
    if meta_channels and version < 15:
        raise ValueError("SGF-metadata encoders need model version >= 15")
    rng = np.random.default_rng(seed)
    w = _Writer(version)
    act = activation
    c, cmid, cg = cfg["trunk"], cfg["mid"], cfg["gpool"]
    w.line(name or f"{config}-synth{seed}")
    w.line(version)
    w.line(num_input_channels)
    w.line(num_global)
    if version >= 13:
        w.line(20.0, 20.0, 20.0, 20.0, 40.0, 0.25, 30.0)
    if version >= 15:
        w.line(1 if meta_channels else 0, 0, 0, 0, 0, 0, 0, 0)
    w.line("trunk")
    w.line(len(cfg["blocks"]), c, cmid, cmid - cg, cmid - cg, cg)
    if version >= 15:
        w.line(0, 0, 0, 0, 0, 0)
    _conv(w, rng, "conv1", 3, num_input_channels, c)
    _matmul(w, rng, "ginputw", num_global, c)
    if meta_channels:
        mrng = np.random.default_rng([seed, 192])
        w.line("sgf_metadata_encoder")
        w.line(192)
        _matmul(w, mrng, "meta.mul1", 192, meta_channels); _matbias(w, mrng, "meta.bias1", meta_channels); _act(w, "meta.act1", act)
        _matmul(w, mrng, "meta.mul2", meta_channels, meta_channels); _matbias(w, mrng, "meta.bias2", meta_channels); _act(w, "meta.act2", act)
        _matmul(w, mrng, "meta.mul3", meta_channels, c, gain=meta_out_gain)
    for i, kind in enumerate(cfg["blocks"]):
        nm = f"block{i}"
        if kind == "r":
            _ordinary(w, rng, nm, c, act)
        elif kind == "g":
            _gpool(w, rng, nm, c, cg, act)
        elif kind == "n":
            _nested(w, rng, nm, c, cmid, None, act)
        elif kind == "N":
            _nested(w, rng, nm, c, cmid, cg, act)
        else:
            raise ValueError(kind)
    _bn(w, rng, "trunk.tipnorm", c); _act(w, "trunk.tipact", act)
    p1, g1, v1, v2 = cfg["p1"], cfg["g1"], cfg["v1"], cfg["v2"]
    ncp = 1 if version < 12 else (4 if version == 16 else 2)
    w.line("policyhead")
    if version >= 17:
        w.line(ncp); w.line(0, 0, 0)
    _conv(w, rng, "p1.w", 1, c, p1)
    _conv(w, rng, "g1.w", 1, c, g1)
    _bn(w, rng, "g1.norm", g1); _act(w, "g1.act", act)
    _matmul(w, rng, "matmulg2w", 3 * g1, p1, gain=0.5)
    _bn(w, rng, "p1.norm", p1); _act(w, "p1.act", act)
    _conv(w, rng, "p2.w", 1, p1, ncp)
    if version >= 15:
        _matmul(w, rng, "matmulpass", 3 * g1, p1)
        _matbias(w, rng, "biaspass", p1)
        _act(w, "passact", act)
        _matmul(w, rng, "matmulpass2", p1, ncp)
    else:
        _matmul(w, rng, "matmulpass", 3 * g1, ncp)
    w.line("valuehead")
    if version >= 17:
        w.line(0, 0, 0)
    _conv(w, rng, "v1.w", 1, c, v1)
    _bn(w, rng, "v1.norm", v1); _act(w, "v1.act", act)
    _matmul(w, rng, "v2.w", 3 * v1, v2); _matbias(w, rng, "v2.b", v2); _act(w, "v2.act", act)
    _matmul(w, rng, "v3.w", v2, 3); _matbias(w, rng, "v3.b", 3)
    nsv = 6 if version >= 9 else 4 if version >= 8 else 2 if version >= 4 else 1
    _matmul(w, rng, "sv3.w", v2, nsv); _matbias(w, rng, "sv3.b", nsv)
    _conv(w, rng, "vownership.w", 1, v1, 1)
    return w.buf.getvalue()


def write_model(path: str, config: str, seed: int = 0, **kw) -> str:
    data = model_bytes(config, seed, **kw)
    if path.endswith(".gz"):
        with gzip.open(path, "wb", compresslevel=1) as f:
            f.write(data)
    else:
        with open(path, "wb") as f:
            f.write(data)
    return path


def synthetic_inputs(n: int, x_len: int = 19, y_len: int = 19, seed: int = 0, board_sizes=None, num_channels: int = 22,
                     num_global: int = 19, nhwc: bool = True):
    """Plausible V7 feature rows without the Go engine: channel 0 on-board mask, channels 1/2 disjoint stones with a
    realistic density, the other planes sparse 0/1, globals small floats.  (Kernel-level inputs only: real rows come from
    fillRowV7.)  board_sizes: optional list of (bx, by) per row, smaller boards sit in the top-left corner as in
    NNInputs::fillRowV7 (nninputs.cpp:2307-2330)."""
    rng = np.random.default_rng(seed)
    sp = np.zeros((n, y_len, x_len, num_channels), np.float32)
    for i in range(n):
        bx, by = (x_len, y_len) if board_sizes is None else board_sizes[i]
        on = np.zeros((y_len, x_len), np.float32)
        on[:by, :bx] = 1.0
        sp[i, :, :, 0] = on
        dens = rng.uniform(0.0, 0.6)
        r = rng.uniform(size=(y_len, x_len))
        sp[i, :, :, 1] = (r < dens / 2) * on
        sp[i, :, :, 2] = ((r >= dens / 2) & (r < dens)) * on
        for c in range(3, num_channels):
            sp[i, :, :, c] = (rng.uniform(size=(y_len, x_len)) < 0.05) * on
    gl = (rng.standard_normal((n, num_global)) * 0.5).astype(np.float32)
    if not nhwc:
        sp = np.ascontiguousarray(sp.transpose(0, 3, 1, 2))
    return sp, gl
