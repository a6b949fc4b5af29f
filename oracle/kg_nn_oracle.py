"""CPU oracle for the NN-evaluator stage of the KataGo self-play hot path (SURVEY.md §8 rows a10-a17).

TEST INFRASTRUCTURE ONLY.  Nothing under katago_b200/ may import this module; only tests/,
__graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs do.  It is a plain numpy fp32
restatement of the reference's Eigen backend and model loader:

  * model file grammar + BN merge            cpp/neuralnet/desc.cpp:40-90,110-155,208-289,382-403,451-535,
                                             566-576,652-666,783-801,1444-1562,1669-1764,2051-2103,2242-2272,
                                             2441-2574
  * transformToReduceActivations             cpp/neuralnet/desc.cpp:627-632,745-758,944-1001,1911-1972,2810
  * forward pass                             cpp/neuralnet/eigenbackend.cpp:124-197 (mask sum, NC bias, pools),
                                             739-762 (BN+act+mask), 780-809 (activations), 1127-1145 (residual),
                                             1183-1229 (gpool residual), 1295-1314 (nested bottleneck),
                                             1909-1947 (trunk), 1992-2036 (policy head), 2079-2114 (value head),
                                             2162-2216 (model), 2445-2628 (getOutput: symmetry, policy optimism)
  * symmetry copies                          cpp/neuralnet/nninputs.cpp:529-597

The reference computes 3x3 convolutions by Winograd F(4x4,3x3) in fp32 (eigenbackend.cpp:448-690); this oracle
uses direct convolution (im2col + sgemm), which is the same function up to fp32 summation order, so agreement
with the reference is ~1e-5 relative, not bitwise (Eigen itself is not under /root/reference - SURVEY.md §8c).

Pinning (see tests/test_oracle_nn.py): (1) the reference's own known-answer test for this path, cpp/tests/tinymodel.cpp - its two
embedded tiny nets, three positions, expected outputs and tolerances (tests/golden/tinymodel.json.gz + models/tiny*.bin.gz, read
from the reference's test source by tests/golden/make_tinymodel_fixtures.py, input rows from the reference's fillRowV7); (2)
tests/golden/torchref_*.npz: outputs of the reference's PyTorch model (python/katago/train/model_pytorch.py) on nets exported by
the reference's exporter; (3) direct-convolution MAC counts equal to those of the reference's own loader.  The device path is
held to the same known-answer test in tests/test_gpu_nn_parity.py.
"""
from __future__ import annotations

import gzip
import io
import math
from dataclasses import dataclass, field
from typing import List, Optional, Tuple

import numpy as np

ACT_IDENTITY, ACT_RELU, ACT_MISH, ACT_SILU = 0, 1, 2, 3
_ACT_NAMES = {"ACTIVATION_IDENTITY": ACT_IDENTITY, "ACTIVATION_RELU": ACT_RELU,
              "ACTIVATION_MISH": ACT_MISH, "ACTIVATION_SILU": ACT_SILU}


# --------------------------------------------------------------------------------------------------------------
# Layer descriptions (loader)
# --------------------------------------------------------------------------------------------------------------

class _Reader:
    """Whitespace-token reader with '@BIN@' little-endian fp32 blocks (desc.cpp:40-90)."""

    def __init__(self, data: bytes, binary: bool):
        self.d = data
        self.p = 0
        self.binary = binary

    def tok(self) -> str:
        d, p = self.d, self.p
        n = len(d)
        while p < n and d[p] in b" \t\r\n":
            p += 1
        s = p
        while p < n and d[p] not in b" \t\r\n":
            p += 1
        if s == p:
            raise ValueError("unexpected end of model file")
        self.p = p
        return d[s:p].decode("ascii")

    def int(self) -> int:
        return int(self.tok())

    def float(self) -> float:
        return float(self.tok())

    def floats(self, n: int, name: str) -> np.ndarray:
        if not self.binary:
            out = np.empty(n, dtype=np.float32)
            for i in range(n):
                out[i] = np.float32(self.tok())
            return out
        at = self.d.find(b"@", self.p)
        if at < 0 or at - self.p > 100 or self.d[at:at + 5] != b"@BIN@":
            raise ValueError(f"{name}: did not find expected header for binary float block")
        s = at + 5
        out = np.frombuffer(self.d, dtype="<f4", count=n, offset=s).astype(np.float32)
        self.p = s + 4 * n
        if not np.all(np.isfinite(out)):
            raise ValueError(f"{name}: non-finite weight")
        return out


@dataclass
class Conv:
    name: str
    ky: int
    kx: int
    cin: int
    cout: int
    w: np.ndarray  # [ky, kx, cin, cout]  (file order, desc.cpp:131-142)

    @staticmethod
    def parse(r: _Reader) -> "Conv":
        name = r.tok()
        ky, kx, cin, cout, dy, dx = r.int(), r.int(), r.int(), r.int(), r.int(), r.int()
        if dy != 1 or dx != 1:
            raise ValueError(f"{name}: dilation unsupported")
        w = r.floats(ky * kx * cin * cout, name).reshape(ky, kx, cin, cout).copy()
        return Conv(name, ky, kx, cin, cout, w)

    def scale_out(self, f: np.ndarray):
        self.w = (self.w * f.reshape(1, 1, 1, -1)).astype(np.float32)


@dataclass
class BN:
    name: str
    c: int
    scale: np.ndarray  # merged scale
    bias: np.ndarray   # merged bias

    @staticmethod
    def parse(r: _Reader) -> "BN":
        name = r.tok()
        c = r.int()
        eps = np.float32(r.float())
        has_scale, has_bias = r.int(), r.int()
        mean = r.floats(c, name)
        var = r.floats(c, name)
        scale = r.floats(c, name) if has_scale else np.ones(c, np.float32)
        bias = r.floats(c, name) if has_bias else np.zeros(c, np.float32)
        # desc.cpp:282-289
        ms = (scale / np.sqrt(var + eps)).astype(np.float32)
        mb = (bias - ms * mean).astype(np.float32)
        return BN(name, c, ms, mb)

    def scale_in(self, f: np.ndarray):           # desc.cpp:291-305
        self.scale = (self.scale * f).astype(np.float32)

    def extract_lt_one(self) -> np.ndarray:      # desc.cpp:307-325
        f = np.ones(self.c, np.float32)
        m = np.abs(self.scale) < 1.0
        f[m] = self.scale[m]
        self.scale = self.scale.copy()
        self.scale[m] = 1.0
        return f

    def extract_lt_one_with_inv(self) -> Tuple[np.ndarray, np.ndarray]:  # desc.cpp:326-353
        f = np.ones(self.c, np.float32)
        inv = np.ones(self.c, np.float32)
        s = self.scale.copy()
        for i in range(self.c):
            a = abs(s[i])
            if a < 0.5:
                f[i] = 0.5
                inv[i] = 2.0
                s[i] = np.float32(s[i] * np.float32(2.0))
            elif a < 1.0:
                f[i] = s[i]
                inv[i] = np.float32(1.0) / s[i]
                s[i] = 1.0
        self.scale = s
        return f, inv


def _parse_act(r: _Reader, version: int) -> int:  # desc.cpp:382-403
    r.tok()
    if version >= 11:
        return _ACT_NAMES[r.tok()]
    return ACT_RELU


@dataclass
class MatMul:
    name: str
    cin: int
    cout: int
    w: np.ndarray  # [cin, cout] file order (desc.cpp:451-479)

    @staticmethod
    def parse(r: _Reader) -> "MatMul":
        name = r.tok()
        cin, cout = r.int(), r.int()
        w = r.floats(cin * cout, name).reshape(cin, cout).copy()
        return MatMul(name, cin, cout, w)

    def scale_out(self, f: np.ndarray):
        self.w = (self.w * f.reshape(1, -1)).astype(np.float32)


@dataclass
class MatBias:
    name: str
    c: int
    w: np.ndarray

    @staticmethod
    def parse(r: _Reader) -> "MatBias":
        name = r.tok()
        c = r.int()
        return MatBias(name, c, r.floats(c, name))


@dataclass
class ResBlock:
    kind = "ordinary_block"
    name: str
    pre_bn: BN
    pre_act: int
    conv1: Conv
    mid_bn: BN
    mid_act: int
    conv2: Conv

    @staticmethod
    def parse(r: _Reader, v: int) -> "ResBlock":
        name = r.tok()
        pre_bn = BN.parse(r); pre_act = _parse_act(r, v)
        conv1 = Conv.parse(r)
        mid_bn = BN.parse(r); mid_act = _parse_act(r, v)
        conv2 = Conv.parse(r)
        return ResBlock(name, pre_bn, pre_act, conv1, mid_bn, mid_act, conv2)

    @property
    def final_conv(self):
        return self.conv2

    def transform(self):  # desc.cpp:627-632
        self.conv1.scale_out(self.mid_bn.extract_lt_one())


@dataclass
class GPoolBlock:
    kind = "gpool_block"
    name: str
    pre_bn: BN
    pre_act: int
    regular_conv: Conv
    gpool_conv: Conv
    gpool_bn: BN
    gpool_act: int
    gpool_to_bias: MatMul
    mid_bn: BN
    mid_act: int
    conv2: Conv

    @staticmethod
    def parse(r: _Reader, v: int) -> "GPoolBlock":  # desc.cpp:652-666
        name = r.tok()
        pre_bn = BN.parse(r); pre_act = _parse_act(r, v)
        regular = Conv.parse(r)
        gconv = Conv.parse(r)
        gbn = BN.parse(r); gact = _parse_act(r, v)
        g2b = MatMul.parse(r)
        mid_bn = BN.parse(r); mid_act = _parse_act(r, v)
        conv2 = Conv.parse(r)
        return GPoolBlock(name, pre_bn, pre_act, regular, gconv, gbn, gact, g2b, mid_bn, mid_act, conv2)

    @property
    def final_conv(self):
        return self.conv2

    def transform(self):  # desc.cpp:745-758
        f = self.mid_bn.extract_lt_one()
        self.regular_conv.scale_out(f)
        self.gpool_to_bias.scale_out(f)
        self.gpool_conv.scale_out(self.gpool_bn.extract_lt_one())


@dataclass
class NestedBlock:
    kind = "nested_bottleneck_block"
    name: str
    pre_bn: BN
    pre_act: int
    pre_conv: Conv
    blocks: list
    post_bn: BN
    post_act: int
    post_conv: Conv

    @staticmethod
    def parse(r: _Reader, v: int) -> "NestedBlock":  # desc.cpp:783-801
        name = r.tok()
        n_inner = r.int()
        pre_bn = BN.parse(r); pre_act = _parse_act(r, v)
        pre_conv = Conv.parse(r)
        blocks = _parse_block_stack(r, v, n_inner)
        post_bn = BN.parse(r); post_act = _parse_act(r, v)
        post_conv = Conv.parse(r)
        return NestedBlock(name, pre_bn, pre_act, pre_conv, blocks, post_bn, post_act, post_conv)

    @property
    def final_conv(self):
        return self.post_conv

    def transform(self):  # desc.cpp:944-1001
        f, inv = self.post_bn.extract_lt_one_with_inv()
        self.pre_conv.scale_out(f)
        for b in self.blocks:
            b.pre_bn.scale_in(inv)
            b.final_conv.scale_out(f)
        for b in self.blocks:
            b.transform()


def _parse_block_stack(r: _Reader, v: int, n: int) -> list:  # desc.cpp:1444-1562
    out = []
    for _ in range(n):
        kind = r.tok()
        if kind == "ordinary_block":
            out.append(ResBlock.parse(r, v))
        elif kind == "gpool_block":
            out.append(GPoolBlock.parse(r, v))
        elif kind == "nested_bottleneck_block":
            out.append(NestedBlock.parse(r, v))
        else:
            raise ValueError(f"unsupported block kind {kind} (transformer nets are out of scope, SURVEY.md §2)")
    return out


@dataclass
class Model:
    name: str = ""
    version: int = 0
    num_input_channels: int = 0
    num_input_global: int = 0
    post: dict = field(default_factory=dict)
    trunk_c: int = 0
    mid_c: int = 0
    regular_c: int = 0
    gpool_c: int = 0
    initial_conv: Optional[Conv] = None
    initial_matmul: Optional[MatMul] = None
    blocks: list = field(default_factory=list)
    tip_bn: Optional[BN] = None
    tip_act: int = ACT_RELU
    # policy head
    policy_out_channels: int = 1
    p1_conv: Optional[Conv] = None
    g1_conv: Optional[Conv] = None
    g1_bn: Optional[BN] = None
    g1_act: int = ACT_RELU
    gpool_to_bias: Optional[MatMul] = None
    p1_bn: Optional[BN] = None
    p1_act: int = ACT_RELU
    p2_conv: Optional[Conv] = None
    gpool_to_pass: Optional[MatMul] = None
    gpool_to_pass_bias: Optional[MatBias] = None
    pass_act: int = ACT_RELU
    gpool_to_pass2: Optional[MatMul] = None
    # value head
    v1_conv: Optional[Conv] = None
    v1_bn: Optional[BN] = None
    v1_act: int = ACT_RELU
    v2_mul: Optional[MatMul] = None
    v2_bias: Optional[MatBias] = None
    v2_act: int = ACT_RELU
    v3_mul: Optional[MatMul] = None
    v3_bias: Optional[MatBias] = None
    sv3_mul: Optional[MatMul] = None
    sv3_bias: Optional[MatBias] = None
    ownership_conv: Optional[Conv] = None

    def transform_to_reduce_activations(self):  # desc.cpp:1911-1972 (+ :2810)
        f, inv = self.tip_bn.extract_lt_one_with_inv()
        self.initial_conv.scale_out(f)
        self.initial_matmul.scale_out(f)
        for b in self.blocks:
            b.pre_bn.scale_in(inv)
            b.final_conv.scale_out(f)
        for b in self.blocks:
            b.transform()


def _expect_zeros(r: _Reader, n: int, what: str):
    for _ in range(n):
        if r.int() != 0:
            raise ValueError(f"unknown/unsupported {what} option")


def parse_model(data: bytes, binary: bool, apply_transform: bool = True) -> Model:
    r = _Reader(data, binary)
    m = Model()
    m.name = r.tok()
    m.version = v = r.int()
    if v < 3 or v > 17:
        raise ValueError(f"unsupported model version {v}")
    m.num_input_channels = r.int()
    m.num_input_global = r.int()
    if v >= 13:  # desc.cpp:2477-2513
        keys = ["tdScoreMultiplier", "scoreMeanMultiplier", "scoreStdevMultiplier", "leadMultiplier",
                "varianceTimeMultiplier", "shorttermValueErrorMultiplier", "shorttermScoreErrorMultiplier"]
        m.post = {k: r.float() for k in keys}
    else:        # desc.cpp:2412-2420
        m.post = dict(tdScoreMultiplier=20.0, scoreMeanMultiplier=20.0, scoreStdevMultiplier=20.0,
                      leadMultiplier=20.0, varianceTimeMultiplier=40.0, shorttermValueErrorMultiplier=0.25,
                      shorttermScoreErrorMultiplier=30.0)
    if v >= 15:
        meta = r.int()
        if meta != 0:
            raise ValueError("SGF-metadata (humanSL) nets are out of scope")
        r.int()  # preferPassAliveUnderSuicideRules
        _expect_zeros(r, 6, "model")
    # trunk (desc.cpp:1669-1764)
    r.tok()
    n_blocks = r.int()
    m.trunk_c, m.mid_c, m.regular_c = r.int(), r.int(), r.int()
    r.int()  # dilated (unused)
    m.gpool_c = r.int()
    if v >= 15:
        if r.int() != 0:
            raise ValueError("RMSNorm trunk tip out of scope")
        _expect_zeros(r, 5, "trunk")
    m.initial_conv = Conv.parse(r)
    m.initial_matmul = MatMul.parse(r)
    m.blocks = _parse_block_stack(r, v, n_blocks)
    m.tip_bn = BN.parse(r)
    m.tip_act = _parse_act(r, v)
    # policy head (desc.cpp:2051-2103)
    r.tok()
    if v >= 17:
        m.policy_out_channels = r.int()
        _expect_zeros(r, 3, "policy")
    elif v == 16:
        m.policy_out_channels = 4
    elif v >= 12:
        m.policy_out_channels = 2
    else:
        m.policy_out_channels = 1
    m.p1_conv = Conv.parse(r)
    m.g1_conv = Conv.parse(r)
    m.g1_bn = BN.parse(r); m.g1_act = _parse_act(r, v)
    m.gpool_to_bias = MatMul.parse(r)
    m.p1_bn = BN.parse(r); m.p1_act = _parse_act(r, v)
    m.p2_conv = Conv.parse(r)
    m.gpool_to_pass = MatMul.parse(r)
    if v >= 15:
        m.gpool_to_pass_bias = MatBias.parse(r)
        m.pass_act = _parse_act(r, v)
        m.gpool_to_pass2 = MatMul.parse(r)
    # value head (desc.cpp:2242-2272)
    r.tok()
    if v >= 17:
        _expect_zeros(r, 3, "value")
    m.v1_conv = Conv.parse(r)
    m.v1_bn = BN.parse(r); m.v1_act = _parse_act(r, v)
    m.v2_mul = MatMul.parse(r); m.v2_bias = MatBias.parse(r); m.v2_act = _parse_act(r, v)
    m.v3_mul = MatMul.parse(r); m.v3_bias = MatBias.parse(r)
    m.sv3_mul = MatMul.parse(r); m.sv3_bias = MatBias.parse(r)
    m.ownership_conv = Conv.parse(r)
    if apply_transform:
        m.transform_to_reduce_activations()
    return m


def load_model(path: str, apply_transform: bool = True) -> Model:
    """File-suffix dispatch as in desc.cpp:2753-2808."""
    with open(path, "rb") as f:
        raw = f.read()
    if path.endswith(".gz"):
        raw = gzip.decompress(raw)
    base = path[:-3] if path.endswith(".gz") else path
    if base.endswith(".txt"):
        return parse_model(raw, False, apply_transform)
    if base.endswith(".bin"):
        return parse_model(raw, True, apply_transform)
    try:
        return parse_model(raw, True, apply_transform)
    except Exception:
        return parse_model(raw, False, apply_transform)


# --------------------------------------------------------------------------------------------------------------
# Forward pass (NHWC; fp32 by default, or float64)
# --------------------------------------------------------------------------------------------------------------

def _f32(x):
    return np.asarray(x, dtype=np.float32)


# The forward pass runs in fp32 by default, as the reference does; dt=np.float64 gives a high-precision reference of the same
# function (same weights, same constants) to measure fp32 implementations against.
def _as(dt, x):
    return np.asarray(x, dtype=dt)


def act_fn(x: np.ndarray, act: int, dt=np.float32) -> np.ndarray:
    """eigenbackend.cpp:780-809."""
    if act == ACT_IDENTITY:
        return x
    if act == ACT_RELU:
        return np.maximum(x, np.float32(0))
    if act == ACT_MISH:
        sp = np.log1p(np.exp(np.minimum(x, np.float32(20)))) + (np.maximum(x, np.float32(20)) - np.float32(20))
        return _as(dt, x * np.tanh(sp))
    if act == ACT_SILU:
        return _as(dt, x / (np.exp(-x) + np.float32(1)))
    raise ValueError(act)


def bn_act_mask(x: np.ndarray, bn: BN, act: int, mask: np.ndarray, dt=np.float32) -> np.ndarray:
    """eigenbackend.cpp:739-762: mask==1 ? act(x*s+b) : 0.   x [N,H,W,C], mask [N,H,W]."""
    y = act_fn(_as(dt, x * bn.scale + bn.bias), act, dt)
    return _as(dt, np.where(mask[..., None] == 1.0, y, np.float32(0)))


def conv2d(x: np.ndarray, c: Conv, dt=np.float32) -> np.ndarray:
    """Zero-padded 'same' cross-correlation, NHWC (eigenbackend.cpp:448-701 computes the same function)."""
    n, h, w, cin = x.shape
    assert cin == c.cin, (c.name, cin, c.cin)
    py, px = c.ky // 2, c.kx // 2
    if c.ky == 1 and c.kx == 1:
        return _as(dt, x.reshape(-1, cin) @ c.w.reshape(cin, c.cout)).reshape(n, h, w, c.cout)
    xp = np.zeros((n, h + 2 * py, w + 2 * px, cin), dt)
    xp[:, py:py + h, px:px + w, :] = x
    out = np.zeros((n * h * w, c.cout), dt)
    for dy in range(c.ky):
        for dx in range(c.kx):
            patch = xp[:, dy:dy + h, dx:dx + w, :].reshape(-1, cin)
            out += patch @ c.w[dy, dx]
    return out.reshape(n, h, w, c.cout)


def gpool(x: np.ndarray, mask: np.ndarray, mask_sum: np.ndarray, dt=np.float32) -> np.ndarray:
    """eigenbackend.cpp:152-177 -> [N, 3C]."""
    n, h, w, c = x.shape
    s = x.reshape(n, -1, c).sum(axis=1, dtype=dt)
    mx = np.maximum((x + (mask[..., None] - np.float32(1))).reshape(n, -1, c).max(axis=1), np.float32(-1.0))
    div = mask_sum.reshape(n, 1)
    sq = np.sqrt(div)
    mean = _as(dt, s / div)
    return _as(dt, np.concatenate([mean, mean * (sq - np.float32(14)) * np.float32(0.1), mx], axis=1))


def vpool(x: np.ndarray, mask_sum: np.ndarray, dt=np.float32) -> np.ndarray:
    """eigenbackend.cpp:179-197 -> [N, 3C]."""
    n, h, w, c = x.shape
    s = x.reshape(n, -1, c).sum(axis=1, dtype=dt)
    div = mask_sum.reshape(n, 1)
    sq = np.sqrt(div)
    mean = _as(dt, s / div)
    a = (sq - np.float32(14))
    return _as(dt, np.concatenate([mean, mean * a * np.float32(0.1),
                                mean * (a * a * np.float32(0.01) - np.float32(0.1))], axis=1))


def _apply_blocks(blocks: list, x: np.ndarray, mask, mask_sum, dt=np.float32) -> np.ndarray:
    for b in blocks:
        if isinstance(b, ResBlock):       # eigenbackend.cpp:1127-1145
            mid = conv2d(bn_act_mask(x, b.pre_bn, b.pre_act, mask, dt), b.conv1, dt)
            x = _as(dt, x + conv2d(bn_act_mask(mid, b.mid_bn, b.mid_act, mask, dt), b.conv2, dt))
        elif isinstance(b, GPoolBlock):   # eigenbackend.cpp:1183-1229
            a = bn_act_mask(x, b.pre_bn, b.pre_act, mask, dt)
            reg = conv2d(a, b.regular_conv, dt)
            g = bn_act_mask(conv2d(a, b.gpool_conv, dt), b.gpool_bn, b.gpool_act, mask, dt)
            bias = _as(dt, gpool(g, mask, mask_sum, dt) @ b.gpool_to_bias.w)
            reg = _as(dt, reg + bias[:, None, None, :])
            x = _as(dt, x + conv2d(bn_act_mask(reg, b.mid_bn, b.mid_act, mask, dt), b.conv2, dt))
        elif isinstance(b, NestedBlock):  # eigenbackend.cpp:1295-1314
            mid = conv2d(bn_act_mask(x, b.pre_bn, b.pre_act, mask, dt), b.pre_conv, dt)
            mid = _apply_blocks(b.blocks, mid, mask, mask_sum, dt)
            x = _as(dt, x + conv2d(bn_act_mask(mid, b.post_bn, b.post_act, mask, dt), b.post_conv, dt))
        else:
            raise TypeError(b)
    return x


def forward_raw(m: Model, spatial: np.ndarray, glob: np.ndarray, return_trunk: bool = False, dtype=np.float32) -> dict:
    """Model::apply (eigenbackend.cpp:2162-2216).  spatial [N,H,W,Cin] NHWC, glob [N,G]; computed in `dtype` (fp32 by default,
    np.float64 for a high-precision reference).

    Returns raw head outputs: policy [N,H,W,Cp], policy_pass [N,Cp], value [N,3], score_value [N,S],
    ownership [N,H,W]."""
    dt = dtype
    x_in = _as(dt, spatial)
    g_in = _as(dt, glob)
    mask = x_in[..., 0].copy()                                   # :2181
    mask_sum = mask.reshape(mask.shape[0], -1).sum(axis=1, dtype=dt)
    # Trunk::apply :1909-1947
    x = conv2d(x_in, m.initial_conv, dt)
    x = _as(dt, x + _as(dt, g_in @ m.initial_matmul.w)[:, None, None, :])
    x = _apply_blocks(m.blocks, x, mask, mask_sum, dt)
    trunk = bn_act_mask(x, m.tip_bn, m.tip_act, mask, dt)
    # PolicyHead::apply :1992-2036
    p1 = conv2d(trunk, m.p1_conv, dt)
    g1 = bn_act_mask(conv2d(trunk, m.g1_conv, dt), m.g1_bn, m.g1_act, mask, dt)
    g1c = gpool(g1, mask, mask_sum, dt)
    p1 = _as(dt, p1 + _as(dt, g1c @ m.gpool_to_bias.w)[:, None, None, :])
    p1 = bn_act_mask(p1, m.p1_bn, m.p1_act, mask, dt)
    policy = conv2d(p1, m.p2_conv, dt)
    if m.version >= 15:
        pp = _as(dt, g1c @ m.gpool_to_pass.w) + m.gpool_to_pass_bias.w
        pp = act_fn(_as(dt, pp), m.pass_act, dt)
        policy_pass = _as(dt, pp @ m.gpool_to_pass2.w)
    else:
        policy_pass = _as(dt, g1c @ m.gpool_to_pass.w)
    # ValueHead::apply :2079-2114
    v1 = bn_act_mask(conv2d(trunk, m.v1_conv, dt), m.v1_bn, m.v1_act, mask, dt)
    v1m = vpool(v1, mask_sum, dt)
    v2 = act_fn(_as(dt, _as(dt, v1m @ m.v2_mul.w) + m.v2_bias.w), m.v2_act, dt)
    value = _as(dt, _as(dt, v2 @ m.v3_mul.w) + m.v3_bias.w)
    score_value = _as(dt, _as(dt, v2 @ m.sv3_mul.w) + m.sv3_bias.w)
    ownership = conv2d(v1, m.ownership_conv, dt)[..., 0]
    out = dict(policy=policy, policy_pass=policy_pass, value=value, score_value=score_value, ownership=ownership)
    if return_trunk:
        out["trunk"] = trunk
    return out


# --------------------------------------------------------------------------------------------------------------
# Symmetry + getOutput packaging
# --------------------------------------------------------------------------------------------------------------

def _sym_index_map(h: int, w: int, symmetry: int, reverse: bool) -> np.ndarray:
    """dst flat index for every src (y,x), as copyWithSymmetry (nninputs.cpp:529-575, C==1 NCHW branch)."""
    transpose = (symmetry & 4) != 0 and h == w
    flip_x = (symmetry & 2) != 0
    flip_y = (symmetry & 1) != 0
    if transpose and not reverse:
        flip_x, flip_y = flip_y, flip_x
    h_stride, w_stride = w, 1
    h_base = w_base = 0
    hs, ws = h_stride, w_stride
    if flip_y:
        h_base = (h - 1) * hs
        hs = -hs
    if flip_x:
        w_base = (w - 1) * ws
        ws = -ws
    if transpose:
        hs, ws = ws, hs
    ys, xs = np.meshgrid(np.arange(h), np.arange(w), indexing="ij")
    return (h_base + ys * hs + w_base + xs * ws).reshape(-1)


def apply_symmetry_nhwc(x: np.ndarray, symmetry: int, reverse: bool = False) -> np.ndarray:
    """x [H,W,C] or [H,W] -> same shape, entries permuted like copyInputsWithSymmetry / copyOutputsWithSymmetry."""
    h, w = x.shape[0], x.shape[1]
    idx = _sym_index_map(h, w, symmetry, reverse)
    flat = x.reshape(h * w, -1)
    out = np.empty_like(flat)
    out[idx] = flat
    return out.reshape(x.shape)


def get_output(m: Model, spatial: np.ndarray, glob: np.ndarray, symmetries=None, policy_optimism=None, dtype=np.float32) -> dict:
    """NeuralNet::getOutput (eigenbackend.cpp:2445-2628): rows given un-symmetrised (as fillRowV7 wrote them, NHWC);
    returns logits with the symmetry already inverted.

    policy [N, H*W+1] (pass last), value [N,3], score_value [N,6-padded: mean, meansq, lead, vartime, stwl, stscore],
    ownership [N,H*W]."""
    dt = dtype
    n, h, w, _ = spatial.shape
    symmetries = [0] * n if symmetries is None else list(symmetries)
    policy_optimism = [0.0] * n if policy_optimism is None else list(policy_optimism)
    sp = np.stack([apply_symmetry_nhwc(_as(dt, spatial[i]), symmetries[i], False) for i in range(n)])
    raw = forward_raw(m, sp, glob, dtype=dt)
    cp = m.policy_out_channels
    policy = np.zeros((n, h * w + 1), dt)
    own = np.zeros((n, h * w), dt)
    for i in range(n):
        po = dt(policy_optimism[i])
        if cp == 2 or (cp == 4 and m.version >= 16):
            p = raw["policy"][i, :, :, 0]
            popt = raw["policy"][i, :, :, 1]
            pt = _as(dt, p + (popt - p) * po)
            pp = raw["policy_pass"][i]
            ppass = dt(pp[0] + (pp[1] - pp[0]) * po)
        else:
            pt = raw["policy"][i, :, :, 0]
            ppass = raw["policy_pass"][i, 0]
        policy[i, :h * w] = apply_symmetry_nhwc(pt, symmetries[i], True).reshape(-1)
        policy[i, h * w] = ppass
        own[i] = apply_symmetry_nhwc(raw["ownership"][i], symmetries[i], True).reshape(-1)
    sv = raw["score_value"]
    sv6 = np.zeros((n, 6), dt)
    if m.version >= 9:
        sv6[:] = sv[:, :6]
    elif m.version >= 8:
        sv6[:, :4] = sv[:, :4]
    elif m.version >= 4:
        sv6[:, 0] = sv[:, 0]; sv6[:, 1] = sv[:, 1]; sv6[:, 2] = sv[:, 0]
    else:
        sv6[:, 0] = sv[:, 0]; sv6[:, 1] = sv[:, 0] * sv[:, 0]; sv6[:, 2] = sv[:, 0]
    return dict(policy=policy, value=raw["value"], score_value=sv6, ownership=own)


# --------------------------------------------------------------------------------------------------------------
# Accounting used by bench.py / DESIGN.md (SURVEY.md §8d: direct-convolution FLOPs)
# --------------------------------------------------------------------------------------------------------------

def iter_convs(m: Model):
    yield m.initial_conv

    def rec(blocks):
        for b in blocks:
            if isinstance(b, ResBlock):
                yield b.conv1; yield b.conv2
            elif isinstance(b, GPoolBlock):
                yield b.regular_conv; yield b.gpool_conv; yield b.conv2
            else:
                yield b.pre_conv
                yield from rec(b.blocks)
                yield b.post_conv
    yield from rec(m.blocks)
    for c in (m.p1_conv, m.g1_conv, m.p2_conv, m.v1_conv, m.ownership_conv):
        yield c


def conv_macs_per_position(m: Model) -> int:
    return sum(c.ky * c.kx * c.cin * c.cout for c in iter_convs(m))
