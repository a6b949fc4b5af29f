"""The 3x3 convolutions' epilogue warpgroup (kgb_conv_wg_epi_kernel: the accumulators go through a shared-memory tile to a
warpgroup of their own, so the next tile's MMAs run under each tile's epilogue) against kgb_conv_wg_kernel, which
KGB_EPILOGUE_WG=0 keeps everywhere: the same bits for every 3x3 epilogue the evaluator launches (the initial conv's per-image bias
included), at several tile counts and under a ragged mixed-size plan, layer by layer and through the chained graph forward, whose
outputs must also equal the same ops run one at a time.  Split mode, b28's 256-column tiles and fp32 streams keep the other
kernel, and no chain wait may give up."""
import ctypes as C
import os
import tempfile

import numpy as np
import pytest

from katago_b200 import NeuralNet, load_library, modelgen, nn_backend

pytestmark = pytest.mark.gpu

OUTPUTS = (("policy", 362), ("value", 3), ("score_value", 6), ("ownership", 361))
_models = {}


def model(cfg):
    if cfg not in _models:
        path = modelgen.write_model(os.path.join(tempfile.mkdtemp(), cfg + ".bin"), cfg, seed=5)
        _models[cfg] = NeuralNet.loadModelFile(path)
    return _models[cfg]


def chain_error():
    v = C.c_int(-1)
    assert load_library().kgb_conv_chain_error(C.byref(v)) == 0
    return v.value


def bits(a):
    return None if a is None else a.view(np.uint32)


def same(a, b):
    return (a is None and b is None) or np.array_equal(bits(a), bits(b))


def both_kernels(monkeypatch, fn):
    """fn() with the epilogue warpgroup allowed, then with KGB_EPILOGUE_WG=0"""
    monkeypatch.delenv("KGB_EPILOGUE_WG", raising=False)
    on = fn()
    monkeypatch.setenv("KGB_EPILOGUE_WG", "0")
    off = fn()
    monkeypatch.delenv("KGB_EPILOGUE_WG")
    return on, off


def layer_data(ky, cin, cout, n, X, Y, seed):
    rng = np.random.default_rng(seed)
    return dict(w=rng.standard_normal((ky, ky, cin, cout)).astype(np.float32) / np.sqrt(ky * ky * cin),
                x=rng.standard_normal((n, Y, X, cin)).astype(np.float32),
                res=rng.standard_normal((n, Y, X, cout)).astype(np.float32),
                ncb=rng.standard_normal((n, cout)).astype(np.float32),
                sc=(0.5 + rng.random(cout)).astype(np.float32), bi=(0.3 * rng.standard_normal(cout)).astype(np.float32))


# (k, cin, cout, kind, ncbias): kind 0 = the gpool unit's raw fp32 conv, 1 = the first conv of a unit, 2 = + fp16 residual stream in
# place, 3 = raw fp16 stream + operand; 3 with ncbias = the initial conv.  n = 8, 42 and 256 19x19 boards are 25, 132 and 800 tiles.
LAYERS = [(3, 192, 192, 0, False), (3, 192, 192, 1, False), (3, 192, 192, 2, False), (3, 128, 192, 2, False),
          (3, 192, 192, 3, False), (3, 22, 384, 3, True), (5, 22, 384, 3, True), (3, 96, 96, 2, False), (3, 160, 160, 1, False)]


@pytest.mark.parametrize("n", [8, 42, 256])
@pytest.mark.parametrize("k,cin,cout,kind,ncbias", LAYERS)
def test_layer_bit_identical(monkeypatch, k, cin, cout, kind, ncbias, n):
    d = layer_data(k, cin, cout, n, 19, 19, seed=k * 1000 + cin + cout + kind + n)
    run = lambda: nn_backend.test_conv_ex(k, k, cin, cout, d["w"], n, 19, 19, True, kind, d["x"], ncbias=d["ncb"] if ncbias else None,
                                          residual=d["res"] if kind == 2 else None, bn_scale=d["sc"], bn_bias=d["bi"], activation=2)
    on, off = both_kernels(monkeypatch, run)
    for name, a, b in zip(("raw", "act"), on[:2], off[:2]):
        assert same(a, b), (name, k, cin, cout, kind, n, float(np.abs(a - b).max()))


@pytest.mark.parametrize("k,cin,cout,kind,ncbias", [(3, 192, 192, 2, False), (3, 192, 192, 1, False), (3, 22, 384, 3, True)])
def test_layer_ragged_plan_bit_identical(monkeypatch, k, cin, cout, kind, ncbias):
    sizes = [(19, 19), (9, 9), (13, 13), (7, 11), (19, 19), (5, 17), (13, 13), (19, 13)] * 12
    n = len(sizes)
    d = layer_data(k, cin, cout, n, 19, 19, seed=7 + kind)
    bxy = np.array(sizes, np.int32)
    for i, (bx, by) in enumerate(sizes):   # zero off the board, as the plan hook wants it
        d["x"][i, by:] = 0.0
        d["x"][i, :, bx:] = 0.0
    sym = (np.arange(n) % 8).astype(np.int32)
    run = lambda: nn_backend.test_conv_plan(k, k, cin, cout, d["w"], n, 19, 19, True, kind, d["x"], bxy, sym, 1,
                                            ncbias=d["ncb"] if ncbias else None, residual=d["res"] if kind == 2 else None,
                                            bn_scale=d["sc"], bn_bias=d["bi"], activation=2)
    on, off = both_kernels(monkeypatch, run)
    assert on[3]["segments"] > 1
    for name, a, b in zip(("raw", "act"), on[:2], off[:2]):
        assert same(a, b), (name, k, cin, cout, kind)


def forward(cfg, fp16, max_batch, batches):
    """Per batch (board sizes or n): the graph forward's outputs, checked bit for bit against the same ops run one at a time; and the
    handle's epilogue-warpgroup launches per forward."""
    import torch
    lm = model(cfg)
    ctx = NeuralNet.createComputeContext([0], 19, 19, fp16, lm)
    h = NeuralNet.createComputeHandle(ctx, lm, max_batch, False, True, 0)
    lib = load_library()
    dev = torch.device("cuda:0")
    res = []
    try:
        wg = lib.kgb_handle_epilogue_wg_launches_per_forward(h._p)
        for boards in batches:
            n = boards if isinstance(boards, int) else len(boards)
            sp, gl = modelgen.synthetic_inputs(n, 19, 19, seed=31 * n, board_sizes=None if isinstance(boards, int) else boards)
            dsp, dgl = torch.from_numpy(sp.reshape(n, -1)).to(dev), torch.from_numpy(gl).to(dev)
            got = []
            for fn in (lib.kgb_forward_device, lib.kgb_test_forward_serial):
                bufs = [torch.full((n, w), float("nan"), device=dev) for _, w in OUTPUTS]
                torch.cuda.synchronize()
                rc = fn(h._p, n, dsp.data_ptr(), dgl.data_ptr(), None, None, *(b.data_ptr() for b in bufs))
                assert rc == 0, lib.kgb_last_error()
                h.sync()
                got.append([b.cpu().numpy() for b in bufs])
            for (k, _), a, b in zip(OUTPUTS, got[0], got[1]):
                assert np.isfinite(a).all() and np.array_equal(bits(a), bits(b)), (cfg, n, k)
            assert chain_error() == 0
            res.append(got[0])
    finally:
        h.free()
        ctx.free()
    return res, wg


def b19(n):
    return [(19, 19)] * n


# b18c384nbt's 3x3 launches: the initial conv, 31 + 31 in ordinary units, 5 + 5 in gpool units.  With 19x19 boards the plan has
# 400 n + 22 rows in 128-row tiles: 26, 132, 133, 792 and 801 tiles below.
B18_3X3 = 73
MIXED = [(9, 9), (13, 13), (19, 19), (19, 13), (13, 13), (19, 19), (9, 9), (19, 19)] * 24


def test_b18_forward_bit_identical(monkeypatch):
    batches = [8, 42, b19(42) + [(9, 9)], b19(253) + [(9, 9)], 256, MIXED]
    (on, wg_on), (off, wg_off) = both_kernels(monkeypatch, lambda: forward("b18c384nbt", True, 256, batches))
    assert (wg_on, wg_off) == (B18_3X3, 0)
    for i, (a, b) in enumerate(zip(on, off)):
        for (k, _), x, y in zip(OUTPUTS, a, b):
            assert np.array_equal(bits(x), bits(y)), (i, k)


def test_b18_fp32_streams_keep_the_other_kernel(monkeypatch):
    """With fp32 streams only the launches without one take the epilogue warpgroup: the 31 first convs of the ordinary units and the
    5 gpool convs, whose raw output is fp32 in every mode; the outputs do not change."""
    monkeypatch.setenv("KGB_STREAM_FP32", "all")
    (on, wg_on), (off, wg_off) = both_kernels(monkeypatch, lambda: forward("b18c384nbt", True, 64, [64]))
    assert (wg_on, wg_off) == (36, 0)
    for (k, _), x, y in zip(OUTPUTS, on[0], off[0]):
        assert np.array_equal(bits(x), bits(y)), k


def test_split_mode_and_b28_keep_the_other_kernel():
    assert forward("b18c384nbt", False, 16, [16])[1] == 0    # fp32-equivalent mode
    assert forward("b28c512nbt", True, 16, [16])[1] == 0     # 256-column tiles
