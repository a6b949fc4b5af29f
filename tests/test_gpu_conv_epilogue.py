"""The wgmma convolution's fused epilogue against the numpy oracle, one launch at a time (kgb_test_conv_epilogue).

The epilogue reads the residual stream from a shared-memory ring of 32-column slices filled by TMA, and the mask and BN constants
from shared memory.  These cases cover what that depends on: both stream dtypes (kind 2 keeps the residual stream in the operand
dtype's mode, kind 4 in fp32), the tightest shared-memory budget (split mode, 256-wide fp32 residual), a partial last M tile in a
launch of more than 132 tiles, every tile width the weight packing produces (64, 128, 160, 192, 224, 256) and a layer of two n
tiles.  The hook itself checks that every pad row of the activated operand comes back zero.  Tolerances are those of
test_gpu_nn_parity.py::test_conv_fused_epilogues.
"""
import numpy as np
import pytest

import kg_nn_oracle as orc

pytestmark = pytest.mark.gpu

CASES = [
    # ky, cin, cout, n, X, Y, kind, fp16
    pytest.param(1, 192, 384, 7, 19, 19, 4, True, id="exit1x1-kind4-two-n-tiles"),
    pytest.param(1, 192, 384, 7, 19, 19, 2, True, id="exit1x1-kind2-fp16-stream"),
    pytest.param(3, 192, 192, 5, 19, 19, 4, True, id="3x3-192-kind4"),
    pytest.param(3, 192, 192, 5, 19, 19, 1, True, id="3x3-192-kind1"),
    pytest.param(3, 192, 192, 5, 19, 19, 3, False, id="3x3-192-kind3-split"),
    pytest.param(3, 256, 256, 3, 19, 19, 2, False, id="3x3-256-split-fp32-residual"),
    pytest.param(3, 256, 256, 3, 19, 19, 4, False, id="3x3-256-split-kind4"),
    pytest.param(3, 64, 64, 70, 19, 19, 2, True, id="partial-last-tile-219-tiles-fp16"),
    pytest.param(3, 64, 64, 70, 19, 19, 4, False, id="partial-last-tile-219-tiles-split"),
    pytest.param(1, 64, 32, 3, 19, 19, 2, True, id="cout32-padded-n64"),
    pytest.param(3, 96, 128, 3, 13, 13, 4, True, id="n128-13x13"),
    pytest.param(1, 128, 320, 3, 19, 19, 4, True, id="n160-two-tiles"),
    pytest.param(1, 128, 448, 3, 19, 19, 2, False, id="n224-two-tiles-split"),
    pytest.param(1, 384, 256, 4, 9, 9, 4, True, id="n256-9x9"),
]


def _reference(x, w, res, sc, bi, ky, cin, cout):
    raw = orc.conv2d(x, orc.Conv("t", ky, ky, cin, cout, w))
    if res is not None:
        raw = raw + res
    z = raw * sc + bi
    return raw, z * np.tanh(np.log1p(np.exp(np.minimum(z, 30.0))))


@pytest.mark.parametrize("ky,cin,cout,n,X,Y,kind,fp16", CASES)
def test_conv_epilogue_from_shared_memory(ky, cin, cout, n, X, Y, kind, fp16):
    from katago_b200 import nn_backend
    rng = np.random.default_rng(1000 * ky + cin + 7 * cout + kind)
    w = (rng.standard_normal((ky, ky, cin, cout)) * np.sqrt(1.0 / (ky * ky * cin))).astype(np.float16).astype(np.float32)
    x = rng.standard_normal((n, Y, X, cin)).astype(np.float16).astype(np.float32)
    res = rng.standard_normal((n, Y, X, cout)).astype(np.float16).astype(np.float32) if kind in (2, 4) else None
    sc = rng.uniform(0.5, 1.5, cout).astype(np.float32)
    bi = rng.uniform(-0.5, 0.5, cout).astype(np.float32)
    raw_ref, act_ref = _reference(x, w, res, sc, bi, ky, cin, cout)
    raw, a = nn_backend.test_conv_epilogue(ky, ky, cin, cout, w, n, X, Y, fp16, kind, x, res, sc, bi, 2)
    tol = 4e-3 if fp16 else 3e-4
    if kind >= 2:
        assert np.abs(raw - raw_ref).max() <= tol * max(1.0, np.abs(raw_ref).max()), np.abs(raw - raw_ref).max()
    else:
        assert raw is None
    assert np.abs(a - act_ref).max() <= tol * max(1.0, np.abs(act_ref).max()), np.abs(a - act_ref).max()
