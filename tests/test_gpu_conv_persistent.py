"""The persistent wgmma convolution at sizes where every CTA runs many tiles, against the numpy oracle.

A launch has at most one CTA per SM, and each CTA walks its tiles with rings (A halo, weights, residual / staging slices, activated
slices) whose stage and phase carry over from one tile to the next, while the previous tile's TMA stores are still in flight.  These
cases make those rings wrap across tile boundaries: the b18c384nbt layer shapes at batch 256 (800 tiles, 6-7 per CTA; 1600 for the
two-n-tile exit 1x1), split mode, an odd number of main-loop steps per tile (3x3 with 64 input channels: 9), slice counts that the
4-slot residual ring does not divide (n_tile 160: 5 slices, 224: 7) and a tile count the grid does not divide, with a partial last
tile.  Tolerances are those of test_gpu_conv_epilogue.py.
"""
import numpy as np
import pytest

import kg_nn_oracle as orc

pytestmark = pytest.mark.gpu

CASES = [
    # ky, cin, cout, n, X, Y, kind, fp16
    pytest.param(3, 192, 192, 256, 19, 19, 1, True, id="3x3-192-kind1-b256"),
    pytest.param(3, 192, 192, 256, 19, 19, 2, True, id="3x3-192-kind2-b256"),
    pytest.param(1, 192, 384, 256, 19, 19, 2, True, id="exit1x1-kind2-b256"),
    pytest.param(1, 384, 192, 256, 19, 19, 3, True, id="entry1x1-kind3-b256"),
    pytest.param(3, 192, 192, 256, 19, 19, 0, True, id="gpool3x3-kind0-b256"),
    pytest.param(3, 192, 192, 128, 19, 19, 4, False, id="3x3-192-kind4-split-b128"),
    pytest.param(3, 64, 64, 200, 19, 19, 2, True, id="3x3-cin64-nine-steps"),
    pytest.param(1, 128, 320, 100, 19, 19, 2, True, id="n160-five-slices"),
    pytest.param(1, 128, 448, 100, 19, 19, 4, True, id="n224-seven-slices"),
    pytest.param(3, 192, 192, 101, 19, 19, 2, True, id="316-tiles-partial-last"),
]


def _mish(z):
    return z * np.tanh(np.log1p(np.exp(np.minimum(z, 30.0))))


@pytest.mark.parametrize("ky,cin,cout,n,X,Y,kind,fp16", CASES)
def test_conv_many_tiles_per_cta(ky, cin, cout, n, X, Y, kind, fp16):
    from katago_b200 import nn_backend
    rng = np.random.default_rng(7 * n + 1000 * ky + cin + 3 * cout + kind)
    w = (rng.standard_normal((ky, ky, cin, cout)) * np.sqrt(1.0 / (ky * ky * cin))).astype(np.float16).astype(np.float32)
    x = rng.standard_normal((n, Y, X, cin)).astype(np.float16).astype(np.float32)
    raw_ref = orc.conv2d(x, orc.Conv("t", ky, ky, cin, cout, w))
    tol = 4e-3 if fp16 else 3e-4
    if kind == 0:
        got = nn_backend.NeuralNet.testEvaluateConv(ky, ky, cin, cout, w, n, X, Y, fp16, x)
        assert np.abs(got - raw_ref).max() <= tol * max(1.0, np.abs(raw_ref).max()), np.abs(got - raw_ref).max()
        return
    res = rng.standard_normal((n, Y, X, cout)).astype(np.float16).astype(np.float32) if kind in (2, 4) else None
    sc = rng.uniform(0.5, 1.5, cout).astype(np.float32)
    bi = rng.uniform(-0.5, 0.5, cout).astype(np.float32)
    if res is not None:
        raw_ref = raw_ref + res
    act_ref = _mish(raw_ref * sc + bi)
    raw, a = nn_backend.test_conv_epilogue(ky, ky, cin, cout, w, n, X, Y, fp16, kind, x, res, sc, bi, 2)
    if kind >= 2:
        assert np.abs(raw - raw_ref).max() <= tol * max(1.0, np.abs(raw_ref).max()), np.abs(raw - raw_ref).max()
    assert np.abs(a - act_ref).max() <= tol * max(1.0, np.abs(act_ref).max()), np.abs(a - act_ref).max()
