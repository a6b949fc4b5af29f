"""The fused nested-block boundary (one launch for a block's exit 1x1 and the next block's entry 1x1) against the two launches it
replaces: the same bits in the trunk stream, the inner stream and the inner operand, exact zeros in masked rows and padded
channels, and whole-net outputs that do not change when KGB_FUSE_BOUNDARY=0 turns the fusion off.
"""
import ctypes as C
import os

import numpy as np
import pytest

from katago_b200 import NeuralNet, load_library, modelgen

pytestmark = pytest.mark.gpu


def _boundary(inner_c, trunk_c, n, X, Y, boards, trunk_fp32, inner_fp32, seed):
    lib = load_library()
    out = np.zeros(6, np.int64)
    bxy = None if boards is None else np.ascontiguousarray(np.array(boards, np.int32).reshape(n, 2))
    rc = lib.kgb_test_conv_boundary(inner_c, trunk_c, n, X, Y, None if bxy is None else bxy.ctypes.data_as(C.POINTER(C.c_int32)),
                                    int(trunk_fp32), int(inner_fp32), C.c_uint32(seed), out.ctypes.data_as(C.POINTER(C.c_int64)))
    assert rc == 0, lib.kgb_last_error()
    return out


MIXED = [(19, 19), (9, 9), (13, 13), (7, 11), (19, 19), (5, 17)]


@pytest.mark.parametrize("inner_c,trunk_c,n,boards,trunk_fp32,inner_fp32", [
    pytest.param(192, 384, 256, None, False, False, id="b18-fp16-b256"),
    pytest.param(192, 384, 1021, None, False, False, id="b18-fp16-partial-last-tile"),
    pytest.param(192, 384, 96, MIXED * 16, False, False, id="b18-fp16-mixed-boards"),
    pytest.param(192, 384, 128, MIXED * 21 + MIXED[:2], True, False, id="b18-fp32-trunk"),
    pytest.param(192, 384, 77, None, True, True, id="b18-fp32-all"),
    pytest.param(64, 128, 50, MIXED * 8 + MIXED[:2], False, False, id="mid_nbt"),
    pytest.param(32, 64, 9, None, False, False, id="tiny_nbt"),
    pytest.param(32, 64, 9, None, True, True, id="tiny_nbt-fp32-all"),
])
def test_boundary_bit_identical(inner_c, trunk_c, n, boards, trunk_fp32, inner_fp32):
    out = _boundary(inner_c, trunk_c, n, 19, 19, boards, trunk_fp32, inner_fp32, seed=n + inner_c)
    assert out[:3].tolist() == [0, 0, 0], f"elements differing from the two launches (trunk.S, inner.S, inner.A): {out[:3]}"
    assert out[3:].tolist() == [0, 0, 0], f"nonzero elements in masked rows / padded channels: {out[3:]}"


def test_boundary_b28_falls_back():
    """b28c512nbt's 256-column entry accumulator is not compiled into the fused kernel: the hook says so instead of running it."""
    lib = load_library()
    out = np.zeros(6, np.int64)
    rc = lib.kgb_test_conv_boundary(256, 512, 8, 19, 19, None, 0, 0, C.c_uint32(1), out.ctypes.data_as(C.POINTER(C.c_int64)))
    assert rc != 0 and b"does not take" in lib.kgb_last_error()


def _forward(path, sp, gl, sym, opt, fuse, streams=None):
    env = {"KGB_FUSE_BOUNDARY": None if fuse else "0", "KGB_STREAM_FP32": streams}
    old = {k: os.environ.get(k) for k in env}
    try:
        for k, v in env.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v
        lm = NeuralNet.loadModelFile(path)
        ctx = NeuralNet.createComputeContext([0], 19, 19, True, lm)
        h = NeuralNet.createComputeHandle(ctx, lm, sp.shape[0], False, True, 0)
        launches = h.launches_per_forward
        got = NeuralNet.getOutput(h, sp.reshape(sp.shape[0], -1), gl, sym, opt)
        h.free(); ctx.free(); lm.free()
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v
    return got, launches


@pytest.mark.parametrize("cfg,n,streams,boundaries", [
    ("tiny_nbt", 5, None, 2),
    ("mid_nbt", 9, None, 3),
    ("b18c384nbt", 64, None, 17),
    ("b18c384nbt", 32, "trunk", 17),
    ("b18c384nbt", 32, "all", 17),
])
def test_net_outputs_unchanged(tmp_path, cfg, n, streams, boundaries):
    path = modelgen.write_model(str(tmp_path / f"{cfg}.bin"), cfg, seed=3)
    boards = [(19, 19), (9, 9), (13, 13), (19, 19), (7, 11)]
    sp, gl = modelgen.synthetic_inputs(n, 19, 19, seed=n, board_sizes=(boards * n)[:n])
    rng = np.random.default_rng(n)
    sym = rng.integers(0, 8, n).astype(np.int32)
    opt = rng.uniform(0, 1, n).astype(np.float32)
    fused, lf = _forward(path, sp, gl, sym, opt, True, streams)
    plain, lp = _forward(path, sp, gl, sym, opt, False, streams)
    assert lp - lf == boundaries
    for k in ("policy", "value", "score_value", "ownership"):
        assert np.isfinite(fused[k]).all()
        assert np.array_equal(fused[k].view(np.uint32), plain[k].view(np.uint32)), k
