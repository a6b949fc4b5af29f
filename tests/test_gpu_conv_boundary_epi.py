"""The fused block boundary's exit-epilogue warpgroup (kgb_conv_pair_epi_kernel: the exit's accumulators go through shared-memory
slots to a warpgroup of its own, so the MMAs run under the exit's epilogue) against kgb_conv_pair_kernel, which
KGB_PAIR_EPILOGUE_WG=0 keeps, and against the two launches that KGB_FUSE_BOUNDARY=0 keeps.  Single launches at several tile counts
and under a ragged mixed-size plan must equal the two launches bit for bit with either kernel; the chained b18 forward must give
the same bits with either kernel and unfused, and equal the same ops run one at a time.  fp32 streams, split mode and b28 keep
the other kernel, and no chain wait may give up."""
import ctypes as C
import os
import tempfile

import numpy as np
import pytest

from katago_b200 import NeuralNet, load_library, modelgen

pytestmark = pytest.mark.gpu

OUTPUTS = (("policy", 362), ("value", 3), ("score_value", 6), ("ownership", 361))
SWITCH = "KGB_PAIR_EPILOGUE_WG"
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
    return a.view(np.uint32)


def b19(n):
    return [(19, 19)] * n


# With 19x19 boards the plan has 400 n + 22 rows in 128-row tiles: 26, 132, 133, 792 and 801 tiles
SIZES = [(b19(8), 26), (b19(42), 132), (b19(42) + [(9, 9)], 133), (b19(253) + [(9, 9)], 792), (b19(256), 801)]
MIXED = [(9, 9), (13, 13), (19, 19), (19, 13), (13, 13), (19, 19), (9, 9), (19, 19)] * 24


def boundary_plan(boards, sym, seed):
    """kgb_test_conv_boundary_plan for b18's boundary (192 inner, 384 trunk channels, fp16 streams) under the ragged plan: the counts
    of elements that differ from the two launches, of nonzero elements off the board, of NaNs and of bytes written past the plan,
    and the plan's (rows, tiles, segments)."""
    lib = load_library()
    boards = np.ascontiguousarray(np.array(boards, np.int32).reshape(-1, 2))
    sym = np.ascontiguousarray(np.array(sym, np.int32))
    out, stats = np.zeros(12, np.int64), np.zeros(3, np.int64)
    rc = lib.kgb_test_conv_boundary_plan(192, 384, len(boards), 19, 19, boards.ctypes.data, sym.ctypes.data, 1, 0, 0, C.c_uint32(seed),
                                         out.ctypes.data, stats.ctypes.data)
    assert rc == 0, lib.kgb_last_error()
    return out, stats


@pytest.mark.parametrize("pair_epi", [True, False], ids=["epi-wg", "old-kernel"])
@pytest.mark.parametrize("boards,tiles", SIZES, ids=[str(t) for _, t in SIZES])
def test_single_launch_bit_identical(monkeypatch, pair_epi, boards, tiles):
    if pair_epi:
        monkeypatch.delenv(SWITCH, raising=False)
    else:
        monkeypatch.setenv(SWITCH, "0")
    out, stats = boundary_plan(boards, np.zeros(len(boards)), seed=tiles)
    assert stats[1] == tiles
    assert out.tolist() == [0] * 12, f"differing / off-board nonzero / NaN / past-the-end counts: {out.tolist()}"


@pytest.mark.parametrize("pair_epi", [True, False], ids=["epi-wg", "old-kernel"])
def test_single_launch_ragged_mixed_sizes(monkeypatch, pair_epi):
    if pair_epi:
        monkeypatch.delenv(SWITCH, raising=False)
    else:
        monkeypatch.setenv(SWITCH, "0")
    boards = [(19, 19), (9, 9), (13, 13), (7, 11), (19, 19), (5, 17), (13, 13), (19, 13)] * 12
    out, stats = boundary_plan(boards, np.arange(len(boards)) % 8, seed=3)
    assert stats[2] > 1
    assert out.tolist() == [0] * 12, f"differing / off-board nonzero / NaN / past-the-end counts: {out.tolist()}"


def forward(cfg, fp16, max_batch, batches):
    """Per batch (board sizes or n): the graph forward's outputs, checked bit for bit against the same ops run one at a time; and the
    handle's fused boundaries per forward that take the exit-epilogue warpgroup."""
    import torch
    lm = model(cfg)
    ctx = NeuralNet.createComputeContext([0], 19, 19, fp16, lm)
    h = NeuralNet.createComputeHandle(ctx, lm, max_batch, False, True, 0)
    lib = load_library()
    dev = torch.device("cuda:0")
    res = []
    try:
        pairs = lib.kgb_handle_pair_epilogue_wg_launches_per_forward(h._p)
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
    return res, pairs


def with_env(monkeypatch, env, fn):
    for k, v in env.items():
        if v is None:
            monkeypatch.delenv(k, raising=False)
        else:
            monkeypatch.setenv(k, v)
    try:
        return fn()
    finally:
        for k in env:
            monkeypatch.delenv(k, raising=False)


def test_b18_forward_bit_identical(monkeypatch):
    """b18c384nbt's 17 boundaries: the exit-epilogue warpgroup, the old fused kernel and the two launches give the same bits"""
    batches = [boards for boards, _ in SIZES] + [MIXED]
    run = lambda: forward("b18c384nbt", True, 256, batches)
    on, n_on = with_env(monkeypatch, {SWITCH: None, "KGB_FUSE_BOUNDARY": None}, run)
    off, n_off = with_env(monkeypatch, {SWITCH: "0", "KGB_FUSE_BOUNDARY": None}, run)
    unfused, n_unfused = with_env(monkeypatch, {SWITCH: None, "KGB_FUSE_BOUNDARY": "0"}, run)
    assert (n_on, n_off, n_unfused) == (17, 0, 0)
    for i in range(len(batches)):
        for (k, _), x, y, z in zip(OUTPUTS, on[i], off[i], unfused[i]):
            assert np.array_equal(bits(x), bits(y)) and np.array_equal(bits(x), bits(z)), (i, k)


@pytest.mark.parametrize("streams", ["trunk", "all"])
def test_fp32_streams_keep_the_other_kernel(monkeypatch, streams):
    res, pairs = with_env(monkeypatch, {"KGB_STREAM_FP32": streams}, lambda: forward("b18c384nbt", True, 16, [16]))
    assert pairs == 0


def test_split_mode_and_b28_keep_the_other_kernel():
    assert forward("b18c384nbt", False, 16, [16])[1] == 0    # fp32-equivalent mode: no fused boundaries
    assert forward("b28c512nbt", True, 16, [16])[1] == 0     # (256, 512) boundaries stay two launches
