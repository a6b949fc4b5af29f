"""Chained convolution launches: in a forward, a convolution that follows another one starts while the previous one's last tiles
still run, and waits per tile for the rows it reads (kgb_conv.cuh, launchConvWG).  The graph forward must give the same bits as
the same ops run one at a time with a stream synchronise after each (kgb_test_forward_serial), at tile counts below, at and just
above one round of CTAs, at the end of the 6th round and in the 7th, on ragged mixed-size batches, in every stream precision, on a
net with two n-tiles per launch, and over replays with rotating inputs; and no flag wait may ever give up."""
import ctypes as C
import os
import tempfile

import numpy as np
import pytest

from katago_b200 import NeuralNet, load_library, modelgen

pytestmark = pytest.mark.gpu

OUTPUTS = (("policy", 362), ("value", 3), ("score_value", 6), ("ownership", 361))
_models = {}


def model(cfg):
    if cfg not in _models:
        path = modelgen.write_model(os.path.join(tempfile.mkdtemp(), cfg + ".bin"), cfg, seed=3)
        _models[cfg] = NeuralNet.loadModelFile(path)
    return _models[cfg]


def chain_error():
    v = C.c_int(-1)
    assert load_library().kgb_conv_chain_error(C.byref(v)) == 0
    return v.value


def chained_launches(cfg, fused):
    """Convolution launches that directly follow another one: of the initial conv, per nested block an entry 1x1, two inner units of
    two 3x3 each and an exit 1x1, and the heads' 1x1, all but the initial conv (it follows the global-input matmul) and each gpool
    unit's second conv (it follows the pooling kernels).  A fused boundary is one launch for an exit and the next entry."""
    blocks = modelgen.CONFIGS[cfg]["blocks"]
    convs = 1 + 6 * len(blocks) + 1 - (len(blocks) - 1 if fused else 0)
    return convs - 1 - blocks.count("N")


def run_case(cfg, fp16, max_batch, batches, replays=1, monkeypatch=None, streams=None, fused=True):
    """batches: list of (board_sizes or n, expected m_tiles or None).  Every batch runs `replays` times through the graph with
    inputs rotating over three seeds, each compared bit for bit with the serial run of the same inputs."""
    import torch
    if streams is not None:
        monkeypatch.setenv("KGB_STREAM_FP32", streams)
    lm = model(cfg)
    ctx = NeuralNet.createComputeContext([0], 19, 19, fp16, lm)
    h = NeuralNet.createComputeHandle(ctx, lm, max_batch, False, True, 0)
    lib = load_library()
    dev = torch.device("cuda:0")
    try:
        # the launches are actually chained, not merely correct
        assert lib.kgb_handle_chained_launches_per_forward(h._p) == chained_launches(cfg, fused)
        for boards, want_tiles in batches:
            n = boards if isinstance(boards, int) else len(boards)
            sizes = None if isinstance(boards, int) else boards
            inputs = []
            for seed in range(3):
                sp, gl = modelgen.synthetic_inputs(n, 19, 19, seed=100 * n + seed, board_sizes=sizes)
                inputs.append((torch.from_numpy(sp.reshape(n, -1)).to(dev), torch.from_numpy(gl).to(dev)))
            outs = {k: [torch.full((n, w), float("nan"), device=dev) for _ in range(2)] for k, w in OUTPUTS}
            torch.cuda.synchronize()
            for r in range(replays):
                dsp, dgl = inputs[r % 3]
                got = []
                for which, fn in enumerate((lib.kgb_forward_device, lib.kgb_test_forward_serial)):
                    bufs = [outs[k][which] for k, _ in OUTPUTS]
                    for b in bufs:
                        b.fill_(float("nan"))
                    torch.cuda.synchronize()
                    rc = fn(h._p, n, dsp.data_ptr(), dgl.data_ptr(), None, None, *(b.data_ptr() for b in bufs))
                    assert rc == 0, lib.kgb_last_error()
                    h.sync()
                    got.append([b.cpu().numpy() for b in bufs])
                for (k, _), a, b in zip(OUTPUTS, got[0], got[1]):
                    assert np.isfinite(b).all(), (cfg, n, k)
                    assert np.array_equal(a.view(np.uint32), b.view(np.uint32)), (cfg, fp16, streams, n, r, k, float(np.abs(a - b).max()))
                assert chain_error() == 0
            if want_tiles is not None:
                assert h.layout_stats()["m_tiles"] == want_tiles
    finally:
        h.free()
        ctx.free()


# With 19x19 boards the plan has 400 n + 22 rows, rounded up to 128; a 9x9 board adds one tile of its own.  On 132 SMs: 132 tiles
# are one round, 792 six and 801 seven.
def b19(n):
    return [(19, 19)] * n


def test_b18_tile_counts_fp16():
    run_case("b18c384nbt", True, 256, [(8, 26), (42, 132), (b19(42) + [(9, 9)], 133), (b19(253) + [(9, 9)], 792), (256, 801)])


def test_b18_replays_rotating_inputs_fp16():
    run_case("b18c384nbt", True, 256, [(256, 801)], replays=20)


def test_b18_ragged_mixed_sizes():
    sizes = [(9, 9), (13, 13), (19, 19), (19, 13), (13, 13), (19, 19), (9, 9), (19, 19)] * 24
    run_case("b18c384nbt", True, 256, [(sizes, None)], replays=3)


def test_b18_fp32_streams(monkeypatch):
    run_case("b18c384nbt", True, 256, [(42, 132), (256, 801)], monkeypatch=monkeypatch, streams="all")


def test_b18_split_mode():
    run_case("b18c384nbt", False, 256, [(42, 132), (256, 801)], fused=False)   # split mode keeps two launches per boundary


def test_b28_two_n_tiles():
    run_case("b28c512nbt", True, 64, [(16, None), (64, None)], replays=2, fused=False)   # b28's boundary shape is not fused
