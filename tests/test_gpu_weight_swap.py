"""GPU tests (H100) of the weight hot-swap behind the C ABI (include/kgb200.h: kgb_handle_stage_weights,
kgb_handle_commit_weights, kgb_nccl_unique_id, kgb_handle_comm_init, kgb_handle_broadcast_staged_weights).

Reference behaviour replaced: the self-play command polls its models directory and builds a fresh NNEvaluator per new net
(cpp/command/selfplay.cpp:142-231,336-352); games move over to it between moves (switchNetsMidGame).  Here a handle keeps
its graphs and buffers and only its weight arena changes; the bar is bit-equality with a handle built from the new file.
The 2-GPU broadcast is exercised by tests/gpu_checks/weight_swap_nccl.py under torchrun (bench.py runs it at N > 1)."""
import numpy as np
import pytest

from katago_b200 import NeuralNet, modelgen
from katago_b200.nn_backend import KGBError, SelfPlay, nccl_unique_id

pytestmark = pytest.mark.gpu


def _handle(path, fp16, batch=8, X=19):
    lm = NeuralNet.loadModelFile(path)
    ctx = NeuralNet.createComputeContext([0], X, X, fp16, lm)
    return lm, ctx, NeuralNet.createComputeHandle(ctx, lm, batch, False, True, 0)


@pytest.mark.parametrize("fp16", [False, True])
@pytest.mark.parametrize("cfg", ["tiny_nbt", "mid_nbt", "tiny_reg"])
def test_staged_and_committed_weights_equal_a_fresh_handle(tmp_path, cfg, fp16):
    a = modelgen.write_model(str(tmp_path / "a.bin"), cfg, seed=11)
    b = modelgen.write_model(str(tmp_path / "b.bin"), cfg, seed=12)
    sp, gl = modelgen.synthetic_inputs(5, 19, 19, seed=3)
    sym = np.array([0, 3, 5, 6, 1])
    lmA, ctxA, hA = _handle(a, fp16)
    lmB, ctxB, hB = _handle(b, fp16)
    outA = NeuralNet.getOutput(hA, sp.reshape(5, -1), gl, sym)
    outB = NeuralNet.getOutput(hB, sp.reshape(5, -1), gl, sym)
    assert hA.weights_bytes == hB.weights_bytes > 0
    assert not np.array_equal(outA["policy"], outB["policy"])
    hA.stage_weights(lmB)
    # staging alone changes nothing: evaluation continues on the old net until the commit
    mid = NeuralNet.getOutput(hA, sp.reshape(5, -1), gl, sym)
    for k in outA:
        assert np.array_equal(mid[k], outA[k]), k
    hA.commit_weights()
    new = NeuralNet.getOutput(hA, sp.reshape(5, -1), gl, sym)
    for k in outB:
        assert np.array_equal(new[k], outB[k]), k
    # and back again: the arena is reusable
    hA.stage_weights(lmA); hA.commit_weights()
    back = NeuralNet.getOutput(hA, sp.reshape(5, -1), gl, sym)
    for k in outA:
        assert np.array_equal(back[k], outA[k]), k
    with pytest.raises(KGBError, match="nothing is staged"):
        hA.commit_weights()
    for o in (hA, hB, ctxA, ctxB, lmA, lmB):
        o.free()


def test_a_net_of_another_architecture_is_refused(tmp_path):
    a = modelgen.write_model(str(tmp_path / "a.bin"), "tiny_nbt", seed=1)
    lmA, ctxA, hA = _handle(a, True)
    sp, gl = modelgen.synthetic_inputs(2, 19, 19, seed=5)
    before = NeuralNet.getOutput(hA, sp.reshape(2, -1), gl)
    for other, kw in (("mid_nbt", {}), ("tiny_reg", {}), ("tiny_nbt", {"activation": "ACTIVATION_RELU"})):
        lm = NeuralNet.loadModelFile(modelgen.write_model(str(tmp_path / "o.bin"), other, seed=2, **kw))
        with pytest.raises(KGBError, match="architecture|layout"):
            hA.stage_weights(lm)
        lm.free()
    after = NeuralNet.getOutput(hA, sp.reshape(2, -1), gl)       # a refused model leaves the live net untouched
    for k in before:
        assert np.array_equal(before[k], after[k]), k
    hA.free(); ctxA.free(); lmA.free()


def test_single_rank_communicator_broadcast_and_commit(tmp_path):
    """NCCL through the library with one rank: id, communicator, broadcast (to itself), commit."""
    a = modelgen.write_model(str(tmp_path / "a.bin"), "tiny_nbt", seed=21)
    b = modelgen.write_model(str(tmp_path / "b.bin"), "tiny_nbt", seed=22)
    lmA, ctxA, hA = _handle(a, True)
    lmB, ctxB, hB = _handle(b, True)
    sp, gl = modelgen.synthetic_inputs(3, 19, 19, seed=8)
    want = NeuralNet.getOutput(hB, sp.reshape(3, -1), gl)
    with pytest.raises(KGBError, match="comm_init first"):
        hA.broadcast_staged_weights(0)
    uid = nccl_unique_id()
    assert len(uid) == 128
    hA.comm_init(uid, 0, 1)
    with pytest.raises(KGBError, match="nothing staged"):
        hA.broadcast_staged_weights(0)
    hA.stage_weights(lmB)
    ms = hA.broadcast_staged_weights(0)
    assert ms >= 0.0
    hA.commit_weights()
    got = NeuralNet.getOutput(hA, sp.reshape(3, -1), gl)
    for k in want:
        assert np.array_equal(got[k], want[k]), k
    for o in (hA, hB, ctxA, ctxB, lmA, lmB):
        o.free()


def test_games_continue_across_a_swap_and_then_search_with_the_new_net(tmp_path):
    """A loop on a swapped handle (evaluation cache emptied) continues from its positions exactly like a loop on a handle that was
    built from the new net and brought to the same positions."""
    a = modelgen.write_model(str(tmp_path / "a.bin"), "tiny_nbt", seed=31)
    b = modelgen.write_model(str(tmp_path / "b.bin"), "tiny_nbt", seed=32)
    lmA, ctxA, hA = _handle(a, False, batch=4, X=9)
    lmB, ctxB, hB = _handle(b, False, batch=4, X=9)
    kw = dict(komi=7.5, multi_stone_suicide_legal=True, seed=5, debug_hold_at_max_visits=True, debug_fixed_symmetry=0, nn_cache_size_power_of_two=12,
              root_ending_bonus_points=0.5, root_prune_useless_moves=True)
    moves = [(2, 2), (6, 6), (2, 6), (6, 2), (4, 4)]
    spA = SelfPlay(hA, 4, 40, **kw)
    spA.play_moves(moves)
    spA.set_search_rand("swap-test")
    spA.run(12)                                   # a search on the old net is under way (tree and cache hold its outputs)
    before = spA.stats()
    hA.stage_weights(lmB)
    hA.commit_weights()
    spA.clear_nn_cache()
    spA.run(12)
    assert spA.stats()["total_visits"] > before["total_visits"]
    # fresh searches on the swapped handle == searches on the handle built from the new net
    spA2 = SelfPlay(hA, 4, 40, **kw); spB = SelfPlay(hB, 4, 40, **kw)
    for s in (spA2, spB):
        s.play_moves(moves)
        s.set_search_rand("swap-test")
        for _ in range(40):
            s.run(8)
            if all(s.game(g)[1]["root_visits"] >= 40 for g in range(4)):
                break
    for g in range(4):
        va, pa, ua = spA2.root_children(g)
        vb, pb, ub = spB.root_children(g)
        assert np.array_equal(va, vb) and np.array_equal(pa, pb) and np.array_equal(ua, ub)
    for o in (spA, spA2, spB, hA, hB, ctxA, ctxB, lmA, lmB):
        o.free()
