"""BASELINE config 4 ("mixed 9/13/19 board sizes ... per-board masking") and the per-game rules of the reference's GameInitializer
(program/play.cpp:330-650) in the device loop: games of different board sizes and ko rules side by side in one loop, one evaluator
frame.  Fixtures: tests/golden/make_mixed_size_fixtures.py (the reference's Search / fillRowV7 with nnXLen = nnYLen = 19 > board)."""
import json
import os

import numpy as np
import pytest

from katago_b200 import NeuralNet, SelfPlay

pytestmark = pytest.mark.gpu


def _snake(name):
    return "".join("_" + ch.lower() if ch.isupper() else ch for ch in name)


def _kwargs(params):
    kw = dict(cpuct_exploration=1.0, cpuct_exploration_log=0.45, cpuct_exploration_base=500.0, fpu_reduction_max=0.2, root_fpu_reduction_max=0.1)
    for k, v in params.items():
        name = "min_visit_prop_for_lcb" if k == "minVisitPropForLCB" else _snake(k)
        kw[name] = (bool(v) if k in ("fpuParentWeightByVisitedPolicy", "useGraphSearch", "useLcbForSelection", "useNonBuggyLcb", "rootPruneUselessMoves")
                    else int(v) if k in ("graphSearchRepBound", "rootNumSymmetriesToSample") else float(v))
    return kw


def _moves(arr):
    return [None if m[0] < 0 else (int(m[0]), int(m[1])) for m in arr]


def test_games_of_different_sizes_and_ko_rules_search_like_the_reference(golden_dir, tmp_models):
    """Six games - 19x19, 9x9 (positional superko), 13x7, 5x5 (situational superko), 7x7 (root move pruning position), 9x9 - in ONE loop with a
    19x19 evaluator frame, each compared with the reference Search run on that board inside a 19x19 NNEvaluator: identical visit counts,
    policies (illegal = everything off the game's own board too), child utilities, NodeStats moments and play selection values.  Exercises
    per game: board masks, score utility and root temperature scaled by the game's own area, superko bans, pass-alive pruning, ending bonus
    read from the frame-indexed ownership, transposition / bias tables."""
    d = np.load(os.path.join(golden_dir, "searchfake_mixed.npz"))
    n, frame, visits = int(d["num_games"]), int(d["frame"]), int(d["visits"])
    lm = NeuralNet.loadModelFile(tmp_models["tiny_reg"])
    ctx = NeuralNet.createComputeContext([0], frame, frame, True, lm)
    h = NeuralNet.createComputeHandle(ctx, lm, 8, False, True, 0)
    sp = SelfPlay(h, n, visits, komi=7.5, multi_stone_suicide_legal=True, early_temperature_moves=0, seed=1, debug_fake_nn=True,
                  debug_hold_at_max_visits=True, **_kwargs(json.loads(str(d["params"]))))
    setups = np.stack([d[f"g{g}_setup"] for g in range(n)])
    sp.set_game_setup(setups, also_current_games=True)
    cur, _ = sp.game_setups()
    assert np.array_equal(cur, setups)
    for g in range(n):
        sp.play_moves_game(g, _moves(d[f"g{g}_moves"]))
    with pytest.raises(Exception, match="off the board"):
        sp.play_moves_game(1, [(12, 3)])                     # game 1 is 9x9
    for _ in range(200):
        sp.run(max(8, visits // 8))
        if all(sp.game(g)[1]["root_visits"] >= visits for g in range(n)):
            break
    for g in range(n):
        X, Y = int(setups[g, 0]), int(setups[g, 1])
        colors, info = sp.game(g)
        assert info["root_visits"] == visits
        assert not colors[Y:, :].any() and not colors[:, X:].any(), "stones off the game's board"
        v, pol, util = sp.root_children(g)
        ref_pol, ref_v, ref_u = d[f"g{g}_policy"], d[f"g{g}_visits"], d[f"g{g}_util"]
        assert np.array_equal(pol < 0, ref_pol < 0), f"game {g}: legality mask differs"
        assert np.abs(pol - ref_pol)[ref_pol >= 0].max() < 2e-6
        assert np.array_equal(v, ref_v), (g, np.nonzero(v != ref_v), v[v != ref_v], ref_v[v != ref_v])
        assert np.abs(util - ref_u)[v > 0].max() < 1e-12
        ch, rt = sp.root_value_stats(g)
        assert np.abs(ch - d[f"g{g}_child_stats"])[v > 0].max() < 1e-9 and np.abs(rt - d[f"g{g}_root_stats"]).max() < 1e-9
        psv, ref_psv = sp.play_selection_values(g), d[f"g{g}_play_selection"]
        assert np.array_equal(psv < 0, ref_psv < 0)
        assert np.abs(psv - ref_psv).max() <= 1e-9 * max(1.0, np.abs(ref_psv).max())
    sp.free(); h.free(); ctx.free()


def test_feature_rows_of_small_boards_inside_the_frame_match_fillRowV7(golden_dir, tmp_models):
    """NNInputs::fillRowV7 with nnXLen = 19 on 9x9, 13x7 and 13x13 boards (the reference run that way) vs the rows three games of one loop
    write: every plane incl. ladders and pass-alive area and all 19 globals bit-exact; plane 0 = the game's board, nothing outside it."""
    names = ["featstream_9x9_in_19", "featstream_13x7_in_19", "featstream_13x13_in_19"]
    fx = [np.load(os.path.join(golden_dir, nm + ".npz")) for nm in names]
    frame = int(fx[0]["frame"])
    lm = NeuralNet.loadModelFile(tmp_models["tiny_reg"])
    ctx = NeuralNet.createComputeContext([0], frame, frame, True, lm)
    h = NeuralNet.createComputeHandle(ctx, lm, 4, False, True, 0)
    steps = min(len(f["steps"]) for f in fx)
    setups = np.array([[int(f["X"]), int(f["Y"]), 0, int(f["multi"])] for f in fx], np.int32)
    checked = 0
    for i in range(steps):
        sp = SelfPlay(h, 3, 8, komi=7.5, multi_stone_suicide_legal=True, seed=1, debug_fake_nn=True)
        sp.set_game_setup(setups, also_current_games=True)
        for g, f in enumerate(fx):
            sp.play_moves_game(g, _moves(f["moves"][:int(f["steps"][i])]))
        sp.run(1)
        for g, f in enumerate(fx):
            row, gl = sp.nn_row(g)
            ref_row, ref_gl = f["rows"][i].astype(np.float32), f["glob"][i]
            for pl in range(22):
                assert np.array_equal(row[:, pl], ref_row[:, pl]), f"{names[g]} step {int(f['steps'][i])} plane {pl}: {np.nonzero(row[:, pl] != ref_row[:, pl])[0][:8]}"
            assert np.array_equal(gl, ref_gl), f"{names[g]} step {int(f['steps'][i])} globals {gl} vs {ref_gl}"
            checked += 1
        sp.free()
    assert checked == 3 * steps
    h.free(); ctx.free()


def test_mixed_size_self_play_runs_games_to_the_end_and_takes_the_next_setup(tmp_models):
    """The real evaluator in the loop, evaluation cache shared by games of different sizes: every slot plays its game to the end on its
    own board, the finished game's score is its own area count with its own komi, and the slot's next game starts with the setup (and
    komi) handed over for it."""
    lm = NeuralNet.loadModelFile(tmp_models["tiny_reg"])
    frame = 13
    ctx = NeuralNet.createComputeContext([0], frame, frame, True, lm)
    h = NeuralNet.createComputeHandle(ctx, lm, 8, False, True, 0)
    n = 6
    sp = SelfPlay(h, n, 12, komi=7.5, max_moves=60, seed=5, use_graph_search=True, value_weight_exponent=0.5, nn_cache_size_power_of_two=12,
                  root_num_symmetries_to_sample=2, debug_hold_at_max_visits=True)
    first = np.array([[5, 5, 0, 1], [7, 7, 1, 0], [9, 9, 2, 1], [13, 13, 0, 1], [9, 5, 0, 0], [13, 7, 3, 1]], np.int32)
    nxt = np.array([[13, 13, 1, 0], [5, 5, 0, 1], [7, 9, 0, 1], [9, 9, 0, 0], [13, 13, 2, 1], [6, 6, 0, 1]], np.int32)
    komi1 = np.array([5.5, 6.0, 7.0, 7.5, -3.5, 0.5], np.float32)
    komi2 = np.array([7.5, 4.5, 6.5, 7.0, 7.5, 2.0], np.float32)
    sp.set_game_setup(first, also_current_games=True); sp.set_komi(komi1, also_current_games=True)
    sp.set_game_setup(nxt); sp.set_komi(komi2)
    with pytest.raises(Exception, match="fit the evaluator's frame"):
        sp.set_game_setup(np.array([[14, 13, 0, 1]] * n, np.int32))
    finished = {}
    for it in range(4000):
        sp.run(8)
        held = np.asarray(sp.root_visits()) >= sp.max_visits
        for g in np.flatnonzero(held):
            colors, info = sp.game(int(g))
            X, Y = (first if int(g) not in finished else nxt)[g, :2]
            assert not colors[Y:, :].any() and not colors[:, X:].any(), (g, X, Y)
            v, pol, _ = sp.root_children(int(g))
            on = np.zeros((frame, frame), bool); on[:Y, :X] = True
            assert (pol[:-1].reshape(frame, frame)[~on] < 0).all() and v[:-1].reshape(frame, frame)[~on].sum() == 0
        sp.release(held.astype(np.uint8))
        sp.run(1)
        for g in np.flatnonzero(held):
            last = sp.last_move(int(g))
            if last["game_over"] and int(g) not in finished:
                finished[int(g)] = last
                cur, lastf = sp.game_setups()
                assert np.array_equal(lastf[g], first[g]) and np.array_equal(cur[g], nxt[g])
                kc, kl = sp.komi_values()
                assert kl[g] == komi1[g] and kc[g] == komi2[g]
                X, Y = first[g, :2]
                fc, fa = np.asarray(last["final_colors"]).reshape(frame, frame), np.asarray(last["final_area"]).reshape(frame, frame)
                assert not fc[Y:, :].any() and not fc[:, X:].any() and not fa[Y:, :].any() and not fa[:, X:].any()
                if not last["no_result"] and not last["hit_move_limit"]:
                    assert last["final_white_minus_black_score"] == komi1[g] - (int((fa == 1).sum()) - int((fa == 2).sum()))
        if len(finished) == n and it > 50:
            break
    assert len(finished) == n, sorted(finished)
    st = sp.stats()
    assert st["games_finished"] >= n and st["nn_cache_hits"] > 0
    sp.free(); h.free(); ctx.free()


def test_games_of_different_sizes_never_share_an_evaluation_cache_entry(tmp_models):
    """NNInputs::getHash contains the board size and the rules (through Board::pos_hash and Rules): the same stones on a 9x9 and on a 13x13
    board, or under two ko rules, are different evaluations."""
    lm = NeuralNet.loadModelFile(tmp_models["tiny_reg"])
    ctx = NeuralNet.createComputeContext([0], 13, 13, True, lm)
    h = NeuralNet.createComputeHandle(ctx, lm, 4, False, True, 0)
    sp = SelfPlay(h, 4, 8, komi=7.5, seed=3, nn_cache_size_power_of_two=10, debug_fixed_symmetry=0)
    sp.set_game_setup(np.array([[9, 9, 0, 1], [13, 13, 0, 1], [9, 9, 1, 1], [9, 9, 0, 1]], np.int32), also_current_games=True)
    sp.play_moves([(2, 2), (3, 3)])
    sp.run(1)
    keys = [tuple(int(k) for k in sp.leaf_cache_key(g)) for g in range(4)]
    assert keys[0] == keys[3] and len({keys[0], keys[1], keys[2]}) == 3, keys
    sp.free(); h.free(); ctx.free()


def test_policy_initialised_openings(tmp_models, golden_dir):
    """PlayUtils::initializeGameUsingPolicy on the device: the first moves of a game are drawn from the net's raw policy, one evaluation per
    move, without holding the slot; the recorder's first turn comes after them.  The kept opening replays to the slot's root position, and at a
    low temperature the draw concentrates on the policy's best move."""
    from katago_b200 import nn_backend
    lm = NeuralNet.loadModelFile(tmp_models["tiny_reg"])
    ctx = NeuralNet.createComputeContext([0], 9, 9, True, lm)
    h = NeuralNet.createComputeHandle(ctx, lm, 64, False, True, 0)
    want = np.array([0, 3, 10, 5, 0, 7, 1, 12], np.int32)
    sp = SelfPlay(h, 8, 16, komi=7.5, seed=11, debug_hold_at_max_visits=True, nn_cache_size_power_of_two=10, root_num_symmetries_to_sample=2, root_noise_enabled=True,
                  use_play_selection=True)
    sizes = np.array([[9, 9, 0, 1]] * 6 + [[7, 7, 0, 1], [9, 5, 0, 1]], np.int32)
    sp.set_game_setup(sizes, also_current_games=True)
    sp.set_policy_init(want, 1.0, also_current_games=True)
    sp.set_policy_init(np.full(8, 2, np.int32), 1.0)                      # the slots' next games
    for _ in range(100):
        sp.run(8)
        if (sp.root_visits() >= 16).all():
            break
    left, cnt, moves = sp.policy_init(max_moves=64)
    assert (left == 0).all() and np.array_equal(cnt, want), (left, cnt)
    for g in range(8):
        colors, info = sp.game(g)
        assert info["move_num"] == want[g] and info["root_visits"] == 16
        X, Y = int(sizes[g, 0]), int(sizes[g, 1])
        assert all(m == (-1, -1) or (0 <= m[0] < X and 0 <= m[1] < Y) for m in moves[g])
        if want[g] > 0:
            rep = nn_backend.board_replay(X, Y, np.array([[[m[0], m[1], 1 + (i % 2)] for i, m in enumerate(moves[g])]], np.int8), True)
            assert np.array_equal(rep["colors"][0, -1], colors[:Y, :X]), g          # the opening leads to the root the search is held at
    with pytest.raises(Exception, match="already started"):
        sp.set_policy_init(want, 1.0, also_current_games=True)
    sp.free()
    h.free(); ctx.free()
    # the draw follows policy ^ (1 / T): a trained net (peaked policy), 128 games draw one move each from the same empty-board evaluation
    lm = NeuralNet.loadModelFile(os.path.join(golden_dir, "models", "g170-b6c96-s175395328-d26788732.bin.gz"))
    ctx = NeuralNet.createComputeContext([0], 9, 9, True, lm)
    h = NeuralNet.createComputeHandle(ctx, lm, 128, False, True, 0)
    ref = SelfPlay(h, 1, 4, komi=7.5, seed=1, debug_hold_at_max_visits=True, debug_fixed_symmetry=0)
    ref.run(2)
    pol = ref.root_children(0)[1]
    ref.free()
    T = 0.5
    sp = SelfPlay(h, 128, 4, komi=7.5, seed=5, debug_hold_at_max_visits=True, debug_fixed_symmetry=0)
    sp.set_policy_init(np.ones(128, np.int32), T, also_current_games=True)
    for _ in range(8):
        sp.run(4)
    _, cnt, moves = sp.policy_init(max_moves=4)
    assert (cnt == 1).all()
    drawn = np.array([m[0][1] * 9 + m[0][0] if m[0][0] >= 0 else 81 for m in moves])
    weights = np.where(pol > 0, pol.astype(np.float64), 0.0) ** (1.0 / T)
    weights /= weights.sum()
    top = np.argsort(-weights)[:4]
    expect, got = float(weights[top].sum()), float(np.isin(drawn, top).mean())
    assert expect > 0.3 and abs(got - expect) < 4 * np.sqrt(expect * (1 - expect) / 128) + 0.02, (got, expect)
    assert (weights[drawn] > 0).all()
    sp.free(); h.free(); ctx.free()
