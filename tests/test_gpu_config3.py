"""BASELINE config 3 at its full size: 19x19, b28c512nbt, 1024 concurrent games, maxVisits 1600.

  * The b28 evaluator at 1024 rows (3200 m-tiles per convolution) in both modes: finite, a row's result independent of its batch
    position (bit for bit), the two modes within fp16 accuracy of each other, and sampled rows against the numpy oracle.
  * The device loop at 1024 games x 1600 visits with the fake net and the evaluation cache shared by all games: 8 slots spread over
    the index range search like the reference's Search (fixture: tests/golden/make_search1600_fixture.py).
  * The real b28 net in the loop: a game's search does not depend on how many other games share the loop.

Every slot that is not sampled starts from a prefix of one of two 19x19 games (the board streams with game-ending pass pairs
dropped, stored in the fixture), of length g mod 150 under the suicide rule the game was recorded with, so the loop holds games
at many stages.  Only one loop is alive at a time."""
import json
import os

import numpy as np
import pytest

import kg_nn_oracle as orc
from katago_b200 import NeuralNet, SelfPlay, modelgen
from test_gpu_mixed_sizes import _kwargs, _moves
from test_gpu_nn_parity import FP16_REL, FP32_TOL, run_cuda

pytestmark = pytest.mark.gpu

GAMES, VISITS = 1024, 1600
KEYS = ("policy", "value", "score_value", "ownership")


def _place(sp, fx, placed):
    """placed: {slot: move array} under multi-stone suicide.  Every other slot g: the first g mod 150 moves of one of the two fill
    games (alternating every 150 slots), under that game's suicide rule."""
    streams = ((fx["fill_multisuicide"], 1), (fx["fill_nosuicide"], 0))
    setups = np.tile(np.array([19, 19, 0, 1], np.int32), (sp.num_games, 1))
    lists = []
    for g in range(sp.num_games):
        if g in placed:
            lists.append(placed[g])
        else:
            moves, multi = streams[(g // 150) % 2]
            setups[g, 3] = multi
            lists.append(moves[:g % 150])
    sp.set_game_setup(setups, also_current_games=True)
    for g, mv in enumerate(lists):
        sp.play_moves_game(g, _moves(mv))


@pytest.fixture(scope="module")
def fixture_1600(golden_dir):
    return np.load(os.path.join(golden_dir, "searchfake_1600.npz"))


@pytest.fixture(scope="module")
def b28_model(tmp_path_factory):
    return modelgen.write_model(str(tmp_path_factory.mktemp("b28") / "b28c512nbt.bin"), "b28c512nbt", seed=0)


# ---- the evaluator at 1024 rows --------------------------------------------------------------------------------------------------

SAMPLED_ROWS = np.array([0, 1, 300, 510, 511, 512, 513, 1023])


@pytest.fixture(scope="module")
def b28_batch1024(b28_model):
    n = GAMES
    sp, gl = modelgen.synthetic_inputs(n, 19, 19, seed=79)
    sym = (np.arange(n) * 3 + 1) % 8
    sp[n // 2:] = sp[:n // 2][::-1]; gl[n // 2:] = gl[:n // 2][::-1]; sym[n // 2:] = sym[:n // 2][::-1]   # second half = first half reversed
    got16 = run_cuda(b28_model, sp, gl, sym, None, True, max_batch=n)
    got32 = run_cuda(b28_model, sp, gl, sym, None, False, max_batch=n)
    idx = SAMPLED_ROWS
    ref = orc.get_output(orc.load_model(b28_model), sp[idx], gl[idx], sym[idx])
    return got16, got32, ref


def test_b28_batch1024_rows_and_modes(b28_batch1024):
    """b28c512nbt at 1024 rows: every output finite; rows 512-1023 (rows 0-511 reversed) give bit-identical results in both modes;
    fp16 mode agrees with fp32-equivalent mode and, on the sampled rows, with the fp32 oracle to fp16 accuracy."""
    got16, got32, ref = b28_batch1024
    h = GAMES // 2
    for k in KEYS:
        for got in (got16, got32):
            assert np.isfinite(got[k]).all(), k
            assert np.array_equal(got[k][h:], got[k][:h][::-1]), k
        assert np.abs(got16[k] - got32[k]).max() <= FP16_REL * max(1.0, np.abs(got32[k]).max()), k
        err16 = np.abs(got16[k][SAMPLED_ROWS] - ref[k]).max()
        print(f"{k}: fp16 mode - fp32 oracle {err16:.3g}")
        assert err16 <= FP16_REL * max(1.0, np.abs(ref[k]).max()), (k, err16)


@pytest.mark.xfail(strict=True, reason="measured on an H100 80GB HBM3 (700 W): up to 6.4e-3 (policy), 3.9e-3 (ownership), 1.2e-3 (score). "
                   "Every b28 layer shape stays within its derived bound in test_gpu_conv_fp64.py: the shortfall is the tensor core's "
                   "truncating fp32 accumulation, which this net amplifies more than b18 (DESIGN section 4)")
def test_b28_batch1024_fp32_equivalent_mode_against_oracle(b28_batch1024):
    """The sampled rows of fp32-equivalent mode within 1e-3 of the fp32 oracle (north star: logits within 1e-3 fp32)."""
    _, got32, ref = b28_batch1024
    errs = {k: float(np.abs(got32[k][SAMPLED_ROWS] - ref[k]).max()) for k in KEYS}
    print("fp32-equivalent mode - fp32 oracle:", {k: f"{v:.3g}" for k, v in errs.items()})
    assert max(errs.values()) <= FP32_TOL, errs


# ---- the search at 1024 games x 1600 visits against the reference -----------------------------------------------------------------

FIXTURE_SLOTS = (0, 1, 255, 511, 512, 767, 1022, 1023)   # slot of fixture case i


def test_search_1024_games_1600_visits_matches_reference(fixture_1600, tmp_models):
    """One loop of 1024 games at 1600 visits with the fake net, the search block bench.py runs (as far as the reference driver
    implements it) and an evaluation cache shared by all games.  The 8 fixture positions sit in slots spread over the index range,
    and each must match the reference's Search like test_tree_search_matches_reference_search_with_fake_net: identical child
    visits, utilities to 1e-12, value moments to 1e-9, play selection values to 1e-9.  The other games hit the cache with entries
    of other games; that must change nothing.  All 1024 games: the root's children hold its visits minus one, no root exceeds
    1600 visits, the visits add up to the loop's total, and nothing is non-finite."""
    d = fixture_1600
    assert int(d["visits"]) == VISITS and int(d["num_cases"]) == len(FIXTURE_SLOTS)
    lm = NeuralNet.loadModelFile(tmp_models["tiny_reg"])
    ctx = NeuralNet.createComputeContext([0], 19, 19, True, lm)
    h = NeuralNet.createComputeHandle(ctx, lm, GAMES, False, True, 0)
    sp = SelfPlay(h, GAMES, VISITS, komi=7.5, multi_stone_suicide_legal=True, early_temperature_moves=0, seed=1, debug_fake_nn=True,
                  debug_hold_at_max_visits=True, nn_cache_size_power_of_two=20, ladder_nodes_per_wave=256,
                  **_kwargs(json.loads(str(d["params"]))))
    _place(sp, d, {s: d[f"c{i}_moves"] for i, s in enumerate(FIXTURE_SLOTS)})
    slots = np.array(FIXTURE_SLOTS)
    for _ in range(100):           # graph search can finish several playouts in a wave, a ladder can stall one: run until the budget is spent
        sp.run(200)
        if (sp.root_visits()[slots] >= VISITS).all():
            break
    st = sp.stats()
    print({k: st[k] for k in ("total_visits", "nn_cache_hits", "nn_cache_stores", "instant_playouts", "stalled_waves", "nodes_allocated")})
    assert st["nn_cache_hits"] > 0
    for i, g in enumerate(FIXTURE_SLOTS):
        v, pol, util = sp.root_children(g)
        assert sp.game(g)[1]["root_visits"] == VISITS, g
        ref_pol = d[f"c{i}_policy"]
        assert np.array_equal(pol < 0, ref_pol < 0), f"slot {g}: legality mask differs"
        assert np.abs(pol - ref_pol)[ref_pol >= 0].max() < 2e-6, g
        ref_v = d[f"c{i}_visits"]
        assert np.array_equal(v, ref_v), (g, np.nonzero(v != ref_v), v[v != ref_v], ref_v[v != ref_v])
        assert np.abs(util - d[f"c{i}_util"])[v > 0].max() < 1e-12, g
        ch, rt = sp.root_value_stats(g)
        assert np.abs(ch - d[f"c{i}_child_stats"])[v > 0].max() < 1e-9 and np.abs(rt - d[f"c{i}_root_stats"]).max() < 1e-9, g
        psv, ref_psv = sp.play_selection_values(g), d[f"c{i}_play_selection"]
        assert np.array_equal(psv < 0, ref_psv < 0), g
        assert np.abs(psv - ref_psv).max() <= 1e-9 * max(1.0, np.abs(ref_psv).max()), g
    rv = sp.root_visits()
    assert (rv >= 1).all() and (rv <= VISITS).all(), (rv.min(), rv.max())
    assert st["total_visits"] == int(rv.sum()) and st["total_moves"] == 0, (st["total_visits"], int(rv.sum()), st["total_moves"])
    for g in range(GAMES):
        v, pol, util = sp.root_children(g)
        ch, rt = sp.root_value_stats(g)
        assert v.sum() == rv[g] - 1, (g, v.sum(), rv[g])
        assert np.isfinite(pol).all() and np.isfinite(util).all() and np.isfinite(ch).all() and np.isfinite(rt).all(), g
    sp.free(); h.free(); ctx.free()


# ---- the real b28 net in the loop: a game does not depend on the others ---------------------------------------------------------

LOOP_SLOTS = (0, 1, 300, 511, 512, 1023)
LOOP_PREFIXES = (0, 19, 57, 88, 121, 149)   # moves of the multisuicide fill game
LOOP_WAVES = 48


def _loop_record(handle, num_games, placed, fx, symmetry=0):
    """Runs LOOP_WAVES waves of a fresh loop with the search block bench.py runs, returns what the slots of `placed` hold."""
    # bench.py's search block; the evaluation cache is off (a hit from another game changes how many playouts a wave finishes), and
    # every game's search generator is seeded with the same string, so root noise and root symmetries do not depend on the slot index
    sp = SelfPlay(handle, num_games, VISITS, komi=7.5, multi_stone_suicide_legal=True, early_temperature_moves=30,
                  cpuct_exploration=1.05, cpuct_exploration_log=0.28, cpuct_exploration_base=500.0, fpu_reduction_max=0.2,
                  root_fpu_reduction_max=0.0, value_weight_exponent=0.5, fpu_parent_weight_by_visited_policy=True,
                  fpu_parent_weight_by_visited_policy_pow=2.0, root_desired_per_child_visits_coeff=2.0,
                  subtree_value_bias_factor=0.30, subtree_value_bias_weight_exponent=0.8, use_graph_search=True, graph_search_rep_bound=11,
                  root_noise_enabled=True, root_dirichlet_noise_total_concentration=10.83, root_dirichlet_noise_weight=0.25,
                  root_policy_temperature=1.1, root_policy_temperature_early=1.5, chosen_move_temperature_halflife=19.0,
                  nn_cache_size_power_of_two=0, root_num_symmetries_to_sample=4, root_ending_bonus_points=0.5, root_prune_useless_moves=True,
                  ko_rule=0, use_play_selection=True, use_lcb_for_selection=True, use_non_buggy_lcb=True, lcb_stdevs=5.0,
                  min_visit_prop_for_lcb=0.15, chosen_move_temperature=0.15, chosen_move_temperature_early=0.75, chosen_move_subtract=0.0,
                  chosen_move_prune=1.0, seed=1234, ladder_nodes_per_wave=256, static_score_utility_factor=0.05,
                  dynamic_score_utility_factor=0.30, dynamic_score_center_zero_weight=0.25, dynamic_score_center_scale=0.50,
                  draw_equivalent_wins_for_white=0.5, debug_hold_at_max_visits=True, debug_fixed_symmetry=symmetry)
    _place(sp, fx, placed)
    sp.set_search_rand("config3$searchThread")
    sp.run(LOOP_WAVES)
    out = {}
    for g in placed:
        v, pol, util = sp.root_children(g)
        ch, rt = sp.root_value_stats(g)
        row, gl = sp.nn_row(g)
        path, valid = sp.leaf_path(g)
        out[g] = dict(visits=v, policy=pol, util=util, child_stats=ch, root_stats=rt, row=row, glob=gl, path=np.array(
            [(-1, -1) if m is None else m for m in path], np.int32).reshape(-1, 2), path_valid=np.array(valid))
    sp.free()
    return out


def test_b28_game_does_not_depend_on_the_other_games(fixture_1600, b28_model):
    """The evaluator's rows do not depend on the rest of the batch, bit for bit, so neither does a game's search.  Six games on
    b28c512nbt in fp16 mode (bench.py's mode), in slots spread over a 1024-game loop at 1600 visits, after 48 waves: root children
    (visits, policy, utilities), value moments, the last wave's feature row and leaf path must equal those of a 6-game loop on a
    handle of the same net with batch size 8."""
    fill = fixture_1600["fill_multisuicide"]
    lists = [fill[:k] for k in LOOP_PREFIXES]
    lm = NeuralNet.loadModelFile(b28_model)
    ctx = NeuralNet.createComputeContext([0], 19, 19, True, lm)
    h = NeuralNet.createComputeHandle(ctx, lm, GAMES, False, True, 0)
    big = _loop_record(h, GAMES, dict(zip(LOOP_SLOTS, lists)), fixture_1600)
    h.free()
    h = NeuralNet.createComputeHandle(ctx, lm, 8, False, True, 0)
    small = _loop_record(h, len(lists), dict(enumerate(lists)), fixture_1600)
    h.free(); ctx.free()
    for i, g in enumerate(LOOP_SLOTS):
        a, b = big[g], small[i]
        assert a["visits"].sum() > 0, g
        for k in a:
            assert np.array_equal(a[k], b[k]), (g, k)
