"""What recording costs: visits/s of the device loop left alone vs. driven by GameRecorder in lockstep (`step`) and with per-game
release (`pump`), same search block, wall clock around whole moves (the recorder's host reads are part of what is measured).

    python tests/gpu_checks/record_overhead.py [config] [games] [visits] [moves]        e.g. b18c384nbt 256 600 3

Prepared in round 1, not yet run on a GPU (DESIGN.md §8 item 4)."""
import json, os, sys, tempfile, time
ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from katago_b200 import NeuralNet, SelfPlay, modelgen
from katago_b200.game_recorder import GameRecorder

cfg = sys.argv[1] if len(sys.argv) > 1 else "b18c384nbt"
games = int(sys.argv[2]) if len(sys.argv) > 2 else 256
visits = int(sys.argv[3]) if len(sys.argv) > 3 else 600
moves = int(sys.argv[4]) if len(sys.argv) > 4 else 3
SEARCH = dict(komi=7.5, cpuct_exploration=1.05, cpuct_exploration_log=0.28, root_fpu_reduction_max=0.0, value_weight_exponent=0.5,
              fpu_parent_weight_by_visited_policy=True, fpu_parent_weight_by_visited_policy_pow=2.0, root_desired_per_child_visits_coeff=2.0,
              subtree_value_bias_factor=0.30, subtree_value_bias_weight_exponent=0.8, use_graph_search=True, root_noise_enabled=True,
              root_dirichlet_noise_total_concentration=10.83, root_dirichlet_noise_weight=0.25, root_policy_temperature=1.1, root_policy_temperature_early=1.5,
              root_num_symmetries_to_sample=4, nn_cache_size_power_of_two=20, use_play_selection=True, use_lcb_for_selection=True,
              use_non_buggy_lcb=True, lcb_stdevs=5.0, min_visit_prop_for_lcb=0.15, chosen_move_temperature=0.15, chosen_move_temperature_early=0.75,
              static_score_utility_factor=0.05, dynamic_score_utility_factor=0.30, dynamic_score_center_zero_weight=0.25, dynamic_score_center_scale=0.50)
path = modelgen.write_model(os.path.join(tempfile.mkdtemp(), cfg + ".bin"), cfg, seed=0)
lm = NeuralNet.loadModelFile(path)
ctx = NeuralNet.createComputeContext([0], 19, 19, True, lm)
h = NeuralNet.createComputeHandle(ctx, lm, games, False, True, 0)
out = {"config": cfg, "games": games, "max_visits": visits, "moves_per_game": moves}


def measure(name, hold, drive):
    sp = SelfPlay(h, games, visits, seed=7, debug_hold_at_max_visits=hold, **SEARCH)
    sp.random_openings(60)
    sp.run(20); h.sync()
    v0, m0, t0 = sp.stats()["total_visits"], sp.stats()["total_moves"], time.time()
    drive(sp)
    h.sync()
    dt = time.time() - t0
    st = sp.stats()
    out[name] = {"visits_per_sec": (st["total_visits"] - v0) / dt, "moves": st["total_moves"] - m0, "seconds": dt}
    sp.free()


def free_running(sp):
    while sp.stats()["total_moves"] < games * moves:
        sp.run(64)


def lockstep(sp):
    rec = GameRecorder(sp, None, 7.5)
    for _ in range(moves):
        rec.step()


def per_game(sp):
    rec = GameRecorder(sp, None, 7.5)
    while rec.moves_recorded < games * moves:
        rec.pump(8)


measure("free_running", False, free_running)
measure("recorder_lockstep", True, lockstep)
measure("recorder_per_game_release", True, per_game)
print(json.dumps(out, indent=1))
