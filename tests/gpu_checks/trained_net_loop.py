"""Tree statistics of the device loop on a TRAINED net (VERDICT r01 "what's weak" 6): a trained policy gives deeper, narrower trees and
more evaluation-cache hits than the random-weight net of the bench, and the select / backup cost follows the depth.
    python tests/gpu_checks/trained_net_loop.py [games] [waves]
Net: g170-b6c96-s175395328-d26788732 (from the reference's test suite, committed under tests/golden/models), 19x19, the search block of
selfplay8mainb18.cfg, 600 visits.  Prints one JSON line."""
import json, os, sys
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from katago_b200 import NeuralNet, SelfPlay
games = int(sys.argv[1]) if len(sys.argv) > 1 else 256
waves = int(sys.argv[2]) if len(sys.argv) > 2 else 1200
mppw = int(sys.argv[3]) if len(sys.argv) > 3 else 0          # max_playouts_per_wave (0 = 16)
model = os.path.join(ROOT, "tests", "golden", "models", "g170-b6c96-s175395328-d26788732.bin.gz")
lm = NeuralNet.loadModelFile(model)
ctx = NeuralNet.createComputeContext([0], 19, 19, True, lm)
h = NeuralNet.createComputeHandle(ctx, lm, games, False, True, 0)
sp = SelfPlay(h, games, 600, komi=7.5, seed=1234, cpuct_exploration=1.05, cpuct_exploration_log=0.28, fpu_reduction_max=0.2, root_fpu_reduction_max=0.0,
              value_weight_exponent=0.5, fpu_parent_weight_by_visited_policy=True, fpu_parent_weight_by_visited_policy_pow=2.0,
              root_desired_per_child_visits_coeff=2.0, subtree_value_bias_factor=0.3, subtree_value_bias_weight_exponent=0.8, use_graph_search=True,
              root_noise_enabled=True, root_policy_temperature=1.1, root_policy_temperature_early=1.5, nn_cache_size_power_of_two=20,
              use_play_selection=True, use_lcb_for_selection=True, use_non_buggy_lcb=True, lcb_stdevs=5.0, min_visit_prop_for_lcb=0.15,
              chosen_move_temperature=0.15, chosen_move_temperature_early=0.75, static_score_utility_factor=0.05, dynamic_score_utility_factor=0.3,
              dynamic_score_center_zero_weight=0.25, dynamic_score_center_scale=0.5, ladder_nodes_per_wave=256, root_num_symmetries_to_sample=4,
              root_ending_bonus_points=0.5, root_prune_useless_moves=True, max_playouts_per_wave=mppw)
sp.random_openings(150)
sp.run(700); h.sync()
import torch
s0 = sp.stats()
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
stream = torch.cuda.ExternalStream(h.stream)
with torch.cuda.stream(stream):
    e0.record(stream)
    sp.run(waves)
    e1.record(stream)
h.sync()
ms = e0.elapsed_time(e1)
s1 = sp.stats()
dv = s1["total_visits"] - s0["total_visits"]
kids = [int((sp.root_children(g)[0] > 0).sum()) for g in range(0, games, 8)]
sel, bak = sp.time_tree_kernels(30)
print(json.dumps({"check": "trained_net_loop", "net": "g170-b6c96 (trained)", "board": "19x19", "games": games, "waves": waves, "ms_per_wave": ms / waves,
                  "visits_per_s": dv / (ms * 1e-3), "avg_leaf_depth": (s1["sum_leaf_depth"] - s0["sum_leaf_depth"]) / max(1, dv),
                  "cache_hit_fraction": (s1["nn_cache_hits"] - s0["nn_cache_hits"]) / max(1, dv),
                  "instant_playout_fraction": (s1["instant_playouts"] - s0["instant_playouts"]) / max(1, dv),
                  "stalled_game_waves_fraction": (s1["stalled_waves"] - s0["stalled_waves"]) / (waves * games),
                  "moves_played": s1["total_moves"] - s0["total_moves"], "games_finished": s1["games_finished"] - s0["games_finished"],
                  "max_playouts_per_wave": mppw, "root_children_mean": float(np.mean(kids)), "ms_select": sel, "ms_backup": bak}))
