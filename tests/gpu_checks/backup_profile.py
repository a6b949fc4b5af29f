"""Where does the backup kernel spend its cycles?  Profiling build (EXTRA_NVCC_FLAGS=-DKGB_PROFILE_DESCENT), bench configuration or, with
`trained`, the trained g170-b6c96 net.  Per game and wave: the warp's total, post-processing before the path update, path length, and inside
recomputeNodeStats: child gathers, first sums + value weighting, utility / moment sums, bias table + writes."""
import os, sys, tempfile
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from katago_b200 import NeuralNet, SelfPlay, modelgen
trained = len(sys.argv) > 1 and sys.argv[1] == "trained"
p = os.path.join(ROOT, "tests", "golden", "models", "g170-b6c96-s175395328-d26788732.bin.gz") if trained else modelgen.write_model(os.path.join(tempfile.mkdtemp(), "b18.bin"), "b18c384nbt", seed=0)
lm = NeuralNet.loadModelFile(p)
ctx = NeuralNet.createComputeContext([0], 19, 19, True, lm)
h = NeuralNet.createComputeHandle(ctx, lm, 256, False, True, 0)
sp = SelfPlay(h, 256, 600, komi=7.5, seed=1234, cpuct_exploration=1.05, cpuct_exploration_log=0.28, fpu_reduction_max=0.2, root_fpu_reduction_max=0.0,
              value_weight_exponent=0.5, fpu_parent_weight_by_visited_policy=True, fpu_parent_weight_by_visited_policy_pow=2.0,
              root_desired_per_child_visits_coeff=2.0, subtree_value_bias_factor=0.3, subtree_value_bias_weight_exponent=0.8, use_graph_search=True,
              root_noise_enabled=True, root_policy_temperature=1.1, root_policy_temperature_early=1.5, nn_cache_size_power_of_two=20,
              use_play_selection=True, use_lcb_for_selection=True, use_non_buggy_lcb=True, lcb_stdevs=5.0, min_visit_prop_for_lcb=0.15,
              chosen_move_temperature=0.15, chosen_move_temperature_early=0.75, static_score_utility_factor=0.05, dynamic_score_utility_factor=0.3,
              dynamic_score_center_zero_weight=0.25, dynamic_score_center_scale=0.5, ladder_nodes_per_wave=256, root_num_symmetries_to_sample=4,
              root_ending_bonus_points=0.5, root_prune_useless_moves=True, max_playouts_per_wave=4 if trained else 0)
sp.random_openings(150)
sp.run(700); h.sync()
sp.debug_cycles(True)
acc = []
for w in range(24):
    sp.run(1); h.sync()
    c = sp.debug_cycles(True).astype(np.float64)
    ok = c[:, 1] > 0
    acc.append(c[ok])
    worst = int(c[:, 0].argmax())
    print(f"wave {w:2d}: slowest warp {c[worst,0]:8.0f} cyc: before the path {c[worst,2]:7.0f}, path length {c[worst,3]:3.0f}, nodes recomputed {c[worst,1]:3.0f}: gathers {c[worst,4]:7.0f} "
          f"sums+weighting {c[worst,5]:7.0f} utility/moment sums {c[worst,6]:7.0f} bias+writes {c[worst,7]:7.0f}")
a = np.concatenate(acc)
n = a[:, 1].sum()
print("game-waves:", len(a), " nodes recomputed per backup %.2f" % a[:, 1].mean(), " warp total mean %.0f cyc, before the path mean %.0f" % (a[:, 0].mean(), a[:, 2].mean()))
for name, col in (("child gathers", 4), ("first sums + value weighting", 5), ("utility / moment sums", 6), ("bias table + writes", 7)):
    print(f"  {name:30s} per node {a[:, col].sum() / n:8.0f} cyc   mean per backup {a[:, col].mean():8.0f}")
print("tree kernels (ms select, ms backup):", sp.time_tree_kernels(30))
