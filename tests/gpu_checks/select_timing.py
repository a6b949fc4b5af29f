"""Which games make the select kernel slow?  Per-wave, per-game clock64 spans (kgb_selfplay_debug_cycles) in the bench configuration.
    python tests/gpu_checks/select_timing.py [waves]"""
import os, sys, tempfile
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from katago_b200 import NeuralNet, SelfPlay, modelgen
waves = int(sys.argv[1]) if len(sys.argv) > 1 else 40
cap = int(sys.argv[2]) if len(sys.argv) > 2 else 256
p = modelgen.write_model(os.path.join(tempfile.mkdtemp(), "b18.bin"), "b18c384nbt", seed=0)
lm = NeuralNet.loadModelFile(p)
ctx = NeuralNet.createComputeContext([0], 19, 19, True, lm)
h = NeuralNet.createComputeHandle(ctx, lm, 256, False, True, 0)
sp = SelfPlay(h, 256, 600, komi=7.5, seed=1234, cpuct_exploration=1.05, cpuct_exploration_log=0.28, fpu_reduction_max=0.2, root_fpu_reduction_max=0.0,
              value_weight_exponent=0.5, fpu_parent_weight_by_visited_policy=True, fpu_parent_weight_by_visited_policy_pow=2.0,
              root_desired_per_child_visits_coeff=2.0, subtree_value_bias_factor=0.3, subtree_value_bias_weight_exponent=0.8, use_graph_search=True,
              root_noise_enabled=True, root_policy_temperature=1.1, root_policy_temperature_early=1.5, nn_cache_size_power_of_two=20,
              use_play_selection=True, use_lcb_for_selection=True, use_non_buggy_lcb=True, lcb_stdevs=5.0, min_visit_prop_for_lcb=0.15,
              chosen_move_temperature=0.15, chosen_move_temperature_early=0.75, static_score_utility_factor=0.05, dynamic_score_utility_factor=0.3,
              dynamic_score_center_zero_weight=0.25, dynamic_score_center_scale=0.5, ladder_nodes_per_wave=cap, root_num_symmetries_to_sample=4)
sp.random_openings(150)
sp.run(700); h.sync()
sp.debug_cycles(True)
rows = []
for w in range(waves):
    sp.run(1); h.sync()
    c = sp.debug_cycles(True).astype(np.float64)
    tot = c[:, 0]
    worst = int(tot.argmax())
    rows.append((tot.max(), tot.mean(), np.median(tot), c[worst, 1], c[worst, 2], c[worst, 3], int((c[:, 1] > 0).sum())))
    print(f"wave {w:3d}: slowest block {tot.max():9.0f} cyc (mean {tot.mean():8.0f}, median {np.median(tot):8.0f}, p90 {np.percentile(tot, 90):8.0f}); slowest: root-advance {c[worst,1]:8.0f} "
          f"warp0 {c[worst,2]:8.0f} ladders {c[worst,3]:8.0f}; games that advanced their root this wave: {int((c[:,1] > 0).sum())}")
    if w < 6:
        print("          slowest block: descent %.0f libs+legal %.0f area %.0f rows %.0f | all games mean: descent %.0f libs+legal %.0f area %.0f rows %.0f ladders %.0f" %
              (c[worst, 4], c[worst, 5], c[worst, 6], c[worst, 7], c[:, 4].mean(), c[:, 5].mean(), c[:, 6].mean(), c[:, 7].mean(), c[:, 3].mean()))
r = np.array(rows)
print("mean over waves: slowest %.0f  mean block %.0f  median block %.0f; waves whose slowest block advanced its root: %d of %d" %
      (r[:, 0].mean(), r[:, 1].mean(), r[:, 2].mean(), int((r[:, 3] > 0).sum()), len(r)))
print("ladder cap", cap, "tree kernels (ms select, ms backup):", sp.time_tree_kernels(30), "stats", sp.stats())
