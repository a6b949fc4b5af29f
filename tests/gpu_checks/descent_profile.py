"""Where does a descent step of the select kernel spend its cycles?  Needs the profiling build of the library:
    EXTRA_NVCC_FLAGS=-DKGB_PROFILE_DESCENT KGB_FORCE_BUILD=1 bash katago_b200/csrc/build.sh
Bench configuration (b18c384nbt random weights, 256 games, 600 visits).  Per game and wave: steps of the descent, cycles in the child
gathers + ordered sums, in the selection arithmetic / argmax, in the move (history + bitboard play), in the new-edge work."""
import os, sys, tempfile
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from katago_b200 import NeuralNet, SelfPlay, modelgen
waves = int(sys.argv[1]) if len(sys.argv) > 1 else 24
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
              dynamic_score_center_zero_weight=0.25, dynamic_score_center_scale=0.5, ladder_nodes_per_wave=256, root_num_symmetries_to_sample=4,
              root_ending_bonus_points=0.5, root_prune_useless_moves=True)
sp.random_openings(150)
sp.run(700); h.sync()
sp.debug_cycles(True)
acc = []
for w in range(waves):
    sp.run(1); h.sync()
    c = sp.debug_cycles(True)
    steps = (c[:, 1] & 0x3ff).astype(np.float64); attempts = ((c[:, 1] >> 10) & 0x3f).astype(np.float64); edge = (c[:, 1] >> 16).astype(np.float64)
    backup = (c[:, 4] >> 32).astype(np.float64); advance = (c[:, 4] & 0xffffffff).astype(np.float64)
    ok = attempts > 0
    acc.append(np.stack([steps, attempts, c[:, 5], c[:, 6], c[:, 7], edge, backup, advance, c[:, 0], c[:, 2], c[:, 3]], 1)[ok])
    worst = int(c[:, 0].argmax())
    print(f"wave {w:2d}: slowest block {c[worst,0]:8d} cyc (warp0 {c[worst,2]:8d}, ladders {c[worst,3]:8d}): playouts {int(attempts[worst])} steps {int(steps[worst]):3d}: gather {c[worst,5]:7d} "
          f"select {c[worst,6]:7d} move {c[worst,7]:7d} edge {int(edge[worst]):7d} in-kernel backup {int(backup[worst]):8d} root advance {int(advance[worst]):8d}")
a_ = np.concatenate(acc)
st = a_[:, 0]
print("games x waves:", len(a_), " mean steps %.2f, mean playouts started per wave %.3f" % (st.mean(), a_[:, 1].mean()))
for name, col in (("gather+sums", 2), ("selection", 3), ("move (hist+board)", 4), ("edge / loop head", 5), ("in-kernel backup", 6), ("root advance", 7)):
    print(f"  {name:18s} mean {a_[:, col].mean():9.0f} cyc   per step {a_[:, col].sum() / st.sum():8.0f}   p99 {np.percentile(a_[:, col], 99):9.0f}   max {a_[:, col].max():9.0f}")
print("  block total mean %.0f, warp0 mean %.0f, ladders mean %.0f; slowest block per wave mean %.0f" % (a_[:, 8].mean(), a_[:, 9].mean(), a_[:, 10].mean(), np.mean([x[:, 8].max() for x in acc])))
print("tree kernels (ms select, ms backup):", sp.time_tree_kernels(30))
