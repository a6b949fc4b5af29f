"""Two game populations on one GPU (VERDICT r01 item 4): loop A's select / backup kernels run while loop B's evaluator owns the tensor
pipes, and vice versa.  Two handles (own stream, own activation buffers, own CUDA graph) x 128 games against one handle x 256 games.
    python tests/gpu_checks/pingpong.py [steps]"""
import json, os, sys, tempfile
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
import torch
from katago_b200 import NeuralNet, SelfPlay, modelgen
steps = int(sys.argv[1]) if len(sys.argv) > 1 else 60
p = modelgen.write_model(os.path.join(tempfile.mkdtemp(), "b18.bin"), "b18c384nbt", seed=0)
lm = NeuralNet.loadModelFile(p)
ctx = NeuralNet.createComputeContext([0], 19, 19, True, lm)
KW = dict(komi=7.5, cpuct_exploration=1.05, cpuct_exploration_log=0.28, fpu_reduction_max=0.2, root_fpu_reduction_max=0.0,
          value_weight_exponent=0.5, fpu_parent_weight_by_visited_policy=True, fpu_parent_weight_by_visited_policy_pow=2.0,
          root_desired_per_child_visits_coeff=2.0, subtree_value_bias_factor=0.3, subtree_value_bias_weight_exponent=0.8, use_graph_search=True,
          root_noise_enabled=True, root_policy_temperature=1.1, root_policy_temperature_early=1.5, nn_cache_size_power_of_two=20,
          use_play_selection=True, use_lcb_for_selection=True, use_non_buggy_lcb=True, lcb_stdevs=5.0, min_visit_prop_for_lcb=0.15,
          chosen_move_temperature=0.15, chosen_move_temperature_early=0.75, static_score_utility_factor=0.05, dynamic_score_utility_factor=0.3,
          dynamic_score_center_zero_weight=0.25, dynamic_score_center_scale=0.5, ladder_nodes_per_wave=256, root_num_symmetries_to_sample=4,
          root_ending_bonus_points=0.5, root_prune_useless_moves=True)


def measure(pops, games_each):
    hs = [NeuralNet.createComputeHandle(ctx, lm, games_each, False, True, 0) for _ in range(pops)]
    sps = [SelfPlay(h, games_each, 600, seed=1234 + 17 * i, **KW) for i, h in enumerate(hs)]
    for sp in sps:
        sp.random_openings(150)
    for _ in range(700):
        for sp in sps:
            sp.run(1)
    for h in hs:
        h.sync()
    streams = [torch.cuda.ExternalStream(h.stream) for h in hs]
    before = [sp.stats() for sp in sps]
    e0 = [torch.cuda.Event(enable_timing=True) for _ in hs]; e1 = [torch.cuda.Event(enable_timing=True) for _ in hs]
    torch.cuda.synchronize()
    for s, e in zip(streams, e0):
        e.record(s)
    for _ in range(steps):
        for sp in sps:
            sp.run(1)
    for s, e in zip(streams, e1):
        e.record(s)
    for h in hs:
        h.sync()
    # all streams start together: the job takes as long as the longest of them
    ms = max(a.elapsed_time(b) for a, b in zip(e0, e1))
    cross = max(e0[0].elapsed_time(b) for b in e1)
    after = [sp.stats() for sp in sps]
    visits = sum(a["total_visits"] - b["total_visits"] for a, b in zip(after, before))
    out = {"populations": pops, "games_each": games_each, "steps": steps, "ms_total": max(ms, cross), "ms_per_round": max(ms, cross) / steps,
           "visits_per_s": visits / (max(ms, cross) * 1e-3)}
    for sp in sps:
        sp.free()
    for h in hs:
        h.free()
    return out


res = [measure(1, 256), measure(2, 128), measure(2, 256), measure(1, 256)]
for r in res:
    print(json.dumps(r))
