"""What uncertainty weighting and noise pruning cost the search's tree kernels, and that the default path is unchanged.

    python tests/gpu_checks/uncertainty_cost.py [--parent TREE] [--out DIR]

1. spSelectKernel / spBackupKernel times (kgb_selfplay_time_tree_kernels, CUDA events, 20 launches each, evaluator skipped) at 256
   games on a random b18c384nbt net (version 15), with the bench search block: switches off, uncertainty on, both on; three
   alternating rounds, median reported.  Noise pruning runs as one warp-uniform pass over the children (values broadcast by shuffle).
2. With --parent TREE (a built checkout of the parent commit): bench.py --steps 20 --warmup 3 --dump-outputs on this tree and on the
   parent, alternating, fp16 and --fp32, three runs each; the dumps must be bit-identical and `value` is listed for both.
The card name and power limit are printed first."""
import argparse, json, os, subprocess, sys, tempfile
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def tree_kernel_times():
    sys.path.insert(0, ROOT)
    from katago_b200 import NeuralNet, SelfPlay, modelgen
    p = modelgen.write_model(os.path.join(tempfile.mkdtemp(), "b18.bin"), "b18c384nbt", seed=0)
    lm = NeuralNet.loadModelFile(p)
    ctx = NeuralNet.createComputeContext([0], 19, 19, True, lm)
    h = NeuralNet.createComputeHandle(ctx, lm, 256, False, True, 0)
    base = dict(komi=7.5, seed=1234, cpuct_exploration=1.05, cpuct_exploration_log=0.28, fpu_reduction_max=0.2, root_fpu_reduction_max=0.0,
                value_weight_exponent=0.5, fpu_parent_weight_by_visited_policy=True, fpu_parent_weight_by_visited_policy_pow=2.0,
                root_desired_per_child_visits_coeff=2.0, subtree_value_bias_factor=0.3, subtree_value_bias_weight_exponent=0.8, use_graph_search=True,
                root_noise_enabled=True, nn_cache_size_power_of_two=20, use_play_selection=True, static_score_utility_factor=0.05,
                dynamic_score_utility_factor=0.3, dynamic_score_center_zero_weight=0.25, dynamic_score_center_scale=0.5, ladder_nodes_per_wave=256)
    variants = {"off": {}, "uncertainty": dict(use_uncertainty=True), "both": dict(use_uncertainty=True, use_noise_pruning=True)}
    loops = {}
    for name, extra in variants.items():
        sp = SelfPlay(h, 256, 600, **base, **extra)
        sp.random_openings(150)
        sp.run(300); h.sync()        # trees of a few hundred nodes, as in steady self-play
        loops[name] = sp
    res = {k: [] for k in variants}
    for _ in range(3):
        for name, sp in loops.items():
            res[name].append(sp.time_tree_kernels(20))
    out = {}
    for name, r in res.items():
        r = np.array(r)
        out[name] = dict(select_ms=float(np.median(r[:, 0])), backup_ms=float(np.median(r[:, 1])), backup_all=r[:, 1].tolist())
        print(f"{name:12s} select {out[name]['select_ms']:.4f} ms  backup {out[name]['backup_ms']:.4f} ms  (backup runs: {', '.join(f'{x:.4f}' for x in r[:, 1])})")
    for sp in loops.values():
        sp.free()
    h.free(); ctx.free()
    return out


def bench_compare(parent, outdir):
    res = {}
    for fp32 in (False, True):
        for rnd in range(3):
            for label, tree in (("branch", ROOT), ("parent", parent)):
                dump = os.path.join(outdir, f"dump_{label}_{'fp32' if fp32 else 'fp16'}_{rnd}")
                cmd = [sys.executable, "bench.py", "--gpus", "1", "--steps", "20", "--warmup", "3", "--dump-outputs", dump] + (["--fp32"] if fp32 else [])
                r = subprocess.run(cmd, cwd=tree, capture_output=True, text=True, timeout=1800)
                line = [ln for ln in r.stdout.splitlines() if ln.startswith("{")][-1]
                res.setdefault((label, fp32), []).append(json.loads(line)["value"])
                print(label, "fp32" if fp32 else "fp16", rnd, json.loads(line)["value"], flush=True)
        for rnd in range(3):
            a, b = (os.path.join(outdir, f"dump_{lab}_{'fp32' if fp32 else 'fp16'}_{rnd}") for lab in ("branch", "parent"))
            names = sorted(os.listdir(a))
            assert names == sorted(os.listdir(b)), (names, os.listdir(b))
            for n in names:
                x, y = np.load(os.path.join(a, n)), np.load(os.path.join(b, n))
                assert x.dtype == y.dtype and x.shape == y.shape and x.tobytes() == y.tobytes(), (n, fp32, rnd)
        print("fp32" if fp32 else "fp16", "dumps bit-identical to the parent in all rounds")
    for k, v in res.items():
        print(k, "values", v)
    return {f"{k[0]}_{'fp32' if k[1] else 'fp16'}": v for k, v in res.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--parent", default="")
    ap.add_argument("--out", default="", help="directory for the bench dumps and uncertainty_cost.json (default: a new temporary one)")
    a = ap.parse_args()
    a.out = a.out or tempfile.mkdtemp(prefix="uncertainty_cost_")
    os.makedirs(a.out, exist_ok=True)
    print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv"], capture_output=True, text=True).stdout, flush=True)
    result = {"tree_kernels": tree_kernel_times()}
    if a.parent:
        result["bench"] = bench_compare(a.parent, a.out)
    with open(os.path.join(a.out, "uncertainty_cost.json"), "w") as f:
        json.dump(result, f, indent=1)
    print("results in", a.out)


if __name__ == "__main__":
    main()
