"""What the SGF-metadata encoder costs a forward pass, and that nets without one compute and launch as before.

    python tests/gpu_checks/meta_cost.py [--parent TREE] [--out DIR]

1. Forward time (kgb_forward_device, CUDA events around 50 forwards after 10 warm-up ones) of a random b18c384nbt and of the same net
   with an encoder (b18c384nbt-meta: 192 -> 384 -> 384 -> 384) at batch 256, fp16 and fp32-equivalent mode, five alternating rounds,
   median reported.  The encoder is three small fp32 matmuls (~0.1 GFLOP against ~18.9 GFLOP of convolutions per forward).
2. With --parent TREE (a built checkout of the parent commit): bench.py --steps 20 --warmup 3 --dump-outputs on this tree and on the
   parent, fp16 and --fp32; the dumps must be bit-identical and gpu_launches equal.
The card name and power limit are printed first."""
import argparse, json, os, subprocess, sys, tempfile
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def forward_times():
    sys.path.insert(0, ROOT)
    import torch
    from katago_b200 import NeuralNet, modelgen
    from katago_b200.nn_backend import load_library
    lib = load_library()
    d = tempfile.mkdtemp()
    paths = {"b18c384nbt": modelgen.write_model(os.path.join(d, "b18.bin"), "b18c384nbt", seed=0),
             "b18c384nbt-meta": modelgen.write_model(os.path.join(d, "b18m.bin"), "b18c384nbt", seed=0, meta_channels=384)}
    n = 256
    sp, gl = modelgen.synthetic_inputs(n, 19, 19, seed=1)
    rows = np.load(os.path.join(ROOT, "tests", "golden", "metarows.npz"))["rows"]
    meta = rows[np.random.default_rng(2).choice(len(rows), n)]
    dev = torch.device("cuda:0")
    t = {k: torch.from_numpy(np.ascontiguousarray(v, np.float32)).to(dev) for k, v in (("sp", sp.reshape(n, -1)), ("gl", gl), ("meta", meta))}
    outs = [torch.empty((n, s), device=dev) for s in (362, 3, 6, 361)]
    out = {}
    for fp16 in (True, False):
        nets = {}
        for name, p in paths.items():
            lm = NeuralNet.loadModelFile(p)
            ctx = NeuralNet.createComputeContext([0], 19, 19, fp16, lm)
            h = NeuralNet.createComputeHandle(ctx, lm, n, False, True, 0)
            nets[name] = (lm, ctx, h)

        def fwd(name):
            h = nets[name][2]
            args = [o.data_ptr() for o in outs]
            if name.endswith("-meta"):
                rc = lib.kgb_forward_device_meta(h._p, n, t["sp"].data_ptr(), t["gl"].data_ptr(), t["meta"].data_ptr(), None, None, *args)
            else:
                rc = lib.kgb_forward_device(h._p, n, t["sp"].data_ptr(), t["gl"].data_ptr(), None, None, *args)
            assert rc == 0, lib.kgb_last_error()

        times = {k: [] for k in nets}
        for _ in range(5):
            for name in nets:
                h = nets[name][2]
                s = torch.cuda.ExternalStream(h.stream)
                for _ in range(10):
                    fwd(name)
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record(s)
                for _ in range(50):
                    fwd(name)
                b.record(s)
                b.synchronize()
                times[name].append(a.elapsed_time(b) / 50)
        mode = "fp16" if fp16 else "fp32"
        for name, v in times.items():
            out[f"{name}_{mode}_ms"] = float(np.median(v))
            out[f"{name}_{mode}_runs"] = v
            out[f"{name}_launches"] = nets[name][2].launches_per_forward
        base, meta_ms = out[f"b18c384nbt_{mode}_ms"], out[f"b18c384nbt-meta_{mode}_ms"]
        print(f"{mode}: b18c384nbt {base:.3f} ms  b18c384nbt-meta {meta_ms:.3f} ms  (+{meta_ms - base:.3f} ms, {100 * (meta_ms / base - 1):+.2f}%)  "
              f"runs {[round(x, 3) for x in times['b18c384nbt']]} / {[round(x, 3) for x in times['b18c384nbt-meta']]}", flush=True)
        for lm, ctx, h in nets.values():
            h.free(); ctx.free(); lm.free()
    return out


def bench_compare(parent, outdir):
    res = {}
    for fp32 in (False, True):
        dumps = {}
        for label, tree in (("branch", ROOT), ("parent", parent)):
            dump = dumps[label] = os.path.join(outdir, f"dump_{label}_{'fp32' if fp32 else 'fp16'}")
            cmd = [sys.executable, "bench.py", "--gpus", "1", "--steps", "20", "--warmup", "3", "--dump-outputs", dump] + (["--fp32"] if fp32 else [])
            r = subprocess.run(cmd, cwd=tree, capture_output=True, text=True, timeout=1800)
            line = json.loads([ln for ln in r.stdout.splitlines() if ln.startswith("{")][-1])
            res[f"{label}_{'fp32' if fp32 else 'fp16'}"] = {k: line.get(k) for k in ("value", "gpu_launches")}
            print(label, "fp32" if fp32 else "fp16", res[f"{label}_{'fp32' if fp32 else 'fp16'}"], flush=True)
        names = sorted(os.listdir(dumps["branch"]))
        assert names == sorted(os.listdir(dumps["parent"]))
        for nm in names:
            x, y = np.load(os.path.join(dumps["branch"], nm)), np.load(os.path.join(dumps["parent"], nm))
            assert x.dtype == y.dtype and x.shape == y.shape and x.tobytes() == y.tobytes(), (nm, fp32)
        mode = "fp32" if fp32 else "fp16"
        assert res[f"branch_{mode}"]["gpu_launches"] == res[f"parent_{mode}"]["gpu_launches"]
        print(mode, "dumps bit-identical to the parent, gpu_launches equal", flush=True)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--parent", default="")
    ap.add_argument("--out", default="", help="directory for the bench dumps and meta_cost.json (default: a new temporary one)")
    a = ap.parse_args()
    a.out = a.out or tempfile.mkdtemp(prefix="meta_cost_")
    os.makedirs(a.out, exist_ok=True)
    print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv"], capture_output=True, text=True).stdout, flush=True)
    result = {"forward": forward_times()}
    if a.parent:
        result["bench"] = bench_compare(a.parent, a.out)
    with open(os.path.join(a.out, "meta_cost.json"), "w") as f:
        json.dump(result, f, indent=1)
    print("results in", a.out)


if __name__ == "__main__":
    main()
