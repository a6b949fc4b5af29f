"""Ragged rows against the reference plan (KGB_RAGGED_ROWS=0), same build, one GPU, alternating, `runs` runs each:
  - forward time of b18c384nbt at batch 256 (device buffers, CUDA events) for three board-size workloads: 19x19 only, BASELINE
    config 4 (9/13/19 with equal probabilities) and the size draw of the stock selfplay8mainb18.cfg (bSizes 7..19, 10% rectangles);
  - the rows each layout uses (layout_stats);
  - the device self-play loop's visits/s on the same net for config 4 and the stock draw.
Prints the card's name and power limit first, then one JSON line per measurement.
    python tests/gpu_checks/ragged_rows.py [runs]"""
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from katago_b200 import NeuralNet, SelfPlay, load_library, modelgen  # noqa: E402

RUNS = int(sys.argv[1]) if len(sys.argv) > 1 else 3
N = 256
STOCK_SIZES = np.array([7, 9, 11, 13, 15, 17, 19, 8, 10, 12, 14, 16, 18])
STOCK_PROBS = np.array([1, 4, 3, 10, 7, 9, 75, 1, 2, 4, 6, 8, 10], float) / 140.0


def draw(workload, n, rng):
    """[n][2] board (x, y) of a workload."""
    if workload == "19x19":
        return np.full((n, 2), 19)
    if workload == "config4":
        s = rng.choice([9, 13, 19], n)
        return np.stack([s, s], 1)
    x = rng.choice(STOCK_SIZES, n, p=STOCK_PROBS)
    y = np.where(rng.uniform(size=n) < 0.10, rng.choice(STOCK_SIZES, n, p=STOCK_PROBS), x)
    return np.stack([x, y], 1)


def emit(rec):
    print(json.dumps(rec), flush=True)


def handle(path, ragged):
    if ragged:
        os.environ.pop("KGB_RAGGED_ROWS", None)
    else:
        os.environ["KGB_RAGGED_ROWS"] = "0"
    lm = NeuralNet.loadModelFile(path)
    ctx = NeuralNet.createComputeContext([0], 19, 19, True, lm)
    h = NeuralNet.createComputeHandle(ctx, lm, N, False, True, 0)
    os.environ.pop("KGB_RAGGED_ROWS", None)
    return lm, ctx, h


def time_forward(h, dev_in, iters=30):
    lib = load_library()
    dsp, dgl, dsym, outs = dev_in

    def run():
        rc = lib.kgb_forward_device(h._p, N, dsp.data_ptr(), dgl.data_ptr(), dsym.data_ptr(), None, *(o.data_ptr() for o in outs))
        assert rc == 0, lib.kgb_last_error()

    for _ in range(3):
        run()
    h.sync()
    stream = torch.cuda.ExternalStream(h.stream)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    for _ in range(iters):
        run()
    e1.record(stream)
    h.sync()
    return e0.elapsed_time(e1) / iters


def main():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    emit({"gpu": q.stdout.strip()})
    path = modelgen.write_model(os.path.join(tempfile.mkdtemp(), "b18c384nbt.bin"), "b18c384nbt", seed=0)
    handles = {r: handle(path, r) for r in (True, False)}
    dev = torch.device("cuda:0")
    rng = np.random.default_rng(7)
    for workload in ("19x19", "config4", "stock"):
        boards = draw(workload, N, rng)
        sp, gl = modelgen.synthetic_inputs(N, 19, 19, seed=3, board_sizes=[tuple(b) for b in boards])
        sym = rng.integers(0, 8, N).astype(np.int32)
        outs = [torch.empty(s, device=dev) for s in ((N, 362), (N, 3), (N, 6), (N, 361))]
        dev_in = (torch.from_numpy(sp.reshape(N, -1)).to(dev), torch.from_numpy(gl).to(dev), torch.from_numpy(sym).to(dev), outs)
        torch.cuda.synchronize()
        for run in range(RUNS):
            for ragged in (True, False):
                h = handles[ragged][2]
                ms = time_forward(h, dev_in)
                emit({"what": "forward", "net": "b18c384nbt", "batch": N, "workload": workload, "ragged": ragged, "run": run,
                      "ms": round(ms, 4), "layout": h.layout_stats(), "frame_rows": N * 400})
    for workload in ("config4", "stock"):
        setups = np.concatenate([draw(workload, N, rng), rng.integers(0, 4, (N, 1)), np.ones((N, 1), int)], 1).astype(np.int32)
        nxt = np.concatenate([draw(workload, N, rng), rng.integers(0, 4, (N, 1)), np.ones((N, 1), int)], 1).astype(np.int32)
        for run in range(RUNS):
            for ragged in (True, False):
                h = handles[ragged][2]
                loop = SelfPlay(h, N, 200, komi=7.5, seed=1 + run, use_graph_search=True, nn_cache_size_power_of_two=16,
                                root_num_symmetries_to_sample=4, root_noise_enabled=True, full_history_rules=True)
                loop.set_game_setup(setups, also_current_games=True)
                loop.set_game_setup(nxt)
                loop.run(20)
                h.sync()
                v0 = loop.stats()["total_visits"]
                t0 = time.perf_counter()
                loop.run(200)
                h.sync()
                dt = time.perf_counter() - t0
                v1 = loop.stats()["total_visits"]
                emit({"what": "loop", "net": "b18c384nbt", "games": N, "workload": workload, "ragged": ragged, "run": run,
                      "visits_per_s": round((v1 - v0) / dt, 1), "layout": h.layout_stats()})
                loop.free()
    for lm, ctx, h in handles.values():
        h.free(); ctx.free(); lm.free()


if __name__ == "__main__":
    main()
