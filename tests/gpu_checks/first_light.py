"""Bring-up checks run on the GPU box (not a pytest file): prints max errors of the CUDA path vs the numpy oracle.
Usage: python tests/gpu_checks/first_light.py [stage ...]"""
import os, sys, time, tempfile
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "oracle"))
import kg_nn_oracle as orc
from katago_b200 import NeuralNet, modelgen

def conv_check(ky, cin, cout, n=2, X=19, Y=19, fp16=True, seed=0):
    rng = np.random.default_rng(seed)
    w = (rng.standard_normal((ky, ky, cin, cout)) * np.sqrt(1.0 / (ky * ky * cin))).astype(np.float32)
    x = rng.standard_normal((n, Y, X, cin)).astype(np.float32)
    if fp16:
        w = w.astype(np.float16).astype(np.float32); x = x.astype(np.float16).astype(np.float32)
    ref = orc.conv2d(x, orc.Conv("t", ky, ky, cin, cout, w))
    got = NeuralNet.testEvaluateConv(ky, ky, cin, cout, w, n, X, Y, fp16, x)
    err = np.abs(got - ref).max()
    print(f"conv {ky}x{ky} {cin}->{cout} n={n} {X}x{Y} fp16={fp16}: max|err|={err:.3e} ref_max={np.abs(ref).max():.3f}", flush=True)
    return err

def model_check(path, n, X, Y, fp16, sizes=None, seed=1):
    m = orc.load_model(path)
    sp, gl = modelgen.synthetic_inputs(n, X, Y, seed=seed, board_sizes=sizes)
    sym = np.arange(n) % 8
    opt = np.linspace(0, 1, n).astype(np.float32)
    t = time.time(); ref = orc.get_output(m, sp, gl, sym, opt); tref = time.time() - t
    lm = NeuralNet.loadModelFile(path)
    ctx = NeuralNet.createComputeContext([0], X, Y, fp16, lm)
    h = NeuralNet.createComputeHandle(ctx, lm, max(n, 4), False, True)
    t = time.time(); got = NeuralNet.getOutput(h, sp.reshape(n, -1), gl, sym, opt); tg = time.time() - t
    t = time.time(); got = NeuralNet.getOutput(h, sp.reshape(n, -1), gl, sym, opt); tg2 = time.time() - t
    res = {}
    for k in ("policy", "value", "score_value", "ownership"):
        res[k] = float(np.abs(got[k] - ref[k]).max())
    print(f"model {os.path.basename(path)} n={n} {X}x{Y} fp16={fp16} "
          f"streams={os.environ.get('KGB_STREAM_FP32','default')}: " + " ".join(f"{k}={v:.3e}" for k, v in res.items()) +
          f" | ref |policy|max={np.abs(ref['policy']).max():.2f} |value|max={np.abs(ref['value']).max():.2f} oracle {tref:.2f}s gpu first {tg:.3f}s second {tg2*1e3:.2f}ms", flush=True)
    h.free(); ctx.free(); lm.free()
    return res

if __name__ == "__main__":
    stages = sys.argv[1:] or ["conv", "model"]
    tmp = tempfile.mkdtemp()
    if "conv" in stages:
        for fp16 in (True, False):
            conv_check(1, 64, 64, fp16=fp16)
            conv_check(3, 64, 64, fp16=fp16)
            conv_check(3, 22, 96, n=3, X=9, Y=9, fp16=fp16)
            conv_check(5, 22, 96, n=3, X=9, Y=9, fp16=fp16)
            conv_check(3, 192, 192, n=5, fp16=fp16)
            conv_check(1, 384, 192, n=9, fp16=fp16)
            conv_check(1, 192, 384, n=4, fp16=fp16)
            conv_check(3, 128, 192, n=8, X=13, Y=7, fp16=fp16)
    if "model" in stages:
        g170 = os.path.join(ROOT, "tests/golden/models/g170-b6c96-s175395328-d26788732.bin.gz")
        paths = {}
        for cfg in ("tiny_reg", "tiny_nbt", "mid_nbt"):
            paths[cfg] = modelgen.write_model(os.path.join(tmp, cfg + ".bin"), cfg, seed=3)
        for fp16 in (True, False):
            model_check(paths["tiny_reg"], 3, 9, 9, fp16)
            model_check(paths["tiny_nbt"], 5, 19, 19, fp16, sizes=[(19, 19), (9, 9), (13, 13), (19, 19), (7, 11)])
            model_check(g170, 4, 19, 19, fp16)
            model_check(g170, 3, 9, 9, fp16)
            model_check(paths["mid_nbt"], 9, 19, 19, fp16)
    if "b18" in stages:
        p = modelgen.write_model(os.path.join(tmp, "b18.bin"), "b18c384nbt", seed=0)
        for streams in ("trunk", "all", "none"):
            os.environ["KGB_STREAM_FP32"] = streams
            model_check(p, 8, 19, 19, True)
        os.environ.pop("KGB_STREAM_FP32")
        model_check(p, 8, 19, 19, False)
