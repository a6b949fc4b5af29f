"""Generates tests/golden/searchfake_uncertainty.npz from the REFERENCE Search with uncertainty-weighted evaluations and noise pruning
(useUncertainty, useNoisePruning), driven by tests/cpp/uncertainty_search_driver.cpp, which this script compiles against the reference
objects oracle/Makefile.ref builds (oracle/_ref/libkgref.a; run `python __graft_entry__.py` first).

The driver's fake net is the hash net of oracle/ref_driver.cpp with hash-derived raw short-term error channels (the device loop's
debug_fake_nn = 2) unless a case says otherwise.  Whether the errors count depends on the model file's version
(NNEvaluator::supportsShorttermError): the cases use nets of versions 15, 12, 9 and 8 written by katago_b200.modelgen (only the
version and the post-processing multipliers matter to the fake net).  Stored per case as in searchfake.npz, plus the root's and every
root child's weightSum / weightSqSum."""
import json, os, subprocess, sys, tempfile
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(HERE, "..", ".."))
import make_search_fixtures as F  # noqa: E402
from katago_b200 import modelgen  # noqa: E402


def model_for(version, directory):
    """The net of a given version the fixture and the device test both use (deterministic)."""
    act = "ACTIVATION_MISH" if version >= 11 else "ACTIVATION_RELU"
    return modelgen.write_model(os.path.join(directory, f"unc_v{version}.bin"), "tiny_reg", seed=20 + version, version=version, activation=act)


UNC = {"useUncertainty": 1, "uncertaintyCoeff": 0.25, "uncertaintyExponent": 1.0, "uncertaintyMaxWeight": 8.0}
PRUNE = {"useNoisePruning": 1, "noisePruneUtilityScale": 0.15, "noisePruningCap": 1e50}
SP = dict(F.SELFPLAY8B18)
GRAPH = dict(F.SELFPLAY8B18, useGraphSearch=1, **F.BIAS, **F.LCB)


def cases():
    p19 = F.prefix_from_stream("boardstream_19x19_multisuicide.npz", 40)
    p9 = F.prefix_from_stream("boardstream_9x9_multisuicide.npz", 12)
    p5 = F.prefix_from_stream("boardstream_5x5_multisuicide.npz", 9)
    # (X, Y, visits, moves, params, model version, fake short-term channels)
    return [
        (9, 9, 400, p9, dict(SP, **UNC), 15, 1),                                                   # uncertainty alone
        (9, 9, 400, p9, dict(SP, **PRUNE), 15, 1),                                                 # noise pruning alone
        (9, 9, 400, p9, dict(SP, **UNC, **PRUNE), 15, 1),                                          # both
        (9, 9, 500, p9, dict(GRAPH, **UNC, **PRUNE), 15, 1),                                       # graph search, bias, LCB
        (9, 9, 400, p9, dict(SP, **dict(UNC, uncertaintyExponent=0.5), **PRUNE), 12, 1),           # version 10-13, sqrt branch
        (9, 9, 400, p9, dict(SP, **dict(UNC, uncertaintyExponent=0.7), **PRUNE), 9, 1),            # version 9, pow branch
        (9, 9, 400, p9, dict(SP, **UNC, **PRUNE), 8, 1),                                           # version 8: weight 1, pruning still acts
        (9, 9, 300, p9, dict(SP, **UNC, rootNumSymmetriesToSample=4), 15, 1),                      # 4 root symmetries, errors averaged
        (9, 9, 300, p9, dict(SP, **UNC, **PRUNE, rootNumSymmetriesToSample=4), 12, 1),
        (5, 5, 600, p5, dict(SP, **UNC, **PRUNE), 15, 1),                                          # reaches terminal positions
        (5, 5, 600, p5, dict(SP, **dict(UNC, uncertaintyExponent=0.7, uncertaintyMaxWeight=3.0)), 15, 1),
        (19, 19, 300, p19, dict(SP, **UNC, **PRUNE), 15, 1),
        (19, 19, 300, p19, dict(GRAPH, **dict(UNC, uncertaintyExponent=0.5), **PRUNE), 15, 1),
        (9, 9, 400, p9, dict(SP, **UNC, **PRUNE), 15, 0),                                          # the fake net's zero channels
        (9, 9, 300, p9, dict(SP, **UNC, **PRUNE, rootNoiseEnabled=1, rootDirichletNoiseTotalConcentration=10.83,
                             rootDirichletNoiseWeight=0.25), 15, 1),                              # root noise: pruning on the noised policy
        (9, 9, 400, p9, dict(SP, **dict(PRUNE, noisePruneUtilityScale=0.05, noisePruningCap=0.5)), 15, 1),
    ]


def build_driver(directory):
    """tests/cpp/uncertainty_search_driver.cpp linked like oracle/Makefile.drivers links the fixture driver (same reference tree, flags and
    libraries)."""
    root = os.path.join(HERE, "..", "..")
    make = ["make", "-s", "-f", "oracle/Makefile.drivers", "--eval", "print-%: ; @echo $($*)"]
    ref, cxxflags, libs = (subprocess.run(make + [f"print-{v}"], cwd=root, capture_output=True, text=True, check=True).stdout.strip()
                           for v in ("REF", "CXXFLAGS", "LIBS"))
    exe = os.path.join(directory, "uncertainty_search_driver")
    subprocess.run(["g++"] + cxxflags.split() + ["-I" + ref, "-I.", "-o", exe, "tests/cpp/uncertainty_search_driver.cpp"] + libs.split(),
                   cwd=root, check=True)
    return exe


def run(driver, X, Y, visits, moves, params, model, fake_shortterm):
    s = " ".join("pass" if m is None else f"{m[0]},{m[1]}" for m in moves)
    out = subprocess.run([driver, model, str(X), str(Y), str(visits), str(fake_shortterm), s] + [f"{k}={float(v)!r}" for k, v in params.items()],
                         capture_output=True, text=True, check=True).stdout
    P = X * Y + 1
    v = np.zeros(P, np.int32); u = np.zeros(P, np.float64); w = np.zeros((P, 2), np.float64); rw = np.zeros(2, np.float64); seed = ""
    for ln in out.splitlines():
        f = ln.split()
        idx = lambda x, y: X * Y if x < 0 else y * X + x
        if f[0] == "child":
            i = idx(int(f[1]), int(f[2])); v[i] = int(f[3]); u[i] = float(f[4]); w[i] = [float(f[5]), float(f[6])]
        elif f[0] == "rootweights":
            rw[:] = [float(f[1]), float(f[2])]
        elif f[0] == "threadseed":
            seed = ln.split(" ", 1)[1]
    return v, u, w, rw, seed


def main():
    store = {}
    with tempfile.TemporaryDirectory() as tmp:
        driver = build_driver(tmp)
        for i, (X, Y, visits, moves, params, version, fake) in enumerate(cases()):
            v, u, w, rw, seed = run(driver, X, Y, visits, moves, params, model_for(version, tmp), fake)
            store[f"c{i}_shape"] = np.array([X, Y, visits], np.int32)
            store[f"c{i}_moves"] = np.array([(-1, -1) if m is None else m for m in moves], np.int8).reshape(-1, 2)
            store[f"c{i}_params"] = np.array(json.dumps(params))
            store[f"c{i}_version"] = np.array(version, np.int32)
            store[f"c{i}_fake_shortterm"] = np.array(fake, np.int32)
            store[f"c{i}_visits"] = v; store[f"c{i}_util"] = u; store[f"c{i}_weights"] = w; store[f"c{i}_root_weights"] = rw
            store[f"c{i}_threadseed"] = np.array(seed)
            print(f"case {i}: {X}x{Y} v{version} {visits} visits, root weight {rw[0]:.4f} / {rw[1]:.4f}, {int((v > 0).sum())} children")
    store["num_cases"] = np.array(len(cases()), np.int32)
    np.savez_compressed(os.path.join(HERE, "searchfake_uncertainty.npz"), **store)


if __name__ == "__main__":
    main()
