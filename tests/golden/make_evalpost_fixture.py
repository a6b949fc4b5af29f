"""Generates tests/golden/evalpost.npz: the REFERENCE NNEvaluator's post-processing of chosen raw net outputs, and what the
reference Search makes of them after one visit (oracle/_ref/kgref_driver searchfake with KGREF_FAKE_TABLE, the table net).

Each row gives the table net one set of raw outputs (policy logits over the evaluator's frame, value logits, the six score-value
channels) and runs the reference Search for 1 visit on a small position, once with Black and once with White to move.  Stored per
row: the raw outputs, the position, rules, model and SearchParams, and from the reference: the root's NNOutput (policy with -1 on
illegal points, win / loss / no-result, score mean, mean square, lead, short-term errors), its NodeStats moments, utility and
weights.  The device loop's table net (debug_fake_nn = 3) is given the same raw outputs: tests/test_gpu_eval_postprocess.py.

The rows reach what the hash nets never do: a no-result logit that dominates (also under superko, where it must be removed),
win = loss, value and policy spreads whose tails underflow in double / float, the largest logit on an illegal point or on pass,
score-stdev logits at and around the softplus branch point 40 and far beyond it, large score means and leads, short-term error
channels for every post-processing version (8, 9, 10, 13, 14, 15) and non-default ModelPostProcessParams, and non-zero
noResultUtilityForWhite / winLossUtilityFactor, and a position where only pass is legal: one side fills the 7x7 board but for two
single-point eyes while the other passes (a pass in a new situation does not end the game), so the only empty points are single-stone
suicides, illegal even with multi-stone suicide legal.

Needs oracle/_ref/kgref_driver (run `python __graft_entry__.py` first)."""
import json, os, subprocess, sys, tempfile
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "..", ".."))
from katago_b200 import modelgen  # noqa: E402

DRIVER = os.path.join(HERE, "..", "..", "oracle", "_ref", "kgref_driver")

# model key -> (version, ModelPostProcessParams multipliers or None for the defaults); the device test writes the same nets
PP_ODD = (20.0, 15.5, 11.25, 7.75, 40.0, 0.3125, 42.5)
MODELS = {"v15": (15, None), "v8": (8, None), "v9": (9, None), "v10": (10, None), "v13": (13, None), "v14": (14, None),
          "v15pp": (15, PP_ODD), "v13pp": (13, PP_ODD)}


def model_for(key, directory):
    version, pp = MODELS[key]
    act = "ACTIVATION_MISH" if version >= 11 else "ACTIVATION_RELU"
    kw = {} if pp is None else {"postprocess": pp}
    return modelgen.write_model(os.path.join(directory, f"evalpost_{key}.bin"), "tiny_reg", seed=30 + version, version=version,
                                activation=act, **kw)


F32 = np.float32
VALUES = {"std": (1.0, -1.0, -30.0), "nr_dom": (-1.0, 0.5, 6.0), "w_eq_l": (0.3, 0.3, -2.0), "spread": (400.0, -400.0, -340.0),
          "mid": (0.2, -0.4, 0.6)}
SCORES = {"std": (0.3, 0.5, -0.2, 0.0, 0.0, 0.0),
          "pre40m": (0.3, float(np.nextafter(F32(40), F32(0))), -0.2, 0.0, 0.0, 0.0),
          "pre40": (0.3, 40.0, -0.2, 0.0, 0.0, 0.0),
          "pre40p": (0.3, float(np.nextafter(F32(40), F32(100))), -0.2, 0.0, 0.0, 0.0),
          "prem40": (0.3, -40.0, -0.2, 0.0, 0.0, 0.0),
          "pre800": (-0.7, 800.0, 0.9, 0.0, 0.0, 0.0),
          "big": (45.0, 3.0, -38.0, 0.0, 0.0, 0.0),
          "st": (0.6, 1.5, -0.45, 0.0, -3.5, 2.75),
          "st_big": (-0.6, 2.0, 0.45, 0.0, 50.0, -45.0)}
UNC = {"useUncertainty": 1, "uncertaintyCoeff": 0.25, "uncertaintyExponent": 1.0, "uncertaintyMaxWeight": 8.0}
BLACK_MOVES, WHITE_MOVES = [(1, 1), (2, 2)], [(1, 1)]      # Black to move after two stones, White after one


def pass_only_moves(side, n=7):
    """The opponent of `side` fills the n x n board but for the eyes (0, 0) and (n-1, n-1) while `side` passes: `side` to move, only pass
    legal."""
    fill = [(x, y) for y in range(n) for x in range(n) if (x, y) not in ((0, 0), (n - 1, n - 1))]
    moves = []
    for p in fill:
        if side == "b":
            moves += [None, p]           # Black passes, White fills; Black to move after White's last stone
        else:
            moves += [p, None]           # Black fills, White passes
    return moves if side == "b" else moves[:-1]


def policy_logits(kind, frame, X, Y, seed):
    """Raw policy logits over the frame (pass last).  (1, 1) is occupied in every row: an illegal point."""
    rng = np.random.default_rng(seed)
    P = frame * frame + 1
    lg = rng.uniform(-4.0, 4.0, P).astype(F32)
    if kind == "equal":
        lg[:] = 0.25
    elif kind == "spike":                     # one legal point 110 above the rest: every other term underflows in float
        lg[:] = -50.0
        lg[3 * frame + 3] = 60.0
    elif kind == "illegalmax":                # the largest logit on an occupied point, far above every legal one
        lg[1 * frame + 1] = 150.0
    elif kind == "passmax":
        lg[P - 1] = 9.0
    elif kind == "pm60":
        lg = rng.uniform(-60.0, 60.0, P).astype(F32)
    return lg


def rows():
    out = []
    add = lambda **r: out.append(dict(dict(frame=7, X=7, Y=7, ko=0, model="v15", params={}, policy="random", value="std", score="std"), **r))
    for k in ("equal", "spike", "illegalmax", "passmax", "pm60", "random"):
        add(policy=k)
    add(frame=19, X=9, Y=9, value="nr_dom")
    add(frame=19, X=7, Y=11, value="mid", score="big")
    add(frame=19, X=9, Y=9, policy="pm60", value="w_eq_l")
    add(frame=19, X=7, Y=11, policy="illegalmax", value="spread")
    for v in ("nr_dom", "w_eq_l", "spread", "mid"):
        add(value=v)
    for ko in (1, 2):
        for v in ("nr_dom", "mid", "spread"):
            add(ko=ko, value=v)
    for s in ("pre40m", "pre40", "pre40p", "prem40", "pre800", "big"):
        add(value="mid", score=s)
    add(ko=1, value="nr_dom", score="big")
    for m in MODELS:
        for s in ("st", "st_big"):
            add(model=m, value="mid", score=s, params=dict(UNC) if MODELS[m][0] >= 9 else {})
    add(value="nr_dom", params={"noResultUtilityForWhite": -0.5})
    add(value="mid", params={"noResultUtilityForWhite": 0.3})
    add(value="mid", params={"noResultUtilityForWhite": 0.3, "winLossUtilityFactor": 0.7}, score="big")
    add(ko=2, value="nr_dom", params={"noResultUtilityForWhite": -0.5})
    add(position="passonly", value="mid", score="big")
    full = []
    for i, r in enumerate(out):
        for side, moves in (("b", BLACK_MOVES), ("w", WHITE_MOVES)):
            if r.get("position") == "passonly":
                moves = pass_only_moves(side, r["X"])
            full.append(dict(r, side=side, moves=moves, seed=1000 + i))
    return full


def name_of(r):
    return (("passonly_" if r.get("position") == "passonly" else "") + f"{r['X']}x{r['Y']}in{r['frame']}_ko{r['ko']}_{r['model']}_pol-{r['policy']}_val-{r['value']}_sc-{r['score']}"
            + "".join(f"_{k}={v}" for k, v in sorted(r["params"].items()) if not k.startswith("uncertainty")) + f"_{r['side']}")


def raw_of(r):
    pol = policy_logits(r["policy"], r["frame"], r["X"], r["Y"], r["seed"])
    return np.concatenate([pol, np.array(VALUES[r["value"]], F32), np.array(SCORES[r["score"]], F32)])


def run_row(r, model, tmpdir):
    frame = r["frame"]
    raw = raw_of(r)
    table = np.concatenate([raw, np.zeros(frame * frame, F32)])       # ownership logits 0
    tpath = os.path.join(tmpdir, "table.txt")
    with open(tpath, "w") as f:
        f.write(" ".join(repr(float(v)) for v in table))
    env = dict(os.environ, KGREF_FAKE_TABLE=tpath, KGREF_NN_LEN=str(frame))
    params = dict(r["params"])
    if r["ko"]:
        params["koRule"] = r["ko"]
    s = " ".join("pass" if m is None else f"{m[0]},{m[1]}" for m in r["moves"])
    out = subprocess.run([DRIVER, "searchfake", model, str(r["X"]), str(r["Y"]), "1", s] + [f"{k}={float(v)!r}" for k, v in params.items()],
                         capture_output=True, text=True, check=True, env=env).stdout
    res = {}
    for ln in out.splitlines():
        f = ln.split()
        if f[0] == "rootvisits":
            assert int(f[1]) == 1, ln
            res["util"] = np.float64(f[3])
        elif f[0] == "rootstats":
            res["rootstats"] = np.array([float(t) for t in f[1:6]], np.float64)
        elif f[0] == "rootweight":
            res["weight"] = np.array([float(t) for t in f[1:3]], np.float64)
        elif f[0] == "nnoutput":
            res["nnout"] = np.array([float(t) for t in f[1:9]], F32)
        elif f[0] == "policy":
            res["policy"] = np.array([float(t) for t in f[1:]], F32)
    assert res["policy"].size == frame * frame + 1
    return raw, res


if __name__ == "__main__":
    rs = rows()
    arrays = {"num_rows": np.int32(len(rs))}
    with tempfile.TemporaryDirectory() as td:
        models = {k: model_for(k, td) for k in MODELS}
        for i, r in enumerate(rs):
            raw, res = run_row(r, models[r["model"]], td)
            meta = {k: r[k] for k in ("frame", "X", "Y", "ko", "model", "params", "side", "moves")}
            meta["name"] = name_of(r)
            arrays[f"r{i}_meta"] = np.array(json.dumps(meta))
            arrays[f"r{i}_raw"] = raw
            for k, v in res.items():
                arrays[f"r{i}_{k}"] = v
    arrays["models"] = np.array(json.dumps(MODELS))
    np.savez_compressed(os.path.join(HERE, "evalpost.npz"), **arrays)
    print(f"wrote {len(rs)} rows")
