"""The loop's evaluation post-processing restated in numpy, with the error model the tests bound it by.

What is restated: NNEvaluator's post-processing of one raw net output (nneval.cpp:960-1051 policy, :1112-1215 value, score and
short-term errors; version >= 4 nets), as the device loop runs it in spBackupKernel, and the utility the search gives that
evaluation (Search::getUtilityFromNN without score utility: (win - loss) * winLossUtilityFactor + noResult * noResultUtilityForWhite).

`exact(row)` computes every quantity in float64 from the float raw outputs, without rounding the results to float.  `device_model(row)`
computes them the way the kernel does: policy in float32 (exp of the float difference to the legal maximum, a 32-lane tree sum with
up to 12 terms per lane, one division), value fields in double then rounded to float, NodeStats moments and utility from the rounded
floats widened back to double.  Mutants of the kernel are flags of `device_model`.

Error model (u = 2^-24, the unit roundoff of float):
- policy, per legal point i with exact probability p_i and a_i = |logit_i - max|: the difference rounds (u * a_i), CUDA expf errs by
  at most 2 ulp (4u); the sum errs by the p-weighted mean of those term errors plus one rounding per level of the summation tree
  (12 per lane + 5 butterfly levels on the device, P - 1 for the reference's sequential sum), the division by one more u.  So
  |p - p_i| <= p_i * (e_i + sum_j p_j e_j + (depth + 1) u) + 2^-147, e_j = u * a_j + 4u; the absolute term covers terms that
  underflow to float denormals or to 0.
- value fields (win, loss, no-result, score mean, mean square, lead, short-term errors): a double result rounded to float, so at most
  1 float ulp of the exact value plus the double error (1e-14 relative here).  The win-loss moment is the difference of two such
  floats: the sum of their bounds.
- utility: the rounding of the floats it is made of, scaled by the factors, plus 1e-14.
Against the reference's own results (evalpost.npz): the legality mask equal, policy within the sum of the two policy bounds, NNOutput
fields within 1 float ulp of each other, NodeStats moments, utility and weights to 1e-12 relative (both sides round the same double
to float, so the float values agree; what remains is double arithmetic)."""
import json
import numpy as np

U = 2.0 ** -24
ABS_POLICY = 2.0 ** -147
DEVICE_SUM_DEPTH = 12 + 5
MUTANTS = ("lead_no_1mn", "meansq_no_1mn", "no_superko_zeroing", "max_over_illegal", "softplus_ge_40", "softplus_no_linear_branch",
           "lead_no_colour_flip", "ignore_no_result_utility", "no_float_round_trip")


def load_rows(path):
    d = np.load(path)
    rows = []
    for i in range(int(d["num_rows"])):
        r = json.loads(str(d[f"r{i}_meta"]))
        for k in ("raw", "util", "rootstats", "weight", "nnout", "policy"):
            r[k] = d[f"r{i}_{k}"]
        rows.append(r)
    return rows


def model_params(key):
    """(version, scoreMean, scoreStdev, lead, shorttermValueError, shorttermScoreError multipliers) of a fixture model key."""
    version, pp = {"v15": (15, None), "v8": (8, None), "v9": (9, None), "v10": (10, None), "v13": (13, None), "v14": (14, None),
                   "v15pp": (15, (20.0, 15.5, 11.25, 7.75, 40.0, 0.3125, 42.5)), "v13pp": (13, (20.0, 15.5, 11.25, 7.75, 40.0, 0.3125, 42.5))}[key]
    pp = pp or (20.0, 20.0, 20.0, 20.0, 40.0, 0.25, 30.0)
    f = [float(np.float32(v)) for v in pp]         # ModelPostProcessParams are floats
    return version, f[1], f[2], f[3], f[5], f[6]


def legal_mask(row):
    """The reference's legality mask (NNOutput policy -1 = illegal); the device test checks that the loop's mask equals it."""
    return np.asarray(row["policy"]) >= 0


def _softplus(x):
    return x if x > 40.0 else float(np.log(1.0 + np.exp(x)))


def _value_part(row, mutant=None):
    """Value, score and short-term fields in double, white's perspective, before rounding to float (nneval.cpp:1112-1215)."""
    raw = np.asarray(row["raw"], np.float32)
    P = row["frame"] ** 2 + 1
    val, sc = [float(v) for v in raw[P:P + 3]], [float(v) for v in raw[P + 3:P + 9]]
    version, mmul, smul, lmul, stv, sts = model_params(row["model"])
    wl, ll, nl = val
    superko = row["ko"] != 0 and mutant != "no_superko_zeroing"
    if superko:
        nl -= 100000.0
    m = max(wl, ll, nl)
    w, l, n = np.exp(wl - m), np.exp(ll - m), np.exp(nl - m)
    if superko:
        n = 0.0
    s = w + l + n
    w, l, n = w / s, l / s, n / s
    mean = sc[0] * mmul
    pre = sc[1]
    if mutant == "softplus_ge_40":
        sd = pre if pre >= 40.0 else float(np.log(1.0 + np.exp(pre)))
    elif mutant == "softplus_no_linear_branch":
        with np.errstate(over="ignore"):
            sd = float(np.log(1.0 + np.exp(pre)))
    else:
        sd = _softplus(pre)
    sd *= smul
    meansq = mean * mean + sd * sd
    mean *= 1.0 - n
    if mutant != "meansq_no_1mn":
        meansq *= 1.0 - n
    lead = sc[2] * lmul * (1.0 if mutant == "lead_no_1mn" else 1.0 - n)
    if version >= 14:
        a, b = _softplus(sc[4] * 0.5), _softplus(sc[5] * 0.5)
        ste, sse = np.sqrt(a * a * stv), np.sqrt(b * b * sts)
    elif version >= 10:
        ste, sse = np.sqrt(_softplus(sc[4]) * stv), np.sqrt(_softplus(sc[5]) * sts)
    else:
        ste, sse = _softplus(sc[4]), _softplus(sc[5]) * 10.0
    if version < 9:
        ste = sse = -1.0
    black = row["side"] == "b"
    flip = -1.0 if black else 1.0
    return dict(win=l if black else w, loss=w if black else l, noresult=n, mean=flip * mean, meansq=meansq,
                lead=(lead if mutant == "lead_no_colour_flip" else flip * lead), st_wl=float(ste), st_score=float(sse))


FIELDS = ("win", "loss", "noresult", "mean", "meansq", "lead", "st_wl", "st_score")


def _utility(row, v, mutant=None):
    wlf = float(row["params"].get("winLossUtilityFactor", 1.0))
    nru = 0.0 if mutant == "ignore_no_result_utility" else float(row["params"].get("noResultUtilityForWhite", 0.0))
    return (v["win"] - v["loss"]) * wlf + v["noresult"] * nru


def _moments(v):
    return np.array([v["win"] - v["loss"], v["noresult"], v["mean"], v["meansq"], v["lead"]], np.float64)


def exact(row):
    """float64 restatement: policy (-1 illegal), value fields (unrounded), moments and utility of the unrounded values."""
    raw = np.asarray(row["raw"], np.float32)
    P = row["frame"] ** 2 + 1
    lg = raw[:P].astype(np.float64)
    legal = legal_mask(row)
    m = lg[legal].max()
    e = np.where(legal, np.exp(np.where(legal, lg - m, 0.0)), 0.0)
    pol = np.where(legal, e / e.sum(), -1.0)
    v = _value_part(row)
    return dict(policy=pol, values=v, moments=_moments(v), utility=_utility(row, v))


def device_model(row, mutant=None):
    """What spBackupKernel computes, restated with float32 where the kernel uses float; `mutant` breaks one step of it."""
    raw = np.asarray(row["raw"], np.float32)
    P = row["frame"] ** 2 + 1
    lg = raw[:P]
    legal = legal_mask(row)
    m = lg.max() if mutant == "max_over_illegal" else lg[legal].max()
    with np.errstate(under="ignore", over="ignore", invalid="ignore", divide="ignore"):
        d = np.where(legal, lg - m, np.float32(0)).astype(np.float32)             # the difference rounds to float, exp is then
        e = np.where(legal, np.exp(d.astype(np.float64)).astype(np.float32), np.float32(0))   # correctly rounded (expf: <= 2 ulp)
        lanes = np.zeros(32, np.float32)
        for i in range(P):                                  # lane i % 32 adds its terms in order, then the butterfly
            lanes[i % 32] = np.float32(lanes[i % 32] + e[i])
        o = 16
        while o:
            lanes = (lanes + lanes[np.arange(32) ^ o]).astype(np.float32)
            o >>= 1
        pol = np.where(legal, (e / lanes[0]).astype(np.float32), np.float32(-1)).astype(np.float32)
    v = _value_part(row, mutant)
    if mutant != "no_float_round_trip":
        v = {k: float(np.float32(x)) for k, x in v.items()}
    return dict(policy=pol.astype(np.float64), values=v, moments=_moments(v), utility=_utility(row, v, mutant))


def _ulp32(x):
    x = np.abs(np.asarray(x, np.float64))
    return np.spacing(np.float32(np.minimum(x, 3.0e38))).astype(np.float64)


def policy_bound(row, ex_policy, depth):
    legal = legal_mask(row)
    raw = np.asarray(row["raw"], np.float32)
    P = row["frame"] ** 2 + 1
    lg = raw[:P].astype(np.float64)
    a = np.abs(lg - lg[legal].max())
    e = U * a + 4 * U
    p = np.where(legal, ex_policy, 0.0)
    sum_err = float((p * e).sum())
    return np.where(legal, p * (e + sum_err + (depth + 1) * U) + ABS_POLICY, 0.0)


def value_bound(x):
    """1 float ulp of the exact value plus the double error."""
    return _ulp32(x) + 1e-14 * np.abs(x) + 1e-300


def moment_bound(ex):
    v = ex["values"]
    b = np.array([value_bound(v["win"]) + value_bound(v["loss"]), value_bound(v["noresult"]), value_bound(v["mean"]),
                  value_bound(v["meansq"]), value_bound(v["lead"])])
    return b


def utility_bound(row, ex):
    v = ex["values"]
    wlf = abs(float(row["params"].get("winLossUtilityFactor", 1.0)))
    nru = abs(float(row["params"].get("noResultUtilityForWhite", 0.0)))
    return wlf * (value_bound(v["win"]) + value_bound(v["loss"])) + nru * value_bound(v["noresult"]) + 1e-14


def _ratio(err, bound):
    err = np.abs(np.asarray(err, np.float64))
    with np.errstate(invalid="ignore", divide="ignore"):
        r = np.where(np.isfinite(err), err / bound, np.inf)
    return float(np.max(r)) if r.size else 0.0


def check(row, got, ex=None):
    """Worst error / bound of every check for one row.  got: dict(policy, moments, utility[, values, root_stats, root_utility,
    root_weight]) - what the device (or a restatement standing in for it) produced; absent keys are not checked."""
    ex = ex or exact(row)
    legal = legal_mask(row)
    out = {}
    pol = np.asarray(got["policy"], np.float64)
    out["mask"] = 0.0 if np.array_equal(pol >= 0, legal) else np.inf
    bd = policy_bound(row, ex["policy"], DEVICE_SUM_DEPTH)
    br = policy_bound(row, ex["policy"], row["frame"] ** 2)
    out["policy_vs_fp64"] = _ratio((pol - ex["policy"])[legal], bd[legal])
    out["policy_vs_ref"] = _ratio((pol - row["policy"].astype(np.float64))[legal], (bd + br)[legal])
    out["moments_vs_fp64"] = _ratio(np.asarray(got["moments"]) - ex["moments"], moment_bound(ex))
    ref_nn = row["nnout"].astype(np.float64)
    ref_mom = np.array([ref_nn[0] - ref_nn[1], ref_nn[2], ref_nn[3], ref_nn[4], ref_nn[5]])
    ulp_ref = np.array([_ulp32(ref_nn[0]) + _ulp32(ref_nn[1]), _ulp32(ref_nn[2]), _ulp32(ref_nn[3]), _ulp32(ref_nn[4]), _ulp32(ref_nn[5])])
    out["moments_vs_ref_nnoutput"] = _ratio(np.asarray(got["moments"]) - ref_mom, ulp_ref + 1e-300)
    stats = got.get("root_stats", got["moments"])
    out["root_stats_vs_ref"] = _ratio(np.asarray(stats) - row["rootstats"], 1e-12 * np.maximum(1.0, np.abs(row["rootstats"])))
    out["utility_vs_fp64"] = _ratio(got["utility"] - ex["utility"], utility_bound(row, ex))
    ru = got.get("root_utility", got["utility"])
    out["utility_vs_ref"] = _ratio(ru - float(row["util"]), 1e-12 * max(1.0, abs(float(row["util"]))))
    if "values" in got:
        gv = got["values"]
        out["shortterm_vs_ref"] = _ratio([gv["st_wl"] - float(ref_nn[6]), gv["st_score"] - float(ref_nn[7])],
                                         np.array([_ulp32(ref_nn[6]), _ulp32(ref_nn[7])]) + 1e-300)
    if "root_weight" in got:
        out["weight_vs_ref"] = _ratio(np.asarray(got["root_weight"]) - row["weight"], 1e-12 * np.maximum(1.0, np.abs(row["weight"])))
    return out
