"""The loop's evaluation post-processing (spBackupKernel: legality-masked policy softmax, win / loss / no-result softmax in double with
the float round trip, superko's no-result removal, score mean / stdev / lead scaled by P(result), short-term errors) and the utility
and NodeStats moments the search takes from it - where the hash nets never reach.

tests/golden/evalpost.npz (tests/golden/make_evalpost_fixture.py) holds raw net outputs chosen per row and what the REFERENCE
NNEvaluator and Search (1 visit) made of them.  The device loop's table net (debug_fake_nn = 3) returns the same raw outputs; every
row is checked against the float64 restatement of tests/evalpost_oracle.py within the bounds of its error model, and against the
reference's own results.  The CPU tests check the restatement against the fixture, rehearse the bounds on a float32 restatement of the
kernel, and show that each mutant of the kernel breaks a bound by 8x or more.

searchfake_wide.npz (tests/golden/make_searchfake_wide_fixture.py) carries the same post-processing through whole searches on the wide
hash net (debug_fake_nn = 4), with the assertions of the narrow net's search fixture.

Mutants applied to the kernel in throwaway builds and run on an H100 against the search tests that existed before these
(test_gpu_board_selfplay.py fake-net and trained-net searches, test_gpu_uncertainty.py, test_gpu_mixed_sizes.py: 91 tests) and
against this file:
  lead without (1 - n)                              old: all pass        new: 13 fail (table rows; 12 wide searches)
  score mean square without (1 - n)                 old: 3 trained-net   new: 13 fail
  no superko removal (no -100000, no zeroing)       old: all pass        new: 5 fail (table rows; wide searches 2, 3, 11, 14)
  utilityFromEval ignores noResultUtilityForWhite   old: all pass        new: 12 fail
Dropping only the zeroing is an equivalent mutant: after the -100000 the no-result exp underflows to 0 anyway.  The wide searches
under superko cannot show the (1 - n) and noResultUtilityForWhite mutants (P(no result) is removed there); those without
noResultUtilityForWhite cannot show the last one."""
import collections
import json
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import evalpost_oracle as eo  # noqa: E402

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "evalpost.npz")


@pytest.fixture(scope="module")
def rows():
    return eo.load_rows(GOLDEN)


def test_fixture_covers_the_rows_the_hash_nets_miss(rows):
    """The no-result-dominant, superko, underflow, softplus-branch, illegal-maximum and utility rows are all there, each both ways."""
    names = [r["name"] for r in rows]
    assert len(names) == len(set(names))
    assert collections.Counter(r["side"] for r in rows) == {"b": len(rows) // 2, "w": len(rows) // 2}
    nr = [r for r in rows if r["ko"] == 0 and eo.exact(r)["values"]["noresult"] > 0.9]
    sk = [r for r in rows if r["ko"] != 0 and max(r["raw"][r["frame"] ** 2 + 1:][:3]) == r["raw"][r["frame"] ** 2 + 3]]
    assert nr and sk and all(float(r["nnout"][2]) == 0.0 for r in sk)
    assert {r["model"] for r in rows} >= {"v8", "v9", "v10", "v13", "v14", "v15", "v15pp", "v13pp"}
    assert {r["params"].get("noResultUtilityForWhite") for r in rows} >= {-0.5, 0.3}
    pre = {float(r["raw"][r["frame"] ** 2 + 1 + 4]) for r in rows}
    assert {float(np.nextafter(np.float32(40), np.float32(0))), 40.0, float(np.nextafter(np.float32(40), np.float32(100))), -40.0, 800.0} <= pre
    assert any((r["policy"] == 0).any() for r in rows), "no policy tail underflows to 0"
    assert any(r["frame"] == 19 and r["X"] == 7 and r["Y"] == 11 for r in rows) and any(r["frame"] == 19 and r["X"] == 9 for r in rows)
    assert {r["side"] for r in rows if eo.legal_mask(r).sum() == 1 and eo.legal_mask(r)[-1]} == {"b", "w"}, "no pass-only position"


def test_float64_restatement_matches_the_reference(rows):
    """The reference's NNOutput and 1-visit NodeStats are within the bounds of the float64 restatement (reference summation depth)."""
    worst = collections.defaultdict(float)
    for r in rows:
        ex = eo.exact(r)
        legal = eo.legal_mask(r)
        ref = r["policy"].astype(np.float64)
        b = eo.policy_bound(r, ex["policy"], r["frame"] ** 2)
        worst["policy"] = max(worst["policy"], float((np.abs(ref - ex["policy"])[legal] / b[legal]).max()))
        v = ex["values"]
        for i, k in enumerate(eo.FIELDS):
            if k.startswith("st_") and v[k] == -1.0:
                assert r["nnout"][i] == -1.0, (r["name"], k)
                continue
            worst[k] = max(worst[k], abs(float(r["nnout"][i]) - v[k]) / float(eo.value_bound(v[k])))
        worst["utility"] = max(worst["utility"], abs(float(r["util"]) - ex["utility"]) / eo.utility_bound(r, ex))
    assert max(worst.values()) <= 1.0, dict(worst)


def test_float32_restatement_stays_well_inside_every_bound(rows):
    """The kernel restated with its own float steps stays within half of the value and utility bounds (rounding to nearest is half
    the ulp they allow) and within the policy bound, and meets the checks against the reference.  The policy has no wider margin: the
    float difference to the maximum that exp takes errs by up to u * |logit - max|, in the kernel and in this restatement alike, and
    that term dominates the bound of the far tail (pm60 rows reach 0.58 of it)."""
    for r in rows:
        ex = eo.exact(r)
        dm = eo.device_model(r)
        res = eo.check(r, dm, ex)
        assert res["policy_vs_fp64"] <= 1.0 and res["moments_vs_fp64"] <= 0.5 and res["utility_vs_fp64"] <= 0.5, (r["name"], res)
        assert all(v <= 1.0 for v in res.values()), (r["name"], res)


# Rows that must show each mutant (named by what makes them able to): every other row cannot, for the reason given.
def _n(r):
    return eo.exact(r)["values"]["noresult"]


SHOWN_BY = {
    # P(no result) must be far from 0 and the lead / stdev not zero: simple-ko rows with a mid or dominant no-result logit
    "lead_no_1mn": lambda r: _n(r) > 0.05,
    "meansq_no_1mn": lambda r: _n(r) > 0.05,
    # superko rows whose no-result logit is not negligible before the removal
    "no_superko_zeroing": lambda r: r["ko"] != 0 and r["raw"][r["frame"] ** 2 + 3] - max(r["raw"][r["frame"] ** 2 + 1:][:2]) > -20,
    # an illegal logit so far above the legal ones that every legal term underflows
    "max_over_illegal": lambda r: r["raw"][1 * r["frame"] + 1] - r["raw"][:r["frame"] ** 2 + 1][eo.legal_mask(r)].max() > 110,
    # the stdev logit overflows exp without the linear branch
    "softplus_no_linear_branch": lambda r: r["raw"][r["frame"] ** 2 + 1 + 4] > 710,
    # Black to move with a lead that survives (1 - n)
    "lead_no_colour_flip": lambda r: r["side"] == "b" and abs(eo.exact(r)["values"]["lead"]) > 1e-3,
    "ignore_no_result_utility": lambda r: r["params"].get("noResultUtilityForWhite", 0.0) != 0.0 and _n(r) > 0.05,
    # every row whose win, loss or no-result is not a float already
    "no_float_round_trip": lambda r: any(float(np.float32(eo.exact(r)["values"][k])) != eo.exact(r)["values"][k] for k in ("win", "loss", "noresult")),
}


@pytest.mark.parametrize("mutant", [m for m in eo.MUTANTS if m != "softplus_ge_40"])
def test_each_mutant_breaks_a_bound_by_8x(rows, mutant):
    shown = [r for r in rows if SHOWN_BY[mutant](r)]
    assert shown, mutant
    for r in shown:
        res = eo.check(r, eo.device_model(r, mutant))
        assert max(res.values()) >= 8.0, (mutant, r["name"], res)


def test_softplus_branch_at_40_is_invisible_in_double(rows):
    """`pre >= 40` instead of `pre > 40` changes only pre = 40 exactly, where log(1 + exp(40)) = 40 + 4.2e-18 rounds to 40 in double:
    an equivalent mutant that no output can show (the rows at 40 - ulp, 40 and 40 + ulp pin both sides of the branch instead)."""
    at40 = [r for r in rows if float(r["raw"][r["frame"] ** 2 + 1 + 4]) == 40.0]
    assert at40
    for r in at40:
        a, b = eo.device_model(r), eo.device_model(r, "softplus_ge_40")
        assert a["values"] == b["values"]


def _snake(k):
    return "".join("_" + c.lower() if c.isupper() else c for c in k)


@pytest.mark.gpu
def test_device_post_processing_matches_float64_and_the_reference(rows, tmp_path):
    """Every row through the loop's table net for one wave (1 visit): legality mask, policy, the root's own evaluation,
    NodeStats moments, utility and weight against the float64 restatement and the reference.  Prints each check's worst error as a
    fraction of its bound.  The short-term errors have no reader of their own: they are checked through the root's weight, which
    the uncertainty rows (versions 9-15, default and other multipliers) derive from them and which must equal the reference's to 1e-12;
    the version-8 rows check that the weight stays 1."""
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
    from make_evalpost_fixture import model_for
    from katago_b200 import NeuralNet, SelfPlay
    groups = collections.defaultdict(list)
    for r in rows:
        groups[(r["frame"], r["model"], json.dumps(r["params"], sort_keys=True))].append(r)
    worst = collections.defaultdict(float)
    failures = []
    models = {}
    for (frame, mkey, pj), grp in groups.items():
        if mkey not in models:
            models[mkey] = NeuralNet.loadModelFile(model_for(mkey, str(tmp_path)))
        lm = models[mkey]
        ctx = NeuralNet.createComputeContext([0], frame, frame, False, lm)
        h = NeuralNet.createComputeHandle(ctx, lm, max(8, len(grp)), False, True, 0)
        kw = {_snake(k): (bool(v) if k == "useUncertainty" else float(v)) for k, v in json.loads(pj).items()}
        # max_visits 2 (the least the loop takes) and one wave: the wave evaluates each unvisited root once, like the reference's
        # 1-visit search
        sp = SelfPlay(h, len(grp), 2, komi=7.5, multi_stone_suicide_legal=True, early_temperature_moves=0, seed=1, debug_fake_nn=3,
                      debug_hold_at_max_visits=True, **kw)
        sp.set_game_setup(np.array([[r["X"], r["Y"], r["ko"], 1] for r in grp], np.int32), also_current_games=True)
        for g, r in enumerate(grp):
            sp.play_moves_game(g, [None if m is None else tuple(m) for m in r["moves"]])
            P = frame * frame + 1
            sp.debug_set_raw_outputs(g, r["raw"][:P], r["raw"][P:P + 3], r["raw"][P + 3:P + 9])
        sp.run(1)
        for g, r in enumerate(grp):
            _, info = sp.game(g)
            assert info["root_visits"] == 1 and info["black_to_move"] == (r["side"] == "b"), (r["name"], info)
            v, pol, _ = sp.root_children(g)
            _, rt = sp.root_value_stats(g)
            nn = sp.root_extra(g)["root_nn_moments"]
            u_nn, u_avg = sp.root_utility(g)
            _, rw = sp.root_weights(g)
            got = dict(policy=pol, moments=nn, utility=u_nn, root_stats=rt, root_utility=u_avg, root_weight=rw)
            res = eo.check(r, got)
            for k, x in res.items():
                worst[k] = max(worst[k], x)
            if max(res.values()) > 1.0:
                failures.append((r["name"], {k: x for k, x in res.items() if x > 1.0}))
        sp.free(); h.free(); ctx.free()
    for lm in models.values():
        lm.free()
    print("worst error / bound: " + " ".join(f"{k}={x:.3g}" for k, x in sorted(worst.items())))
    assert not failures, failures[:10]


# ---- the wide hash net: the same post-processing backed up through whole searches ------------------------------------------------
WIDE_GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "searchfake_wide.npz")
BRANCHES = ("P(no result) > 0.05", "superko removes P(no result) > 0.05", "stdev logit > 40", "policy term underflows to 0 in float")


def test_wide_fixture_reaches_every_branch():
    """The reference's own evaluations in searchfake_wide.npz took every branch the narrow hash net never reaches, so the fixture cannot
    drift back into the narrow range."""
    d = np.load(WIDE_GOLDEN)
    n = int(d["num_cases"])
    assert n >= 16
    total = sum(d[f"c{i}_branches"] for i in range(n))
    assert (total > 0).all(), dict(zip(BRANCHES, total.tolist()))
    params = [json.loads(str(d[f"c{i}_params"])) for i in range(n)]
    assert {p.get("koRule", 0) for p in params} == {0, 1, 2}
    assert any(p.get("useGraphSearch") for p in params) and any(p.get("rootNumSymmetriesToSample", 1) == 4 for p in params)
    assert any(p.get("rootEndingBonusPoints") and p.get("rootPruneUselessMoves") for p in params)
    assert any(p.get("staticScoreUtilityFactor") for p in params) and sum(p.get("noResultUtilityForWhite", 0.0) != 0.0 for p in params) >= 8
    assert any(json.loads(str(d[f"c{i}_device"])).get("nn_cache_size_power_of_two") for i in range(n))
    assert any(int(d[f"c{i}_shape"][3]) == 19 and int(d[f"c{i}_shape"][0]) == 9 for i in range(n))


def _wide_kwargs(params):
    kw = dict(cpuct_exploration=1.0, cpuct_exploration_log=0.45, cpuct_exploration_base=500.0, fpu_reduction_max=0.2, root_fpu_reduction_max=0.1)
    for k, v in params.items():
        if k == "minVisitPropForLCB":
            kw["min_visit_prop_for_lcb"] = float(v)
        elif k == "koRule":
            kw["ko_rule"] = int(v)
        elif k in ("fpuParentWeightByVisitedPolicy", "useGraphSearch", "useLcbForSelection", "useNonBuggyLcb", "rootPruneUselessMoves"):
            kw[_snake(k)] = bool(v)
        elif k in ("graphSearchRepBound", "rootNumSymmetriesToSample"):
            kw[_snake(k)] = int(v)
        else:
            kw[_snake(k)] = float(v)
    return kw


@pytest.mark.gpu
@pytest.mark.parametrize("case", range(16))
def test_wide_hash_net_searches_match_the_reference(tmp_models, case):
    """Whole searches on the wide hash net (debug_fake_nn = 4; P(no result) up to ~1, superko removing it, noResultUtilityForWhite,
    stdev logits past 40, underflowing policy tails): root visit counts identical to the reference Search's, child utilities to 1e-12,
    NodeStats moments of the root and its children to 1e-9, play selection values - the assertions of the narrow net's fixture."""
    from katago_b200 import NeuralNet, SelfPlay
    d = np.load(WIDE_GOLDEN)
    X, Y, visits, frame = (int(v) for v in d[f"c{case}_shape"])
    params = json.loads(str(d[f"c{case}_params"]))
    kw = dict(_wide_kwargs(params), **json.loads(str(d[f"c{case}_device"])))
    lm = NeuralNet.loadModelFile(tmp_models["tiny_reg"])
    ctx = NeuralNet.createComputeContext([0], frame or X, frame or Y, True, lm)
    h = NeuralNet.createComputeHandle(ctx, lm, 4, False, True, 0)
    sp = SelfPlay(h, 3, visits, komi=7.5, multi_stone_suicide_legal=True, early_temperature_moves=0, seed=1, debug_fake_nn=4,
                  debug_hold_at_max_visits=True, **kw)
    if frame:
        sp.set_game_setup(np.array([[X, Y, params.get("koRule", 0), 1]] * 3, np.int32), also_current_games=True)
    sp.play_moves([None if m[0] < 0 else (int(m[0]), int(m[1])) for m in d[f"c{case}_moves"]])
    sp.set_search_rand(str(d[f"c{case}_thread_seed"]))
    for _ in range(100):
        sp.run(max(8, visits // 8))
        if all(sp.game(g)[1]["root_visits"] >= visits for g in range(3)):
            break
    for g in range(3):
        v, pol, util = sp.root_children(g)
        assert sp.game(g)[1]["root_visits"] == visits
        ref_pol = d[f"c{case}_policy"]
        assert np.array_equal(pol < 0, ref_pol < 0), "legality mask differs"
        assert np.abs(pol - ref_pol)[ref_pol >= 0].max() < 2e-6
        ref_v = d[f"c{case}_visits"]
        assert np.array_equal(v, ref_v), (np.nonzero(v != ref_v), v[v != ref_v], ref_v[v != ref_v])
        assert np.abs(util - d[f"c{case}_util"])[v > 0].max() < 1e-12
        ch, rt = sp.root_value_stats(g)
        assert np.abs(ch - d[f"c{case}_child_stats"])[v > 0].max() < 1e-9 and np.abs(rt - d[f"c{case}_root_stats"]).max() < 1e-9
        psv, ref_psv = sp.play_selection_values(g), d[f"c{case}_play_selection"]
        assert np.array_equal(psv < 0, ref_psv < 0)
        assert np.abs(psv - ref_psv).max() <= 1e-9 * max(1.0, np.abs(ref_psv).max())
    sp.free(); h.free(); ctx.free()
