"""Uncertainty-weighted evaluations and noise pruning in the device loop's search (DESIGN.md row a20), on the GPU: against the
reference's own Search with the fake net (tests/golden/searchfake_uncertainty.npz, make_uncertainty_fixture.py), with and without
the evaluation cache, and end to end through the gatekeeper with the stock gatekeeper1.cfg search block."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from katago_b200 import NeuralNet, SelfPlay

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BOOL_KEYS = ("fpuParentWeightByVisitedPolicy", "useGraphSearch", "useLcbForSelection", "useNonBuggyLcb", "useUncertainty", "useNoisePruning",
             "rootNoiseEnabled")


def _kwargs(params):
    snake = lambda k: "min_visit_prop_for_lcb" if k == "minVisitPropForLCB" else "".join("_" + c.lower() if c.isupper() else c for c in k)
    return {snake(k): bool(v) if k in BOOL_KEYS else int(v) if k in ("graphSearchRepBound", "rootNumSymmetriesToSample") else float(v)
            for k, v in params.items()}


def _search(d, case, model, cache_pow2=0, games=2):
    X, Y, visits = (int(v) for v in d[f"c{case}_shape"])
    lm = NeuralNet.loadModelFile(model)
    ctx = NeuralNet.createComputeContext([0], X, Y, True, lm)
    h = NeuralNet.createComputeHandle(ctx, lm, 4, False, True, 0)
    sp = SelfPlay(h, games, visits, komi=7.5, multi_stone_suicide_legal=True, early_temperature_moves=0, seed=1,
                  debug_fake_nn=2 if int(d[f"c{case}_fake_shortterm"]) else 1, debug_hold_at_max_visits=True,
                  nn_cache_size_power_of_two=cache_pow2, **_kwargs(json.loads(str(d[f"c{case}_params"]))))
    sp.play_moves([None if m[0] < 0 else (int(m[0]), int(m[1])) for m in d[f"c{case}_moves"]])
    sp.set_search_rand(str(d[f"c{case}_threadseed"]))
    for _ in range(100):
        sp.run(max(8, visits // 8))
        if all(sp.game(g)[1]["root_visits"] >= visits for g in range(games)):
            break
    out = []
    for g in range(games):
        v, _, util = sp.root_children(g)
        assert sp.game(g)[1]["root_visits"] == visits
        out.append((v, util) + sp.root_weights(g))
    sp.free(); h.free(); ctx.free()
    return out


@pytest.fixture(scope="module")
def fixture_and_models(golden_dir, tmp_path_factory):
    sys.path.insert(0, golden_dir)
    import make_uncertainty_fixture as U
    d = np.load(os.path.join(golden_dir, "searchfake_uncertainty.npz"))
    tmp = str(tmp_path_factory.mktemp("uncmodels"))
    return d, {v: U.model_for(v, tmp) for v in (8, 9, 12, 15)}


@pytest.mark.parametrize("case", range(16))
def test_search_with_uncertainty_and_noise_pruning_matches_reference_search(fixture_and_models, case):
    """Root child visit counts identical to the reference Search in every case.  Each switch alone: child utilities to 1e-12, the
    root's and children's weightSum / weightSqSum to 1e-9 relative (noise pruning's 1 - exp(-utilityGap / noisePruneUtilityScale)
    magnifies a last-bit difference between the device's exp and the host's when the gap is small: 3e-10 seen on a root).  Both
    switches together: utilities and weights agree to 1e-7 relative only (up to 1.3e-8 seen); where the larger difference comes
    from is not pinned down yet, the visit counts are unaffected.  Cases with graph search (3, 12) also run with the evaluation
    cache on: the cache holds the short-term errors, so a hit recomputes the same weight."""
    d, models = fixture_and_models
    model = models[int(d[f"c{case}_version"])]
    ref_v, ref_u, ref_w, ref_rw = (d[f"c{case}_{k}"] for k in ("visits", "util", "weights", "root_weights"))
    params = json.loads(str(d[f"c{case}_params"]))
    both = bool(params.get("useUncertainty")) and bool(params.get("useNoisePruning")) and int(d[f"c{case}_version"]) >= 9
    utol, wtol = (1e-7, 1e-7) if both else (1e-12, 1e-9)
    for cache in ((0, 12) if case in (3, 12) else (0,)):
        for v, util, w, rw in _search(d, case, model, cache):
            assert np.array_equal(v, ref_v), (cache, np.nonzero(v != ref_v), v[v != ref_v], ref_v[v != ref_v])
            assert np.abs(util - ref_u)[v > 0].max() < utol, np.abs(util - ref_u)[v > 0].max()
            assert np.abs(w - ref_w)[v > 0].max() < wtol * max(1.0, np.abs(ref_w).max()), np.abs(w - ref_w)[v > 0].max()
            assert np.abs(rw - ref_rw).max() < wtol * max(1.0, np.abs(ref_rw).max()), (rw, ref_rw)
    if int(d[f"c{case}_version"]) >= 9 and params.get("useUncertainty"):
        assert ref_rw[0] != ref_v.sum() + 1       # the weights really act: not one per visit


@pytest.mark.parametrize("switches", ["uncertainty", "pruning", "both"])
def test_games_are_the_same_with_and_without_the_cache(fixture_and_models, switches):
    """With uncertainty weighting and / or noise pruning on, games are move for move the same with the evaluation cache on and off: the
    cache keeps the short-term errors, and the weight is recomputed from them with the search's own score centre.  The hash net with raw
    short-term error channels on a version-15 model (weights act); the board of every game at move 6 is compared (with the cache, playouts
    finish inside the select kernel, so games advance at another pace per wave)."""
    _, models = fixture_and_models
    lm = NeuralNet.loadModelFile(models[15])
    ctx = NeuralNet.createComputeContext([0], 9, 9, True, lm)
    h = NeuralNet.createComputeHandle(ctx, lm, 4, False, True, 0)
    kw = dict(komi=7.5, seed=5, debug_fake_nn=2, early_temperature_moves=3, value_weight_exponent=0.5, use_graph_search=True,
              static_score_utility_factor=0.05, dynamic_score_utility_factor=0.3, dynamic_score_center_zero_weight=0.25,
              dynamic_score_center_scale=0.5, subtree_value_bias_factor=0.3, subtree_value_bias_weight_exponent=0.8,
              use_uncertainty=switches != "pruning", use_noise_pruning=switches != "uncertainty")
    boards, hits = {}, {}
    for cache in (0, 14):
        sp = SelfPlay(h, 4, 80, nn_cache_size_power_of_two=cache, **kw)
        seen = {}
        for _ in range(4000):
            sp.run(1)
            for g in range(4):
                colors, info = sp.game(g)
                if info["move_num"] == 6 and g not in seen:
                    seen[g] = colors.copy()
            if len(seen) == 4:
                break
        assert len(seen) == 4
        boards[cache], hits[cache] = seen, sp.stats()["nn_cache_hits"]
        sp.free()
    h.free(); ctx.free()
    assert hits[14] > 0 and hits[0] == 0
    for g in range(4):
        assert np.array_equal(boards[0][g], boards[14][g]), g


def test_gatekeeper_runs_with_the_stock_gatekeeper1_search_block(tmp_path, golden_dir):
    """gatekeeper_cli.py with the search block of gatekeeper1.cfg (useUncertainty = true): runs clean, says nothing about uncertainty;
    once with the trained g170 net (version 8: weight 1) against itself and once with two random version-15 nets, where the weights act."""
    from katago_b200 import modelgen
    sys.path.insert(0, os.path.dirname(__file__))
    from test_uncertainty_search import GATEKEEPER1_SEARCH
    g170 = os.path.join(golden_dir, "models", "g170-b6c96-s175395328-d26788732.bin.gz")
    pairs = {"g170": (g170, g170)}
    v15 = [modelgen.write_model(str(tmp_path / f"v15_{i}.bin.gz"), "tiny_nbt", seed=40 + i) for i in range(2)]
    pairs["v15"] = tuple(v15)
    for name, (accepted, candidate) in pairs.items():
        base = tmp_path / name
        for sub in ("test", "accepted", "rejected", "sgf", "selfplay"):
            (base / sub).mkdir(parents=True)
        os.makedirs(base / "test" / "cand-s1", exist_ok=True)
        os.symlink(candidate, base / "test" / "cand-s1" / "model.bin.gz")
        os.makedirs(base / "accepted" / "acc-s0", exist_ok=True)
        os.symlink(accepted, base / "accepted" / "acc-s0" / "model.bin.gz")
        cfg = dict(GATEKEEPER1_SEARCH, maxVisits="24", numGamesPerGating="8", numGameThreads="8", bSizes="9", koRules="SIMPLE",
                   maxMovesPerGame="120", nnCacheSizePowerOfTwo="14")
        (base / "g.cfg").write_text("".join(f"{k} = {v}\n" for k, v in cfg.items()))
        r = subprocess.run([sys.executable, "-m", "katago_b200.gatekeeper_cli", "-config", str(base / "g.cfg"), "-test-models-dir", str(base / "test"),
                            "-accepted-models-dir", str(base / "accepted"), "-rejected-models-dir", str(base / "rejected"),
                            "-sgf-output-dir", str(base / "sgf"), "-selfplay-dir", str(base / "selfplay"), "-quit-if-no-nets-to-test",
                            "-no-autoreject-old-models", "-games-per-gpu", "8"],
                           cwd=ROOT, capture_output=True, text=True, timeout=900)
        assert r.returncode == 0, r.stderr[-3000:]
        assert "ncertainty" not in r.stderr and "NoisePruning" not in r.stderr, r.stderr[-3000:]
        print(name, r.stderr.strip().splitlines()[-1])
