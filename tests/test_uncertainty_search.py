"""Uncertainty-weighted evaluations and noise pruning (DESIGN.md row a20), the parts that need no GPU: the device loop's short-term error
post-processing and evaluation weight (the same __host__ __device__ code through kgb_test_uncertainty_weight) against a restatement of
the reference's formulas, and the configuration keys through the Python and the C++ loaders and the match commands."""
import json
import os
import subprocess

import numpy as np
import pytest

from katago_b200 import match_cli
from katago_b200 import selfplay_cli as C
from katago_b200.nn_backend import uncertainty_weight

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def reference_loader(tmp_path_factory):
    """tests/cpp/uncertainty_search_driver.cpp (the reference's own configuration loader mapped by integration/b200params.h), built where
    the reference objects and sources are (oracle/Makefile.ref); None elsewhere."""
    if not os.path.exists(os.path.join(ROOT, "oracle", "_ref", "libkgref.a")):
        return None
    import sys
    sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
    import make_uncertainty_fixture as U
    try:
        return U.build_driver(str(tmp_path_factory.mktemp("refloader")))
    except subprocess.CalledProcessError:      # reference sources absent: the objects alone cannot be compiled against
        return None


def _softplus(x):
    return x if x > 40.0 else np.log(1.0 + np.exp(x))


def _errors(version, raw_wl, raw_se, vm, sm):
    """nneval.cpp:1161-1178 and 1217-1226: the errors as NNOutput keeps them (float), -1 below version 9."""
    if version < 9:
        return np.float32(-1.0), np.float32(-1.0)
    if version >= 14:
        a, b = _softplus(raw_wl * 0.5), _softplus(raw_se * 0.5)
        wl, se = np.sqrt(a * a * vm), np.sqrt(b * b * sm)
    elif version >= 10:
        wl, se = np.sqrt(_softplus(raw_wl) * vm), np.sqrt(_softplus(raw_se) * sm)
    else:
        wl, se = _softplus(raw_wl), _softplus(raw_se) * 10.0
    return np.float32(wl), np.float32(se)


def _weight(wl, se, coeff, exponent, max_weight, wlf, sf, df, dscale, center, sqrt_area, score_mean):
    """Search::computeWeightFromNNOutput with getApproxScoreUtilityDerivative and ScoreValue::whiteDScoreValueDScoreSmoothNoDrawAdjust."""
    two_over_pi = 0.63661977236758134308

    def d(score, c, scale):
        adj, s = score - c, scale * sqrt_area
        return s / (s * s + adj * adj) * two_over_pi
    sm = float(np.float32(score_mean))
    u = wlf * float(wl) + (d(sm, 0.0, 2.0) * sf + d(sm, center, dscale) * df) * float(se)
    powered = u if exponent == 1.0 else np.sqrt(u) if exponent == 0.5 else u ** exponent
    return coeff / (powered + coeff / max_weight)


@pytest.mark.parametrize("version", [8, 9, 12, 15])
@pytest.mark.parametrize("exponent", [1.0, 0.5, 0.7])
def test_shortterm_errors_and_weight_match_the_reference_formulas(version, exponent):
    rng = np.random.default_rng(version * 10 + int(exponent * 10))
    n = 64
    raw_wl, raw_se = rng.uniform(-6, 6, n), rng.uniform(-6, 6, n)
    raw_wl[:2] = [45.0, -45.0]                      # both sides of the softplus cut-off
    vm, sm = 0.25, 30.0
    center, score_mean = rng.uniform(-10, 10, n), rng.uniform(-40, 40, n)
    kw = dict(value_error_multiplier=vm, score_error_multiplier=sm, coeff=0.25, exponent=exponent, max_weight=8.0, win_loss_utility_factor=1.0,
              static_score_utility_factor=0.1, dynamic_score_utility_factor=0.3, dynamic_score_center_scale=0.75, sqrt_board_area=13.0)
    wl, se, w = uncertainty_weight(np.full(n, version), raw_wl, raw_se, center=center, white_score_mean=score_mean, **kw)
    for i in range(n):
        ewl, ese = _errors(version, raw_wl[i], raw_se[i], vm, sm)
        assert wl[i] == float(ewl) and se[i] == float(ese), (i, wl[i], ewl, se[i], ese)
        if version >= 9:
            ew = _weight(ewl, ese, 0.25, exponent, 8.0, 1.0, 0.1, 0.3, 0.75, center[i], 13.0, score_mean[i])
            assert abs(w[i] - ew) <= 1e-14 * ew, (i, w[i], ew)
            assert 0.0 < w[i] <= 8.0
    if version < 9:
        assert (wl == -1.0).all() and (se == -1.0).all()


def test_weight_without_score_utility_and_at_zero_error():
    """Only the win/loss term is left with both score factors 0; zero uncertainty gives the maximum weight."""
    _, _, w = uncertainty_weight([15, 15], [-200.0, 2.0], [-200.0, 2.0], coeff=0.25, max_weight=8.0)
    assert w[0] == 8.0
    ewl, _ = _errors(15, 2.0, 2.0, 0.25, 30.0)
    assert abs(w[1] - 0.25 / (float(ewl) + 0.25 / 8.0)) <= 1e-15


GATEKEEPER1_SEARCH = {
    "maxVisits": "150", "numSearchThreads": "1", "nnCacheSizePowerOfTwo": "21", "chosenMoveTemperatureEarly": "0.5", "chosenMoveTemperatureHalflife": "19",
    "chosenMoveTemperature": "0.2", "chosenMoveSubtract": "0", "chosenMovePrune": "1", "useLcbForSelection": "true", "lcbStdevs": "5.0",
    "minVisitPropForLCB": "0.15", "winLossUtilityFactor": "1.0", "staticScoreUtilityFactor": "0.00", "dynamicScoreUtilityFactor": "0.25",
    "dynamicScoreCenterZeroWeight": "0.25", "dynamicScoreCenterScale": "0.50", "noResultUtilityForWhite": "0.0", "drawEquivalentWinsForWhite": "0.5",
    "rootEndingBonusPoints": "0.5", "rootPruneUselessMoves": "true", "cpuctExploration": "1.1", "cpuctExplorationLog": "0.0", "fpuReductionMax": "0.2",
    "rootFpuReductionMax": "0.1", "valueWeightExponent": "0.5", "subtreeValueBiasFactor": "0.35", "subtreeValueBiasWeightExponent": "0.8",
    "useNonBuggyLcb": "true", "useGraphSearch": "true", "useUncertainty": "true", "uncertaintyExponent": "1.0", "uncertaintyCoeff": "0.25",
}
CASES = {
    "gatekeeper1": (GATEKEEPER1_SEARCH, dict(use_uncertainty=True, uncertainty_coeff=0.25, uncertainty_exponent=1.0, uncertainty_max_weight=8.0,
                                             use_noise_pruning=False, noise_prune_utility_scale=0.15, noise_pruning_cap=1e50)),
    "every_key": ({"maxVisits": "100", "numSearchThreads": "1", "useUncertainty": "true", "uncertaintyCoeff": "0.3", "uncertaintyExponent": "0.7",
                   "uncertaintyMaxWeight": "5.5", "useNoisePruning": "true", "noisePruneUtilityScale": "0.2", "noisePruningCap": "3.5"},
                  dict(use_uncertainty=True, uncertainty_coeff=0.3, uncertainty_exponent=0.7, uncertainty_max_weight=5.5, use_noise_pruning=True,
                       noise_prune_utility_scale=0.2, noise_pruning_cap=3.5)),
    "absent": ({"maxVisits": "100", "numSearchThreads": "1"},
               dict(use_uncertainty=False, uncertainty_coeff=0.25, uncertainty_exponent=1.0, uncertainty_max_weight=8.0, use_noise_pruning=False,
                    noise_prune_utility_scale=0.15, noise_pruning_cap=1e50)),
}


@pytest.fixture(scope="module")
def cpp_host(tmp_path_factory):
    exe = tmp_path_factory.mktemp("cpphost") / "b200_selfplay"
    subprocess.run(["g++", "-std=c++17", "-O1", "-Wall", "-Wextra", "-Werror", "-I", ROOT, os.path.join(ROOT, "integration", "b200_selfplay_main.cpp"), "-o", str(exe),
                    "-L", os.path.join(ROOT, "katago_b200"), "-lkgb200", "-lz", "-Wl,-rpath," + os.path.join(ROOT, "katago_b200")], check=True)
    return str(exe)


@pytest.mark.parametrize("which", list(CASES))
def test_uncertainty_and_noise_pruning_keys_map_in_both_loaders(tmp_path, cpp_host, reference_loader, which):
    settings, expected = CASES[which]
    path = tmp_path / "c.cfg"
    path.write_text("".join(f"{k} = {v}\n" for k, v in settings.items()))
    kw, _, report = C.selfplay_kwargs_from_cfg(C.parse_cfg(str(path)))
    mine = json.loads(subprocess.run([cpp_host, "-config", str(path), "-print-config"], capture_output=True, text=True, check=True).stdout)
    for k, v in expected.items():
        assert kw[k] == v, (k, kw[k], v)
        assert float(mine[k]) == float(v), (k, mine[k], v)
    nb = " ".join(report["not_built"])
    assert "useUncertainty" not in nb and "useNoisePruning" not in nb and "uncertainty" not in nb.lower()
    if reference_loader:                # the reference's own loader, mapped by integration/b200params.h
        ref = json.loads(subprocess.run([reference_loader, "paramsmap", str(path)], capture_output=True, text=True, check=True).stdout)
        for k, v in expected.items():
            assert float(ref[k]) == float(v), (k, ref[k], v)
        assert not any("ncertainty" in u or "NoisePruning" in u for u in ref["unsupported"]), ref["unsupported"]


def test_match_keys_per_bot_and_the_default_note():
    cfg = {"numBots": "2", "botName0": "a", "botName1": "b", "maxVisits": "50", "useUncertainty": "false", "useUncertainty1": "true",
           "uncertaintyCoeff1": "0.3", "useNoisePruning0": "true"}
    kws = [C.selfplay_kwargs_from_cfg(match_cli.bot_cfg(cfg, i))[0] for i in range(2)]
    assert kws[0]["use_uncertainty"] is False and kws[1]["use_uncertainty"] is True
    assert kws[0]["uncertainty_coeff"] == 0.25 and kws[1]["uncertainty_coeff"] == 0.3
    assert kws[0]["use_noise_pruning"] is True and kws[1]["use_noise_pruning"] is False
    assert match_cli.match_default_note(cfg) is None
    note = match_cli.match_default_note({"maxVisits": "50"})
    assert "useUncertainty and useNoisePruning not set" in note and "katago match defaults them to true" in note
    assert "useUncertainty = true, useNoisePruning = true" in note
    note = match_cli.match_default_note({"useUncertainty1": "true"})
    assert note.startswith("[config] useNoisePruning not set") and "useUncertainty" not in note


def test_match_commands_log_the_default_note(tmp_path, tmp_models):
    """Both match commands say once that the switches are off when the configuration leaves them out (and then stop: no GPU here)."""
    cfg = tmp_path / "m.cfg"
    cfg.write_text(f"numBots = 2\nbotName0 = a\nbotName1 = b\nnnModelFile = {tmp_models['tiny_reg']}\nnumGamesTotal = 2\nmaxVisits = 10\nbSizes = 9\n")
    exe = os.path.join(ROOT, "katago_b200", "b200_match")
    runs = [subprocess.run(["python", "-m", "katago_b200.match_cli", "-config", str(cfg), "-sgf-output-dir", str(tmp_path / "py")], cwd=ROOT,
                           capture_output=True, text=True, timeout=300)]
    if os.path.exists(exe):
        runs.append(subprocess.run([exe, "-config", str(cfg), "-sgf-output-dir", str(tmp_path / "cpp")], capture_output=True, text=True, timeout=300))
    for r in runs:
        assert r.stderr.count("useUncertainty and useNoisePruning not set: off here") == 1, r.stderr[-2000:]
