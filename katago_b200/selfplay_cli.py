"""`python -m katago_b200.selfplay_cli` - the reference's `katago selfplay` command (command/selfplay.cpp) on the device loop
(SURVEY.md §8f row 3, first slice).

    python -m katago_b200.selfplay_cli -models-dir DIR -output-dir DIR -config selfplay.cfg [-max-games-total N]
                                       [-override-config "key=value,key=value"] [-games-per-gpu N] [-strict]

Same arguments and the same output layout as the reference (`<output-dir>/<model name>/tdata/<16 hex>.npz` and `.../sgfs/<16 hex>.sgfs`,
selfplay.cpp:177-225),
and it reads the reference's own .cfg files: every search / rules / data key the device loop implements is mapped to its
`kgb_selfplay_config` field (`selfplay_kwargs_from_cfg`), every other key is reported - either as irrelevant here (logging, thread
and device placement of the reference's CPU threads) or as NOT BUILT (options that change the data distribution: forks, cheap
searches, handicap games, ...).  `-strict` turns the second group into an error.

The reference randomises rules, board size and komi per game (GameInitializer); the device loop takes them per game slot
(kgb_selfplay_set_game_setup / set_komi), so list-valued
keys (`koRules`, `bSizes`, ...) are drawn per game like the reference does (game_initializer.py); values the loop lacks are left out (reported).
Under torchrun (one process per GPU) the ranks split `-max-games-total`, use LOCAL_RANK's GPU and their own seeds, and write into the
same tdata directory (`shard_plan`); there is no collective on this path.
There is no CPU fallback: without an H100 the command fails when it creates the evaluator."""
import argparse
import glob
import os
import sys

# reference key -> (SelfPlay keyword, converter)
_B = lambda s: s.strip().lower() in ("true", "1", "yes")
_SEARCH_KEYS = {
    "maxVisits": ("max_visits", int),
    "cpuctExploration": ("cpuct_exploration", float), "cpuctExplorationLog": ("cpuct_exploration_log", float),
    "cpuctExplorationBase": ("cpuct_exploration_base", float), "fpuReductionMax": ("fpu_reduction_max", float),
    "rootFpuReductionMax": ("root_fpu_reduction_max", float), "fpuLossProp": ("fpu_loss_prop", float), "rootFpuLossProp": ("root_fpu_loss_prop", float),
    "fpuParentWeight": ("fpu_parent_weight", float), "fpuParentWeightByVisitedPolicy": ("fpu_parent_weight_by_visited_policy", _B),
    "fpuParentWeightByVisitedPolicyPow": ("fpu_parent_weight_by_visited_policy_pow", float), "valueWeightExponent": ("value_weight_exponent", float),
    "cpuctUtilityStdevPrior": ("cpuct_utility_stdev_prior", float), "cpuctUtilityStdevPriorWeight": ("cpuct_utility_stdev_prior_weight", float),
    "cpuctUtilityStdevScale": ("cpuct_utility_stdev_scale", float), "rootDesiredPerChildVisitsCoeff": ("root_desired_per_child_visits_coeff", float),
    "subtreeValueBiasFactor": ("subtree_value_bias_factor", float), "subtreeValueBiasWeightExponent": ("subtree_value_bias_weight_exponent", float),
    "useGraphSearch": ("use_graph_search", _B), "graphSearchRepBound": ("graph_search_rep_bound", int),
    "rootNoiseEnabled": ("root_noise_enabled", _B), "rootDirichletNoiseTotalConcentration": ("root_dirichlet_noise_total_concentration", float),
    "rootDirichletNoiseWeight": ("root_dirichlet_noise_weight", float), "rootPolicyTemperature": ("root_policy_temperature", float),
    "rootPolicyTemperatureEarly": ("root_policy_temperature_early", float), "chosenMoveTemperature": ("chosen_move_temperature", float),
    "chosenMoveTemperatureEarly": ("chosen_move_temperature_early", float), "chosenMoveTemperatureHalflife": ("chosen_move_temperature_halflife", float),
    "chosenMoveTemperatureOnlyBelowProb": ("chosen_move_temperature_only_below_prob", float),
    "chosenMoveSubtract": ("chosen_move_subtract", float), "chosenMovePrune": ("chosen_move_prune", float),
    "useLcbForSelection": ("use_lcb_for_selection", _B), "lcbStdevs": ("lcb_stdevs", float), "minVisitPropForLCB": ("min_visit_prop_for_lcb", float),
    "useNonBuggyLcb": ("use_non_buggy_lcb", _B), "winLossUtilityFactor": ("win_loss_utility_factor", float),
    "staticScoreUtilityFactor": ("static_score_utility_factor", float), "dynamicScoreUtilityFactor": ("dynamic_score_utility_factor", float),
    "dynamicScoreCenterZeroWeight": ("dynamic_score_center_zero_weight", float), "dynamicScoreCenterScale": ("dynamic_score_center_scale", float),
    "noResultUtilityForWhite": ("no_result_utility_for_white", float), "drawEquivalentWinsForWhite": ("draw_equivalent_wins_for_white", float),
    "rootNumSymmetriesToSample": ("root_num_symmetries_to_sample", int), "nnCacheSizePowerOfTwo": ("nn_cache_size_power_of_two", int),
    "maxMovesPerGame": ("max_moves", int),
    "rootEndingBonusPoints": ("root_ending_bonus_points", float), "rootPruneUselessMoves": ("root_prune_useless_moves", _B),
    "useUncertainty": ("use_uncertainty", _B), "uncertaintyCoeff": ("uncertainty_coeff", float),
    "uncertaintyExponent": ("uncertainty_exponent", float), "uncertaintyMaxWeight": ("uncertainty_max_weight", float),
    "useNoisePruning": ("use_noise_pruning", _B), "noisePruneUtilityScale": ("noise_prune_utility_scale", float),
    "noisePruningCap": ("noise_pruning_cap", float),
}
# keys that only place or log the reference's own CPU threads / evaluator servers: nothing to do here
_IRRELEVANT_PREFIXES = ("log", "cuda", "trt", "opencl", "eigen", "metal", "numNNServerThreads", "nnMaxBatchSize", "nnMutexPool", "numSearchThreads",
                        "maxDataQueueSize", "nnRandomize", "numVirtualLossesPerThread", "gpuToUse", "homeDataDir")
# neutral values: the option is switched off, so not having it changes nothing
_NEUTRAL = {"sekiForkHackProb": 0.0,
            "handicapAsymmetricPlayoutProb": 0.0, "normalAsymmetricPlayoutProb": 0.0,
            "switchNetsMidGame": True, "fancyKomiVarying": False,
            "handicapProb": 0.0,
            "drawRandRadius": 0.0, "noResultStdev": 0.0, "compensateAfterPolicyInitProb": 0.0}
_REFERENCE_DEFAULTS = {
    "cpuct_exploration": 1.0, "cpuct_exploration_log": 0.45, "cpuct_exploration_base": 500.0, "fpu_reduction_max": 0.2, "root_fpu_reduction_max": 0.1,
    "win_loss_utility_factor": 1.0, "no_result_utility_for_white": 0.0, "static_score_utility_factor": 0.1, "dynamic_score_utility_factor": 0.3,
    "dynamic_score_center_zero_weight": 0.2, "dynamic_score_center_scale": 0.75, "draw_equivalent_wins_for_white": 0.5, "value_weight_exponent": 0.25,
    "fpu_parent_weight_by_visited_policy": True, "fpu_parent_weight_by_visited_policy_pow": 2.0, "fpu_parent_weight": 0.0, "fpu_loss_prop": 0.0,
    "root_fpu_loss_prop": 0.0, "cpuct_utility_stdev_prior": 0.40, "cpuct_utility_stdev_prior_weight": 2.0, "cpuct_utility_stdev_scale": 0.0,
    "root_desired_per_child_visits_coeff": 0.0, "subtree_value_bias_factor": 0.45, "subtree_value_bias_weight_exponent": 0.85, "use_graph_search": True,
    "graph_search_rep_bound": 11, "root_noise_enabled": False, "root_dirichlet_noise_total_concentration": 10.83, "root_dirichlet_noise_weight": 0.25,
    "root_policy_temperature": 1.0, "root_policy_temperature_early": 1.0, "chosen_move_temperature_halflife": 19.0, "use_lcb_for_selection": True,
    "use_non_buggy_lcb": False, "lcb_stdevs": 5.0, "min_visit_prop_for_lcb": 0.15, "chosen_move_temperature": 0.10, "chosen_move_temperature_early": 0.50,
    "chosen_move_temperature_only_below_prob": 1.0, "chosen_move_subtract": 0.0, "chosen_move_prune": 1.0, "nn_cache_size_power_of_two": 0,
    "root_num_symmetries_to_sample": 1, "root_ending_bonus_points": 0.5, "root_prune_useless_moves": True,
    "use_uncertainty": False, "uncertainty_coeff": 0.25, "uncertainty_exponent": 1.0, "uncertainty_max_weight": 8.0,
    "use_noise_pruning": False, "noise_prune_utility_scale": 0.15, "noise_pruning_cap": 1e50,
}
# options the reference switches ON by default and the loop does not have: reported even when the key is absent (none at present)
_DEFAULT_ON_NOT_BUILT = {}
_KO_RULES = {"SIMPLE": 0, "POSITIONAL": 1, "SITUATIONAL": 2, "SPIGHT": 3}


def parse_cfg(path_or_text, is_text=False):
    """KataGo .cfg: `key = value` lines, `#` comments (core/config_parser.cpp).  `@include` is not supported.  Later keys win."""
    text = path_or_text if is_text else open(path_or_text).read()
    out = {}
    for n, raw in enumerate(text.splitlines(), 1):
        line = raw.split("#", 1)[0].strip()
        if not line:
            continue
        if line.startswith("@"):
            raise ValueError(f"line {n}: '{line.split()[0]}' directives are not supported")
        if "=" not in line:
            raise ValueError(f"line {n}: expected 'key = value', got {raw!r}")
        k, v = line.split("=", 1)
        out[k.strip()] = v.strip()
    return out


def _supported_values(cfg, key, supported, report, default):
    """The values of a list-valued key that the loop can play, in the order listed.  The reference draws one per game (GameInitializer,
    program/play.cpp:83-650) and so does this command (katago_b200/game_initializer.py); values the loop does not have are left out of
    the draw and named under "fixed"."""
    if key not in cfg:
        return [default]
    vals = [v.strip() for v in cfg[key].split(",") if v.strip()]
    ok = [v for v in vals if v.upper() in supported or v.lower() in supported]
    if not ok:
        raise ValueError(f"{key} = {cfg[key]}: none of these is built (supported: {sorted(supported)}); pass an explicit single value")
    dropped = [v for v in vals if v not in ok]
    if dropped:
        report["fixed"].append(f"{key}: the reference draws one of [{cfg[key]}] per game; {', '.join(dropped)} not built, this loop draws from [{', '.join(ok)}]")
    return ok


def selfplay_kwargs_from_cfg(cfg, strict=False):
    """(kwargs for nn_backend.SelfPlay, data settings, report) from a parsed reference .cfg.
    report: {"mapped": [...], "irrelevant": [...], "fixed": [...], "not_built": [...]}."""
    report = {"mapped": [], "irrelevant": [], "fixed": [], "not_built": []}
    kw = {}
    used = set()
    for key, (name, conv) in _SEARCH_KEYS.items():
        if key in cfg:
            kw[name] = conv(cfg[key])
            used.add(key); report["mapped"].append(key)
    # Keys that are absent get the defaults of the reference's own loader (Setup::loadParams, program/setup.cpp, as a self-play
    # command sees them), not the loop's: tests/test_selfplay_cli.py compares both loaders on the same files.
    by_policy = kw.get("fpu_parent_weight_by_visited_policy", True)
    if by_policy:        # setup.cpp:501-513: the power is read only with the flag, the plain weight only without it
        kw.pop("fpu_parent_weight", None)
    else:
        kw.pop("fpu_parent_weight_by_visited_policy_pow", None)
    # three defaults follow other keys (setup.cpp:575-583): the early root temperature the plain one, the root's fpu loss proportion the tree's,
    # and the root fpu reduction is 0 once root noise is on
    if "root_policy_temperature" in kw:
        kw.setdefault("root_policy_temperature_early", kw["root_policy_temperature"])
    if "fpu_loss_prop" in kw:
        kw.setdefault("root_fpu_loss_prop", kw["fpu_loss_prop"])
    if kw.get("root_noise_enabled", False):
        kw.setdefault("root_fpu_reduction_max", 0.0)
    for name, ref_default in _REFERENCE_DEFAULTS.items():
        kw.setdefault(name, ref_default)
    if not by_policy:
        kw["fpu_parent_weight_by_visited_policy_pow"] = 1.0
    kw["use_play_selection"] = True                       # Search::getChosenMoveLoc always goes through the play selection values
    # rules, board size and komi: drawn per game like the reference's GameInitializer does (game_initializer.py); the loop's own
    # configuration carries the first listed ko / suicide rule as its default
    kos = [_KO_RULES[v.upper()] for v in _supported_values(cfg, "koRules", set(_KO_RULES), report, "SIMPLE")]
    kw["ko_rule"] = kos[0]
    _supported_values(cfg, "scoringRules", {"AREA"}, report, "AREA")
    _supported_values(cfg, "taxRules", {"NONE"}, report, "NONE")
    _supported_values(cfg, "hasButtons", {"false"}, report, "false")
    suicides = [_B(v) for v in _supported_values(cfg, "multiStoneSuicideLegals", {"false", "true"}, report, "true")]
    kw["multi_stone_suicide_legal"] = suicides[0]
    edges = [int(v) for v in _supported_values(cfg, "bSizes", {str(s) for s in range(2, 20)}, report, "19")]
    all_edges = [v.strip() for v in cfg.get("bSizes", "19").split(",") if v.strip()]
    rel = [float(v) for v in cfg["bSizeRelProbs"].split(",") if v.strip()] if "bSizeRelProbs" in cfg else [1.0] * len(all_edges)
    if len(rel) != len(all_edges):
        raise ValueError(f"bSizeRelProbs has {len(rel)} entries, bSizes has {len(all_edges)}")
    rel = [pr for v, pr in zip(all_edges, rel) if v in {str(e) for e in edges}]
    from .game_initializer import board_size_distribution
    sizes, size_probs = board_size_distribution(edges, rel, float(cfg.get("allowRectangleProb", 0.0)))
    size = max(edges)                                     # the evaluator's frame holds the largest board
    used.update(("koRules", "scoringRules", "taxRules", "hasButtons", "multiStoneSuicideLegals", "bSizes", "bSizeRelProbs", "allowRectangleProb"))
    komi = float(cfg["komiMean"]) if "komiMean" in cfg else 7.5
    used.update(("komiMean", "komiAuto", "komiStdev", "komiBigStdevProb", "komiBigStdev", "komiBiggerStdevProb", "komiBiggerStdev", "komiAllowIntegerProb"))
    # komiAuto (fair komi of the empty board found by search, play.cpp:1563-1575) and lead targets (play.cpp:2290-2324): komi-bisection searches
    # on a side loop (komi_search.py)
    komi_search = dict(komi_auto=_B(cfg.get("komiAuto", "false")), compensate_komi_visits=int(cfg.get("compensateKomiVisits", 20)),
                       estimate_lead_prob=float(cfg.get("estimateLeadProb", 0.0)), estimate_lead_visits=int(cfg.get("estimateLeadVisits", 6)))
    used.update(("compensateKomiVisits", "estimateLeadProb", "estimateLeadVisits"))
    data = {"board_size": size, "komi": komi,
            "data_board_len": int(cfg.get("dataBoardLen", size)), "max_rows_per_train_file": int(cfg.get("maxRowsPerTrainFile", 20000)),
            "first_file_rand_min_prop": float(cfg.get("firstFileRandMinProp", 1.0)), "num_game_threads": int(cfg.get("numGameThreads", 256))}
    data["komi_search"] = komi_search
    # forked games (Play::maybeForkGame, play.cpp:2413-2508; fork_play.py)
    data["forks"] = dict(early_fork_game_prob=float(cfg.get("earlyForkGameProb", 0.0)), early_fork_game_expected_move_prop=float(cfg.get("earlyForkGameExpectedMoveProp", 0.0)),
                         fork_game_prob=float(cfg.get("forkGameProb", 0.0)), fork_game_min_choices=int(cfg.get("forkGameMinChoices", 1)),
                         early_fork_game_max_choices=int(cfg.get("earlyForkGameMaxChoices", 1)), fork_game_max_choices=int(cfg.get("forkGameMaxChoices", 1)),
                         fork_compensate_komi_prob=float(cfg.get("forkCompensateKomiProb", cfg.get("handicapCompensateKomiProb", 0.0))))
    data["side_position_prob"] = float(cfg.get("forkSidePositionProb", 0.0))      # PlaySettings::sidePositionProb (playsettings.cpp: cfg key forkSidePositionProb)
    used.add("forkSidePositionProb")
    used.update(("earlyForkGameProb", "earlyForkGameExpectedMoveProp", "forkGameProb", "forkGameMinChoices", "earlyForkGameMaxChoices", "forkGameMaxChoices",
                 "forkCompensateKomiProb", "handicapCompensateKomiProb"))
    data["game_init"] = dict(sizes=sizes, size_probs=size_probs, ko_rules=kos, multi_stone_suicide_legals=suicides, komi_mean=komi,
                             komi_stdev=float(cfg.get("komiStdev", 0.0)), komi_big_stdev_prob=float(cfg.get("komiBigStdevProb", 0.0)),
                             komi_big_stdev=float(cfg.get("komiBigStdev", 10.0)), komi_bigger_stdev_prob=float(cfg.get("komiBiggerStdevProb", 0.0)),
                             komi_bigger_stdev=float(cfg.get("komiBiggerStdev", 30.0)), komi_allow_integer_prob=float(cfg.get("komiAllowIntegerProb", 1.0)))
    used.update(("dataBoardLen", "maxRowsPerTrainFile", "firstFileRandMinProp", "numGameThreads"))
    # PlaySettings the recorder implements (program/playsettings.cpp): surprise weighting of the finished game's rows
    data["policy_surprise_data_weight"] = float(cfg.get("policySurpriseDataWeight", 0.0))
    data["value_surprise_data_weight"] = float(cfg.get("valueSurpriseDataWeight", 0.0))
    data["use_search_value_surprise"] = _B(cfg.get("useSearchValueSurprise", "false"))
    used.update(("policySurpriseDataWeight", "valueSurpriseDataWeight", "useSearchValueSurprise"))
    # search limits per move (getSearchLimitsThisMove, program/play.cpp:1093-1223): cheap searches and reduced visits, drawn by the recorder
    data["play_settings"] = dict(
        cheap_search_prob=float(cfg.get("cheapSearchProb", 0.0)), cheap_search_visits=int(cfg.get("cheapSearchVisits", 0)),
        cheap_search_target_weight=float(cfg.get("cheapSearchTargetWeight", 0.0)), reduce_visits=_B(cfg.get("reduceVisits", "false")),
        reduce_visits_threshold=float(cfg.get("reduceVisitsThreshold", 100.0)), reduce_visits_threshold_lookback=int(cfg.get("reduceVisitsThresholdLookback", 1)),
        reduced_visits_min=int(cfg.get("reducedVisitsMin", 0)), reduced_visits_weight=float(cfg.get("reducedVisitsWeight", 1.0)))
    used.update(("cheapSearchProb", "cheapSearchVisits", "cheapSearchTargetWeight", "reduceVisits", "reduceVisitsThreshold", "reduceVisitsThresholdLookback",
                 "reducedVisitsMin", "reducedVisitsWeight"))
    # policy-initialised openings (initializeGameUsingPolicy): the device draws the moves, the host the count per game
    data["policy_init"] = dict(enabled=_B(cfg.get("initGamesWithPolicy", "false")), area_prop=float(cfg.get("policyInitAreaProp", 0.04)),
                               temperature=float(cfg.get("policyInitAreaTemperature", 1.0)))
    used.update(("initGamesWithPolicy", "policyInitAreaProp", "policyInitAreaTemperature"))
    if data["policy_init"]["enabled"] and float(cfg.get("compensateAfterPolicyInitProb", 0.0)) > 0:
        pass          # reported below through _NEUTRAL (komi compensation after the opening needs searches before the game: not built)
    if data["play_settings"]["cheap_search_prob"] > 0 and data["play_settings"]["cheap_search_target_weight"] <= 0:
        report["fixed"].append("cheapSearchProb: the reference keeps the previous move's tree for cheap searches it does not record; this loop starts every move on a cleared tree")
    if data["data_board_len"] < size:
        raise ValueError(f"dataBoardLen = {data['data_board_len']} but bSizes goes up to {size}: the data frame must hold the largest board")
    data["board_size"] = size = data["data_board_len"]    # rows are written in the data frame, so the evaluator's frame is that (nnXLen = dataBoardLen)
    for key, val in cfg.items():
        if key in used or key in ("numGamesPerGating", "numGamesTotal", "numBots", "allowResignation", "resignThreshold", "resignConsecTurns"):   # read by the gatekeeper / match commands themselves
            continue
        if key.startswith(_IRRELEVANT_PREFIXES):
            report["irrelevant"].append(key)
            continue
        neutral = _NEUTRAL.get(key, None)
        if neutral is not None:
            cur = _B(val) if isinstance(neutral, bool) else float(val)
            if cur == neutral:
                continue
        report["not_built"].append(f"{key} = {val}")
    for key, val in _DEFAULT_ON_NOT_BUILT.items():
        if key not in cfg:
            report["not_built"].append(f"{key} = {val} (the reference's default)")
    if strict and report["not_built"]:
        raise ValueError("options that are not built: " + "; ".join(report["not_built"]))
    return kw, data, report


class SlotSetups:
    """Host side of the per-game setup: draws from a GameInitializer and hands them to the loop (SelfPlay.set_game_setup / set_komi)."""

    def __init__(self, init, num_games, policy_init=None, fair_komi=None, forks=None, searcher=None):
        self.init, self.n = init, num_games
        self.fair_komi = fair_komi            # KomiSearcher for komiAuto, or None
        self.forks, self.searcher = forks, searcher      # fork_play.ForkManager and the side loop its komi compensation runs on
        self.fork_next = [None] * num_games   # the forked position the slot's NEXT game starts from (its setup and komi are the ones handed over)
        self.serial = [0] * num_games
        self.policy_init = policy_init if policy_init and policy_init.get("enabled") and policy_init.get("area_prop", 0) > 0 else None
        self.setups, self.komis = init.draw_many(num_games)
        self.openings = self._openings(self.setups)

    def _opening_len(self, x, y):
        """numInitialMovesToPlay (playutils.cpp:243-250, gamma shape 1): floor of an exponential with mean area * policyInitAreaProp."""
        import math
        return int(math.floor(self.init.rand.expovariate(1.0) * x * y * self.policy_init["area_prop"])) if self.policy_init else 0

    def _openings(self, setups):
        import numpy as np
        return np.array([self._opening_len(int(q[0]), int(q[1])) for q in setups], np.int32)

    def start(self, sp):
        """A fresh loop: the drawn values become the games in progress (none has started), new ones are drawn for the games after them."""
        sp.set_game_setup(self.setups, also_current_games=True)
        sp.set_komi(self.komis, also_current_games=True)
        if self.policy_init:
            sp.set_policy_init(self.openings, self.policy_init["temperature"], also_current_games=True)
        self.setups, self.komis = self.init.draw_many(self.n)
        self.openings = self._openings(self.setups)
        sp.set_game_setup(self.setups)
        sp.set_komi(self.komis)
        if self.policy_init:
            sp.set_policy_init(self.openings, self.policy_init["temperature"])
        if self.fair_komi is not None:
            for slot in range(self.n):
                self._ask_fair_komi(sp, slot)

    def _ask_fair_komi(self, sp, slot):
        """komiAuto: the komi at which the net calls the empty board of the slot's NEXT game even (makeGameFairForEmptyBoard, play.cpp:1563-1575)
        becomes the mean the komi noise is drawn around.  Searched on the side loop while the slot's current game is played; the answer
        replaces the komi handed over so far (drawn around komiMean) unless that game has started meanwhile."""
        from .komi_search import adjust_komi_to_even
        x, y, ko, suicide = (int(v) for v in self.setups[slot])
        self.serial[slot] += 1
        serial = self.serial[slot]

        def done(fair):
            if self.serial[slot] != serial:
                return
            self.komis[slot] = self.init.draw_komi(x, y, mean=fair)
            sp.set_komi(self.komis)
        self.fair_komi.submit(adjust_komi_to_even(self.init.komi_mean, x, y, self.init.rand), (x, y, ko, suicide), [], done)

    def game_started(self, sp, rec, slot):
        """The slot's next game has begun on the device (empty board, the setup handed over): if it is a forked game, play the fork's moves into the
        slot and tell the recorder; then draw for the game after it."""
        fork, self.fork_next[slot] = self.fork_next[slot], None
        if fork is not None:
            sp.play_moves_game(slot, [None if m[0] < 0 else m for m in fork["moves"]])
            rec.start_from(slot, fork["moves"], mode=2)
        self.redraw(sp, slot)

    def redraw(self, sp, slot):
        fork = self.forks.pop() if self.forks is not None else None
        if fork is not None:
            # GameInitializer's initialPosition branch (play.cpp:497-526): the forked game's board, rules and komi, komi noise redrawn around it,
            # with probability forkCompensateKomiProb first adjusted to even at the forked position; no policy-initialised opening
            x, y, ko, suicide = fork["setup"]
            self.serial[slot] += 1
            self.setups[slot] = (x, y, ko, suicide)
            self.komis[slot] = self.init.draw_komi(x, y, mean=fork["komi"])
            self.fork_next[slot] = fork
            if self.searcher is not None and self.init.rand.random() < float(self.forks.s.get("fork_compensate_komi_prob", 0.0)):
                from .komi_search import adjust_komi_to_even
                serial = self.serial[slot]

                def done(fair, slot=slot, x=x, y=y):
                    if self.serial[slot] == serial and self.fork_next[slot] is fork:
                        self.komis[slot] = self.init.draw_komi(x, y, mean=fair)
                        sp.set_komi(self.komis)
                self.searcher.submit(adjust_komi_to_even(fork["komi"], x, y, self.init.rand), fork["setup"], fork["moves"], done)
            sp.set_game_setup(self.setups)
            sp.set_komi(self.komis)
            if self.policy_init:
                self.openings[slot] = 0
                sp.set_policy_init(self.openings, self.policy_init["temperature"])
            return
        x, y, ko, suicide, komi = self.init.draw()
        self.setups[slot] = (x, y, ko, suicide)
        self.komis[slot] = komi
        if self.fair_komi is not None:
            self._ask_fair_komi(sp, slot)
        sp.set_game_setup(self.setups)
        sp.set_komi(self.komis)
        if self.policy_init:
            self.openings[slot] = self._opening_len(x, y)
            sp.set_policy_init(self.openings, self.policy_init["temperature"])


def _game_hash(seed, slot, index):
    """FinishedGameData::gameHash: 128 bits that identify the game (two draws of the game's Rand in the reference).  splitmix64 of
    (seed, slot, index), so ranks and slots never repeat one."""
    def mix(z):
        z = (z + 0x9E3779B97F4A7C15) & (2 ** 64 - 1)
        z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & (2 ** 64 - 1)
        z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & (2 ** 64 - 1)
        return z ^ (z >> 31)
    a = mix(mix(seed & (2 ** 64 - 1)) ^ (slot << 32) ^ index)
    return a, mix(a)


def newest_model(models_dir):
    """The reference polls the models dir for the newest net (command/selfplay.cpp:150-176); this takes the newest once."""
    files = [f for ext in ("*.bin.gz", "*.bin", "*.txt.gz", "*.txt") for f in glob.glob(os.path.join(models_dir, ext))]
    files += [f for f in glob.glob(os.path.join(models_dir, "*", "model.bin.gz"))]
    if not files:
        raise FileNotFoundError(f"no model file in {models_dir}")
    return max(files, key=os.path.getmtime)


def shard_plan(rank, world_size, max_games_total, seed):
    """One process per GPU (torchrun): games are independent, so ranks share nothing - each plays its own games on its own GPU with its
    own seeds and writes its own files into the common tdata directory (names come from the writer's Rand, so they must not collide).
    Returns (games this rank should finish, loop seed, writer seed string)."""
    if not (0 <= rank < world_size):
        raise ValueError("rank out of range")
    games = 0 if max_games_total <= 0 else max_games_total // world_size + (1 if rank < max_games_total % world_size else 0)
    return games, seed * 1000003 + rank, f"selfplay{seed}:rank{rank}of{world_size}"


class SgfSink:
    """<model dir>/sgfs/<16 hex>.sgfs: one game record per line, like the reference's self-play (command/selfplay.cpp:178, 225;
    program/selfplaymanager.cpp:377)."""

    def __init__(self, sgf_dir, name_seed, b_name, w_name):
        from .npz_writer import RowRand
        os.makedirs(sgf_dir, exist_ok=True)
        r = RowRand(name_seed)
        lo, hi = r.next_uint(), r.next_uint()
        self.path = os.path.join(sgf_dir, "%016X.sgfs" % (lo | (hi << 32)))
        self.b_name, self.w_name, self.count = b_name, w_name, 0

    def add(self, slot, data):
        from .npz_writer import write_sgf
        with open(self.path, "a") as f:
            f.write(write_sgf(data, self.b_name, self.w_name) + "\n")
        self.count += 1


def model_name_of(model_path):
    return os.path.basename(os.path.dirname(model_path)) if os.path.basename(model_path) == "model.bin.gz" else os.path.basename(model_path).split(".")[0]


class ModelOutputs:
    """<output-dir>/<model name>/{tdata,sgfs}: one writer per net, as the reference keeps one per NNEvaluator (selfplay.cpp:178-225).
    switch_to() closes the files of the previous net and opens the new net's."""

    def __init__(self, output_dir, data, board_len, writer_seed, writer_cls):
        self.output_dir, self.data, self.L, self.writer_seed, self.writer_cls = output_dir, data, board_len, writer_seed, writer_cls
        self.writer = self.sgfs = self.model_name = None
        self.rows_total, self.dirs, self.generation = 0, [], 0

    def switch_to(self, model_path):
        self.close()
        self.model_name = model_name_of(model_path)
        tdata = os.path.join(self.output_dir, self.model_name, "tdata")
        os.makedirs(tdata, exist_ok=True)
        seed = self.writer_seed if self.generation == 0 else f"{self.writer_seed}:net{self.generation}"
        self.writer = self.writer_cls(tdata, self.data["max_rows_per_train_file"], self.data["first_file_rand_min_prop"], self.L, seed)
        self.sgfs = SgfSink(os.path.join(self.output_dir, self.model_name, "sgfs"), seed + ":sgfs", self.model_name, self.model_name)
        self.dirs.append(tdata)
        self.generation += 1

    def add_game(self, slot, data):
        self.writer.write_game(data)
        self.sgfs.add(slot, data)

    def close(self):
        if self.writer is not None:
            self.writer.flush_if_nonempty()
            self.rows_total += self.writer.row_count
            self.writer = None


class BackgroundStage:
    """Loads a model file and stages it into a live handle (ComputeHandle.stage_weights) on a side thread."""

    def __init__(self, handle, path, more_handles=()):
        import threading
        self.path, self.error = path, None

        def work():
            try:
                from .nn_backend import NeuralNet
                lm = NeuralNet.loadModelFile(path)
                try:
                    handle.stage_weights(lm)
                    for hx in more_handles:          # the side loops of the komi searches play the same net
                        hx.stage_weights(lm)
                finally:
                    lm.free()
            except Exception as e:      # reported by the loop
                self.error = e
        self._t = threading.Thread(target=work, daemon=True)
        self._t.start()

    def done(self):
        return not self._t.is_alive()


class ModelPoller:
    """The models directory is looked at every `seconds` (the reference: 20, selfplay.cpp:336-352); poll() returns the path of a net
    that is newer than the one in use, once."""

    def __init__(self, models_dir, current, seconds):
        import time
        self.models_dir, self.current, self.seconds, self._clock = models_dir, current, seconds, time.monotonic
        self.next = self._clock() + seconds
        self.previous = current

    def forget(self, path):
        """`path` could not be used: report it again at a later poll."""
        if self.current == path:
            self.current = self.previous

    def poll(self, force=False):
        if not force and self._clock() < self.next:
            return None
        self.next = self._clock() + self.seconds
        try:
            newest = newest_model(self.models_dir)
        except FileNotFoundError:
            return None
        if newest == self.current or os.path.getmtime(newest) <= os.path.getmtime(self.current):
            return None
        self.previous, self.current = self.current, newest
        return newest


def main(argv=None):
    ap = argparse.ArgumentParser(prog="katago_b200.selfplay_cli", description="Self-play data generation on the H100 device loop", prefix_chars="-")
    ap.add_argument("-models-dir", required=True)
    ap.add_argument("-output-dir", required=True)
    ap.add_argument("-config", required=True)
    ap.add_argument("-max-games-total", type=int, default=0, help="stop after this many finished games (0 = run until interrupted)")
    ap.add_argument("-override-config", default="", help="key=value,key=value")
    ap.add_argument("-games-per-gpu", type=int, default=256, help="concurrent games (the evaluator batch); numGameThreads is capped by it")
    ap.add_argument("-strict", action="store_true", help="fail if the config asks for an option that is not built")
    ap.add_argument("-seed", type=int, default=0)
    ap.add_argument("-per-game-release", action="store_true", help="record and release every game as soon as its own search is finished "
                    "(GameRecorder.pump) instead of moving all games in lockstep")
    ap.add_argument("-max-playouts-per-wave", type=int, default=4, help="playouts a game may finish inside one wave without needing the evaluator (cache hits, "
                    "graph-search catch-ups); the wave lasts as long as its slowest game, so the bound keeps one long descent from holding up "
                    "the others; results do not depend on it")
    ap.add_argument("-model-poll-seconds", type=float, default=20.0, help="how often the models directory is checked for a newer net")
    ap.add_argument("-nccl-weights", action="store_true", help="under torchrun: rank 0 alone polls and reads new nets, the packed weights reach the other GPUs by ncclBroadcast")
    ap.add_argument("-model-poll-waves", type=int, default=64, help="with -nccl-weights: recorder iterations between two (collective) polls")
    a = ap.parse_args(argv)
    cfg = parse_cfg(a.config)
    for kv in [s for s in a.override_config.split(",") if s.strip()]:
        k, v = kv.split("=", 1)
        cfg[k.strip()] = v.strip()
    kw, data, report = selfplay_kwargs_from_cfg(cfg, strict=a.strict)
    import time
    log = lambda msg: print(msg, file=sys.stderr, flush=True)          # the reference's own log lines (command/selfplay.cpp, program/selfplaymanager.cpp)
    log("Self Play Engine starting...")
    t_start = time.time()
    log_games_every = int(cfg.get("logGamesEvery", 50))
    for line in report["fixed"]:
        print("[config] " + line, file=sys.stderr)
    if report["not_built"]:
        print("[config] NOT BUILT, ignored: " + "; ".join(report["not_built"]), file=sys.stderr)

    from .nn_backend import KGBError, NeuralNet, SelfPlay          # loads libkgb200; fails loudly without an H100
    from .npz_writer import RowRand, TrainingDataWriter
    from .game_recorder import GameRecorder
    model_path = newest_model(a.models_dir)
    L = data["board_size"]
    games = min(a.games_per_gpu, data["num_game_threads"])
    rank, world, gpu = int(os.environ.get("RANK", "0")), int(os.environ.get("WORLD_SIZE", "1")), int(os.environ.get("LOCAL_RANK", "0"))
    my_games, loop_seed, writer_seed = shard_plan(rank, world, a.max_games_total, a.seed)
    lm = NeuralNet.loadModelFile(model_path)
    ctx = NeuralNet.createComputeContext([gpu], L, L, True, lm)
    h = NeuralNet.createComputeHandle(ctx, lm, games, False, True, gpu)
    max_visits = kw.pop("max_visits", 600)
    sp = SelfPlay(h, games, max_visits, komi=data["komi"], seed=loop_seed, debug_hold_at_max_visits=True, max_playouts_per_wave=a.max_playouts_per_wave, **kw)
    outputs = ModelOutputs(a.output_dir, data, L, writer_seed, TrainingDataWriter)
    outputs.switch_to(model_path)
    log(f"Found new neural net {outputs.model_name}")
    log(f"Loaded latest neural net {outputs.model_name} from: {model_path}")
    log("Loaded all config stuff, starting self play")
    # board size, ko / suicide rule and komi of every game: drawn on the host like the reference's GameInitializer, applied by the device
    # when the slot's next game starts.  `slots` always holds what has been handed to the device for each slot's NEXT game.
    from .game_initializer import GameInitializer
    init = GameInitializer(seed=loop_seed ^ 0x47616D65, **data["game_init"])
    # komi-bisection searches (komiAuto, estimateLeadProb) run on side loops of their own (komi_search.KomiSearcher), one per visit count
    from .komi_search import KomiSearcher
    ks = data["komi_search"]
    if a.nccl_weights and world > 1 and (ks["komi_auto"] or ks["estimate_lead_prob"] > 0):
        raise ValueError("komiAuto / estimateLeadProb with -nccl-weights: the side loops' handles are not part of the weight broadcast yet")
    aux = {"handles": [], "loops": [], "fair": None, "lead": None, "side": None}

    def make_aux(context, model, seed_offset):
        """(fair-komi searcher, lead searcher) on fresh handles of `model`; the previous ones are dropped."""
        for lp in aux["loops"]:
            lp.free()
        for hx in aux["handles"]:
            hx.free()
        aux.update(handles=[], loops=[], fair=None, lead=None, side=None)
        side_kw = KomiSearcher.noiseless_kwargs(kw)
        side_kw["max_moves"] = int(kw.get("max_moves", 0) or 2 * L * L) + 8
        fork_needs_loop = forks.enabled and not (ks["komi_auto"] or ks["estimate_lead_prob"] > 0)      # the fork's evaluations need some side loop
        for name, want, visits in (("fair", ks["komi_auto"] or fork_needs_loop, ks["compensate_komi_visits"]), ("lead", ks["estimate_lead_prob"] > 0, ks["estimate_lead_visits"])):
            if not want:
                continue
            n_side = max(4, min(32, games // 4))
            hx = NeuralNet.createComputeHandle(context, model, n_side, False, True, gpu)
            lp = SelfPlay(hx, n_side, max(2, visits), komi=data["komi"], seed=loop_seed + 104729 + seed_offset, debug_hold_at_max_visits=True, **side_kw)
            aux["handles"].append(hx); aux["loops"].append(lp)
            aux[name] = KomiSearcher(lp)
        if data["side_position_prob"] > 0:      # side positions are searched like the game's own turns: the loop's parameters, noise and all, full visits
            n_side = max(4, min(32, games // 4))
            hx = NeuralNet.createComputeHandle(context, model, n_side, False, True, gpu)
            full_kw = dict(kw); full_kw["max_moves"] = side_kw["max_moves"]
            lp = SelfPlay(hx, n_side, max_visits, komi=data["komi"], seed=loop_seed + 1299709 + seed_offset, debug_hold_at_max_visits=True, **full_kw)
            aux["handles"].append(hx); aux["loops"].append(lp)
            aux["side"] = KomiSearcher(lp)
    from .fork_play import ForkManager
    forks = ForkManager(data["forks"], __import__("random").Random(loop_seed ^ 0x466F726B))
    make_aux(ctx, lm, 0)
    fork_searcher = lambda: aux["lead"] or aux["fair"]       # where fork evaluations and their komi compensation run
    slots = SlotSetups(init, games, data["policy_init"], fair_komi=aux["fair"] if ks["komi_auto"] else None, forks=forks if forks.enabled else None, searcher=fork_searcher())
    slots.start(sp)

    counts = {"started": games, "finished": 0, "moves": 0}

    def log_stats():
        """SelfplayManager::countOneGameStarted's periodic block (selfplaymanager.cpp:290-303), from the device counters."""
        st = sp.stats()
        log(f"Games finished: {counts['finished']}")
        log(f"Moves played: {st['total_moves']}")
        log(f"Data rows: {outputs.rows_total + (outputs.writer.row_count if outputs.writer is not None else 0)}")
        rows_nn = st["total_visits"] - st["nn_cache_hits"] - st["instant_playouts"]
        log(f"NN rows: {rows_nn}")
        log(f"NN batches: {max(1, rows_nn // max(1, games))}")
        log(f"NN avg batch size: {float(games)}")
        log(f"NN cache hits: {st['nn_cache_hits']}")

    def on_game(slot, finished):
        outputs.add_game(slot, finished)
        counts["finished"] += 1
        if forks.enabled and fork_searcher() is not None and not finished.end_no_result:        # Play::maybeForkGame on the finished game
            all_moves = list(finished.start_moves) + list(finished.moves)
            ko = {"SIMPLE": 0, "POSITIONAL": 1, "SITUATIONAL": 2, "SPIGHT": 3}[finished.ko_rule]
            setup = (finished.x_size, finished.y_size, ko, int(finished.multi_stone_suicide_legal))
            job = forks.job(all_moves, setup, finished.komi, L)
            if job is not None:
                # (a fork at the game length cap would be over before its first search: play_moves_game restarts the slot)
                cap = int(kw.get("max_moves", 0) or 2 * finished.x_size * finished.y_size)
                fork_searcher().submit(job, setup, [], lambda moves, setup=setup, komi=finished.komi, cap=cap: forks.add(moves, setup, komi) if moves and len(moves) < cap else None)

    def on_game_start(slot):
        counts["started"] += 1          # the slot's next game started on the device when the previous one ended
        if counts["started"] % log_games_every == 0:
            log(f"Started {counts['started']} games with {outputs.model_name}")
        if counts["started"] % max(1000, log_games_every * 100) == 0:
            log_stats()
        slots.game_started(sp, rec, slot)      # a forked game gets its position; then the draw for the game after it
    rec = GameRecorder(sp, None, data["komi"], draw_equivalent_wins_for_white=kw.get("draw_equivalent_wins_for_white", 0.5), on_game=on_game,
                       game_hash_fn=lambda slot, index: _game_hash(loop_seed, slot, index),
                       policy_surprise_data_weight=data["policy_surprise_data_weight"], value_surprise_data_weight=data["value_surprise_data_weight"],
                       use_search_value_surprise=data["use_search_value_surprise"], weight_rand=RowRand(writer_seed + ":weights"),
                       play_settings=data["play_settings"], policy_init=data["policy_init"]["enabled"], lead_estimator=aux["lead"], estimate_lead_prob=ks["estimate_lead_prob"], on_game_start=on_game_start, side_searcher=aux["side"], side_position_prob=data["side_position_prob"], limits_rand=__import__("random").Random(loop_seed ^ 0x4C696D69))
    # New nets (command/selfplay.cpp:336-352 modelLoadLoop: re-poll the models directory every 20 s; :142-231 load the newest one).
    # Default: every rank polls and reads the file itself.  -nccl-weights: rank 0 polls, reads and packs; the packed weights reach
    # the other GPUs by the library's ncclBroadcast (dist_weights.WeightBroadcaster) - the poll is then a collective, every
    # `-model-poll-waves` recorder iterations.  Games move over between two waves (the reference's switchNetsMidGame = true) and a
    # finished game's rows go to the directory of the net in use when it ended (selfplay.cpp:276-319).
    poller = ModelPoller(a.models_dir, model_path, a.model_poll_seconds)
    wb = None
    if a.nccl_weights and world > 1:
        import torch
        import torch.distributed as dist
        from .dist_weights import WeightBroadcaster
        torch.cuda.set_device(gpu)
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        dist.init_process_group("nccl", device_id=torch.device("cuda", gpu))
        wb = WeightBroadcaster(h, 0, torch.device("cuda", gpu))
    swaps, iters, done, stager, stager_error = 0, 0, False, None, None
    try:
        while True:
            done = a.max_games_total > 0 and rec.games_written >= my_games
            if wb is None and done:
                break
            if not done:
                if a.per_game_release:
                    rec.pump(8)
                else:
                    rec.step()
            for searcher in (aux["fair"], aux["lead"], aux["side"]):       # the side loops advance with the main loop
                if searcher is not None:
                    searcher.step(8)
            iters += 1
            if wb is None:
                # reading and packing a net takes the host ~0.1-0.2 s for a b18: done on a side thread (the library call releases the
                # GIL), the waves keep coming; the swap itself is one device copy ordered between two waves
                if stager is None:
                    p_ = poller.poll()
                    if p_ is not None:
                        stager = BackgroundStage(h, p_, aux["handles"])
                    continue
                if not stager.done():
                    continue
                new_path, stager_error, stager = stager.path, stager.error, None
                if stager_error is None:
                    h.commit_weights()
                    sp.clear_nn_cache()
                    for hx, lp in zip(aux["handles"], aux["loops"]):
                        hx.commit_weights(); lp.clear_nn_cache()
                    swaps += 1
                    outputs.switch_to(new_path)
                    log(f"Model loading loop thread loaded new neural net {outputs.model_name}"); log(f"Game loop changing midgame to new neural net: {outputs.model_name} (swap {swaps})")
                    continue
            elif iters % a.model_poll_waves == 0 or done:
                # collective: [all ranks done?] and rank 0's verdict on the models directory
                import torch.distributed as dist
                box = [poller.poll(force=True) if rank == 0 else None, done]
                everyone = [None] * world
                dist.all_gather_object(everyone, box)
                if all(e[1] for e in everyone):
                    break
                new_path = everyone[0][0]
            else:
                new_path = None
            if new_path is None:
                continue
            try:
                if wb is None:
                    raise stager_error
                else:
                    new_lm = NeuralNet.loadModelFile(new_path) if rank == 0 else None
                    wb.update(new_lm)
                sp.clear_nn_cache()
            except Exception as e:
                if wb is not None:
                    raise
                if not (isinstance(e, KGBError) and any(w in str(e) for w in ("architecture", "layout", "largest convolution"))):
                    # e.g. a file that is still being written: keep playing the current net, look again at the next poll
                    print(f"[model] {new_path}: {e}; keeping {outputs.model_name}", file=sys.stderr)
                    poller.forget(new_path)
                    continue
                # another architecture: the reference builds a new NNEvaluator for any net; here that means a new handle and loop, and
                # the games in flight are dropped (their finished predecessors are already written)
                print(f"[model] {new_path}: {e}; rebuilding the evaluator (games in progress are abandoned)", file=sys.stderr)
                for lp in aux["loops"]:
                    lp.free()
                for hx in aux["handles"]:
                    hx.free()
                aux.update(handles=[], loops=[], fair=None, lead=None, side=None)
                sp.free(); h.free(); ctx.free()
                lm = NeuralNet.loadModelFile(new_path)
                ctx = NeuralNet.createComputeContext([gpu], L, L, True, lm)
                h = NeuralNet.createComputeHandle(ctx, lm, games, False, True, gpu)
                sp = SelfPlay(h, games, max_visits, komi=data["komi"], seed=loop_seed + 7919 * (swaps + 1), debug_hold_at_max_visits=True, max_playouts_per_wave=a.max_playouts_per_wave, **kw)
                make_aux(ctx, lm, swaps + 1)               # (lead jobs of games that ended under the old evaluator are dropped with it)
                slots.fair_komi = aux["fair"] if ks["komi_auto"] else None
                slots.searcher = fork_searcher()
                slots.start(sp)
                written = rec.games_written
                rec = GameRecorder(sp, None, data["komi"], draw_equivalent_wins_for_white=kw.get("draw_equivalent_wins_for_white", 0.5), on_game=on_game,
                                   game_hash_fn=lambda slot, index, s_=swaps + 1: _game_hash(loop_seed + 7919 * s_, slot, index),
                                   policy_surprise_data_weight=data["policy_surprise_data_weight"], value_surprise_data_weight=data["value_surprise_data_weight"],
                                   use_search_value_surprise=data["use_search_value_surprise"], weight_rand=RowRand(writer_seed + f":weights{swaps + 1}"),
                                   play_settings=data["play_settings"], policy_init=data["policy_init"]["enabled"], lead_estimator=aux["lead"], estimate_lead_prob=ks["estimate_lead_prob"], on_game_start=on_game_start, side_searcher=aux["side"], side_position_prob=data["side_position_prob"], limits_rand=__import__("random").Random(loop_seed ^ (0x4C696D69 + swaps + 1)))
                rec.games_written = written
            swaps += 1
            outputs.switch_to(new_path)
            log(f"Model loading loop thread loaded new neural net {outputs.model_name}"); log(f"Game loop changing midgame to new neural net: {outputs.model_name} (swap {swaps})")
    except KeyboardInterrupt:
        pass
    for searcher in (aux["lead"], aux["side"]):      # finished games whose lead searches / side positions are still running
        if searcher is not None and rec.games_waiting_for_lead > 0:
            searcher.drain()
    outputs.close()
    log_stats()
    log(f"Total games: {counts['started']}")
    log(f"Total selfplay runtime (seconds): {time.time() - t_start}")
    log("All cleaned up, quitting")
    print(f"{rec.games_written} games, {outputs.rows_total} rows -> {', '.join(outputs.dirs)}")
    for lp in aux["loops"]:
        lp.free()
    for hx in aux["handles"]:
        hx.free()
    sp.free(); h.free(); ctx.free()
    return 0


if __name__ == "__main__":
    sys.exit(main())
