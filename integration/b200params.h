// kgb_selfplay_config from the reference's own SearchParams + Rules (search/searchparams.h, game/rules.h): the C++ side of what
// katago_b200/selfplay_cli.py does from a .cfg file, for a maintainer who parses the configuration with the reference's own
// Setup::loadSingleParams (program/setup.cpp) and wants the device loop to run the same search (INTEGRATION.md §6).
//
// Reference-side glue: includes the reference's headers.  `unsupported` receives one line per option that is set to something the
// device loop does not implement (the loop then runs WITHOUT it) - the caller decides whether that is an error.
#pragma once
#include <sstream>
#include <string>
#include <vector>

#include "../include/kgb200.h"
#include "game/rules.h"
#include "search/searchparams.h"

namespace b200 {

inline kgb_selfplay_config configFromSearchParams(const SearchParams& p, const Rules& rules, int numGames, int maxMovesPerGame, uint64_t seed,
                                                  int nnCacheSizePowerOfTwo, std::vector<std::string>* unsupported = nullptr) {
  kgb_selfplay_config c = {};
  auto no = [&](bool bad, const std::string& what) { if(bad && unsupported) unsupported->push_back(what); };
  auto num = [](double v) { std::ostringstream s; s << v; return s.str(); };

  c.num_games = numGames;
  c.max_visits = p.maxVisits > 1000000000LL ? 0 : (int32_t)p.maxVisits;
  no(p.maxVisits > 1000000000LL, "maxVisits is not set (the loop needs a visit budget per move)");
  c.max_moves = maxMovesPerGame;
  c.seed = seed;
  c.nn_cache_size_power_of_two = nnCacheSizePowerOfTwo;

  // rules (area scoring, no tax, no button, no handicap bonus)
  c.komi = rules.komi;
  c.multi_stone_suicide_legal = rules.multiStoneSuicideLegal ? 1 : 0;
  c.ko_rule = rules.koRule == Rules::KO_POSITIONAL ? 1 : rules.koRule == Rules::KO_SITUATIONAL ? 2 : rules.koRule == Rules::KO_SPIGHT ? 3 : 0;
  c.full_history_rules = 1;
  no(rules.scoringRule != Rules::SCORING_AREA, "scoringRule = " + Rules::writeScoringRule(rules.scoringRule));
  no(rules.taxRule != Rules::TAX_NONE, "taxRule = " + Rules::writeTaxRule(rules.taxRule));
  no(rules.hasButton, "hasButton = true");
  no(rules.whiteHandicapBonusRule != Rules::WHB_ZERO, "whiteHandicapBonus = " + Rules::writeWhiteHandicapBonusRule(rules.whiteHandicapBonusRule));
  no(rules.friendlyPassOk, "friendlyPassOk = true");

  // utility
  c.win_loss_utility_factor = p.winLossUtilityFactor;
  c.static_score_utility_factor = p.staticScoreUtilityFactor;
  c.dynamic_score_utility_factor = p.dynamicScoreUtilityFactor;
  c.dynamic_score_center_zero_weight = p.dynamicScoreCenterZeroWeight;
  c.dynamic_score_center_scale = p.dynamicScoreCenterScale;
  c.no_result_utility_for_white = p.noResultUtilityForWhite;
  c.draw_equivalent_wins_for_white = p.drawEquivalentWinsForWhite;
  // selection
  c.cpuct_exploration = p.cpuctExploration;
  c.cpuct_exploration_log = p.cpuctExplorationLog;
  c.cpuct_exploration_base = p.cpuctExplorationBase;
  c.cpuct_utility_stdev_prior = p.cpuctUtilityStdevPrior;
  c.cpuct_utility_stdev_prior_weight = p.cpuctUtilityStdevPriorWeight;
  c.cpuct_utility_stdev_scale = p.cpuctUtilityStdevScale;
  c.fpu_reduction_max = p.fpuReductionMax;
  c.fpu_loss_prop = p.fpuLossProp;
  c.fpu_parent_weight_by_visited_policy = p.fpuParentWeightByVisitedPolicy ? 1 : 0;
  c.fpu_parent_weight_by_visited_policy_pow = p.fpuParentWeightByVisitedPolicyPow;
  c.fpu_parent_weight = p.fpuParentWeight;
  c.root_fpu_reduction_max = p.rootFpuReductionMax;
  c.root_fpu_loss_prop = p.rootFpuLossProp;
  c.root_desired_per_child_visits_coeff = p.rootDesiredPerChildVisitsCoeff;
  // backup
  c.value_weight_exponent = p.valueWeightExponent;
  c.subtree_value_bias_factor = p.subtreeValueBiasFactor;
  c.subtree_value_bias_weight_exponent = p.subtreeValueBiasWeightExponent;
  c.use_uncertainty = p.useUncertainty ? 1 : 0;
  c.uncertainty_coeff = p.uncertaintyCoeff;
  c.uncertainty_exponent = p.uncertaintyExponent;
  c.uncertainty_max_weight = p.uncertaintyMaxWeight;
  c.use_noise_pruning = p.useNoisePruning ? 1 : 0;
  c.noise_prune_utility_scale = p.noisePruneUtilityScale;
  c.noise_pruning_cap = p.noisePruningCap;
  // graph search
  c.use_graph_search = p.useGraphSearch ? 1 : 0;
  c.graph_search_rep_bound = p.graphSearchRepBound;
  // root
  c.root_noise_enabled = p.rootNoiseEnabled ? 1 : 0;
  c.root_dirichlet_noise_total_concentration = p.rootDirichletNoiseTotalConcentration;
  c.root_dirichlet_noise_weight = p.rootDirichletNoiseWeight;
  c.root_policy_temperature = p.rootPolicyTemperature;
  c.root_policy_temperature_early = p.rootPolicyTemperatureEarly;
  c.root_num_symmetries_to_sample = p.rootNumSymmetriesToSample;
  // move choice (Search::getChosenMoveLoc)
  c.use_play_selection = 1;
  c.chosen_move_temperature = p.chosenMoveTemperature;
  c.chosen_move_temperature_early = p.chosenMoveTemperatureEarly;
  c.chosen_move_temperature_halflife = p.chosenMoveTemperatureHalflife;
  c.chosen_move_temperature_only_below_prob = p.chosenMoveTemperatureOnlyBelowProb;
  c.chosen_move_subtract = p.chosenMoveSubtract;
  c.chosen_move_prune = p.chosenMovePrune;
  c.use_lcb_for_selection = p.useLcbForSelection ? 1 : 0;
  c.lcb_stdevs = p.lcbStdevs;
  c.min_visit_prop_for_lcb = p.minVisitPropForLCB;
  c.use_non_buggy_lcb = p.useNonBuggyLcb ? 1 : 0;
  c.root_ending_bonus_points = p.rootEndingBonusPoints;
  c.root_prune_useless_moves = p.rootPruneUselessMoves ? 1 : 0;

  // options of the reference's search that the device loop does not have: reported when they are switched on
  no(p.policyOptimism != 0.0, "policyOptimism = " + num(p.policyOptimism));
  no(p.rootPolicyOptimism != 0.0, "rootPolicyOptimism = " + num(p.rootPolicyOptimism));
  no(p.graphSearchCatchUpLeakProb != 0.0, "graphSearchCatchUpLeakProb = " + num(p.graphSearchCatchUpLeakProb));
  no(p.rootSymmetryPruning, "rootSymmetryPruning = true");
  no(p.conservativePass, "conservativePass = true");
  no(p.fillDameBeforePass, "fillDameBeforePass = true");
  no(p.wideRootNoise != 0.0, "wideRootNoise = " + num(p.wideRootNoise));
  no(p.enablePassingHacks, "enablePassingHacks = true");
  no(p.enableMorePassingHacks, "enableMorePassingHacks = true");
  no(p.playoutDoublingAdvantage != 0.0, "playoutDoublingAdvantage = " + num(p.playoutDoublingAdvantage));
  no(p.avoidRepeatedPatternUtility != 0.0, "avoidRepeatedPatternUtility = " + num(p.avoidRepeatedPatternUtility));
  no(p.nnPolicyTemperature != 1.0f, "nnPolicyTemperature = " + num(p.nnPolicyTemperature));
  no(p.antiMirror, "antiMirror = true");
  no(p.ignorePreRootHistory, "ignorePreRootHistory = true");
  no(p.ignoreAllHistory, "ignoreAllHistory = true");
  no(p.useEvalCache, "useEvalCache = true");
  no(p.futileVisitsThreshold != 0.0, "futileVisitsThreshold = " + num(p.futileVisitsThreshold));
  no(p.numThreads > 1, "numSearchThreads = " + num(p.numThreads) + " (one playout per game is in flight; the games are the parallelism)");
  no(p.maxPlayouts < p.maxVisits, "maxPlayouts = " + num((double)p.maxPlayouts));
  no(p.maxTime < 1e20, "maxTime = " + num(p.maxTime));
  return c;
}

}  // namespace b200
