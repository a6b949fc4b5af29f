// Configuration of the C++ hosts (b200_selfplay_main.cpp, b200_gatekeeper_main.cpp): the reference's .cfg files by their own key names ->
// kgb_selfplay_config and the per-game draws, the newest net of a models directory.  Plain C++17.
#pragma once
#include <cctype>
#include <cerrno>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <dirent.h>
#include <fstream>
#include <map>
#include <sstream>
#include <string>
#include <sys/stat.h>
#include <vector>

#include "b200_gameinit.h"

namespace b200host {

inline const char*& programName() { static const char* name = "b200"; return name; }
[[noreturn]] inline void die(const std::string& what) { std::fprintf(stderr, "%s: %s\n", programName(), what.c_str()); std::exit(1); }

inline std::string lower(std::string s) { for(char& c : s) c = (char)std::tolower((unsigned char)c); return s; }      // (the reference's stock files write True / False)

inline std::string trim(const std::string& s) {
  size_t a = s.find_first_not_of(" \t\r\n"), b = s.find_last_not_of(" \t\r\n");
  return a == std::string::npos ? "" : s.substr(a, b - a + 1);
}

// key = value lines, '#' comments (core/config_parser.cpp: the subset without @include and quoting)
struct Cfg {
  std::map<std::string, std::string> kv;
  mutable std::map<std::string, bool> used;
  void line(const std::string& raw, const std::string& where) {
    std::string s = trim(raw.substr(0, raw.find('#')));
    if(s.empty()) return;
    size_t eq = s.find('=');
    if(eq == std::string::npos) die(where + ": expected key = value, got '" + s + "'");
    kv[trim(s.substr(0, eq))] = trim(s.substr(eq + 1));
  }
  void load(const std::string& path) {
    std::ifstream in(path);
    if(!in) die("cannot read config file " + path);
    std::string l; int n = 0;
    while(std::getline(in, l)) line(l, path + ":" + std::to_string(++n));
  }
  void overrides(const std::string& list) {
    std::stringstream ss(list); std::string item;
    while(std::getline(ss, item, ',')) line(item, "-override-config");
  }
  bool has(const std::string& k) const { return kv.count(k) > 0; }
  double num(const std::string& k, double dflt) const {
    used[k] = true;
    auto it = kv.find(k);
    if(it == kv.end()) return dflt;
    char* end = nullptr;
    double v = std::strtod(it->second.c_str(), &end);
    if(end == it->second.c_str() || *end) die("config key " + k + ": not a number: '" + it->second + "'");
    return v;
  }
  bool flag(const std::string& k, bool dflt) const {
    used[k] = true;
    auto it = kv.find(k);
    if(it == kv.end()) return dflt;
    if(lower(it->second) == "true") return true;
    if(lower(it->second) == "false") return false;
    die("config key " + k + ": expected true or false, got '" + it->second + "'");
  }
  std::vector<std::string> list(const std::string& k, const std::string& dflt) const {      // comma-separated values
    std::vector<std::string> out; std::stringstream ss(str(k, dflt)); std::string item;
    while(std::getline(ss, item, ',')) { item = trim(item); if(!item.empty()) out.push_back(item); }
    if(out.empty()) die("config key " + k + ": no value");
    return out;
  }
  std::string str(const std::string& k, const std::string& dflt) const { used[k] = true; auto it = kv.find(k); return it == kv.end() ? dflt : it->second; }
  // Options of the reference that neither host of the device loop has (katago_b200/selfplay_cli.py reports the same ones): fine while they keep their
  // neutral value, else listed as NOT BUILT - the loop then runs WITHOUT them, or, with -strict, not at all.
  mutable std::vector<std::string> notBuilt;
  void neutral(const std::string& k, const std::string& value) const {
    used[k] = true;
    auto it = kv.find(k);
    if(it == kv.end()) return;
    if(value == "true" || value == "false") { if(lower(it->second) == value) return; }
    else { char* end = nullptr; const double v = std::strtod(it->second.c_str(), &end); if(end != it->second.c_str() && !*end && v == std::atof(value.c_str())) return; }
    notBuilt.push_back(k + " = " + it->second);
  }
  // a list-valued key of which the loop has only some values: the others are left out of the per-game draw and named
  std::vector<std::string> supportedOf(const std::string& k, const std::string& dflt, const std::vector<std::string>& supported) const {
    std::vector<std::string> ok, dropped;
    for(const std::string& v : list(k, dflt)) {
      bool have = false;
      for(const std::string& sup : supported) have = have || sup == v || sup == lower(v);
      (have ? ok : dropped).push_back(v);
    }
    if(ok.empty()) die("config key " + k + " = " + str(k, dflt) + ": none of these is built");
    if(!dropped.empty()) { std::string d; for(const std::string& v : dropped) d += (d.empty() ? "" : ", ") + v; notBuilt.push_back(k + ": the reference draws one of [" + str(k, dflt) + "] per game; " + d + " not built"); }
    return ok;
  }
};

inline int koRuleOf(const std::string& ko) {
  const int r = ko == "SIMPLE" ? 0 : ko == "POSITIONAL" ? 1 : ko == "SITUATIONAL" ? 2 : ko == "SPIGHT" ? 3 : -1;
  if(r < 0) die("koRules: SIMPLE, POSITIONAL, SITUATIONAL or SPIGHT, got '" + ko + "'");
  return r;
}
inline bool boolOf(const std::string& key, const std::string& v) {
  if(lower(v) == "true") return true;
  if(lower(v) == "false") return false;
  die("config key " + key + ": expected true or false, got '" + v + "'");
}

// SearchParams and Rules by their cfg names -> kgb_selfplay_config (defaults of absent keys: the reference loader's for a self-play command, program/setup.cpp:445-760, like katago_b200/selfplay_cli.py)
inline kgb_selfplay_config configFromCfg(const Cfg& c, int numGames) {
  kgb_selfplay_config k = {};
  k.num_games = numGames;
  k.max_visits = (int32_t)c.num("maxVisits", 0);
  if(k.max_visits <= 0) die("maxVisits must be set: the loop needs a visit budget per move");
  k.max_moves = (int32_t)c.num("maxMovesPerGame", 0);        // 0 = 2 * X * Y
  k.seed = (uint64_t)c.num("searchRandSeed", 1.0);
  k.nn_cache_size_power_of_two = (int32_t)c.num("nnCacheSizePowerOfTwo", 0);
  k.komi = (float)c.num("komiMean", 7.5);
  // rules, board size and komi are drawn per game (b200_gameinit.h); the loop's own configuration carries the first listed values
  k.ko_rule = koRuleOf(c.list("koRules", "SIMPLE")[0]);
  k.multi_stone_suicide_legal = boolOf("multiStoneSuicideLegals", c.list("multiStoneSuicideLegals", "true")[0]) ? 1 : 0;
  c.supportedOf("scoringRules", "AREA", {"AREA"}); c.supportedOf("taxRules", "NONE", {"NONE"}); c.supportedOf("hasButtons", "false", {"false"});
  c.neutral("handicapProb", "0.0"); c.neutral("compensateAfterPolicyInitProb", "0.0"); c.neutral("sekiForkHackProb", "0.0");
  c.neutral("handicapAsymmetricPlayoutProb", "0.0"); c.neutral("normalAsymmetricPlayoutProb", "0.0"); c.neutral("switchNetsMidGame", "true");
  c.neutral("fancyKomiVarying", "false"); c.neutral("drawRandRadius", "0.0"); c.neutral("noResultStdev", "0.0");

  k.win_loss_utility_factor = c.num("winLossUtilityFactor", 1.0);
  k.static_score_utility_factor = c.num("staticScoreUtilityFactor", 0.1);
  k.dynamic_score_utility_factor = c.num("dynamicScoreUtilityFactor", 0.3);
  k.dynamic_score_center_zero_weight = c.num("dynamicScoreCenterZeroWeight", 0.2);
  k.dynamic_score_center_scale = c.num("dynamicScoreCenterScale", 0.75);
  k.no_result_utility_for_white = c.num("noResultUtilityForWhite", 0.0);
  k.draw_equivalent_wins_for_white = c.num("drawEquivalentWinsForWhite", 0.5);
  k.cpuct_exploration = c.num("cpuctExploration", 1.0);
  k.cpuct_exploration_log = c.num("cpuctExplorationLog", 0.45);
  k.cpuct_exploration_base = c.num("cpuctExplorationBase", 500.0);
  k.cpuct_utility_stdev_prior = c.num("cpuctUtilityStdevPrior", 0.4);
  k.cpuct_utility_stdev_prior_weight = c.num("cpuctUtilityStdevPriorWeight", 2.0);
  k.cpuct_utility_stdev_scale = c.num("cpuctUtilityStdevScale", 0.0);
  k.fpu_reduction_max = c.num("fpuReductionMax", 0.2);
  k.fpu_loss_prop = c.num("fpuLossProp", 0.0);
  k.fpu_parent_weight_by_visited_policy = c.flag("fpuParentWeightByVisitedPolicy", true) ? 1 : 0;
  // setup.cpp:501-513: the power is read only with the flag, the plain weight only without it
  k.fpu_parent_weight_by_visited_policy_pow = k.fpu_parent_weight_by_visited_policy ? c.num("fpuParentWeightByVisitedPolicyPow", 2.0) : 1.0;
  k.fpu_parent_weight = k.fpu_parent_weight_by_visited_policy ? 0.0 : c.num("fpuParentWeight", 0.0);
  k.root_fpu_reduction_max = c.num("rootFpuReductionMax", c.flag("rootNoiseEnabled", false) ? 0.0 : 0.1);   // setup.cpp:578-583
  k.root_fpu_loss_prop = c.num("rootFpuLossProp", k.fpu_loss_prop);
  k.root_desired_per_child_visits_coeff = c.num("rootDesiredPerChildVisitsCoeff", 0.0);
  k.value_weight_exponent = c.num("valueWeightExponent", 0.25);
  k.subtree_value_bias_factor = c.num("subtreeValueBiasFactor", 0.45);
  k.subtree_value_bias_weight_exponent = c.num("subtreeValueBiasWeightExponent", 0.85);
  k.use_graph_search = c.flag("useGraphSearch", true) ? 1 : 0;
  k.graph_search_rep_bound = (int32_t)c.num("graphSearchRepBound", 11);
  k.root_noise_enabled = c.flag("rootNoiseEnabled", false) ? 1 : 0;
  k.root_dirichlet_noise_total_concentration = c.num("rootDirichletNoiseTotalConcentration", 10.83);
  k.root_dirichlet_noise_weight = c.num("rootDirichletNoiseWeight", 0.25);
  k.root_policy_temperature = c.num("rootPolicyTemperature", 1.0);
  k.root_policy_temperature_early = c.num("rootPolicyTemperatureEarly", k.root_policy_temperature);
  k.root_num_symmetries_to_sample = (int32_t)c.num("rootNumSymmetriesToSample", 1);
  k.use_play_selection = 1;
  k.early_temperature_moves = 30;            // (only read without use_play_selection; the value the Python host passes)
  k.chosen_move_temperature = c.num("chosenMoveTemperature", 0.1);
  k.chosen_move_temperature_early = c.num("chosenMoveTemperatureEarly", 0.5);
  k.chosen_move_temperature_halflife = c.num("chosenMoveTemperatureHalflife", 19.0);
  k.chosen_move_temperature_only_below_prob = c.num("chosenMoveTemperatureOnlyBelowProb", 1.0);
  k.chosen_move_subtract = c.num("chosenMoveSubtract", 0.0);
  k.chosen_move_prune = c.num("chosenMovePrune", 1.0);
  k.use_lcb_for_selection = c.flag("useLcbForSelection", true) ? 1 : 0;
  k.lcb_stdevs = c.num("lcbStdevs", 5.0);
  k.min_visit_prop_for_lcb = c.num("minVisitPropForLCB", 0.15);
  k.use_non_buggy_lcb = c.flag("useNonBuggyLcb", false) ? 1 : 0;
  k.root_ending_bonus_points = c.num("rootEndingBonusPoints", 0.5);
  k.root_prune_useless_moves = c.flag("rootPruneUselessMoves", true) ? 1 : 0;
  k.use_uncertainty = c.flag("useUncertainty", false) ? 1 : 0;
  k.uncertainty_coeff = c.num("uncertaintyCoeff", 0.25);
  k.uncertainty_exponent = c.num("uncertaintyExponent", 1.0);
  k.uncertainty_max_weight = c.num("uncertaintyMaxWeight", 8.0);
  k.use_noise_pruning = c.flag("useNoisePruning", false) ? 1 : 0;
  k.noise_prune_utility_scale = c.num("noisePruneUtilityScale", 0.15);
  k.noise_pruning_cap = c.num("noisePruningCap", 1e50);
  k.max_playouts_per_wave = (int32_t)c.num("b200MaxPlayoutsPerWave", 4);
  k.debug_hold_at_max_visits = 1;       // a slot whose search is finished waits for this host to read its move
  return k;
}

// -print-config: the mapped fields as JSON (tests/test_abi_and_loader.py compares them with the reference's own loader through
// integration/b200params.h, `kgref_driver paramsmap`)
inline void printConfig(const kgb_selfplay_config& c) {
  std::printf("{");
#define FI(f) std::printf("\"" #f "\":%lld,", (long long)c.f)
#define FD(f) std::printf("\"" #f "\":%.17g,", (double)c.f)
  FI(num_games); FI(max_visits); FI(max_moves); FI(multi_stone_suicide_legal); FD(komi); FD(cpuct_exploration); FD(cpuct_exploration_log); FD(cpuct_exploration_base);
  FD(fpu_reduction_max); FD(root_fpu_reduction_max); FD(win_loss_utility_factor); FD(no_result_utility_for_white);
  FD(static_score_utility_factor); FD(dynamic_score_utility_factor); FD(dynamic_score_center_zero_weight); FD(dynamic_score_center_scale);
  FD(draw_equivalent_wins_for_white); FD(value_weight_exponent); FI(fpu_parent_weight_by_visited_policy); FD(fpu_parent_weight_by_visited_policy_pow);
  FD(fpu_parent_weight); FD(fpu_loss_prop); FD(root_fpu_loss_prop); FD(cpuct_utility_stdev_prior); FD(cpuct_utility_stdev_prior_weight);
  FD(cpuct_utility_stdev_scale); FD(root_desired_per_child_visits_coeff); FD(subtree_value_bias_factor); FD(subtree_value_bias_weight_exponent);
  FI(use_graph_search); FI(graph_search_rep_bound); FI(root_noise_enabled); FD(root_dirichlet_noise_total_concentration); FD(root_dirichlet_noise_weight);
  FD(root_policy_temperature); FD(root_policy_temperature_early); FD(chosen_move_temperature_halflife); FI(use_play_selection); FI(use_lcb_for_selection);
  FI(use_non_buggy_lcb); FD(lcb_stdevs); FD(min_visit_prop_for_lcb); FD(chosen_move_temperature); FD(chosen_move_temperature_early);
  FD(chosen_move_temperature_only_below_prob); FD(chosen_move_subtract); FD(chosen_move_prune); FI(nn_cache_size_power_of_two);
  FI(root_num_symmetries_to_sample); FI(ko_rule); FD(root_ending_bonus_points); FI(root_prune_useless_moves);
  FI(max_playouts_per_wave); FI(use_uncertainty); FD(uncertainty_coeff); FD(uncertainty_exponent); FD(uncertainty_max_weight);
  FI(use_noise_pruning); FD(noise_prune_utility_scale); FD(noise_pruning_cap);
#undef FI
#undef FD
  std::printf("\"debug_hold_at_max_visits\":%d}\n", (int)c.debug_hold_at_max_visits);
}

// The newest net of a models directory (command/selfplay.cpp:150-176 LoadModel::findLatestModel; as katago_b200/selfplay_cli.py newest_model):
// <dir>/*.bin.gz | *.bin | *.txt.gz | *.txt and <dir>/<name>/model.bin.gz, by modification time.
inline bool endsWith(const std::string& s, const std::string& suffix) { return s.size() >= suffix.size() && s.compare(s.size() - suffix.size(), suffix.size(), suffix) == 0; }
inline std::string newestModel(const std::string& dir) {
  std::string best; double bestTime = -1;
  auto consider = [&](const std::string& path) {
    struct stat st;
    if(stat(path.c_str(), &st) != 0 || !S_ISREG(st.st_mode)) return;
    const double t = (double)st.st_mtim.tv_sec + 1e-9 * (double)st.st_mtim.tv_nsec;
    if(t > bestTime) { bestTime = t; best = path; }
  };
  DIR* d = opendir(dir.c_str());
  if(!d) die("cannot read the models directory " + dir);
  while(dirent* e = readdir(d)) {
    const std::string name = e->d_name;
    if(name == "." || name == "..") continue;
    if(endsWith(name, ".bin.gz") || endsWith(name, ".bin") || endsWith(name, ".txt.gz") || endsWith(name, ".txt")) consider(dir + "/" + name);
    consider(dir + "/" + name + "/model.bin.gz");
  }
  closedir(d);
  if(best.empty()) die("no model file in " + dir);
  return best;
}
// the net's name in the output tree: <name>/model.bin.gz -> name, else the file name up to its first dot
inline std::string modelNameOf(const std::string& path) {
  const size_t slash = path.find_last_of('/');
  const std::string base = slash == std::string::npos ? path : path.substr(slash + 1);
  if(base == "model.bin.gz" && slash != std::string::npos && slash > 0) {
    const size_t prev = path.find_last_of('/', slash - 1);
    return path.substr(prev == std::string::npos ? 0 : prev + 1, slash - (prev == std::string::npos ? 0 : prev + 1));
  }
  return base.substr(0, base.find('.'));
}


// board size, ko / suicide rule and komi of every game (b200_gameinit.h) from bSizes / bSizeRelProbs / allowRectangleProb, koRules,
// multiStoneSuicideLegals, komiMean, komiStdev ...; *dataLen = the evaluator's frame (dataBoardLen, at least the largest board)
inline b200::GameInitializer::Config gameInitConfigFromCfg(const Cfg& cfg, int* dataLen) {
  b200::GameInitializer::Config gi;
  for(const std::string& v : cfg.list("bSizes", "19")) { gi.edges.push_back(std::atoi(v.c_str())); if(gi.edges.back() < 2 || gi.edges.back() > 19) die("bSizes: 2..19"); }
  if(cfg.has("bSizeRelProbs")) for(const std::string& v : cfg.list("bSizeRelProbs", "")) gi.relProbs.push_back(std::atof(v.c_str()));
  else gi.relProbs.assign(gi.edges.size(), 1.0);
  if(gi.relProbs.size() != gi.edges.size()) die("bSizeRelProbs has " + std::to_string(gi.relProbs.size()) + " entries, bSizes has " + std::to_string(gi.edges.size()));
  gi.allowRectangleProb = cfg.num("allowRectangleProb", 0.0);
  gi.koRules.clear(); for(const std::string& v : cfg.list("koRules", "SIMPLE")) gi.koRules.push_back(koRuleOf(v));
  gi.multiStoneSuicideLegals.clear(); for(const std::string& v : cfg.list("multiStoneSuicideLegals", "true")) gi.multiStoneSuicideLegals.push_back(boolOf("multiStoneSuicideLegals", v) ? 1 : 0);
  gi.komiMean = cfg.num("komiMean", 7.5); gi.komiStdev = cfg.num("komiStdev", 0.0); gi.komiBigStdevProb = cfg.num("komiBigStdevProb", 0.0);
  gi.komiBigStdev = cfg.num("komiBigStdev", 10.0); gi.komiBiggerStdevProb = cfg.num("komiBiggerStdevProb", 0.0); gi.komiBiggerStdev = cfg.num("komiBiggerStdev", 30.0);
  gi.komiAllowIntegerProb = cfg.num("komiAllowIntegerProb", 1.0);
  int maxEdge = 0; for(int e : gi.edges) maxEdge = std::max(maxEdge, e);
  const int edge = (int)cfg.num("dataBoardLen", maxEdge);
  if(edge < maxEdge) die("dataBoardLen = " + std::to_string(edge) + " but bSizes goes up to " + std::to_string(maxEdge) + ": the data frame must hold the largest board");
  if(edge > 19) die("dataBoardLen: at most 19");
  *dataLen = edge;
  return gi;
}

// The search keys a bot of a match can have of its own (`maxVisits0` overrides the shared `maxVisits` for bot 0: Setup::loadParams with
// SETUP_FOR_MATCH, program/setup.cpp) - the keys configFromCfg reads
inline const std::vector<std::string>& searchKeys() {
  static const std::vector<std::string> keys = {
    "maxVisits", "cpuctExploration", "cpuctExplorationLog", "cpuctExplorationBase", "fpuReductionMax", "rootFpuReductionMax", "fpuLossProp", "rootFpuLossProp",
    "fpuParentWeight", "fpuParentWeightByVisitedPolicy", "fpuParentWeightByVisitedPolicyPow", "valueWeightExponent", "cpuctUtilityStdevPrior",
    "cpuctUtilityStdevPriorWeight", "cpuctUtilityStdevScale", "rootDesiredPerChildVisitsCoeff", "subtreeValueBiasFactor", "subtreeValueBiasWeightExponent",
    "useGraphSearch", "graphSearchRepBound", "rootNoiseEnabled", "rootDirichletNoiseTotalConcentration", "rootDirichletNoiseWeight", "rootPolicyTemperature",
    "rootPolicyTemperatureEarly", "chosenMoveTemperature", "chosenMoveTemperatureEarly", "chosenMoveTemperatureHalflife", "chosenMoveTemperatureOnlyBelowProb",
    "chosenMoveSubtract", "chosenMovePrune", "useLcbForSelection", "lcbStdevs", "minVisitPropForLCB", "useNonBuggyLcb", "winLossUtilityFactor",
    "staticScoreUtilityFactor", "dynamicScoreUtilityFactor", "dynamicScoreCenterZeroWeight", "dynamicScoreCenterScale", "noResultUtilityForWhite",
    "drawEquivalentWinsForWhite", "rootNumSymmetriesToSample", "nnCacheSizePowerOfTwo", "maxMovesPerGame", "rootEndingBonusPoints", "rootPruneUselessMoves",
    "useUncertainty", "uncertaintyCoeff", "uncertaintyExponent", "uncertaintyMaxWeight", "useNoisePruning", "noisePruneUtilityScale", "noisePruningCap"};
  return keys;
}
// The configuration bot `idx` of a match sees: a search key with the bot's index appended overrides the shared one; keys of other bots, bot
// names and model files are left out (katago_b200/match_cli.py bot_cfg)
inline Cfg botCfg(const Cfg& cfg, int idx) {
  Cfg out;
  auto perBot = [](const std::string& base) {
    if(base == "botName" || base == "nnModelFile") return true;
    for(const std::string& k : searchKeys()) if(k == base) return true;
    return false;
  };
  for(const auto& e : cfg.kv) {
    const std::string& k = e.first;
    size_t digits = k.size();
    while(digits > 0 && std::isdigit((unsigned char)k[digits - 1])) digits--;
    if(k == "botName" || k == "nnModelFile" || (digits < k.size() && digits > 0 && perBot(k.substr(0, digits)))) continue;
    out.kv[k] = e.second;
  }
  for(const std::string& k : searchKeys()) { auto it = cfg.kv.find(k + std::to_string(idx)); if(it != cfg.kv.end()) out.kv[k] = it->second; }
  return out;
}

inline void makeDirsFor(const std::string& path) {       // mkdir -p
  for(size_t i = 1; i <= path.size(); i++)
    if(i == path.size() || path[i] == '/') { const std::string p = path.substr(0, i); if(mkdir(p.c_str(), 0777) != 0 && errno != EEXIST) die("cannot create " + p); }
}

// keys that only place or log the reference's own CPU threads and evaluator servers: nothing to do here
inline void markIrrelevantKeys(const Cfg& cfg) {
  static const char* irrelevant[] = {"log", "cuda", "trt", "opencl", "eigen", "numNNServerThreads", "nnMaxBatchSize", "nnMutexPool", "numSearchThreads",
                                     "maxDataQueueSize", "nnRandomize", "numVirtualLossesPerThread", "gpuToUse", "homeDataDir"};
  for(const auto& e : cfg.kv)
    for(const char* prefix : irrelevant)
      if(e.first.compare(0, std::strlen(prefix), prefix) == 0) cfg.used[e.first] = true;
}

}  // namespace b200host
