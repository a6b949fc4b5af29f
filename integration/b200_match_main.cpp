// `katago match` (command/match.cpp) for two named bots as a C++-only host of the device loops: the stand-alone twin of katago_b200/match_cli.py.
//
//   b200_match -config match.cfg -sgf-output-dir DIR [-log-file FILE] [-games-per-gpu N] [-override-config k=v,..] [-seed N] [-gpu I]
//
// numBots = 2, botName0 / botName1, nnModelFile0 / nnModelFile1 (or one nnModelFile), numGamesTotal; a search key with the bot's index appended
// (maxVisits0 ...) overrides the shared one for that bot.  The bots alternate colours, every game's board size / rules / komi come from the
// reference's per-game keys, one game record per line goes to <sgf-output-dir>/<16 hex>.sgfs (integration/b200_match.h: two device loops, one per
// net).  Plain C++17 over the C ABI - no CUDA headers, no reference headers, no Python.
#include "b200_config.h"
#include "b200_match.h"

using namespace b200host;

int main(int argc, char** argv) {
  programName() = "b200_match";
  std::string cfgPath, sgfDir, logFile, overrides;
  int gamesPerGpu = 128, gpu = 0; long seed = 0;
  for(int i = 1; i < argc; i++) {
    const std::string k = argv[i];
    auto next = [&]() { if(i + 1 >= argc) die("missing value after " + k); return std::string(argv[++i]); };
    if(k == "-config") cfgPath = next();
    else if(k == "-sgf-output-dir") sgfDir = next();
    else if(k == "-log-file") logFile = next();
    else if(k == "-games-per-gpu") gamesPerGpu = std::atoi(next().c_str());
    else if(k == "-override-config") overrides = next();
    else if(k == "-seed") seed = std::atol(next().c_str());
    else if(k == "-gpu") gpu = std::atoi(next().c_str());
    else if(k == "-help" || k == "--help") { std::printf("usage: %s -config FILE -sgf-output-dir DIR [-log-file FILE] [-games-per-gpu N] [-override-config k=v,...] [-seed N] [-gpu I]\n", argv[0]); return 0; }
    else die("unknown argument " + k);
  }
  if(cfgPath.empty() || sgfDir.empty()) die("-config and -sgf-output-dir are required (-help)");
  Cfg cfg;
  cfg.load(cfgPath);
  cfg.overrides(overrides);
  std::ofstream logf;
  if(!logFile.empty()) logf.open(logFile, std::ios::app);
  auto log = [&](const std::string& s) { std::fprintf(stderr, "%s\n", s.c_str()); if(logf.is_open()) { logf << s << "\n"; logf.flush(); } };
  auto check = [](int rc, const char* what) { if(rc != 0) die(std::string(what) + ": " + kgb_last_error()); };

  if((int)cfg.num("numBots", 2) != 2) die("match: exactly two bots are built (numBots = 2)");
  for(const char* k : {"secondaryBots", "extraPairs", "includeBots"}) if(cfg.has(k)) die(std::string("match: ") + k + " is not built");
  std::string names[2], files[2];
  for(int i = 0; i < 2; i++) {
    if(!cfg.has("botName" + std::to_string(i))) die("If more than one bot, must specify botName0, botName1,... individually");
    names[i] = cfg.str("botName" + std::to_string(i), "");
    files[i] = cfg.str("nnModelFile" + std::to_string(i), cfg.str("nnModelFile", ""));
    if(files[i].empty()) die("match: nnModelFile0 / nnModelFile1 (or nnModelFile) required");
  }
  const long total = (long)cfg.num("numGamesTotal", 0);
  if(total <= 0) die("match: numGamesTotal must be positive");
  const int games = (int)std::max(2L, std::min(std::min((long)gamesPerGpu, (long)cfg.num("numGameThreads", gamesPerGpu)), total));
  check(kgb_global_init(), "kgb_global_init");
  log("Match Engine starting...");
  {
    // the reference's katago match loads its bots with SETUP_FOR_MATCH, where both default to true (program/setup.cpp:522-544); an unset
    // key stays off here, so that existing match configurations keep playing the same games (katago_b200/match_cli.py match_default_note)
    std::vector<std::string> absent;
    for(const std::string k : {"useUncertainty", "useNoisePruning"}) {
      bool set = cfg.has(k);
      for(const auto& kv : cfg.kv)
        set = set || (kv.first.size() > k.size() && kv.first.compare(0, k.size(), k) == 0 &&
                      kv.first.find_first_not_of("0123456789", k.size()) == std::string::npos);
      if(!set) absent.push_back(k);
    }
    if(!absent.empty()) {
      std::string line = "[config] " + absent[0] + (absent.size() > 1 ? " and " + absent[1] : "") +
                         " not set: off here, while the reference's katago match defaults " + (absent.size() > 1 ? "them" : "it") + " to true; set ";
      for(size_t i = 0; i < absent.size(); i++) line += (i ? ", " : "") + absent[i] + " = true";
      log(line + " to search like it");
    }
  }

  kgb_model* models[2]; kgb_context* ctxs[2]; kgb_handle* handles[2];
  std::unique_ptr<b200::GameSlots> loops[2];
  b200::MatchPlay::Settings ms;
  ms.numGamesTotal = total; ms.drawEquivalentWinsForWhite = 0.5; ms.noResultUtilityForWhite = 0.0;
  ms.allowResignation = cfg.flag("allowResignation", false); ms.resignThreshold = cfg.num("resignThreshold", -0.90); ms.resignConsecTurns = (int)cfg.num("resignConsecTurns", 5);
  int edge = 19;
  b200::GameInitializer::Config gi;
  for(int i = 0; i < 2; i++) {
    Cfg mine = botCfg(cfg, i);
    mine.kv.erase("numBots"); mine.kv.erase("numGamesTotal");
    if(!mine.has("maxVisits")) mine.kv["maxVisits"] = "500";
    if(i == 0) gi = gameInitConfigFromCfg(mine, &edge);
    kgb_selfplay_config c = configFromCfg(mine, games);
    if(i == 0) { markIrrelevantKeys(mine); for(const std::string& what : mine.notBuilt) log("[config] NOT BUILT, ignored: " + what); }
    c.seed = (uint64_t)(seed * 7919 + 31 * i + 1); c.max_playouts_per_wave = 0;
    ms.maxVisits[i] = c.max_visits;
    check(kgb_model_load_file(files[i].c_str(), nullptr, &models[i]), "loading a model");
    check(kgb_context_create(&gpu, 1, edge, edge, 1, models[i], &ctxs[i]), "creating an evaluator context");
    check(kgb_handle_create(ctxs[i], models[i], games, 0, /*inputs_nhwc=*/1, gpu, &handles[i]), "creating an evaluator handle");
    loops[i].reset(new b200::GameSlots(handles[i], c, edge, edge));
    log("Loaded neural net " + std::to_string(i) + " from: " + files[i] + " for bot " + names[i] + " (maxVisits " + std::to_string(c.max_visits) + ")");
  }
  makeDirsFor(sgfDir);
  b200::RowRand nameRand("match" + std::to_string(seed));
  const uint64_t lo = nameRand.nextUInt(), hi = nameRand.nextUInt();
  char sgfName[32];
  std::snprintf(sgfName, sizeof(sgfName), "%016llX.sgfs", (unsigned long long)(lo | (hi << 32)));
  std::ofstream sgfs(sgfDir + "/" + sgfName, std::ios::app);
  if(!sgfs) die("cannot write the game records");

  long wins[2] = {0, 0}, draws = 0;
  b200::GameInitializer init(gi, (uint64_t)seed ^ 0x4D617463ULL);
  {
    b200::MatchPlay* mpPtr = nullptr;
    b200::MatchPlay mp(*loops[0], *loops[1], names[0], names[1], ms, &init,
                       [&](int, const b200::FinishedGame& game, const std::string& bName, const std::string& wName, const std::string& result) {
      sgfs << b200::writeSgf(game, bName, wName) << "\n";
      sgfs.flush();
      if(result[0] == 'B') wins[bName == names[0] ? 0 : 1]++;
      else if(result[0] == 'W') wins[wName == names[0] ? 0 : 1]++;
      else draws++;
      log("Game " + std::to_string(mpPtr->gamesTallied() - 1) + ": " + bName + " (black) vs " + wName + " (white): " + result + " in " + std::to_string(game.moves.size()) + " moves");
    });
    mpPtr = &mp;
    mp.run((int)cfg.num("b200WavesPerPoll", 8), nullptr);
    char buf[256];
    std::snprintf(buf, sizeof(buf), "Match finished: %s %ld wins, %s %ld wins, %ld draws or void; points %.1f - %.1f in %ld games", names[0].c_str(), wins[0], names[1].c_str(), wins[1], draws,
                  mp.winPoints(0), mp.winPoints(1), mp.gamesTallied());
    log(buf);
  }
  for(int i = 0; i < 2; i++) { loops[i].reset(); kgb_handle_free(handles[i]); kgb_context_free(ctxs[i]); kgb_model_free(models[i]); }
  kgb_global_cleanup();
  return 0;
}
