// oracle/ref_driver.cpp - TEST INFRASTRUCTURE.  Links against the unmodified reference (oracle/_ref/libkgref.a) and
// dumps golden fixtures / answers parity queries straight from the reference's own classes.  Never shipped or timed as
// product.  Built by oracle/Makefile.drivers into oracle/_ref/kgref_driver.
//
//   kgref_driver searchfake MODELFILE X Y MAXVISITS "x,y x,y pass ..." [STATIC DYNAMIC ZEROWEIGHT SCALE]
//       reference Search (search/search.cpp) with the deterministic hash-based fake net defined below as its NeuralNet
//       backend (this file IS the backend TU of the driver); prints the root children's visit counts.  The device loop
//       has the same fake net (kgb_selfplay_config.debug_fake_nn) so tree parity is tested without any real net.  With env
//       KGREF_FAKE_TABLE=<file> the net is the table net instead: fixed raw outputs read from the file (debug_fake_nn = 3); with
//       KGREF_FAKE_WIDE=1 the wide hash net (debug_fake_nn = 4), and the counts of the branches its evaluations took.
//   kgref_driver featstream X Y MULTISUICIDE KOMI "x,y x,y pass ..." EVERY OUT.bin
//       NNInputs::fillRowV7 (neuralnet/nninputs.cpp:2288-2731) rows along a game played through BoardHistory with the rule
//       subset of the device loop (area scoring, simple ko, no tax): after every EVERY-th move writes the NHWC row + globals.
//   kgref_driver ladderrows IN.txt OUT.bin
//       fillRowV7 rows of many positions (one per line of IN.txt) and the time of each position's slowest ladder search.
//   kgref_driver boardstream X Y NMOVES SEED MULTISUICIDE OUT.bin
//       random legal move stream on a reference Board (game/board.h): after every move records the board, ko, capture
//       counters, pos_hash, per-stone liberty counts, the legality mask of the player to move next and the Benson pass-alive /
//       territory area (Board::calculateArea, all flags on).
#include <fstream>

#include "game/board.h"
#include "game/boardhistory.h"
#include "game/rules.h"
#include "neuralnet/nninputs.h"
#include "neuralnet/nninterface.h"
#include "neuralnet/nneval.h"
#include "search/search.h"
#include "search/searchnode.h"
#include "search/distributiontable.h"
#include "core/fancymath.h"
#include "dataio/numpywrite.h"
#include "dataio/trainingwrite.h"
#include "program/play.h"
#include "program/playutils.h"
#include "dataio/sgf.h"
#include "program/setup.h"
#include "core/config_parser.h"
#include "integration/b200params.h"
#include "core/logger.h"
#include "core/timer.h"

#include <cstdint>
#include <cstdio>
#include <cstring>
#include <fstream>
#include <iostream>
#include <sstream>
#include <vector>

using namespace std;

namespace Version {  // main.cpp normally defines these (cpp/main.h)
  std::string getKataGoVersion() { return "ref_driver"; }
  std::string getKataGoVersionForHelp() { return "ref_driver"; }
  std::string getKataGoVersionFullInfo() { return "ref_driver"; }
  std::string getGitRevision() { return "<none>"; }
  std::string getGitRevisionWithBackend() { return "<none>"; }
}

struct Lcg {  // driver-local PRNG (the move stream only needs to be reproducible, not KataGo's Rand)
  uint64_t s;
  explicit Lcg(uint64_t seed) : s(seed * 0x9E3779B97F4A7C15ULL + 12345) {}
  uint32_t next() { s = s * 6364136223846793005ULL + 1442695040888963407ULL; return (uint32_t)(s >> 33); }
};

template <class T> static void put(ofstream& o, T v) { o.write((const char*)&v, sizeof(T)); }

static int cmdBoardStream(int argc, char** argv) {
  if(argc != 8) { cerr << "usage: boardstream X Y NMOVES SEED MULTISUICIDE OUT" << endl; return 1; }
  int X = atoi(argv[2]), Y = atoi(argv[3]), nMoves = atoi(argv[4]);
  uint64_t seed = strtoull(argv[5], NULL, 10);
  bool multi = atoi(argv[6]) != 0;
  Board::initHash();
  Board board(X, Y);
  Lcg rng(seed);
  ofstream out(argv[7], ios::binary);
  put<int32_t>(out, X); put<int32_t>(out, Y); put<int32_t>(out, nMoves); put<int32_t>(out, multi ? 1 : 0);
  Player pla = P_BLACK;
  for(int step = 0; step < nMoves; step++) {
    vector<Loc> legal;
    for(int y = 0; y < Y; y++)
      for(int x = 0; x < X; x++) {
        Loc loc = Location::getLoc(x, y, X);
        if(board.isLegal(loc, pla, multi)) legal.push_back(loc);
      }
    Loc mv;
    if(legal.empty() || rng.next() % 40 == 0) mv = Board::PASS_LOC;
    else mv = legal[rng.next() % legal.size()];
    board.playMoveAssumeLegal(mv, pla);
    int8_t mx = -1, my = -1;
    if(mv != Board::PASS_LOC) { mx = (int8_t)Location::getX(mv, X); my = (int8_t)Location::getY(mv, X); }
    put<int8_t>(out, mx); put<int8_t>(out, my); put<int8_t>(out, (int8_t)pla);
    int8_t kx = -1, ky = -1;
    if(board.ko_loc != Board::NULL_LOC) { kx = (int8_t)Location::getX(board.ko_loc, X); ky = (int8_t)Location::getY(board.ko_loc, X); }
    put<int8_t>(out, kx); put<int8_t>(out, ky);
    put<int16_t>(out, (int16_t)board.numBlackCaptures); put<int16_t>(out, (int16_t)board.numWhiteCaptures);
    put<uint64_t>(out, board.pos_hash.hash0); put<uint64_t>(out, board.pos_hash.hash1);
    Player next = getOpp(pla);
    for(int y = 0; y < Y; y++)
      for(int x = 0; x < X; x++) {
        Loc loc = Location::getLoc(x, y, X);
        put<uint8_t>(out, (uint8_t)board.colors[loc]);
      }
    for(int y = 0; y < Y; y++)
      for(int x = 0; x < X; x++) {
        Loc loc = Location::getLoc(x, y, X);
        int libs = (board.colors[loc] == P_BLACK || board.colors[loc] == P_WHITE) ? board.getNumLiberties(loc) : 0;
        put<uint8_t>(out, (uint8_t)std::min(libs, 255));
      }
    for(int y = 0; y < Y; y++)
      for(int x = 0; x < X; x++) {
        Loc loc = Location::getLoc(x, y, X);
        put<uint8_t>(out, board.isLegal(loc, next, multi) ? 1 : 0);
      }
    // Board::calculateArea as fillRowV7 calls it for area scoring / no tax (nninputs.cpp:2375-2382): all three flags on
    Color area[Board::MAX_ARR_SIZE];
    board.calculateArea(area, true, true, true, multi);
    for(int y = 0; y < Y; y++)
      for(int x = 0; x < X; x++) put<uint8_t>(out, (uint8_t)area[Location::getLoc(x, y, X)]);
    pla = next;
  }
  return 0;
}


// ------------------------------------------------------------------------------------------------------------
// Fake NeuralNet backend of this driver: logits are exact dyadic rationals derived from an order-independent integer hash of
// the stone planes (features 1,2) and the sign of selfKomi, so the CUDA side reproduces them bit-for-bit.
// ------------------------------------------------------------------------------------------------------------
static inline uint64_t splitmix64(uint64_t x) {
  x += 0x9E3779B97F4A7C15ULL;
  x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ULL;
  x = (x ^ (x >> 27)) * 0x94D049BB133111EBULL;
  return x ^ (x >> 31);
}
// The table net (env KGREF_FAKE_TABLE=<file> of searchfake): every evaluation returns the raw outputs listed in the file, whatever the
// position - policy logits [nnXLen*nnYLen+1], value logits [3], score-value channels [6], ownership logits [nnXLen*nnYLen], as text floats
// (the device loop's debug_fake_nn = 3 is given the same numbers)
static std::vector<float> fakeTable;
// The wide hash net (env KGREF_FAKE_WIDE=1 of searchfake; the device loop's debug_fake_nn = 4): the same hash with wider output
// ranges, and how many of its evaluations took each branch of the post-processing that the narrow net never reaches: P(no result)
// > 0.05; superko removing a no-result probability > 0.05; stdev logit > 40 (linear softplus branch); a policy term whose exp
// underflows to 0 in float
static bool fakeWide = false;
static bool fakeSuperko = false;
static long long wideBranches[4] = {0, 0, 0, 0};
#ifndef KGREF_EXTERNAL_BACKEND   // kgref_driver_b200 (oracle/Makefile.drivers) links integration/b200backend.cpp instead: the same commands on a real net
struct LoadedModel { ModelDesc modelDesc; };
struct ComputeContext { int nnXLen, nnYLen; };
struct ComputeHandle { int nnXLen, nnYLen; };
struct InputBuffers { int dummy; };
void NeuralNet::globalInitialize() {}
void NeuralNet::globalCleanup() {}
void NeuralNet::printDevices() {}
LoadedModel* NeuralNet::loadModelFile(const string& file, const string& expectedSha256) {
  LoadedModel* m = new LoadedModel();
  ModelDesc::loadFromFileMaybeGZipped(file, m->modelDesc, expectedSha256);
  return m;
}
void NeuralNet::freeLoadedModel(LoadedModel* m) { delete m; }
const ModelDesc& NeuralNet::getModelDesc(const LoadedModel* m) { return m->modelDesc; }
ComputeContext* NeuralNet::createComputeContext(const std::vector<int>&, Logger*, int nnXLen, int nnYLen, const string&, enabled_t, const LoadedModel*, ConfigParser&) {
  ComputeContext* c = new ComputeContext(); c->nnXLen = nnXLen; c->nnYLen = nnYLen; return c;
}
void NeuralNet::freeComputeContext(ComputeContext* c) { delete c; }
ComputeHandle* NeuralNet::createComputeHandle(ComputeContext* c, const LoadedModel*, Logger*, int, bool, bool inputsUseNHWC, int, int) {
  if(!inputsUseNHWC) throw StringError("fake backend wants NHWC");
  ComputeHandle* h = new ComputeHandle(); h->nnXLen = c->nnXLen; h->nnYLen = c->nnYLen; return h;
}
void NeuralNet::freeComputeHandle(ComputeHandle* h) { delete h; }
bool NeuralNet::isUsingFP16(const ComputeHandle*) { return false; }
bool NeuralNet::setIsWarmup(const ComputeHandle*, bool) { return false; }
InputBuffers* NeuralNet::createInputBuffers(const LoadedModel*, int, int, int) { return new InputBuffers(); }
void NeuralNet::freeInputBuffers(InputBuffers* b) { delete b; }
void NeuralNet::getOutput(ComputeHandle* h, InputBuffers*, int n, NNResultBuf** inputBufs, vector<NNOutput*>& outputs) {
  const int xy = h->nnXLen * h->nnYLen;
  if(!fakeTable.empty()) {
    if(fakeTable.size() != (size_t)(2 * xy + 10)) throw StringError("KGREF_FAKE_TABLE: wrong number of values for the frame");
    for(int r = 0; r < n; r++) {
      NNOutput* o = outputs[r];
      const float* t = fakeTable.data();
      std::copy(t, t + xy + 1, o->policyProbs);
      t += xy + 1;
      o->whiteWinProb = t[0]; o->whiteLossProb = t[1]; o->whiteNoResultProb = t[2];
      o->whiteScoreMean = t[3]; o->whiteScoreMeanSq = t[4]; o->whiteLead = t[5];
      o->varTimeLeft = t[6]; o->shorttermWinlossError = t[7]; o->shorttermScoreError = t[8];
      if(o->whiteOwnerMap != NULL) std::copy(t + 9, t + 9 + xy, o->whiteOwnerMap);
    }
    return;
  }
  for(int r = 0; r < n; r++) {
    const float* sp = inputBufs[r]->rowSpatialBuf.data();
    const float* gl = inputBufs[r]->rowGlobalBuf.data();
    uint64_t hsh = 0;
    for(int pos = 0; pos < xy; pos++) {
      int s = sp[pos * 22 + 1] != 0.0f ? 1 : sp[pos * 22 + 2] != 0.0f ? 2 : 0;
      if(s) hsh += splitmix64((uint64_t)pos * 4 + s);
    }
    if(gl[5] < 0.0f) hsh ^= 0xABCDEFULL;
    // a net that answers differently per requested symmetry (always in the original orientation), for rootNumSymmetriesToSample
    if(inputBufs[r]->symmetry != 0) hsh ^= splitmix64(0x5151ULL + (uint64_t)inputBufs[r]->symmetry);
    NNOutput* o = outputs[r];
    float maxLogit = -1e30f;
    for(int i = 0; i <= xy; i++) {
      uint32_t u = (uint32_t)(splitmix64(hsh + (uint64_t)(i + 1) * 0x9E3779B97F4A7C15ULL) >> 48);
      float logit = fakeWide ? (float)u * (3.0f / 4096.0f) - 24.0f : (float)u * (1.0f / 8192.0f) - 4.0f;
      if(fakeWide && (u & 15u) == 0u) logit -= 96.0f;
      if(i == xy) logit -= 3.0f;
      o->policyProbs[i] = logit;
      maxLogit = std::max(maxLogit, logit);
    }
    if(fakeWide) {
      o->whiteWinProb = (float)(uint32_t)(splitmix64(hsh ^ 0x1111ULL) >> 48) * (3.0f / 16384.0f) - 6.0f;
      o->whiteLossProb = (float)(uint32_t)(splitmix64(hsh ^ 0x2222ULL) >> 48) * (3.0f / 16384.0f) - 6.0f;
      o->whiteNoResultProb = (float)(uint32_t)(splitmix64(hsh ^ 0x8888ULL) >> 48) * (3.0f / 16384.0f) - 6.0f;
      o->whiteScoreMean = (float)(uint32_t)(splitmix64(hsh ^ 0x3333ULL) >> 48) * (3.0f / 32768.0f) - 3.0f;
      o->whiteScoreMeanSq = (float)(uint32_t)(splitmix64(hsh ^ 0x4444ULL) >> 48) * (1.0f / 1024.0f) - 8.0f;
      o->whiteLead = (float)(uint32_t)(splitmix64(hsh ^ 0x5555ULL) >> 48) * (3.0f / 32768.0f) - 3.0f;
      o->varTimeLeft = 0; o->shorttermWinlossError = 0; o->shorttermScoreError = 0;
      const double w = o->whiteWinProb, l = o->whiteLossProb, nr = o->whiteNoResultProb, m = std::max(std::max(w, l), nr);
      const double pNoResult = exp(nr - m) / (exp(w - m) + exp(l - m) + exp(nr - m));
      if(pNoResult > 0.05) { wideBranches[0]++; if(fakeSuperko) wideBranches[1]++; }
      if(o->whiteScoreMeanSq > 40.0f) wideBranches[2]++;
      bool underflow = false;
      for(int i = 0; i <= xy; i++) underflow = underflow || expf(o->policyProbs[i] - maxLogit) == 0.0f;
      if(underflow) wideBranches[3]++;
    }
    else {
    o->whiteWinProb = (float)(uint32_t)(splitmix64(hsh ^ 0x1111ULL) >> 48) * (1.0f / 8192.0f) - 4.0f;
    o->whiteLossProb = (float)(uint32_t)(splitmix64(hsh ^ 0x2222ULL) >> 48) * (1.0f / 8192.0f) - 4.0f;
    o->whiteNoResultProb = -30.0f;
    // raw score head: mean in [-1,1) (x scoreMeanMultiplier 20 = +-20 points), stdev pre-softplus in [-2,2), lead like mean
    o->whiteScoreMean = (float)(uint32_t)(splitmix64(hsh ^ 0x3333ULL) >> 48) * (1.0f / 32768.0f) - 1.0f;
    o->whiteScoreMeanSq = (float)(uint32_t)(splitmix64(hsh ^ 0x4444ULL) >> 48) * (1.0f / 16384.0f) - 2.0f;
    o->whiteLead = (float)(uint32_t)(splitmix64(hsh ^ 0x5555ULL) >> 48) * (1.0f / 32768.0f) - 1.0f;
    o->varTimeLeft = 0; o->shorttermWinlossError = 0; o->shorttermScoreError = 0;
    }
    // raw ownership logits in [-4,4) per point (mover's perspective; NNEvaluator applies tanh and the colour flip, nneval.cpp:1233-1250):
    // about half of the points end beyond |tanh| = 0.95, where Search::getEndingWhiteScoreBonus acts
    if(o->whiteOwnerMap != NULL)
      for(int i = 0; i < xy; i++)
        o->whiteOwnerMap[i] = (float)(uint32_t)(splitmix64(hsh + (uint64_t)(i + 1) * 0xD1B54A32D192ED03ULL) >> 48) * (1.0f / 8192.0f) - 4.0f;
  }
}
bool NeuralNet::testEvaluateConv(const ConvLayerDesc*, int, int, int, bool, bool, const std::vector<float>&, std::vector<float>&) { return false; }
bool NeuralNet::testEvaluateBatchNorm(const BatchNormLayerDesc*, int, int, int, bool, bool, const std::vector<float>&, const std::vector<float>&, std::vector<float>&) { return false; }
bool NeuralNet::testEvaluateResidualBlock(const ResidualBlockDesc*, int, int, int, bool, bool, const std::vector<float>&, const std::vector<float>&, std::vector<float>&) { return false; }
bool NeuralNet::testEvaluateGlobalPoolingResidualBlock(const GlobalPoolingResidualBlockDesc*, int, int, int, bool, bool, const std::vector<float>&, const std::vector<float>&, std::vector<float>&) { return false; }

#endif

static int cmdSearchFake(int argc, char** argv) {
  if(argc < 7) { cerr << "usage: searchfake MODELFILE X Y MAXVISITS MOVES [key=value ...]" << endl; return 1; }
  string modelFile = argv[2];
  int X = atoi(argv[3]), Y = atoi(argv[4]), maxVisits = atoi(argv[5]);
  Board::initHash();
  ScoreValue::initTables();
  Logger logger(nullptr, false, false, false);
  ConfigParser cfg;
  // KGREF_NN_CACHE_POW2 = -1 switches NNEvaluator's evaluation cache off (it is keyed by the situation, not the history: with a real net a
  // transposition then returns the output computed for another move order - fine for play, but not what a cache-less search sees)
  if(getenv("KGREF_FAKE_TABLE")) {
#ifdef KGREF_EXTERNAL_BACKEND
    cerr << "KGREF_FAKE_TABLE needs the driver's own fake backend" << endl; return 1;
#endif
    std::ifstream in(getenv("KGREF_FAKE_TABLE"));
    float v;
    while(in >> v) fakeTable.push_back(v);
    if(fakeTable.empty()) { cerr << "KGREF_FAKE_TABLE: no values read" << endl; return 1; }
  }
  fakeWide = getenv("KGREF_FAKE_WIDE") && atoi(getenv("KGREF_FAKE_WIDE")) != 0;
  const int cachePow2 = getenv("KGREF_NN_CACHE_POW2") ? atoi(getenv("KGREF_NN_CACHE_POW2")) : 10;
  // KGREF_NN_LEN = L: the evaluator's frame is L x L while the board is X x Y (nnXLen > board size: padded rows + mask, nneval.cpp:874-883;
  // BASELINE config 4 "mixed board sizes"); move positions and the policy are then indexed in the frame (NNPos::locToPos)
  const int nnLenEnv = getenv("KGREF_NN_LEN") ? atoi(getenv("KGREF_NN_LEN")) : 0;
  const int NX = nnLenEnv > 0 ? nnLenEnv : X, NY = nnLenEnv > 0 ? nnLenEnv : Y;
  if(NX < X || NY < Y) { cerr << "KGREF_NN_LEN smaller than the board" << endl; return 1; }
  NNEvaluator* nnEval = new NNEvaluator("fake", modelFile, "", &logger, 4, NX, NY, NX == X && NY == Y, true, cachePow2, 8, false, "", enabled_t::False, 1,
                                        vector<int>{0}, "seed", false, 0, true, cfg);
  nnEval->spawnServerThreads();
  // Reference SearchParams restricted to what the device loop implements (DESIGN.md §8): everything else at its default.
  int koRuleOverride = 0;
  SearchParams params;
  params.maxVisits = maxVisits;
  params.numThreads = 1;
  params.cpuctExploration = 1.0; params.cpuctExplorationLog = 0.45; params.cpuctExplorationBase = 500;
  params.fpuReductionMax = 0.2; params.rootFpuReductionMax = 0.1;
  params.staticScoreUtilityFactor = 0.0; params.dynamicScoreUtilityFactor = 0.0;
  params.valueWeightExponent = 0.0;
  params.rootNoiseEnabled = false;
  for(int i = 7; i < argc; i++) {   // SearchParams overrides, by their cfg names
    string kv = argv[i];
    size_t eq = kv.find('=');
    if(eq == string::npos) { cerr << "bad override " << kv << endl; return 1; }
    string k = kv.substr(0, eq); double v = atof(kv.substr(eq + 1).c_str());
    if(k == "staticScoreUtilityFactor") params.staticScoreUtilityFactor = v;
    else if(k == "dynamicScoreUtilityFactor") params.dynamicScoreUtilityFactor = v;
    else if(k == "dynamicScoreCenterZeroWeight") params.dynamicScoreCenterZeroWeight = v;
    else if(k == "dynamicScoreCenterScale") params.dynamicScoreCenterScale = v;
    else if(k == "valueWeightExponent") params.valueWeightExponent = v;
    else if(k == "fpuParentWeightByVisitedPolicy") params.fpuParentWeightByVisitedPolicy = v != 0;
    else if(k == "fpuParentWeightByVisitedPolicyPow") params.fpuParentWeightByVisitedPolicyPow = v;
    else if(k == "fpuParentWeight") params.fpuParentWeight = v;
    else if(k == "fpuLossProp") params.fpuLossProp = v;
    else if(k == "rootFpuLossProp") params.rootFpuLossProp = v;
    else if(k == "fpuReductionMax") params.fpuReductionMax = v;
    else if(k == "rootFpuReductionMax") params.rootFpuReductionMax = v;
    else if(k == "cpuctExploration") params.cpuctExploration = v;
    else if(k == "cpuctExplorationLog") params.cpuctExplorationLog = v;
    else if(k == "cpuctUtilityStdevScale") params.cpuctUtilityStdevScale = v;
    else if(k == "cpuctUtilityStdevPrior") params.cpuctUtilityStdevPrior = v;
    else if(k == "cpuctUtilityStdevPriorWeight") params.cpuctUtilityStdevPriorWeight = v;
    else if(k == "rootDesiredPerChildVisitsCoeff") params.rootDesiredPerChildVisitsCoeff = v;
    else if(k == "rootNumSymmetriesToSample") params.rootNumSymmetriesToSample = (int)v;
    else if(k == "koRule") koRuleOverride = (int)v;
    else if(k == "useLcbForSelection") params.useLcbForSelection = v != 0;
    else if(k == "useNonBuggyLcb") params.useNonBuggyLcb = v != 0;
    else if(k == "lcbStdevs") params.lcbStdevs = v;
    else if(k == "minVisitPropForLCB") params.minVisitPropForLCB = v;
    else if(k == "chosenMoveSubtract") params.chosenMoveSubtract = v;
    else if(k == "chosenMovePrune") params.chosenMovePrune = v;
    else if(k == "rootPolicyTemperature") params.rootPolicyTemperature = v;
    else if(k == "rootPolicyTemperatureEarly") params.rootPolicyTemperatureEarly = v;
    else if(k == "chosenMoveTemperatureHalflife") params.chosenMoveTemperatureHalflife = v;
    else if(k == "useGraphSearch") params.useGraphSearch = v != 0;
    else if(k == "graphSearchRepBound") params.graphSearchRepBound = (int)v;
    else if(k == "subtreeValueBiasFactor") params.subtreeValueBiasFactor = v;
    else if(k == "subtreeValueBiasWeightExponent") params.subtreeValueBiasWeightExponent = v;
    else if(k == "rootEndingBonusPoints") params.rootEndingBonusPoints = v;
    else if(k == "rootPruneUselessMoves") params.rootPruneUselessMoves = v != 0;
    else if(k == "noResultUtilityForWhite") params.noResultUtilityForWhite = v;
    else if(k == "winLossUtilityFactor") params.winLossUtilityFactor = v;
    else if(k == "drawEquivalentWinsForWhite") params.drawEquivalentWinsForWhite = v;
    else if(k == "useUncertainty") params.useUncertainty = v != 0;
    else if(k == "uncertaintyCoeff") params.uncertaintyCoeff = v;
    else if(k == "uncertaintyExponent") params.uncertaintyExponent = v;
    else if(k == "uncertaintyMaxWeight") params.uncertaintyMaxWeight = v;
    else { cerr << "unknown override " << k << endl; return 1; }
  }
  Rules rules;  // defaults, then the rule subset of the loop
  rules.koRule = koRuleOverride == 1 ? Rules::KO_POSITIONAL : koRuleOverride == 2 ? Rules::KO_SITUATIONAL : Rules::KO_SIMPLE;
  fakeSuperko = rules.koRule != Rules::KO_SIMPLE;
  rules.scoringRule = Rules::SCORING_AREA; rules.taxRule = Rules::TAX_NONE;
  rules.multiStoneSuicideLegal = true; rules.hasButton = false; rules.whiteHandicapBonusRule = Rules::WHB_ZERO;
  rules.friendlyPassOk = false; rules.komi = 7.5f;
  Board board(X, Y);
  Player pla = P_BLACK;
  BoardHistory hist(board, pla, rules, 0, false);
  {
    std::istringstream in(argv[6]);
    string tok;
    while(in >> tok) {
      Loc loc;
      if(tok == "pass") loc = Board::PASS_LOC;
      else { int x, y; if(sscanf(tok.c_str(), "%d,%d", &x, &y) != 2) { cerr << "bad move " << tok << endl; return 1; } loc = Location::getLoc(x, y, X); }
      if(!hist.isLegal(board, loc, pla)) { cerr << "illegal move " << tok << endl; return 1; }
      hist.makeBoardMoveAssumeLegal(board, loc, pla, NULL);
      pla = getOpp(pla);
    }
  }
  Search* search = new Search(params, nnEval, &logger, "searchfake");
  search->setPosition(pla, board, hist);
  search->runWholeSearch(pla);
  const SearchNode* root = search->rootNode;
  SearchNodeState st = (SearchNodeState)root->state.load();
  ConstSearchNodeChildrenReference children = root->getChildren(st);
  cout << "rootvisits " << root->stats.visits.load() << " utilityAvg " << Global::strprintf("%.17g", root->stats.utilityAvg.load()) << endl;
 {
    std::ostringstream ss;   // makeSeed(search, 0) (search.cpp:24-36): the seed string of search thread 0's Rand
    ss << "searchfake" << "$searchThread$" << 0 << "$" << board.pos_hash << "$" << hist.moveHistory.size() << "$" << search->numSearchesBegun;
    cout << "threadseed " << ss.str() << endl;
  }
 cout << "rootstats " << Global::strprintf("%.17g %.17g %.17g %.17g %.17g", root->stats.winLossValueAvg.load(), root->stats.noResultValueAvg.load(),
                                            root->stats.scoreMeanAvg.load(), root->stats.scoreMeanSqAvg.load(), root->stats.leadAvg.load()) << endl;
  cout << "recentScoreCenter " << Global::strprintf("%.17g", search->recentScoreCenter) << endl;
  for(int i = 0; i < children.getCapacity(); i++) {
    const SearchChildPointer& cp = children[i];
    const SearchNode* child = cp.getIfAllocated();
    if(child == NULL) break;
    Loc loc = cp.getMoveLoc();
    int x = loc == Board::PASS_LOC ? -1 : Location::getX(loc, X), y = loc == Board::PASS_LOC ? -1 : Location::getY(loc, X);
    cout << "child " << x << " " << y << " " << cp.getEdgeVisits() << " " << Global::strprintf("%.17g", child->stats.utilityAvg.load())
         << " " << Global::strprintf("%.17g %.17g %.17g %.17g %.17g", child->stats.winLossValueAvg.load(), child->stats.noResultValueAvg.load(),
                                     child->stats.scoreMeanAvg.load(), child->stats.scoreMeanSqAvg.load(), child->stats.leadAvg.load()) << endl;
  }
  {
    vector<Loc> locs; vector<double> psv;
    bool suc = search->getPlaySelectionValues(locs, psv, 0.0);
    cout << "playselection " << (suc ? 1 : 0);
    for(size_t i = 0; i < locs.size(); i++) {
      int x = locs[i] == Board::PASS_LOC ? -1 : Location::getX(locs[i], X), y = locs[i] == Board::PASS_LOC ? -1 : Location::getY(locs[i], X);
      cout << " " << x << " " << y << " " << Global::strprintf("%.17g", psv[i]);
    }
    cout << endl;
  }
  cout << "rootweight " << Global::strprintf("%.17g %.17g", root->stats.weightSum.load(), root->stats.weightSqSum.load()) << endl;
  const NNOutput* nn = root->getNNOutput();
  // the root's own evaluation as NNEvaluator post-processed it (nneval.cpp:1112-1215; white's perspective, floats)
  cout << "nnoutput " << Global::strprintf("%.9g %.9g %.9g %.9g %.9g %.9g %.9g %.9g", nn->whiteWinProb, nn->whiteLossProb, nn->whiteNoResultProb,
                                           nn->whiteScoreMean, nn->whiteScoreMeanSq, nn->whiteLead, nn->shorttermWinlossError, nn->shorttermScoreError) << endl;
  cout << "policy";
  for(int i = 0; i <= NX * NY; i++) cout << " " << Global::strprintf("%.9g", nn->getPolicyProbsMaybeNoised()[i]);
  cout << endl;
  {   // what Play::runGame records for this turn (program/play.cpp:848-948): value / Q / policy targets, surprise and entropies
    ReportedSearchValues rv;
    if(search->getNodeValues(root, rv))
      cout << "valuetargets " << Global::strprintf("%.9g %.9g %.9g %.9g", (float)rv.winValue, (float)rv.lossValue, (float)rv.noResultValue, (float)rv.expectedScore) << endl;
    double surprise = 0, searchEntropy = 0, policyEntropy = 0;
    if(search->getPolicySurpriseAndEntropy(surprise, searchEntropy, policyEntropy))
      cout << "surprise " << Global::strprintf("%.17g %.17g %.17g", surprise, searchEntropy, policyEntropy) << endl;
    for(int i = 0; i < children.getCapacity(); i++) {
      const SearchChildPointer& cp = children[i];
      const SearchNode* child = cp.getIfAllocated();
      if(child == NULL) break;
      ReportedSearchValues cv;
      if(!search->getNodeValues(child, cv) || cv.visits <= 0) continue;
      Loc loc = cp.getMoveLoc();
      int x = loc == Board::PASS_LOC ? -1 : Location::getX(loc, X), y = loc == Board::PASS_LOC ? -1 : Location::getY(loc, X);
      cout << "qtarget " << x << " " << y << " " << Global::strprintf("%.9g %.9g", (float)cv.winLossValue, (float)cv.expectedScore) << " " << cv.visits << endl;
    }
    if(children.getCapacity() > 0 && children[0].getIfAllocated() != NULL) {   // a 1-visit search has no child to take targets from
      vector<PolicyTargetMove> pt; vector<Loc> locsBuf; vector<double> psvBuf;
      Play::extractPolicyTarget(pt, search, root, locsBuf, psvBuf);
      cout << "policytarget";
      for(const PolicyTargetMove& m : pt) {
        int x = m.loc == Board::PASS_LOC ? -1 : Location::getX(m.loc, X), y = m.loc == Board::PASS_LOC ? -1 : Location::getY(m.loc, X);
        cout << " " << x << " " << y << " " << m.policyTarget;
      }
      cout << endl;
    }
  }
  if(fakeWide)
    cout << "widebranches " << wideBranches[0] << " " << wideBranches[1] << " " << wideBranches[2] << " " << wideBranches[3] << endl;
  delete search;
  delete nnEval;
  return 0;
}

// svsamples N SEED: N pseudo-random argument tuples and ScoreValue::expectedWhiteScoreValue of each (text, %.17g)
static int cmdSVSamples(int argc, char** argv) {
  if(argc != 4) { cerr << "usage: svsamples N SEED" << endl; return 1; }
  int n = atoi(argv[2]);
  Lcg rng(strtoull(argv[3], NULL, 10));
  ScoreValue::initTables();
  auto unit = [&]() { return (double)rng.next() / 2147483648.0; };
  for(int i = 0; i < n; i++) {
    static const double areas[4] = {19.0, 9.0, 13.0, 9.539392014169456};
    double sqrtArea = areas[rng.next() % 4];
    double mean = (unit() - 0.5) * (i % 7 == 0 ? 1200.0 : 80.0);
    double stdev = unit() * (i % 5 == 0 ? 600.0 : 30.0);
    if(i % 11 == 0) stdev = 0.0;
    double center = (i % 3 == 0) ? 0.0 : (unit() - 0.5) * 40.0;
    double scale = (i % 3 == 0) ? 2.0 : 0.25 + unit();
    double v = ScoreValue::expectedWhiteScoreValue(mean, stdev, center, scale, sqrtArea);
    cout << Global::strprintf("%.17g %.17g %.17g %.17g %.17g %.17g", mean, stdev, center, scale, sqrtArea, v) << endl;
  }
  return 0;
}

// vwtable: the value-weighting CDF table built the way Search's constructor builds it (search.cpp:131-137: the reference's
// DistributionTable over the reference's FancyMath::tdistcdf, 3 degrees of freedom), 2000 lines of %.17g
static int cmdVWTable(int, char**) {
  DistributionTable table(
    [](double z) { return FancyMath::tdistpdf(z, 3.0); },
    [](double z) { return FancyMath::tdistcdf(z, 3.0); },
    -50.0, 50.0, 2000);
  for(int i = 0; i < table.size; i++) cout << Global::strprintf("%.17g", table.cdfTable[i]) << endl;
  return 0;
}

// rootnoise SEEDSTRING POLICYSIZE POLICYSEED CONCENTRATION WEIGHT: Search::addDirichletNoise (searchhelpers.cpp:121-147) with
// Rand(SEEDSTRING) on a pseudo-random policy (some moves illegal = -1); prints the policy before and after.
static int cmdRootNoise(int argc, char** argv) {
  if(argc != 7) { cerr << "usage: rootnoise SEEDSTRING POLICYSIZE POLICYSEED CONCENTRATION WEIGHT" << endl; return 1; }
  Rand rand(argv[2]);
  int n = atoi(argv[3]);
  Lcg rng(strtoull(argv[4], NULL, 10));
  SearchParams params;
  params.rootDirichletNoiseTotalConcentration = atof(argv[5]);
  params.rootDirichletNoiseWeight = atof(argv[6]);
  vector<float> p(NNPos::MAX_NN_POLICY_SIZE, -1.0f);
  double sum = 0.0;
  for(int i = 0; i < n; i++) {
    bool legal = i == n - 1 || rng.next() % 5 != 0;
    if(legal) { double v = pow((double)rng.next() / 2147483648.0, 6.0) + 1e-7; p[i] = (float)v; sum += v; }
  }
  for(int i = 0; i < n; i++) if(p[i] >= 0) p[i] = (float)(p[i] / sum);
  cout << "in";
  for(int i = 0; i < n; i++) cout << " " << Global::strprintf("%.9g", p[i]);
  cout << endl;
  Search::addDirichletNoise(params, rand, n, p.data());
  cout << "out";
  for(int i = 0; i < n; i++) cout << " " << Global::strprintf("%.9g", p[i]);
  cout << endl;
  return 0;
}

// chooseidx SEEDSTRING N PROBSEED TEMPERATURE ONLYBELOWPROB COUNT: COUNT consecutive Search::chooseIndexWithTemperature draws
// (searchhelpers.cpp:12-76) from Rand(SEEDSTRING) over N pseudo-random relative weights (some zero); prints weights and draws.
static int cmdChooseIdx(int argc, char** argv) {
  if(argc != 8) { cerr << "usage: chooseidx SEEDSTRING N PROBSEED TEMPERATURE ONLYBELOWPROB COUNT" << endl; return 1; }
  Rand rand(argv[2]);
  int n = atoi(argv[3]);
  Lcg rng(strtoull(argv[4], NULL, 10));
  double temperature = atof(argv[5]), onlyBelow = atof(argv[6]);
  int count = atoi(argv[7]);
  vector<double> w(n);
  for(int i = 0; i < n; i++) w[i] = (rng.next() % 4 == 0) ? 0.0 : ceil(pow((double)rng.next() / 2147483648.0, 4.0) * 300.0);
  w[rng.next() % n] = 250.0;
  cout << "weights";
  for(int i = 0; i < n; i++) cout << " " << Global::strprintf("%.17g", w[i]);
  cout << endl << "draws";
  for(int i = 0; i < count; i++) cout << " " << Search::chooseIndexWithTemperature(rand, w.data(), n, temperature, onlyBelow, NULL);
  cout << endl;
  return 0;
}

// histstream X Y KORULE(0 simple,1 positional,2 situational,3 spight) MULTISUICIDE SEED NGAMES MAXMOVES OUT
//   random games through the reference's BoardHistory (area scoring): moves are drawn from BoardHistory::isLegal, passes with
//   probability 1/7 (also consecutive ones), until the history says the game is over.  Per move: flags (finished, noResult,
//   passWouldEndPhase for the next player), hist.isLegal of every point for the next player, hist.superKoBanned.
static int cmdHistStream(int argc, char** argv) {
  if(argc != 10) { cerr << "usage: histstream X Y KORULE MULTISUICIDE SEED NGAMES MAXMOVES OUT" << endl; return 1; }
  int X = atoi(argv[2]), Y = atoi(argv[3]), koRule = atoi(argv[4]);
  bool multi = atoi(argv[5]) != 0;
  Lcg rng(strtoull(argv[6], NULL, 10));
  int nGames = atoi(argv[7]), maxMoves = atoi(argv[8]);
  Board::initHash();
  ScoreValue::initTables();
  Rules rules;
  rules.koRule = koRule == 0 ? Rules::KO_SIMPLE : koRule == 1 ? Rules::KO_POSITIONAL : koRule == 2 ? Rules::KO_SITUATIONAL : Rules::KO_SPIGHT;
  rules.scoringRule = Rules::SCORING_AREA; rules.taxRule = Rules::TAX_NONE;
  rules.multiStoneSuicideLegal = multi; rules.hasButton = false; rules.whiteHandicapBonusRule = Rules::WHB_ZERO;
  rules.friendlyPassOk = false; rules.komi = 7.5f;
  ofstream out(argv[9], ios::binary);
  put<int32_t>(out, X); put<int32_t>(out, Y); put<int32_t>(out, koRule); put<int32_t>(out, multi ? 1 : 0); put<int32_t>(out, nGames); put<int32_t>(out, maxMoves);
  for(int gi = 0; gi < nGames; gi++) {
    Board board(X, Y);
    Player pla = P_BLACK;
    BoardHistory hist(board, pla, rules, 0, false);
    vector<char> rec;
    int n = 0;
    while(n < maxMoves && !hist.isGameFinished) {
      vector<Loc> legal;
      for(int y = 0; y < Y; y++) for(int x = 0; x < X; x++) { Loc l = Location::getLoc(x, y, X); if(hist.isLegal(board, l, pla)) legal.push_back(l); }
      Loc mv = (legal.empty() || rng.next() % 7 == 0) ? Board::PASS_LOC : legal[rng.next() % legal.size()];
      hist.makeBoardMoveAssumeLegal(board, mv, pla, NULL);
      pla = getOpp(pla);
      rec.push_back(mv == Board::PASS_LOC ? -1 : (char)Location::getX(mv, X));
      rec.push_back(mv == Board::PASS_LOC ? -1 : (char)Location::getY(mv, X));
      char flags = (hist.isGameFinished ? 1 : 0) | (hist.isNoResult ? 2 : 0) | (hist.passWouldEndPhase(board, pla) ? 4 : 0);
      rec.push_back(flags);
      for(int y = 0; y < Y; y++) for(int x = 0; x < X; x++) rec.push_back(hist.isLegal(board, Location::getLoc(x, y, X), pla) ? 1 : 0);
      for(int y = 0; y < Y; y++) for(int x = 0; x < X; x++) rec.push_back(hist.superKoBanned[Location::getLoc(x, y, X)] ? 1 : 0);
      n++;
    }
    put<int32_t>(out, n);
    out.write(rec.data(), rec.size());
  }
  return 0;
}

// repbound X Y NMOVES SEED BOUND: random legal move stream (like boardstream); after every move prints x y pla and
// Board::simpleRepetitionBoundGt(moveLoc, BOUND) on the board after the move (game/board.cpp:2853-2888).
static int cmdRepBound(int argc, char** argv) {
  if(argc != 7) { cerr << "usage: repbound X Y NMOVES SEED BOUND" << endl; return 1; }
  int X = atoi(argv[2]), Y = atoi(argv[3]), nMoves = atoi(argv[4]), bound = atoi(argv[6]);
  Lcg rng(strtoull(argv[5], NULL, 10));
  Board::initHash();
  Board board(X, Y);
  Player pla = P_BLACK;
  for(int step = 0; step < nMoves; step++) {
    vector<Loc> legal;
    for(int y = 0; y < Y; y++) for(int x = 0; x < X; x++) { Loc l = Location::getLoc(x, y, X); if(board.isLegal(l, pla, true)) legal.push_back(l); }
    Loc mv = (legal.empty() || rng.next() % 30 == 0) ? Board::PASS_LOC : legal[rng.next() % legal.size()];
    board.playMoveAssumeLegal(mv, pla);
    int x = mv == Board::PASS_LOC ? -1 : Location::getX(mv, X), y = mv == Board::PASS_LOC ? -1 : Location::getY(mv, X);
    cout << x << " " << y << " " << (int)pla << " " << (board.simpleRepetitionBoundGt(mv, bound) ? 1 : 0) << endl;
    pla = getOpp(pla);
  }
  return 0;
}

// npyheader ROWS: the 256-byte NumPy headers the reference's NumpyBuffer writes (dataio/numpywrite.cpp:97-226) for the seven arrays of a
// training .npz with ROWS rows (trainingwrite.cpp:854-886), as hex, one line per array: name hex
static int cmdNpyHeader(int argc, char** argv) {
  if(argc != 3) { cerr << "usage: npyheader ROWS" << endl; return 1; }
  int64_t rows = atoll(argv[2]);
  const int64_t maxRows = rows > 4 ? rows : 4;
  auto dump = [&](const char* name, const char* hdr) {
    cout << name << " ";
    for(int i = 0; i < 256; i++) cout << Global::strprintf("%02x", (unsigned)(unsigned char)hdr[i]);
    cout << endl;
  };
  { NumpyBuffer<uint8_t> b({maxRows, 22, 46}); b.prepareHeaderWithNumRows(rows); dump("binaryInputNCHWPacked", (const char*)b.dataIncludingHeader); }
  { NumpyBuffer<float> b({maxRows, 19}); b.prepareHeaderWithNumRows(rows); dump("globalInputNC", (const char*)b.dataIncludingHeader); }
  { NumpyBuffer<int16_t> b({maxRows, 2, 362}); b.prepareHeaderWithNumRows(rows); dump("policyTargetsNCMove", (const char*)b.dataIncludingHeader); }
  { NumpyBuffer<float> b({maxRows, 80}); b.prepareHeaderWithNumRows(rows); dump("globalTargetsNC", (const char*)b.dataIncludingHeader); }
  { NumpyBuffer<int8_t> b({maxRows, 842}); b.prepareHeaderWithNumRows(rows); dump("scoreDistrN", (const char*)b.dataIncludingHeader); }
  { NumpyBuffer<int8_t> b({maxRows, 5, 19, 19}); b.prepareHeaderWithNumRows(rows); dump("valueTargetsNCHW", (const char*)b.dataIncludingHeader); }
  { NumpyBuffer<int16_t> b({maxRows, 3, 362}); b.prepareHeaderWithNumRows(rows); dump("qValueTargetsNCMove", (const char*)b.dataIncludingHeader); }
  return 0;
}

// addrow X Y DATALEN NTURNS SEED NORESULT BONUS OUT.json [PASSALIVE]: TrainingWriteBuffers::addRow (dataio/trainingwrite.cpp:448-852) on a synthetic
// finished game: NTURNS random legal moves, random value / Q / policy targets, Benson ownership of the final board, random scoring
// plane; one row per turn with every optional argument toggled by the turn index.  Dumps each row's arguments and the seven
// buffers the reference filled.  The row Rand is Rand("addrow"+SEED), shared by all rows like the writer's own.
static int cmdAddRow(int argc, char** argv) {
  if(argc != 10 && argc != 11) { cerr << "usage: addrow X Y DATALEN NTURNS SEED NORESULT BONUS OUT.json [PASSALIVE]" << endl; return 1; }
  // PASSALIVE = 1: multi-stone suicide illegal, history flagged alwaysComputePassAliveUnderSuicideRules (global target 68, trainingwrite.cpp:702)
  const bool passAliveFlag = argc == 11 && atoi(argv[10]) != 0;
  const int X = atoi(argv[2]), Y = atoi(argv[3]), D = atoi(argv[4]), nTurns = atoi(argv[5]);
  const string seedStr = argv[6];
  const bool endNoResult = atoi(argv[7]) != 0;
  const float bonus = (float)atof(argv[8]);
  Board::initHash();
  ScoreValue::initTables();
  Rules rules;
  rules.koRule = Rules::KO_SIMPLE; rules.scoringRule = Rules::SCORING_AREA; rules.taxRule = Rules::TAX_NONE;
  rules.multiStoneSuicideLegal = !passAliveFlag; rules.hasButton = false; rules.whiteHandicapBonusRule = Rules::WHB_ZERO;
  rules.friendlyPassOk = false; rules.komi = 7.0f;
  Lcg rng(strtoull(seedStr.c_str(), NULL, 10));
  auto unif = [&]() { return (float)((rng.next() & 0xFFFFFF) / 16777216.0); };

  Board board(X, Y);
  Player pla = P_BLACK;
  BoardHistory hist(board, pla, rules, 0, passAliveFlag);
  const BoardHistory startHist = hist;
  vector<Board> boards; vector<BoardHistory> hists; vector<Player> plas;
  bool prevPass = false;
  for(int t = 0; t < nTurns; t++) {
    boards.push_back(board); hists.push_back(hist); plas.push_back(pla);
    vector<Loc> legal;
    for(int y = 0; y < Y; y++) for(int x = 0; x < X; x++) { Loc l = Location::getLoc(x, y, X); if(hist.isLegal(board, l, pla)) legal.push_back(l); }
    Loc mv = (legal.empty() || (!prevPass && rng.next() % 30 == 0)) ? Board::PASS_LOC : legal[rng.next() % legal.size()];
    if(prevPass && mv == Board::PASS_LOC && !legal.empty()) mv = legal[0];
    prevPass = mv == Board::PASS_LOC;
    hist.makeBoardMoveAssumeLegal(board, mv, pla, NULL);
    pla = getOpp(pla);
  }
  boards.push_back(board);   // posHistForFutureBoards has one board per value target (trainingwrite.cpp:782)
  BoardHistory endHist = hist;
  if(endNoResult) { endHist.isGameFinished = true; endHist.isNoResult = true; }
  else if(nTurns % 2 == 0) endHist.isGameFinished = true;
  endHist.whiteBonusScore += bonus;

  vector<ValueTargets> vts(nTurns + 1);
  for(auto& v : vts) {
    float a = unif(), b = unif() * (1.0f - a);
    v.win = a; v.loss = b; v.noResult = 1.0f - a - b;
    v.score = (unif() - 0.5f) * (rng.next() % 5 == 0 ? 1300.0f : 60.0f);
    v.hasLead = rng.next() % 4 != 0;
    v.lead = (unif() - 0.5f) * (rng.next() % 5 == 0 ? 1300.0f : 50.0f);
  }
  if(nTurns % 3 == 0) vts.back().score = 0.5f * (float)((int)(rng.next() % 41) - 20);   // finished games have half-integer scores
  if(strtoull(seedStr.c_str(), NULL, 10) % 10 == 9) vts.back().score = 500.5f;   // beyond either end of the score distribution (colours alternate)

  Color fullArea[Board::MAX_ARR_SIZE], ownership[Board::MAX_ARR_SIZE];
  float scoring[Board::MAX_ARR_SIZE];
  board.calculateArea(fullArea, true, true, true, true);
  board.calculateArea(ownership, false, false, false, true);
  for(int i = 0; i < Board::MAX_ARR_SIZE; i++) scoring[i] = 0.0f;
  for(int y = 0; y < Y; y++) for(int x = 0; x < X; x++) {
    Loc l = Location::getLoc(x, y, X);
    const uint32_t k = rng.next() % 6;
    scoring[l] = k == 0 ? 1.0f : k == 1 ? -1.0f : k == 2 ? 0.0f : k == 3 ? (float)((int)(rng.next() % 241) - 120) / 120.0f : unif() * 2.0f - 1.0f;
    if(scoring[l] > 1.0f) scoring[l] = 1.0f;
    if(scoring[l] < -1.0f) scoring[l] = -1.0f;
  }
  Hash128 gameHash(((uint64_t)rng.next() << 32) ^ ((uint64_t)rng.next() << 11) ^ rng.next(), ((uint64_t)rng.next() << 33) ^ ((uint64_t)rng.next() << 9) ^ rng.next());

  TrainingWriteBuffers buf(7, nTurns, NNInputs::NUM_FEATURES_SPATIAL_V7, NNInputs::NUM_FEATURES_GLOBAL_V7, D, D, false);
  Rand rowRand("addrow" + seedStr);
  const int P = D * D + 1, A = D * D, SD = A * 2 + NNPos::EXTRA_SCORE_DISTR_RADIUS * 2, packed = (A + 7) / 8;

  ofstream out(argv[9]);
  auto f9 = [](double v) { return Global::strprintf("%.9g", v); };
  auto f17 = [](double v) { return Global::strprintf("%.17g", v); };
  auto locJson = [&](Loc l) { return l == Board::PASS_LOC ? string("-1,-1") : Global::intToString(Location::getX(l, X)) + "," + Global::intToString(Location::getY(l, X)); };
  out << "{\"X\":" << X << ",\"Y\":" << Y << ",\"dataLen\":" << D << ",\"seed\":\"" << seedStr << "\",\"gameHash\":[" << gameHash.hash0 << "," << gameHash.hash1 << "],\n";
  out << "\"valueTargets\":[";
  for(size_t i = 0; i < vts.size(); i++) out << (i ? "," : "") << "[" << f9(vts[i].win) << "," << f9(vts[i].loss) << "," << f9(vts[i].noResult) << "," << f9(vts[i].score) << "," << (vts[i].hasLead ? 1 : 0) << "," << f9(vts[i].lead) << "]";
  out << "],\n\"boards\":[";
  for(size_t i = 0; i < boards.size(); i++) {
    out << (i ? "," : "") << "[";
    for(int y = 0; y < Y; y++) for(int x = 0; x < X; x++) out << ((y || x) ? "," : "") << (int)boards[i].colors[Location::getLoc(x, y, X)];
    out << "]";
  }
  auto plane = [&](const char* name, auto fn) {
    out << "],\n\"" << name << "\":[";
    for(int y = 0; y < Y; y++) for(int x = 0; x < X; x++) out << ((y || x) ? "," : "") << fn(Location::getLoc(x, y, X));
  };
  plane("finalOwnership", [&](Loc l) { return Global::intToString((int)ownership[l]); });
  plane("finalFullArea", [&](Loc l) { return Global::intToString((int)fullArea[l]); });
  plane("finalWhiteScoring", [&](Loc l) { return f9(scoring[l]); });
  out << "],\n\"endFinished\":" << (endHist.isGameFinished ? 1 : 0) << ",\"endNoResult\":" << (endHist.isNoResult ? 1 : 0) << ",\"endWhiteBonus\":" << f9(endHist.whiteBonusScore)
      << ",\"startHistMoves\":" << startHist.moveHistory.size() << ",\n\"rows\":[\n";

  vector<QValueTargets> qts(nTurns + 1);
  for(int t = 0; t < nTurns; t++) {
    const Board& b = boards[t]; const BoardHistory& h = hists[t]; const Player p = plas[t];
    vector<Loc> legal;
    for(int y = 0; y < Y; y++) for(int x = 0; x < X; x++) { Loc l = Location::getLoc(x, y, X); if(h.isLegal(b, l, p)) legal.push_back(l); }
    legal.push_back(Board::PASS_LOC);
    vector<PolicyTargetMove> pt0, pt1;
    for(Loc l : legal) {
      if(rng.next() % 3 == 0) pt0.push_back(PolicyTargetMove(l, (int16_t)(rng.next() % 600)));
      if(rng.next() % 5 == 0) pt1.push_back(PolicyTargetMove(l, (int16_t)(rng.next() % 2)));
      if(rng.next() % 3 == 0) {
        const uint32_t k = rng.next() % 8;
        float wl = k == 0 ? 1.0f : k == 1 ? -1.0f : k == 2 ? 0.0f : unif() * 2.0f - 1.0f;
        float sc = k == 3 ? 500.0f : k == 4 ? -500.0f : k == 5 ? (float)((int)(rng.next() % 81) - 40) * 0.5f : (unif() - 0.5f) * 80.0f;
        int64_t visits = k == 6 ? 100000 : k == 7 ? -3 : (int64_t)(rng.next() % 700);
        qts[t].targets.push_back(QValueTargetMove(l, wl, sc, visits));
      }
    }
    const bool hasP0 = t % 7 != 3, hasP1 = t % 2 == 0, hasOwn = t % 5 != 4, hasFuture = t % 3 != 2, hasScoring = t % 4 != 1;
    const bool hitTurnLimit = (nTurns + (int)strtoull(seedStr.c_str(), NULL, 10)) % 2 == 1, isSide = false;
    const float targetWeight = unif(), valueTargetWeight = rng.next() % 3 == 0 ? 1.0f : unif(), tdValueTargetWeight = rng.next() % 3 == 0 ? 1.0f : unif(), leadFactor = unif();
    const int64_t unreduced = 100 + rng.next() % 2000;
    const double policySurprise = unif() * 2.0, policyEntropy = unif() * 3.0, searchEntropy = unif() * 3.0;
    NNRawStats raw; raw.whiteWinLoss = unif() * 2.0 - 1.0; raw.whiteScoreMean = (unif() - 0.5) * 40.0; raw.policyEntropy = unif() * 4.0;
    const int numBehind = (int)(rng.next() % 3), numExtraBlack = (int)(rng.next() % 3), mode = (int)(rng.next() % 4);
    const double drawEq = 0.5 + 0.1 * (int)(rng.next() % 3);
    vector<ChangedNeuralNet*> changed;
    ChangedNeuralNet dummy("x", 3);
    if(t % 6 == 5) changed.push_back(&dummy);
    ReanalysisData re;
    if(t % 8 == 6) { re.wasReanalyzed = true; re.selectionPolicySurprise = unif(); re.selectionValueSurprise = unif(); re.originalNumVisits = 50 + rng.next() % 100; }
    const int rowsBefore = (int)buf.curRows;
    buf.addRow(b, h, p, startHist, endHist, t, targetWeight, unreduced, hasP0 ? &pt0 : NULL, hasP1 ? &pt1 : NULL, policySurprise, policyEntropy, searchEntropy,
               vts, qts, t, valueTargetWeight, tdValueTargetWeight, leadFactor, raw, &board, fullArea, hasOwn ? ownership : NULL, hasScoring ? scoring : NULL,
               hasFuture ? &boards : NULL, isSide, numBehind, drawEq, C_EMPTY, 0.0, gameHash, changed, hitTurnLimit, numExtraBlack, mode, NULL, rowRand, re);
    const int r = rowsBefore;
    out << (t ? ",\n" : "") << "{\"turnIdx\":" << t << ",\"nextPlayer\":" << (int)p << ",\"targetWeight\":" << f9(targetWeight) << ",\"unreducedNumVisits\":" << unreduced;
    auto ptJson = [&](const char* name, const vector<PolicyTargetMove>* v) {
      out << ",\"" << name << "\":";
      if(!v) { out << "null"; return; }
      out << "[";
      for(size_t i = 0; i < v->size(); i++) out << (i ? "," : "") << "[" << locJson((*v)[i].loc) << "," << (*v)[i].policyTarget << "]";
      out << "]";
    };
    ptJson("policyTarget0", hasP0 ? &pt0 : NULL); ptJson("policyTarget1", hasP1 ? &pt1 : NULL);
    out << ",\"qTargets\":[";
    for(size_t i = 0; i < qts[t].targets.size(); i++) { const QValueTargetMove& q = qts[t].targets[i]; out << (i ? "," : "") << "[" << locJson(q.loc) << "," << f9(q.winLoss) << "," << f9(q.score) << "," << q.visits << "]"; }
    out << "],\"policySurprise\":" << f17(policySurprise) << ",\"policyEntropy\":" << f17(policyEntropy) << ",\"searchEntropy\":" << f17(searchEntropy)
        << ",\"valueTargetWeight\":" << f9(valueTargetWeight) << ",\"tdValueTargetWeight\":" << f9(tdValueTargetWeight) << ",\"leadTargetWeightFactor\":" << f9(leadFactor)
        << ",\"nnRawStats\":[" << f17(raw.whiteWinLoss) << "," << f17(raw.whiteScoreMean) << "," << f17(raw.policyEntropy) << "]"
        << ",\"hasOwnership\":" << (hasOwn ? 1 : 0) << ",\"hasFutureBoards\":" << (hasFuture ? 1 : 0) << ",\"hasScoring\":" << (hasScoring ? 1 : 0)
        << ",\"isSidePosition\":" << (isSide ? 1 : 0) << ",\"numNeuralNetsBehindLatest\":" << numBehind << ",\"drawEquivalentWinsForWhite\":" << f17(drawEq)
        << ",\"numChangedNeuralNets\":" << changed.size() << ",\"hitTurnLimit\":" << (hitTurnLimit ? 1 : 0) << ",\"numExtraBlack\":" << numExtraBlack << ",\"mode\":" << mode
        << ",\"reanalysis\":[" << (re.wasReanalyzed ? 1 : 0) << "," << f9(re.selectionPolicySurprise) << "," << f9(re.selectionValueSurprise) << "," << re.originalNumVisits << "]"
        << ",\"selfKomi\":" << f9(h.currentSelfKomi(p, drawEq)) << ",\"areaScoringOrEncore2\":" << ((h.encorePhase == 2 || h.rules.scoringRule == Rules::SCORING_AREA) ? 1 : 0)
        << ",\"initialTurnNumber\":" << h.initialTurnNumber << ",\"whiteBonusScore\":" << f9(h.whiteBonusScore)
        << ",\"alwaysComputePassAliveUnderSuicideRules\":" << (h.alwaysComputePassAliveUnderSuicideRules ? 1 : 0);
    out << ",\n \"out_binaryInputNCHWPacked\":\"";
    for(int i = 0; i < NNInputs::NUM_FEATURES_SPATIAL_V7 * packed; i++) out << Global::strprintf("%02x", (unsigned)buf.binaryInputNCHWPacked.data[(size_t)r * NNInputs::NUM_FEATURES_SPATIAL_V7 * packed + i]);
    out << "\"";
    auto arr = [&](const char* name, auto* data, size_t n, bool isFloat) {
      out << ",\n \"" << name << "\":[";
      for(size_t i = 0; i < n; i++) { out << (i ? "," : ""); if(isFloat) out << f9((double)data[i]); else out << (long long)data[i]; }
      out << "]";
    };
    arr("out_globalInputNC", buf.globalInputNC.data + (size_t)r * NNInputs::NUM_FEATURES_GLOBAL_V7, NNInputs::NUM_FEATURES_GLOBAL_V7, true);
    arr("out_policyTargetsNCMove", buf.policyTargetsNCMove.data + (size_t)r * 2 * P, 2 * P, false);
    arr("out_globalTargetsNC", buf.globalTargetsNC.data + (size_t)r * 80, 80, true);
    arr("out_scoreDistrN", buf.scoreDistrN.data + (size_t)r * SD, SD, false);
    arr("out_valueTargetsNCHW", buf.valueTargetsNCHW.data + (size_t)r * 5 * A, 5 * A, false);
    arr("out_qValueTargetsNCMove", buf.qValueTargetsNCMove.data + (size_t)r * 3 * P, 3 * P, false);
    out << "}";
  }
  out << "\n]}\n";
  return 0;
}

// writegame X Y DATALEN NTURNS SEED MAXROWS FIRSTFILEPROP NORESULT OUT.json: TrainingDataWriter::writeGame (dataio/trainingwrite.cpp:1097-1325)
// on a synthetic FinishedGameData (main-line rows; no side positions) through the writer's text sink: fractional and multiple target
// weights, reanalysed turns that skip the outcome targets, net changes, file splits at MAXROWS / the randomised first-file size.
// Dumps the game and the text the writer emitted (every flush = one block of the seven arrays).
static int cmdWriteGame(int argc, char** argv) {
  if(argc != 11) { cerr << "usage: writegame X Y DATALEN NTURNS SEED MAXROWS FIRSTFILEPROP NORESULT OUT.json" << endl; return 1; }
  const int X = atoi(argv[2]), Y = atoi(argv[3]), D = atoi(argv[4]), nTurns = atoi(argv[5]);
  const string seedStr = argv[6];
  const int maxRows = atoi(argv[7]);
  const double firstFileProp = atof(argv[8]);
  const bool endNoResult = atoi(argv[9]) != 0;
  Board::initHash();
  ScoreValue::initTables();
  Rules rules;
  rules.koRule = Rules::KO_SIMPLE; rules.scoringRule = Rules::SCORING_AREA; rules.taxRule = Rules::TAX_NONE;
  rules.multiStoneSuicideLegal = true; rules.hasButton = false; rules.whiteHandicapBonusRule = Rules::WHB_ZERO;
  const uint64_t seedNum = strtoull(seedStr.c_str(), NULL, 10);
  const double drawEq = 0.5 + 0.1 * (double)(seedNum % 3);
  rules.friendlyPassOk = false; rules.komi = (seedNum % 2) ? 7.0f : 6.5f;
  Lcg rng(seedNum);
  auto unif = [&]() { return (float)((rng.next() & 0xFFFFFF) / 16777216.0); };

  FinishedGameData data;
  Board board(X, Y);
  Player pla = P_BLACK;
  BoardHistory hist(board, pla, rules, 0, false);
  // KGREF_START_MOVES = S: the game's first S moves (random legal ones) happen before the training period - they are its startHist, like a
  // policy-initialised opening or a forked game's position (startTurnIdx = S in the record, start-history length S in the rows)
  vector<string> startMoveStrs;
  for(int i = 0, S = getenv("KGREF_START_MOVES") ? atoi(getenv("KGREF_START_MOVES")) : 0; i < S; i++) {
    vector<Loc> legal;
    for(int y = 0; y < Y; y++) for(int x = 0; x < X; x++) { Loc l = Location::getLoc(x, y, X); if(hist.isLegal(board, l, pla)) legal.push_back(l); }
    if(legal.empty()) break;
    const Loc mv = legal[rng.next() % legal.size()];
    startMoveStrs.push_back(Global::intToString(Location::getX(mv, X)) + "," + Global::intToString(Location::getY(mv, X)));
    hist.makeBoardMoveAssumeLegal(board, mv, pla, NULL);
    pla = getOpp(pla);
  }
  data.startBoard = board; data.startHist = hist; data.startPla = pla;
  vector<Board> boards; vector<BoardHistory> hists; vector<Player> plas; vector<vector<Loc>> legalByTurn; vector<string> moveStrs, packedHex; vector<vector<float>> globalRows;
  auto inputRows = [&](const Board& b, const BoardHistory& h, Player p, string& hex, vector<float>& rowGlobal) {
    MiscNNInputParams ip; ip.drawEquivalentWinsForWhite = drawEq;
    vector<float> rowBin((size_t)NNInputs::NUM_FEATURES_SPATIAL_V7 * D * D);
    rowGlobal.assign(NNInputs::NUM_FEATURES_GLOBAL_V7, 0.0f);
    NNInputs::fillRowV7(b, h, p, ip, D, D, false, rowBin.data(), rowGlobal.data());
    hex.clear();
    const int A = D * D, packed = (A + 7) / 8;
    for(int c = 0; c < NNInputs::NUM_FEATURES_SPATIAL_V7; c++) for(int bb = 0; bb < packed; bb++) {
      unsigned v = 0;
      for(int k = 0; k < 8; k++) { const int idx = bb * 8 + k; if(idx < A && rowBin[(size_t)c * A + idx] != 0.0f) v |= 1u << (7 - k); }
      hex += Global::strprintf("%02x", v);
    }
  };
  bool prevPass = false;
  for(int t = 0; t < nTurns; t++) {
    boards.push_back(board); hists.push_back(hist); plas.push_back(pla);
    {   // the input rows addRow will compute for this turn (fillRowV7, NCHW, the game's drawEquivalentWinsForWhite), packed like packBits
      string hex; vector<float> rowGlobal;
      inputRows(board, hist, pla, hex, rowGlobal);
      packedHex.push_back(hex); globalRows.push_back(rowGlobal);
    }
    vector<Loc> legal;
    for(int y = 0; y < Y; y++) for(int x = 0; x < X; x++) { Loc l = Location::getLoc(x, y, X); if(hist.isLegal(board, l, pla)) legal.push_back(l); }
    Loc mv = (legal.empty() || (!prevPass && rng.next() % 30 == 0)) ? Board::PASS_LOC : legal[rng.next() % legal.size()];
    if(prevPass && mv == Board::PASS_LOC && !legal.empty()) mv = legal[0];
    prevPass = mv == Board::PASS_LOC;
    legal.push_back(Board::PASS_LOC);
    legalByTurn.push_back(legal);
    moveStrs.push_back(mv == Board::PASS_LOC ? string("-1,-1") : Global::intToString(Location::getX(mv, X)) + "," + Global::intToString(Location::getY(mv, X)));
    hist.makeBoardMoveAssumeLegal(board, mv, pla, NULL);
    pla = getOpp(pla);
  }
  boards.push_back(board);
  data.finalFullArea = new Color[Board::MAX_ARR_SIZE];
  data.finalOwnership = new Color[Board::MAX_ARR_SIZE];
  data.finalSekiAreas = new bool[Board::MAX_ARR_SIZE];
  data.finalWhiteScoring = new float[Board::MAX_ARR_SIZE];
  std::fill(data.finalSekiAreas, data.finalSekiAreas + Board::MAX_ARR_SIZE, false);
  ValueTargets finalTargets;
  if(endNoResult) {
    hist.isGameFinished = true; hist.isNoResult = true; hist.winner = C_EMPTY;
    std::fill(data.finalFullArea, data.finalFullArea + Board::MAX_ARR_SIZE, C_EMPTY);
    std::fill(data.finalOwnership, data.finalOwnership + Board::MAX_ARR_SIZE, C_EMPTY);
    finalTargets.win = 0.0f; finalTargets.loss = 0.0f; finalTargets.noResult = 1.0f; finalTargets.score = 0.0f;
  }
  else {   // what Play::runGame does at the end of a game (program/play.cpp:1989-2000)
    hist.endAndScoreGameNow(board, data.finalOwnership);
    board.calculateArea(data.finalFullArea, true, true, true, hist.suicideLegalForPassAlive());
    finalTargets.win = (float)ScoreValue::whiteWinsOfWinner(hist.winner, drawEq);
    finalTargets.loss = 1.0f - finalTargets.win; finalTargets.noResult = 0.0f;
    finalTargets.score = (float)ScoreValue::whiteScoreDrawAdjust(hist.finalWhiteMinusBlackScore, drawEq, hist);
    finalTargets.hasLead = true; finalTargets.lead = finalTargets.score;
  }
  NNInputs::fillScoring(board, data.finalOwnership, false, data.finalWhiteScoring);
  data.endHist = hist;
  data.hitTurnLimit = false;
  data.gameHash = Hash128(((uint64_t)rng.next() << 32) ^ ((uint64_t)rng.next() << 11) ^ rng.next(), ((uint64_t)rng.next() << 33) ^ ((uint64_t)rng.next() << 9) ^ rng.next());
  data.drawEquivalentWinsForWhite = drawEq;
  data.playoutDoublingAdvantagePla = C_EMPTY; data.playoutDoublingAdvantage = 0.0;
  data.numExtraBlack = 0; data.mode = (int)(rng.next() % 3); data.hasFullData = true;
  data.trainingWeight = rng.next() % 2 == 0 ? 1.0 : 0.75;
  const int numChanges = (int)(rng.next() % 3);
  for(int i = 0; i < numChanges; i++) data.changedNeuralNets.push_back(new ChangedNeuralNet("net" + Global::intToString(i), (int)((i + 1) * nTurns / 3)));
  const bool withReanalysis = rng.next() % 2 == 0;
  for(int t = 0; t < nTurns; t++) {
    static const float weights[8] = {0.0f, 1.0f, 1.0f, 0.35f, 1.6f, 2.0f, 0.9f, 3.25f};
    const float w = weights[rng.next() % 8];
    data.targetWeightByTurn.push_back(w); data.targetWeightByTurnUnrounded.push_back(w);
    vector<PolicyTargetMove>* pt = new vector<PolicyTargetMove>();
    QValueTargets q;
    for(Loc l : legalByTurn[t]) {
      if(rng.next() % 3 == 0) pt->push_back(PolicyTargetMove(l, (int16_t)(1 + rng.next() % 600)));
      if(rng.next() % 4 == 0) q.targets.push_back(QValueTargetMove(l, unif() * 2.0f - 1.0f, (unif() - 0.5f) * 80.0f, (int64_t)(rng.next() % 700)));
    }
    data.policyTargetsByTurn.push_back(PolicyTarget(pt, 100 + rng.next() % 2000));
    data.whiteQValueTargetsByTurn.push_back(q);
    data.policySurpriseByTurn.push_back(unif() * 2.0); data.policyEntropyByTurn.push_back(unif() * 3.0); data.searchEntropyByTurn.push_back(unif() * 3.0);
    ValueTargets v;
    float a = unif(), b = unif() * (1.0f - a);
    v.win = a; v.loss = b; v.noResult = 1.0f - a - b; v.score = (unif() - 0.5f) * 60.0f; v.hasLead = rng.next() % 4 != 0; v.lead = (unif() - 0.5f) * 50.0f;
    data.whiteValueTargetsByTurn.push_back(v);
    NNRawStats raw; raw.whiteWinLoss = unif() * 2.0 - 1.0; raw.whiteScoreMean = (unif() - 0.5) * 40.0; raw.policyEntropy = unif() * 4.0;
    data.nnRawStatsByTurn.push_back(raw);
    if(withReanalysis) {
      ReanalysisData re;
      if(rng.next() % 4 == 0) {
        re.wasReanalyzed = true; re.usedOutcomeTargets = rng.next() % 2 == 0; re.selectionPolicySurprise = unif(); re.selectionValueSurprise = unif();
        re.originalNumVisits = 50 + rng.next() % 100; re.numNeuralNetChangesSoFar = numChanges > 0 ? (int)(rng.next() % (numChanges + 1)) : 0;
      }
      data.reanalysisByTurn.push_back(re);
    }
  }
  data.whiteValueTargetsByTurn.push_back(finalTargets);

  // side positions (trainingwrite.cpp:1258-1323): an alternative move from a main-line position, searched on its own
  struct SideDump { string hex; vector<float> global; };
  vector<SideDump> sideDumps;
  const int numSide = (int)(seedNum % 4);
  for(int k = 0; k < numSide; k++) {
    const int t = (int)(rng.next() % nTurns);
    Board b = boards[t]; BoardHistory h = hists[t]; Player p = plas[t];
    const vector<Loc>& legal = legalByTurn[t];
    const Loc alt = legal[rng.next() % legal.size()];
    h.makeBoardMoveAssumeLegal(b, alt, p, NULL);
    p = getOpp(p);
    if(h.isGameFinished) continue;
    SidePosition* sp = new SidePosition(b, h, p, numChanges > 0 ? (int)(rng.next() % (numChanges + 1)) : 0);
    static const float sw[4] = {1.0f, 0.4f, 2.0f, 1.5f};
    sp->targetWeight = sw[rng.next() % 4]; sp->targetWeightUnrounded = sp->targetWeight;
    sp->unreducedNumVisits = 50 + rng.next() % 900;
    for(int y = 0; y < Y; y++) for(int x = 0; x < X; x++) {
      const Loc l = Location::getLoc(x, y, X);
      if(!h.isLegal(b, l, p)) continue;
      if(rng.next() % 3 == 0) sp->policyTarget.push_back(PolicyTargetMove(l, (int16_t)(1 + rng.next() % 300)));
      if(rng.next() % 5 == 0) sp->whiteQValueTargets.targets.push_back(QValueTargetMove(l, unif() * 2.0f - 1.0f, (unif() - 0.5f) * 60.0f, (int64_t)(rng.next() % 300)));
    }
    sp->policySurprise = unif() * 2.0; sp->policyEntropy = unif() * 3.0; sp->searchEntropy = unif() * 3.0;
    float a = unif(), bb = unif() * (1.0f - a);
    sp->whiteValueTargets.win = a; sp->whiteValueTargets.loss = bb; sp->whiteValueTargets.noResult = 1.0f - a - bb;
    sp->whiteValueTargets.score = (unif() - 0.5f) * 60.0f; sp->whiteValueTargets.hasLead = rng.next() % 2 == 0; sp->whiteValueTargets.lead = (unif() - 0.5f) * 40.0f;
    sp->nnRawStats.whiteWinLoss = unif() * 2.0 - 1.0; sp->nnRawStats.whiteScoreMean = (unif() - 0.5) * 40.0; sp->nnRawStats.policyEntropy = unif() * 4.0;
    SideDump sd; inputRows(b, h, p, sd.hex, sd.global);
    sideDumps.push_back(sd);
    data.sidePositions.push_back(sp);
  }

  data.bName = "b200-black"; data.wName = "b200-white"; data.handicapForSgf = 0;
  ostringstream sgf;   // what SelfplayManager writes next to the training rows (program/selfplaymanager.cpp:377)
  WriteSgf::writeSgf(sgf, data.bName, data.wName, data.endHist, &data, false, true);

  ostringstream sink;
  {
    TrainingDataWriter writer(&sink, 7, maxRows, firstFileProp, D, D, 1, "writegame" + seedStr);
    writer.writeGame(data);
    writer.flushIfNonempty();
  }

  ofstream out(argv[10]);
  auto f9 = [](double v) { return Global::strprintf("%.9g", v); };
  auto f17 = [](double v) { return Global::strprintf("%.17g", v); };
  auto locJson = [&](Loc l) { return l == Board::PASS_LOC ? string("-1,-1") : Global::intToString(Location::getX(l, X)) + "," + Global::intToString(Location::getY(l, X)); };
  out << "{\"X\":" << X << ",\"Y\":" << Y << ",\"dataLen\":" << D << ",\"seed\":\"" << seedStr << "\",\"maxRows\":" << maxRows << ",\"firstFileMinRandProp\":" << f17(firstFileProp)
      << ",\"gameHash\":[" << data.gameHash.hash0 << "," << data.gameHash.hash1 << "],\"komi\":" << f9(rules.komi) << ",\"drawEquivalentWinsForWhite\":" << f17(drawEq)
      << ",\"mode\":" << data.mode << ",\"trainingWeight\":" << f17(data.trainingWeight) << ",\"hitTurnLimit\":0,\"numExtraBlack\":0"
      << ",\"endFinished\":" << (data.endHist.isGameFinished ? 1 : 0) << ",\"endNoResult\":" << (data.endHist.isNoResult ? 1 : 0)
      << ",\"winner\":" << (int)data.endHist.winner << ",\"finalWhiteMinusBlackScore\":" << f9(data.endHist.finalWhiteMinusBlackScore) << ",\n";
  out << "\"sgf\":\"";
  for(char ch : sgf.str()) { if(ch == '\n') out << "\\n"; else if(ch == '"' || ch == '\\') out << '\\' << ch; else out << ch; }
  out << "\",\n\"changedNeuralNetNames\":[";
  for(size_t i = 0; i < data.changedNeuralNets.size(); i++) out << (i ? "," : "") << "\"" << data.changedNeuralNets[i]->name << "\"";
  out << "],\n\"changedNeuralNetTurns\":[";
  for(size_t i = 0; i < data.changedNeuralNets.size(); i++) out << (i ? "," : "") << data.changedNeuralNets[i]->turnIdx;
  out << "],\n\"startMoves\":[";
  for(size_t i = 0; i < startMoveStrs.size(); i++) out << (i ? "," : "") << "[" << startMoveStrs[i] << "]";
  out << "],\n\"moves\":[";
  for(size_t i = 0; i < moveStrs.size(); i++) out << (i ? "," : "") << "[" << moveStrs[i] << "]";
  out << "],\n\"valueTargets\":[";
  for(size_t i = 0; i < data.whiteValueTargetsByTurn.size(); i++) { const ValueTargets& v = data.whiteValueTargetsByTurn[i]; out << (i ? "," : "") << "[" << f9(v.win) << "," << f9(v.loss) << "," << f9(v.noResult) << "," << f9(v.score) << "," << (v.hasLead ? 1 : 0) << "," << f9(v.lead) << "]"; }
  out << "],\n\"boards\":[";
  for(size_t i = 0; i < boards.size(); i++) {
    out << (i ? "," : "") << "[";
    for(int y = 0; y < Y; y++) for(int x = 0; x < X; x++) out << ((y || x) ? "," : "") << (int)boards[i].colors[Location::getLoc(x, y, X)];
    out << "]";
  }
  auto plane = [&](const char* name, auto fn) {
    out << "],\n\"" << name << "\":[";
    for(int y = 0; y < Y; y++) for(int x = 0; x < X; x++) out << ((y || x) ? "," : "") << fn(Location::getLoc(x, y, X));
  };
  plane("finalOwnership", [&](Loc l) { return Global::intToString((int)data.finalOwnership[l]); });
  plane("finalFullArea", [&](Loc l) { return Global::intToString((int)data.finalFullArea[l]); });
  plane("finalWhiteScoring", [&](Loc l) { return f9(data.finalWhiteScoring[l]); });
  out << "],\n\"turns\":[\n";
  for(int t = 0; t < nTurns; t++) {
    out << (t ? ",\n" : "") << "{\"packedInput\":\"" << packedHex[t] << "\",\"globalInput\":[";
    for(size_t i = 0; i < globalRows[t].size(); i++) out << (i ? "," : "") << f9(globalRows[t][i]);
    out << "],\"nextPlayer\":" << (int)plas[t] << ",\"targetWeight\":" << f9(data.targetWeightByTurn[t]) << ",\"unreducedNumVisits\":" << data.policyTargetsByTurn[t].unreducedNumVisits << ",\"policyTarget\":[";
    const vector<PolicyTargetMove>& pt = *data.policyTargetsByTurn[t].policyTargets;
    for(size_t i = 0; i < pt.size(); i++) out << (i ? "," : "") << "[" << locJson(pt[i].loc) << "," << pt[i].policyTarget << "]";
    out << "],\"qTargets\":[";
    const vector<QValueTargetMove>& q = data.whiteQValueTargetsByTurn[t].targets;
    for(size_t i = 0; i < q.size(); i++) out << (i ? "," : "") << "[" << locJson(q[i].loc) << "," << f9(q[i].winLoss) << "," << f9(q[i].score) << "," << q[i].visits << "]";
    out << "],\"policySurprise\":" << f17(data.policySurpriseByTurn[t]) << ",\"policyEntropy\":" << f17(data.policyEntropyByTurn[t]) << ",\"searchEntropy\":" << f17(data.searchEntropyByTurn[t])
        << ",\"nnRawStats\":[" << f17(data.nnRawStatsByTurn[t].whiteWinLoss) << "," << f17(data.nnRawStatsByTurn[t].whiteScoreMean) << "," << f17(data.nnRawStatsByTurn[t].policyEntropy) << "]";
    if(withReanalysis) { const ReanalysisData& re = data.reanalysisByTurn[t]; out << ",\"reanalysis\":[" << (re.wasReanalyzed ? 1 : 0) << "," << (re.usedOutcomeTargets ? 1 : 0) << "," << f9(re.selectionPolicySurprise) << "," << f9(re.selectionValueSurprise) << "," << re.originalNumVisits << "," << re.numNeuralNetChangesSoFar << "]"; }
    out << "}";
  }
  out << "\n],\n\"sidePositions\":[";
  for(size_t k = 0; k < data.sidePositions.size(); k++) {
    const SidePosition* sp = data.sidePositions[k];
    out << (k ? ",\n" : "\n") << "{\"packedInput\":\"" << sideDumps[k].hex << "\",\"globalInput\":[";
    for(size_t i = 0; i < sideDumps[k].global.size(); i++) out << (i ? "," : "") << f9(sideDumps[k].global[i]);
    out << "],\"nextPlayer\":" << (int)sp->pla << ",\"turnIdx\":" << sp->hist.moveHistory.size() << ",\"targetWeight\":" << f9(sp->targetWeight)
        << ",\"unreducedNumVisits\":" << sp->unreducedNumVisits << ",\"numNeuralNetChangesSoFar\":" << sp->numNeuralNetChangesSoFar << ",\"policyTarget\":[";
    for(size_t i = 0; i < sp->policyTarget.size(); i++) out << (i ? "," : "") << "[" << locJson(sp->policyTarget[i].loc) << "," << sp->policyTarget[i].policyTarget << "]";
    out << "],\"qTargets\":[";
    const vector<QValueTargetMove>& q = sp->whiteQValueTargets.targets;
    for(size_t i = 0; i < q.size(); i++) out << (i ? "," : "") << "[" << locJson(q[i].loc) << "," << f9(q[i].winLoss) << "," << f9(q[i].score) << "," << q[i].visits << "]";
    const ValueTargets& v = sp->whiteValueTargets;
    out << "],\"valueTargets\":[" << f9(v.win) << "," << f9(v.loss) << "," << f9(v.noResult) << "," << f9(v.score) << "," << (v.hasLead ? 1 : 0) << "," << f9(v.lead) << "]"
        << ",\"policySurprise\":" << f17(sp->policySurprise) << ",\"policyEntropy\":" << f17(sp->policyEntropy) << ",\"searchEntropy\":" << f17(sp->searchEntropy)
        << ",\"nnRawStats\":[" << f17(sp->nnRawStats.whiteWinLoss) << "," << f17(sp->nnRawStats.whiteScoreMean) << "," << f17(sp->nnRawStats.policyEntropy) << "]}";
  }
  out << "\n],\n\"dump\":\"";
  for(char c : sink.str()) { if(c == '\n') out << "\\n"; else if(c == '"' || c == '\\') out << '\\' << c; else out << c; }
  out << "\"}\n";
  return 0;
}

// paramsmap CFG KORULE: the reference's own configuration loader (ConfigParser + Setup::loadSingleParams, program/setup.cpp) on a .cfg,
// mapped onto the device loop's configuration by integration/b200params.h; prints the mapped fields and the options it reports as
// not implemented.  tests/test_selfplay_cli.py compares this with katago_b200/selfplay_cli.py's own mapping of the same file.
static int cmdParamsMap(int argc, char** argv) {
  if(argc != 4) { cerr << "usage: paramsmap CFG KORULE" << endl; return 1; }
  const string cfgPath = argv[2];
  ConfigParser cfg(cfgPath);
  SearchParams p = Setup::loadSingleParams(cfg, Setup::SETUP_FOR_OTHER);
  Rules rules;
  const int ko = atoi(argv[3]);
  rules.koRule = ko == 1 ? Rules::KO_POSITIONAL : ko == 2 ? Rules::KO_SITUATIONAL : ko == 3 ? Rules::KO_SPIGHT : Rules::KO_SIMPLE;
  rules.scoringRule = Rules::SCORING_AREA; rules.taxRule = Rules::TAX_NONE; rules.multiStoneSuicideLegal = false; rules.hasButton = false;
  rules.whiteHandicapBonusRule = Rules::WHB_ZERO; rules.friendlyPassOk = false; rules.komi = 7.5f;
  vector<string> unsupported;
  const kgb_selfplay_config c = b200::configFromSearchParams(p, rules, 256, cfg.contains("maxMovesPerGame") ? cfg.getInt("maxMovesPerGame", 0, 100000) : 0, 1,
                                                             cfg.contains("nnCacheSizePowerOfTwo") ? cfg.getInt("nnCacheSizePowerOfTwo", -1, 48) : 0, &unsupported);
  auto d = [](double v) { return Global::strprintf("%.17g", v); };
  cout << "{";
#define FI(f) cout << "\"" #f "\":" << (long long)c.f << ","
#define FD(f) cout << "\"" #f "\":" << d(c.f) << ","
  FI(max_visits); FI(max_moves); FI(multi_stone_suicide_legal); FD(komi); FD(cpuct_exploration); FD(cpuct_exploration_log); FD(cpuct_exploration_base);
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
#undef FI
#undef FD
  cout << "\"unsupported\":[";
  for(size_t i = 0; i < unsupported.size(); i++) cout << (i ? "," : "") << "\"" << unsupported[i] << "\"";
  cout << "]}" << endl;
  return 0;
}

// rungame MODELFILE SIZE MAXVISITS MAXMOVES SEED POLICYSURPRISEWEIGHT VALUESURPRISEWEIGHT USESEARCHVALUESURPRISE: one whole game of the
// reference's own Play::runGame (program/play.cpp:1534-2354) with the fake net, full data recording, no cheap searches / forks / policy
// init, so that every turn enters the surprise weighting with weight 1.  Dumps what the weighting and the value surprise are computed
// from (per turn: value targets, raw net win / loss / noResult, policy surprise) and what runGame made of them (valueSurpriseByTurn,
// targetWeightByTurnUnrounded, targetWeightByTurn).  With SLOTLOG ROWSOUT: also what the device loop's getters would have exposed for
// every finished root search of the game (one JSON line per event, the format of tests/mock/kgb200_mock.cpp) and the rows the
// reference's own TrainingDataWriter makes of the game - the whole host chain of the recorder against a real reference game.
static int cmdRunGame(int argc, char** argv) {
  if(argc != 10 && argc != 12) { cerr << "usage: rungame MODELFILE SIZE MAXVISITS MAXMOVES SEED PSW VSW USESEARCHVALUESURPRISE [SLOTLOG ROWSOUT]" << endl; return 1; }
  const bool wantLog = argc == 12;
  const string modelFile = argv[2];
  const int L = atoi(argv[3]), maxVisits = atoi(argv[4]), maxMoves = atoi(argv[5]);
  const string seed = argv[6];
  Board::initHash();
  ScoreValue::initTables();
  Logger logger(nullptr, false, false, false);
  ConfigParser cfg;
  NNEvaluator* nnEval = new NNEvaluator("fake", modelFile, "", &logger, 4, L, L, true, true, 10, 8, false, "", enabled_t::False, 1,
                                        vector<int>{0}, "seed", false, 0, true, cfg);
  nnEval->spawnServerThreads();
  SearchParams params;
  params.maxVisits = maxVisits; params.numThreads = 1;
  params.rootNoiseEnabled = true; params.chosenMoveTemperature = 0.5; params.chosenMoveTemperatureEarly = 0.9;
  PlaySettings ps;
  ps.policySurpriseDataWeight = atof(argv[7]); ps.valueSurpriseDataWeight = atof(argv[8]); ps.useSearchValueSurprise = atoi(argv[9]) != 0;
  ps.forSelfPlay = true; ps.recordTimePerMove = false;
  ps.noResolveTargetWeights = wantLog;   // the chain test leaves the weights fractional: the writer's own Rand then decides the extra rows
  // search limits per move (getSearchLimitsThisMove, play.cpp:1093-1223): KGREF_REDUCE = "threshold,lookback,minVisits,weight", KGREF_CHEAP = "prob,visits,weight"
  if(getenv("KGREF_REDUCE")) {
    double thr, w; int look, mn;
    if(sscanf(getenv("KGREF_REDUCE"), "%lf,%d,%d,%lf", &thr, &look, &mn, &w) != 4) { cerr << "bad KGREF_REDUCE" << endl; return 1; }
    ps.reduceVisits = true; ps.reduceVisitsThreshold = thr; ps.reduceVisitsThresholdLookback = look; ps.reducedVisitsMin = mn; ps.reducedVisitsWeight = (float)w;
    ps.noResolveTargetWeights = true;
  }
  if(getenv("KGREF_CHEAP")) {
    double pr, w; int v;
    if(sscanf(getenv("KGREF_CHEAP"), "%lf,%d,%lf", &pr, &v, &w) != 3) { cerr << "bad KGREF_CHEAP" << endl; return 1; }
    ps.cheapSearchProb = pr; ps.cheapSearchVisits = v; ps.cheapSearchTargetWeight = (float)w;
    ps.noResolveTargetWeights = true;
  }
  if(getenv("KGREF_RESIGN")) {   // allowResignation (play.cpp:1903-1929): "threshold,consecTurns"
    double thr; int consec;
    if(sscanf(getenv("KGREF_RESIGN"), "%lf,%d", &thr, &consec) != 2) { cerr << "bad KGREF_RESIGN" << endl; return 1; }
    ps.allowResignation = true; ps.resignThreshold = thr; ps.resignConsecTurns = consec;
    ps.forSelfPlay = false;      // runGame refuses to record full training data together with resignation
  }
  vector<double> rootWinLoss; vector<int64_t> rootVisitsByTurn;
  Rules rules;
  rules.koRule = Rules::KO_SIMPLE; rules.scoringRule = Rules::SCORING_AREA; rules.taxRule = Rules::TAX_NONE; rules.multiStoneSuicideLegal = true;
  rules.hasButton = false; rules.whiteHandicapBonusRule = Rules::WHB_ZERO; rules.friendlyPassOk = false; rules.komi = 6.5f;
  Board board(L, L);
  Player pla = P_BLACK;
  BoardHistory hist(board, pla, rules, 0, false);
  ExtraBlackAndKomi ebk; ebk.extraBlack = 0; ebk.komiMean = 6.5f; ebk.komiStdev = 0.0f;
  OtherGameProperties other; other.allowPolicyInit = false;
  MatchPairer::BotSpec spec; spec.botIdx = 0; spec.botName = "fake"; spec.nnEval = nnEval; spec.baseParams = params;
  MatchPairer::BotSpec specW = spec;
  Rand gameRand("rungame" + seed);
  vector<vector<double>> raw;
  vector<string> rootEvents; vector<int> movePos;
  auto onEachMove = [&](const Board& b, const BoardHistory& h, Player p, Loc loc, const vector<double>&, const vector<double>&, const vector<double>&, const Search* bot) {
    const ReportedSearchValues v = bot->getRootRawNNValuesRequireSuccess();
    raw.push_back(vector<double>{v.winValue, v.lossValue, v.noResultValue});
    rootWinLoss.push_back(bot->getRootValuesRequireSuccess().winLossValue);      // what runGame appends to historicalMctsWinLossValues
    rootVisitsByTurn.push_back(bot->getRootVisits());
    if(!wantLog) return;
    // what the device loop's getters expose for a finished root search (the event format of tests/mock/kgb200_mock.cpp)
    const int P = L * L + 1;
    auto g17 = [](double x) { return Global::strprintf("%.17g", x); };
    vector<int> colors, edgeVisits(P, 0), nodeVisits(P, 0);
    vector<double> childStats((size_t)P * 5, 0.0), psv(P, -1.0);
    vector<float> policy(P, -1.0f);
    for(int y = 0; y < L; y++) for(int x = 0; x < L; x++) colors.push_back((int)b.colors[Location::getLoc(x, y, L)]);
    const SearchNode* root = bot->rootNode;
    ConstSearchNodeChildrenReference children = root->getChildren();
    auto posOf = [&](Loc l) { return l == Board::PASS_LOC ? L * L : Location::getY(l, L) * L + Location::getX(l, L); };
    for(int i = 0; i < children.getCapacity(); i++) {
      const SearchChildPointer& cp = children[i];
      const SearchNode* child = cp.getIfAllocated();
      if(child == NULL) break;
      const int pos = posOf(cp.getMoveLoc());
      edgeVisits[pos] = (int)cp.getEdgeVisits(); nodeVisits[pos] = (int)child->stats.visits.load();
      childStats[(size_t)pos * 5 + 0] = child->stats.winLossValueAvg.load(); childStats[(size_t)pos * 5 + 1] = child->stats.noResultValueAvg.load();
      childStats[(size_t)pos * 5 + 2] = child->stats.scoreMeanAvg.load(); childStats[(size_t)pos * 5 + 3] = child->stats.scoreMeanSqAvg.load();
      childStats[(size_t)pos * 5 + 4] = child->stats.leadAvg.load();
    }
    const NNOutput* nn = root->getNNOutput();
    for(int i = 0; i < P; i++) policy[i] = nn->getPolicyProbsMaybeNoised()[i];
    { vector<Loc> locs; vector<double> vals; bot->getPlaySelectionValues(locs, vals, 0.0); for(size_t i = 0; i < locs.size(); i++) psv[posOf(locs[i])] = vals[i]; }
    MiscNNInputParams ip; ip.drawEquivalentWinsForWhite = params.drawEquivalentWinsForWhite;
    vector<float> rowSp((size_t)L * L * 22), rowGl(19);
    NNInputs::fillRowV7(b, h, p, ip, L, L, true, rowSp.data(), rowGl.data());
    std::ostringstream o;
    auto arr = [&](const char* name, auto& vec, bool last = false) {
      o << "\"" << name << "\":[";
      for(size_t i = 0; i < vec.size(); i++) o << (i ? "," : "") << g17((double)vec[i]);
      o << "]" << (last ? "" : ",");
    };
    vector<double> rs{root->stats.winLossValueAvg.load(), root->stats.noResultValueAvg.load(), root->stats.scoreMeanAvg.load(), root->stats.scoreMeanSqAvg.load(), root->stats.leadAvg.load()};
    vector<double> rn{(double)nn->whiteWinProb - (double)nn->whiteLossProb, (double)nn->whiteNoResultProb, (double)nn->whiteScoreMean, (double)nn->whiteScoreMeanSq, (double)nn->whiteLead};
    o << "{\"ev\":\"root\",\"slot\":0,\"move_num\":" << h.moveHistory.size() << ",\"black_to_move\":" << (p == P_BLACK ? 1 : 0) << ",\"root_visits\":" << bot->getRootVisits() << ",";
    arr("colors", colors); arr("edge_visits", edgeVisits); arr("node_visits", nodeVisits); arr("policy", policy); arr("child_stats", childStats);
    arr("psv", psv); arr("root_stats", rs); arr("root_nn", rn); arr("row_spatial", rowSp); arr("row_global", rowGl, true);
    o << "}";
    rootEvents.push_back(o.str()); movePos.push_back(posOf(loc));
  };
  FinishedGameData* g = Play::runGame(board, pla, hist, ebk, spec, specW, "rungame" + seed, true, true, logger, false, false, maxMoves,
                                      []() { return false; }, nullptr, ps, other, gameRand, nullptr, onEachMove);
  auto d = [](double v) { return Global::strprintf("%.17g", v); };
  if(ps.allowResignation) {    // no training data in this mode: the root values and how the game ended
    cout << "{\"size\":" << L << ",\"turns\":" << rootWinLoss.size() << ",\"hitTurnLimit\":" << (g->hitTurnLimit ? 1 : 0) << ",\"rootWinLoss\":[";
    for(size_t i = 0; i < rootWinLoss.size(); i++) cout << (i ? "," : "") << d(rootWinLoss[i]);
    cout << "],\"resigned\":" << (g->endHist.isResignation ? 1 : 0) << ",\"winner\":" << (int)g->endHist.winner << ",\"gameFinished\":" << (g->endHist.isGameFinished ? 1 : 0)
         << ",\"moves\":" << g->endHist.moveHistory.size() << "}" << endl;
    delete g; delete nnEval;
    return 0;
  }
  const size_t n = g->targetWeightByTurn.size();
  if(raw.size() != n) { cerr << "onEachMove count " << raw.size() << " != turns " << n << endl; return 1; }
  cout << "{\"size\":" << L << ",\"turns\":" << n << ",\"policySurpriseDataWeight\":" << d(ps.policySurpriseDataWeight) << ",\"valueSurpriseDataWeight\":" << d(ps.valueSurpriseDataWeight)
       << ",\"useSearchValueSurprise\":" << (ps.useSearchValueSurprise ? 1 : 0) << ",\"hitTurnLimit\":" << (g->hitTurnLimit ? 1 : 0);
  auto arr = [&](const char* name, auto fn, size_t count) {
    cout << ",\n\"" << name << "\":[";
    for(size_t i = 0; i < count; i++) cout << (i ? "," : "") << fn(i);
    cout << "]";
  };
  arr("valueTargets", [&](size_t i) { const ValueTargets& v = g->whiteValueTargetsByTurn[i]; return "[" + d(v.win) + "," + d(v.loss) + "," + d(v.noResult) + "," + d(v.score) + "]"; }, n + 1);
  arr("rawNN", [&](size_t i) { return "[" + d(raw[i][0]) + "," + d(raw[i][1]) + "," + d(raw[i][2]) + "]"; }, n);
  arr("policySurprise", [&](size_t i) { return d(g->policySurpriseByTurn[i]); }, n);
  arr("valueSurprise", [&](size_t i) { return d(g->valueSurpriseByTurn[i]); }, n);
  arr("targetWeightUnrounded", [&](size_t i) { return d(g->targetWeightByTurnUnrounded[i]); }, n);
  arr("targetWeight", [&](size_t i) { return d(g->targetWeightByTurn[i]); }, n);
  arr("rootWinLoss", [&](size_t i) { return d(rootWinLoss[i]); }, n);
  arr("rootVisits", [&](size_t i) { return Global::int64ToString(rootVisitsByTurn[i]); }, n);
  cout << ",\n\"resigned\":" << (g->endHist.isResignation ? 1 : 0) << ",\"winner\":" << (int)g->endHist.winner << ",\"gameFinished\":" << (g->endHist.isGameFinished ? 1 : 0);
  cout << "}" << endl;
  if(wantLog) {
    ofstream lg(argv[10]);
    for(size_t t = 0; t < n; t++) {
      lg << rootEvents[t] << "\n";
      const bool lastMove = t + 1 == n;
      lg << "{\"ev\":\"move\",\"slot\":0,\"pos\":" << movePos[t] << ",\"flags\":"
         << (lastMove ? (1 | ((g->endHist.isGameFinished && g->endHist.isNoResult) ? 2 : 0) | (g->hitTurnLimit ? 4 : 0)) : 0)
         << ",\"move_num\":" << t << ",\"game_index\":0,\"game_hash\":[" << g->gameHash.hash0 << "," << g->gameHash.hash1 << "],\"score\":";
      if(lastMove) {   // the outcome as runGame determined it (play.cpp:1989-2027): score, final position, ownership
        BoardHistory h2 = g->endHist; Board b2 = g->endHist.getRecentBoard(0); Color area[Board::MAX_ARR_SIZE];
        h2.endAndScoreGameNow(b2, area);
        lg << Global::strprintf("%.9g", h2.finalWhiteMinusBlackScore) << ",\"final_colors\":[";
        for(int y = 0; y < L; y++) for(int x = 0; x < L; x++) lg << ((y || x) ? "," : "") << (int)b2.colors[Location::getLoc(x, y, L)];
        lg << "],\"final_area\":[";
        for(int y = 0; y < L; y++) for(int x = 0; x < L; x++) lg << ((y || x) ? "," : "") << (int)g->finalOwnership[Location::getLoc(x, y, L)];
        lg << "]}\n";
      }
      else lg << "0,\"final_colors\":[],\"final_area\":[]}\n";
    }
    ofstream rows(argv[11]);
    TrainingDataWriter writer(&rows, 7, 100000, 1.0, L, L, 1, "chain-test");
    writer.writeGame(*g);
    writer.flushIfNonempty();
  }
  delete g;
  delete nnEval;
  return 0;
}

// tinyfeatures DIAGRAMFILE X Y: the inputs of the reference's tiny-net known-answer test (tests/tinymodel.cpp): Board::parseBoard on the
// diagram, Tromp-Taylor-ish rules, black to move, no history; prints the fillRowV7 row on a 19x19 frame (NHWC) and which policy
// positions are legal - what NNEvaluator::evaluate feeds the backend and masks the policy with.
static int cmdTinyFeatures(int argc, char** argv) {
  if(argc != 5) { cerr << "usage: tinyfeatures DIAGRAMFILE X Y" << endl; return 1; }
  Board::initHash();
  ScoreValue::initTables();
  const int X = atoi(argv[3]), Y = atoi(argv[4]), L = 19;
  std::ifstream in(argv[2]);
  std::stringstream ss; ss << in.rdbuf();
  Board board = Board::parseBoard(X, Y, ss.str());
  const Player pla = P_BLACK;
  const Rules rules = Rules::getTrompTaylorish();
  const BoardHistory hist(board, pla, rules, 0, false);
  MiscNNInputParams ip;
  vector<float> sp((size_t)L * L * NNInputs::NUM_FEATURES_SPATIAL_V7), gl(NNInputs::NUM_FEATURES_GLOBAL_V7);
  NNInputs::fillRowV7(board, hist, pla, ip, L, L, true, sp.data(), gl.data());
  cout << "{\"spatial\":[";
  for(size_t i = 0; i < sp.size(); i++) cout << (i ? "," : "") << sp[i];
  cout << "],\"global\":[";
  for(size_t i = 0; i < gl.size(); i++) cout << (i ? "," : "") << Global::strprintf("%.9g", gl[i]);
  cout << "],\"legal\":[";
  for(int pos = 0; pos < L * L; pos++) {
    const int x = pos % L, y = pos / L;
    const bool legal = x < X && y < Y && hist.isLegal(board, Location::getLoc(x, y, X), pla);
    cout << (pos ? "," : "") << (legal ? 1 : 0);
  }
  cout << ",1],\"komi\":" << rules.komi << ",\"koRuleSimple\":" << (rules.koRule == Rules::KO_SIMPLE ? 1 : 0) << "}" << endl;
  return 0;
}

static int cmdFeatStream(int argc, char** argv) {
  if(argc != 9 && argc != 10) { cerr << "usage: featstream X Y MULTISUICIDE KOMI MOVES EVERY OUT [KORULE 0 simple 1 positional 2 situational]" << endl; return 1; }
  int X = atoi(argv[2]), Y = atoi(argv[3]);
  bool multi = atoi(argv[4]) != 0;
  float komi = (float)atof(argv[5]);
  int every = atoi(argv[7]);
  Board::initHash();
  ScoreValue::initTables();
  Rules rules;
  rules.koRule = Rules::KO_SIMPLE; rules.scoringRule = Rules::SCORING_AREA; rules.taxRule = Rules::TAX_NONE;
  if(argc == 10) rules.koRule = atoi(argv[9]) == 1 ? Rules::KO_POSITIONAL : atoi(argv[9]) == 2 ? Rules::KO_SITUATIONAL : Rules::KO_SIMPLE;
  rules.multiStoneSuicideLegal = multi; rules.hasButton = false; rules.whiteHandicapBonusRule = Rules::WHB_ZERO;
  rules.friendlyPassOk = false; rules.komi = komi;
  Board board(X, Y);
  Player pla = P_BLACK;
  BoardHistory hist(board, pla, rules, 0, false);
  ofstream out(argv[8], ios::binary);
  // MOVES may be "random:SEED:N": N random legal moves (BoardHistory::isLegal), 1/40 passes but never two in a row;
  // the generated list is written to OUT.moves so the other side can replay it.
  string movesArg = argv[6];
  if(movesArg.rfind("random:", 0) == 0) {
    uint64_t seed = 0; int count = 0;
    sscanf(movesArg.c_str(), "random:%lu:%d", &seed, &count);
    Lcg rng(seed);
    Board b2(X, Y); Player p2 = P_BLACK; BoardHistory h2(b2, p2, rules, 0, false);
    string gen; bool prevPass = false;
    for(int i = 0; i < count; i++) {
      vector<Loc> legal;
      for(int y = 0; y < Y; y++) for(int x = 0; x < X; x++) { Loc l = Location::getLoc(x, y, X); if(h2.isLegal(b2, l, p2)) legal.push_back(l); }
      Loc mv;
      if(legal.empty() || (!prevPass && rng.next() % 40 == 0)) { if(prevPass) break; mv = Board::PASS_LOC; }
      else mv = legal[rng.next() % legal.size()];
      prevPass = mv == Board::PASS_LOC;
      gen += prevPass ? "pass " : (Global::intToString(Location::getX(mv, X)) + "," + Global::intToString(Location::getY(mv, X)) + " ");
      h2.makeBoardMoveAssumeLegal(b2, mv, p2, NULL);
      p2 = getOpp(p2);
    }
    movesArg = gen;
    ofstream mo(string(argv[8]) + ".moves");
    mo << gen << endl;
  }
  std::istringstream in(movesArg);
  string tok;
  int n = 0, written = 0;
  // KGREF_NN_LEN = L: rows for an L x L evaluator frame with the X x Y board in its corner (see searchfake)
  const int nnLenEnv = getenv("KGREF_NN_LEN") ? atoi(getenv("KGREF_NN_LEN")) : 0;
  const int NX = nnLenEnv > 0 ? nnLenEnv : X, NY = nnLenEnv > 0 ? nnLenEnv : Y;
  if(NX < X || NY < Y) { cerr << "KGREF_NN_LEN smaller than the board" << endl; return 1; }
  vector<float> rowBin(NNInputs::NUM_FEATURES_SPATIAL_V7 * NX * NY), rowGlobal(NNInputs::NUM_FEATURES_GLOBAL_V7);
  auto dump = [&]() {
    MiscNNInputParams params;
    NNInputs::fillRowV7(board, hist, pla, params, NX, NY, true, rowBin.data(), rowGlobal.data());
    put<int32_t>(out, n);
    out.write((const char*)rowBin.data(), rowBin.size() * sizeof(float));
    out.write((const char*)rowGlobal.data(), rowGlobal.size() * sizeof(float));
    written++;
  };
  dump();
  while(in >> tok) {
    Loc loc;
    if(tok == "pass") loc = Board::PASS_LOC;
    else { int x, y; if(sscanf(tok.c_str(), "%d,%d", &x, &y) != 2) { cerr << "bad move " << tok << endl; return 1; } loc = Location::getLoc(x, y, X); }
    if(!hist.isLegal(board, loc, pla)) { cerr << "illegal move " << tok << " at " << n << endl; return 1; }
    hist.makeBoardMoveAssumeLegal(board, loc, pla, NULL);
    pla = getOpp(pla);
    n++;
    if(hist.isGameFinished) break;
    if(n % every == 0) dump();
  }
  cerr << "wrote " << written << " rows" << endl;
  return 0;
}

// ladderrows IN.txt OUT.bin: the fillRowV7 row of many positions in one process (tests/golden/make_ladder_fixtures.py).  Each line of
// IN.txt is "X Y NX NY KORULE MULTISUICIDE move move ..." (moves "x,y" or "pass"), replayed through BoardHistory with the rules of
// featstream (area scoring, no tax, komi 7.5); the row is written for an NX x NY frame with the board in its corner.  Per position OUT.bin
// holds: int32 status (0, or 1 = a move was illegal), float32 microseconds of the slowest single ladder search of the final position (the
// public Board::searchIsLadderCaptured / searchIsLadderCapturedAttackerFirst2Libs on a fresh copy, best of 3 runs: a search that
// reaches the 25 000-node budget takes orders of magnitude longer than the rest, and the reference offers no other view of its node
// count), int32 x, y of a stone of that chain, then the NX*NY*22 spatial values as uint8 (every V7 plane is 0/1) and 19 float32 globals.
static int cmdLadderRows(int argc, char** argv) {
  if(argc != 4) { cerr << "usage: ladderrows IN.txt OUT.bin" << endl; return 1; }
  Board::initHash();
  ScoreValue::initTables();
  ifstream in(argv[2]);
  ofstream out(argv[3], ios::binary);
  string line;
  int count = 0;
  while(getline(in, line)) {
    std::istringstream ls(line);
    int X, Y, NX, NY, koRule, multi;
    if(!(ls >> X >> Y >> NX >> NY >> koRule >> multi)) continue;
    if(NX < X || NY < Y) { cerr << "frame smaller than the board: " << line << endl; return 1; }
    Rules rules;
    rules.koRule = koRule == 1 ? Rules::KO_POSITIONAL : koRule == 2 ? Rules::KO_SITUATIONAL : koRule == 3 ? Rules::KO_SPIGHT : Rules::KO_SIMPLE;
    rules.scoringRule = Rules::SCORING_AREA; rules.taxRule = Rules::TAX_NONE;
    rules.multiStoneSuicideLegal = multi != 0; rules.hasButton = false; rules.whiteHandicapBonusRule = Rules::WHB_ZERO;
    rules.friendlyPassOk = false; rules.komi = 7.5f;
    Board board(X, Y);
    Player pla = P_BLACK;
    BoardHistory hist(board, pla, rules, 0, false);
    int32_t status = 0;
    string tok;
    while(ls >> tok) {
      Loc loc;
      if(tok == "pass") loc = Board::PASS_LOC;
      else { int x, y; if(sscanf(tok.c_str(), "%d,%d", &x, &y) != 2) { cerr << "bad move " << tok << endl; return 1; } loc = Location::getLoc(x, y, X); }
      if(hist.isGameFinished || !hist.isLegal(board, loc, pla)) { status = 1; break; }
      hist.makeBoardMoveAssumeLegal(board, loc, pla, NULL);
      pla = getOpp(pla);
    }
    float slowest = 0.0f;
    int32_t sx = -1, sy = -1;
    vector<Loc> buf, working;
    for(int y = 0; y < Y && status == 0; y++)
      for(int x = 0; x < X; x++) {
        const Loc loc = Location::getLoc(x, y, X);
        if(board.colors[loc] != P_BLACK && board.colors[loc] != P_WHITE) continue;
        const int libs = board.getNumLiberties(loc);
        if(libs != 1 && libs != 2) continue;
        if(board.chain_head[loc] != loc) continue;   // one search per chain
        double best = 1e30;
        for(int rep = 0; rep < 3; rep++) {
          Board copy(board);
          ClockTimer timer;
          if(libs == 1) copy.searchIsLadderCaptured(loc, true, buf);
          else copy.searchIsLadderCapturedAttackerFirst2Libs(loc, buf, working);
          best = std::min(best, timer.getSeconds());
        }
        if(best * 1e6 > slowest) { slowest = (float)(best * 1e6); sx = x; sy = y; }
      }
    vector<float> sp((size_t)NNInputs::NUM_FEATURES_SPATIAL_V7 * NX * NY), gl(NNInputs::NUM_FEATURES_GLOBAL_V7);
    if(status == 0) {
      MiscNNInputParams params;
      NNInputs::fillRowV7(board, hist, pla, params, NX, NY, true, sp.data(), gl.data());
    }
    vector<uint8_t> bits(sp.size());
    for(size_t i = 0; i < sp.size(); i++) bits[i] = sp[i] != 0.0f ? 1 : 0;
    put<int32_t>(out, status); put<float>(out, slowest); put<int32_t>(out, sx); put<int32_t>(out, sy);
    out.write((const char*)bits.data(), bits.size());
    out.write((const char*)gl.data(), gl.size() * sizeof(float));
    count++;
  }
  cerr << "wrote " << count << " rows" << endl;
  return 0;
}

// computelead MODELFILE X Y VISITS KOMI MOVES: PlayUtils::computeLead (program/playutils.cpp:612-660) of the position after MOVES at KOMI, one bot,
// the driver's default search parameters (as in searchfake), no evaluation cache, symmetry 0 - the komi-bisection searches that
// katago_b200/komi_search.py restates as jobs on a side loop.  Prints "lead <value>" and, for the same position,
// "evenkomi <value>" = KOMI - lead.  With kgref_driver_b200 the evaluator is libkgb200 (GPU box).
static int cmdComputeLead(int argc, char** argv) {
  if(argc != 8) { cerr << "usage: computelead MODELFILE X Y VISITS KOMI MOVES" << endl; return 1; }
  const string modelFile = argv[2];
  const int X = atoi(argv[3]), Y = atoi(argv[4]), visits = atoi(argv[5]);
  const float komi = (float)atof(argv[6]);
  Board::initHash();
  ScoreValue::initTables();
  Logger logger(nullptr, false, false, false);
  ConfigParser cfg;
  NNEvaluator* nnEval = new NNEvaluator("lead", modelFile, "", &logger, 4, X, Y, true, true, -1, 8, false, "", enabled_t::False, 1,
                                        vector<int>{0}, "seed", false, 0, true, cfg);
  nnEval->spawnServerThreads();
  SearchParams params;
  params.maxVisits = 1000;
  params.numThreads = 1;
  params.cpuctExploration = 1.0; params.cpuctExplorationLog = 0.45; params.cpuctExplorationBase = 500;
  params.fpuReductionMax = 0.2; params.rootFpuReductionMax = 0.1;
  params.staticScoreUtilityFactor = 0.0; params.dynamicScoreUtilityFactor = 0.0;
  params.valueWeightExponent = 0.0;
  params.rootNoiseEnabled = true;            // computeLead switches the root noise off itself (getNoiselessParams)
  params.rootEndingBonusPoints = 0.0; params.rootPruneUselessMoves = false; params.subtreeValueBiasFactor = 0.0; params.useGraphSearch = false;
  params.useLcbForSelection = false; params.cpuctUtilityStdevScale = 0.0; params.useUncertainty = false; params.useNoisePruning = false;
  Rules rules;
  rules.koRule = Rules::KO_SIMPLE; rules.scoringRule = Rules::SCORING_AREA; rules.taxRule = Rules::TAX_NONE;
  rules.multiStoneSuicideLegal = true; rules.hasButton = false; rules.whiteHandicapBonusRule = Rules::WHB_ZERO;
  rules.friendlyPassOk = false; rules.komi = komi;
  Board board(X, Y);
  Player pla = P_BLACK;
  BoardHistory hist(board, pla, rules, 0, false);
  {
    std::istringstream in(argv[7]);
    string tok;
    while(in >> tok) {
      Loc loc;
      if(tok == "pass") loc = Board::PASS_LOC;
      else { int x, y; if(sscanf(tok.c_str(), "%d,%d", &x, &y) != 2) { cerr << "bad move " << tok << endl; return 1; } loc = Location::getLoc(x, y, X); }
      if(!hist.isLegal(board, loc, pla)) { cerr << "illegal move " << tok << endl; return 1; }
      hist.makeBoardMoveAssumeLegal(board, loc, pla, NULL);
      pla = getOpp(pla);
    }
  }
  Search* bot = new Search(params, nnEval, &logger, "computelead");
  OtherGameProperties props;
  const float lead = PlayUtils::computeLead(bot, bot, board, hist, pla, visits, props);
  cout << "lead " << Global::strprintf("%.9g", lead) << endl;
  cout << "evenkomi " << Global::strprintf("%.9g", komi - lead) << endl;
  delete bot;
  delete nnEval;
  return 0;
}

// komitable MODELFILE X Y VISITS KOMI_LO KOMI_HI MOVES: for every half-integer komi in [KOMI_LO, KOMI_HI], PlayUtils::getWhiteScoreValues
// (program/playutils.cpp:389-417: the noiseless VISITS-visit search that evalKomi runs) of the position after MOVES - one line
// "komi lead winLoss" each.  The bot is the one computelead uses, so the table is the function the komi bisection of computeLead sees
// (its searches do not depend on each other: no noise, symmetry 0, a cleared tree for every komi).  tests/golden/make_komitable_fixture.py.
static int cmdKomiTable(int argc, char** argv) {
  if(argc != 9) { cerr << "usage: komitable MODELFILE X Y VISITS KOMI_LO KOMI_HI MOVES" << endl; return 1; }
  const string modelFile = argv[2];
  const int X = atoi(argv[3]), Y = atoi(argv[4]), visits = atoi(argv[5]);
  const double lo = atof(argv[6]), hi = atof(argv[7]);
  Board::initHash();
  ScoreValue::initTables();
  Logger logger(nullptr, false, false, false);
  ConfigParser cfg;
  NNEvaluator* nnEval = new NNEvaluator("lead", modelFile, "", &logger, 4, X, Y, true, true, -1, 8, false, "", enabled_t::False, 1,
                                        vector<int>{0}, "seed", false, 0, true, cfg);
  nnEval->spawnServerThreads();
  SearchParams params;                       // the same bot as cmdComputeLead
  params.maxVisits = 1000;
  params.numThreads = 1;
  params.cpuctExploration = 1.0; params.cpuctExplorationLog = 0.45; params.cpuctExplorationBase = 500;
  params.fpuReductionMax = 0.2; params.rootFpuReductionMax = 0.1;
  params.staticScoreUtilityFactor = 0.0; params.dynamicScoreUtilityFactor = 0.0;
  params.valueWeightExponent = 0.0;
  params.rootNoiseEnabled = true;
  params.rootEndingBonusPoints = 0.0; params.rootPruneUselessMoves = false; params.subtreeValueBiasFactor = 0.0; params.useGraphSearch = false;
  params.useLcbForSelection = false; params.cpuctUtilityStdevScale = 0.0; params.useUncertainty = false; params.useNoisePruning = false;
  Rules rules;
  rules.koRule = Rules::KO_SIMPLE; rules.scoringRule = Rules::SCORING_AREA; rules.taxRule = Rules::TAX_NONE;
  rules.multiStoneSuicideLegal = true; rules.hasButton = false; rules.whiteHandicapBonusRule = Rules::WHB_ZERO;
  rules.friendlyPassOk = false; rules.komi = 7.5f;
  Board board(X, Y);
  Player pla = P_BLACK;
  BoardHistory hist(board, pla, rules, 0, false);
  {
    std::istringstream in(argv[8]);
    string tok;
    while(in >> tok) {
      Loc loc;
      if(tok == "pass") loc = Board::PASS_LOC;
      else { int x, y; if(sscanf(tok.c_str(), "%d,%d", &x, &y) != 2) { cerr << "bad move " << tok << endl; return 1; } loc = Location::getLoc(x, y, X); }
      if(!hist.isLegal(board, loc, pla)) { cerr << "illegal move " << tok << endl; return 1; }
      hist.makeBoardMoveAssumeLegal(board, loc, pla, NULL);
      pla = getOpp(pla);
    }
  }
  Search* bot = new Search(params, nnEval, &logger, "computelead");
  OtherGameProperties props;
  for(double k = lo; k <= hi + 1e-9; k += 0.5) {
    hist.setKomi((float)k);
    const ReportedSearchValues v = PlayUtils::getWhiteScoreValues(bot, board, hist, pla, visits, props);
    cout << Global::strprintf("%.1f %.17g %.17g", k, v.lead, v.winLossValue) << "\n";
  }
  delete bot;
  delete nnEval;
  return 0;
}

// gameinit CFGFILE N SEED: N games of the reference's GameInitializer::createGame (program/play.cpp:330-650) on the given .cfg: per game
// "X Y koRule multiStoneSuicide komi" - the per-game draws katago_b200/game_initializer.py restates (board size with rectangle probability,
// rules, komi noise scaled by the board, linear rounding, integer komi allowed with probability komiAllowIntegerProb).
static int cmdGameInit(int argc, char** argv) {
  if(argc != 5) { cerr << "usage: gameinit CFGFILE N SEED" << endl; return 1; }
  Board::initHash();
  ScoreValue::initTables();
  Logger logger(nullptr, false, false, false);
  ConfigParser cfg(argv[2]);
  GameInitializer gi(cfg, logger, argv[4]);
  PlaySettings ps;
  const int n = atoi(argv[3]);
  for(int i = 0; i < n; i++) {
    Board board; Player pla; BoardHistory hist; ExtraBlackAndKomi ebk; OtherGameProperties props;
    gi.createGame(board, pla, hist, ebk, NULL, ps, props, NULL, false);
    cout << board.x_size << " " << board.y_size << " " << hist.rules.koRule << " " << (hist.rules.multiStoneSuicideLegal ? 1 : 0) << " "
         << Global::strprintf("%.1f", hist.rules.komi) << "\n";
  }
  return 0;
}

int main(int argc, char** argv) {
  if(argc < 2) { cerr << "usage: kgref_driver <boardstream|...> ..." << endl; return 1; }
  string cmd = argv[1];
  if(cmd == "boardstream") return cmdBoardStream(argc, argv);
  if(cmd == "searchfake") return cmdSearchFake(argc, argv);
  if(cmd == "svsamples") return cmdSVSamples(argc, argv);
  if(cmd == "vwtable") return cmdVWTable(argc, argv);
  if(cmd == "rootnoise") return cmdRootNoise(argc, argv);
  if(cmd == "chooseidx") return cmdChooseIdx(argc, argv);
  if(cmd == "histstream") return cmdHistStream(argc, argv);
  if(cmd == "repbound") return cmdRepBound(argc, argv);
  if(cmd == "npyheader") return cmdNpyHeader(argc, argv);
  if(cmd == "addrow") return cmdAddRow(argc, argv);
  if(cmd == "writegame") return cmdWriteGame(argc, argv);
  if(cmd == "paramsmap") return cmdParamsMap(argc, argv);
  if(cmd == "rungame") return cmdRunGame(argc, argv);
  if(cmd == "tinyfeatures") return cmdTinyFeatures(argc, argv);
  if(cmd == "featstream") return cmdFeatStream(argc, argv);
  if(cmd == "ladderrows") return cmdLadderRows(argc, argv);
  if(cmd == "computelead") return cmdComputeLead(argc, argv);
  if(cmd == "komitable") return cmdKomiTable(argc, argv);
  if(cmd == "gameinit") return cmdGameInit(argc, argv);
  cerr << "unknown command " << cmd << endl;
  return 1;
}
