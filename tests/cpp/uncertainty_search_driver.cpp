// tests/cpp/uncertainty_search_driver.cpp - TEST INFRASTRUCTURE for tests/golden/make_uncertainty_fixture.py.  Links against the unmodified
// reference (oracle/_ref/libkgref.a, built by oracle/Makefile.ref) and runs the reference's own Search with uncertainty-weighted
// evaluations and noise pruning on the device loop's hash fake net; the generator compiles it when it regenerates the fixture.
//
//   uncertainty_search_driver MODELFILE X Y MAXVISITS FAKE_SHORTTERM "x,y x,y pass ..." [key=value ...]
//       FAKE_SHORTTERM = 0: the fake net of oracle/ref_driver.cpp (debug_fake_nn = 1, short-term error channels 0);
//       1: the same net with hash-derived raw short-term error channels in [-2,2) (debug_fake_nn = 2).  Whether the errors count is
//       NNEvaluator::supportsShorttermError, i.e. the version of MODELFILE.  Prints the root children's edge visits, utilities and
//       weight sums, the root's weight sums and the seed string of the search thread's Rand.
//   uncertainty_search_driver paramsmap CFG
//       the reference's own loader (ConfigParser + Setup::loadSingleParams, SETUP_FOR_OTHER) on CFG, mapped by integration/b200params.h:
//       the uncertainty and noise-pruning fields of kgb_selfplay_config and the options reported as not implemented, as JSON.
#include "core/config_parser.h"
#include "core/logger.h"
#include "integration/b200params.h"
#include "program/setup.h"
#include "game/board.h"
#include "game/boardhistory.h"
#include "game/rules.h"
#include "neuralnet/nneval.h"
#include "neuralnet/nninputs.h"
#include "neuralnet/nninterface.h"
#include "search/search.h"
#include "search/searchnode.h"

#include <cstdint>
#include <cstdio>
#include <iostream>
#include <sstream>
#include <vector>

using namespace std;

namespace Version {  // main.cpp normally defines these (cpp/main.h)
  std::string getKataGoVersion() { return "uncertainty_search_driver"; }
  std::string getKataGoVersionForHelp() { return "uncertainty_search_driver"; }
  std::string getKataGoVersionFullInfo() { return "uncertainty_search_driver"; }
  std::string getGitRevision() { return "<none>"; }
  std::string getGitRevisionWithBackend() { return "<none>"; }
}

static bool fakeShortterm = false;

// The fake NeuralNet backend: the hash net of oracle/ref_driver.cpp and of the device loop's spFakeNNKernel (exact dyadic outputs from an
// order-independent hash of the stone planes, the sign of selfKomi and the symmetry), plus the short-term error channels of debug_fake_nn = 2.
static inline uint64_t splitmix64(uint64_t x) {
  x += 0x9E3779B97F4A7C15ULL;
  x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ULL;
  x = (x ^ (x >> 27)) * 0x94D049BB133111EBULL;
  return x ^ (x >> 31);
}
static inline float hashUnit(uint64_t h, float scale, float offset) { return (float)(uint32_t)(splitmix64(h) >> 48) * scale + offset; }
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
  for(int r = 0; r < n; r++) {
    const float* sp = inputBufs[r]->rowSpatialBuf.data();
    const float* gl = inputBufs[r]->rowGlobalBuf.data();
    uint64_t hsh = 0;
    for(int pos = 0; pos < xy; pos++) {
      const int s = sp[pos * 22 + 1] != 0.0f ? 1 : sp[pos * 22 + 2] != 0.0f ? 2 : 0;
      if(s) hsh += splitmix64((uint64_t)pos * 4 + s);
    }
    if(gl[5] < 0.0f) hsh ^= 0xABCDEFULL;
    if(inputBufs[r]->symmetry != 0) hsh ^= splitmix64(0x5151ULL + (uint64_t)inputBufs[r]->symmetry);
    NNOutput* o = outputs[r];
    for(int i = 0; i <= xy; i++) {
      float logit = hashUnit(hsh + (uint64_t)(i + 1) * 0x9E3779B97F4A7C15ULL, 1.0f / 8192.0f, -4.0f);
      if(i == xy) logit -= 3.0f;
      o->policyProbs[i] = logit;
    }
    o->whiteWinProb = hashUnit(hsh ^ 0x1111ULL, 1.0f / 8192.0f, -4.0f);
    o->whiteLossProb = hashUnit(hsh ^ 0x2222ULL, 1.0f / 8192.0f, -4.0f);
    o->whiteNoResultProb = -30.0f;
    o->whiteScoreMean = hashUnit(hsh ^ 0x3333ULL, 1.0f / 32768.0f, -1.0f);
    o->whiteScoreMeanSq = hashUnit(hsh ^ 0x4444ULL, 1.0f / 16384.0f, -2.0f);
    o->whiteLead = hashUnit(hsh ^ 0x5555ULL, 1.0f / 32768.0f, -1.0f);
    o->varTimeLeft = 0;
    o->shorttermWinlossError = fakeShortterm ? hashUnit(hsh ^ 0x6666ULL, 1.0f / 16384.0f, -2.0f) : 0.0f;
    o->shorttermScoreError = fakeShortterm ? hashUnit(hsh ^ 0x7777ULL, 1.0f / 16384.0f, -2.0f) : 0.0f;
    if(o->whiteOwnerMap != NULL)
      for(int i = 0; i < xy; i++) o->whiteOwnerMap[i] = hashUnit(hsh + (uint64_t)(i + 1) * 0xD1B54A32D192ED03ULL, 1.0f / 8192.0f, -4.0f);
  }
}
bool NeuralNet::testEvaluateConv(const ConvLayerDesc*, int, int, int, bool, bool, const std::vector<float>&, std::vector<float>&) { return false; }
bool NeuralNet::testEvaluateBatchNorm(const BatchNormLayerDesc*, int, int, int, bool, bool, const std::vector<float>&, const std::vector<float>&, std::vector<float>&) { return false; }
bool NeuralNet::testEvaluateResidualBlock(const ResidualBlockDesc*, int, int, int, bool, bool, const std::vector<float>&, const std::vector<float>&, std::vector<float>&) { return false; }
bool NeuralNet::testEvaluateGlobalPoolingResidualBlock(const GlobalPoolingResidualBlockDesc*, int, int, int, bool, bool, const std::vector<float>&, const std::vector<float>&, std::vector<float>&) { return false; }

static int paramsMap(const string& cfgPath) {
  ConfigParser cfg(cfgPath);
  const SearchParams p = Setup::loadSingleParams(cfg, Setup::SETUP_FOR_OTHER);
  Rules rules;
  rules.koRule = Rules::KO_SIMPLE; rules.scoringRule = Rules::SCORING_AREA; rules.taxRule = Rules::TAX_NONE; rules.multiStoneSuicideLegal = false;
  rules.hasButton = false; rules.whiteHandicapBonusRule = Rules::WHB_ZERO; rules.friendlyPassOk = false; rules.komi = 7.5f;
  vector<string> unsupported;
  const kgb_selfplay_config c = b200::configFromSearchParams(p, rules, 256, 0, 1, 0, &unsupported);
  cout << Global::strprintf("{\"use_uncertainty\":%d,\"uncertainty_coeff\":%.17g,\"uncertainty_exponent\":%.17g,\"uncertainty_max_weight\":%.17g,"
                            "\"use_noise_pruning\":%d,\"noise_prune_utility_scale\":%.17g,\"noise_pruning_cap\":%.17g,\"unsupported\":[",
                            c.use_uncertainty, c.uncertainty_coeff, c.uncertainty_exponent, c.uncertainty_max_weight, c.use_noise_pruning,
                            c.noise_prune_utility_scale, c.noise_pruning_cap);
  for(size_t i = 0; i < unsupported.size(); i++) cout << (i ? "," : "") << "\"" << unsupported[i] << "\"";
  cout << "]}" << endl;
  return 0;
}

int main(int argc, char** argv) {
  if(argc == 3 && string(argv[1]) == "paramsmap") return paramsMap(argv[2]);
  if(argc < 7) { cerr << "usage: uncertainty_search_driver MODELFILE X Y MAXVISITS FAKE_SHORTTERM MOVES [key=value ...]" << endl; return 1; }
  const string modelFile = argv[1];
  const int X = atoi(argv[2]), Y = atoi(argv[3]), maxVisits = atoi(argv[4]);
  fakeShortterm = atoi(argv[5]) != 0;
  Board::initHash();
  ScoreValue::initTables();
  Logger logger(nullptr, false, false, false);
  ConfigParser cfg;
  NNEvaluator* nnEval = new NNEvaluator("fake", modelFile, "", &logger, 4, X, Y, true, true, 10, 8, false, "", enabled_t::False, 1,
                                        vector<int>{0}, "seed", false, 0, true, cfg);
  nnEval->spawnServerThreads();
  // the defaults of oracle/ref_driver.cpp's searchfake (the parameter subset of the device loop), then the overrides by their cfg names
  SearchParams params;
  params.maxVisits = maxVisits;
  params.numThreads = 1;
  params.cpuctExploration = 1.0; params.cpuctExplorationLog = 0.45; params.cpuctExplorationBase = 500;
  params.fpuReductionMax = 0.2; params.rootFpuReductionMax = 0.1;
  params.staticScoreUtilityFactor = 0.0; params.dynamicScoreUtilityFactor = 0.0;
  params.valueWeightExponent = 0.0;
  params.rootNoiseEnabled = false;
  for(int i = 7; i < argc; i++) {
    const string kv = argv[i];
    const size_t eq = kv.find('=');
    if(eq == string::npos) { cerr << "bad override " << kv << endl; return 1; }
    const string k = kv.substr(0, eq);
    const double v = atof(kv.substr(eq + 1).c_str());
    if(k == "staticScoreUtilityFactor") params.staticScoreUtilityFactor = v;
    else if(k == "dynamicScoreUtilityFactor") params.dynamicScoreUtilityFactor = v;
    else if(k == "dynamicScoreCenterZeroWeight") params.dynamicScoreCenterZeroWeight = v;
    else if(k == "dynamicScoreCenterScale") params.dynamicScoreCenterScale = v;
    else if(k == "valueWeightExponent") params.valueWeightExponent = v;
    else if(k == "fpuParentWeightByVisitedPolicy") params.fpuParentWeightByVisitedPolicy = v != 0;
    else if(k == "fpuParentWeightByVisitedPolicyPow") params.fpuParentWeightByVisitedPolicyPow = v;
    else if(k == "fpuReductionMax") params.fpuReductionMax = v;
    else if(k == "rootFpuReductionMax") params.rootFpuReductionMax = v;
    else if(k == "cpuctExploration") params.cpuctExploration = v;
    else if(k == "cpuctExplorationLog") params.cpuctExplorationLog = v;
    else if(k == "rootDesiredPerChildVisitsCoeff") params.rootDesiredPerChildVisitsCoeff = v;
    else if(k == "rootNumSymmetriesToSample") params.rootNumSymmetriesToSample = (int)v;
    else if(k == "useLcbForSelection") params.useLcbForSelection = v != 0;
    else if(k == "useNonBuggyLcb") params.useNonBuggyLcb = v != 0;
    else if(k == "lcbStdevs") params.lcbStdevs = v;
    else if(k == "minVisitPropForLCB") params.minVisitPropForLCB = v;
    else if(k == "chosenMoveSubtract") params.chosenMoveSubtract = v;
    else if(k == "chosenMovePrune") params.chosenMovePrune = v;
    else if(k == "useGraphSearch") params.useGraphSearch = v != 0;
    else if(k == "subtreeValueBiasFactor") params.subtreeValueBiasFactor = v;
    else if(k == "subtreeValueBiasWeightExponent") params.subtreeValueBiasWeightExponent = v;
    else if(k == "rootNoiseEnabled") params.rootNoiseEnabled = v != 0;
    else if(k == "rootDirichletNoiseTotalConcentration") params.rootDirichletNoiseTotalConcentration = v;
    else if(k == "rootDirichletNoiseWeight") params.rootDirichletNoiseWeight = v;
    else if(k == "useUncertainty") params.useUncertainty = v != 0;
    else if(k == "uncertaintyCoeff") params.uncertaintyCoeff = v;
    else if(k == "uncertaintyExponent") params.uncertaintyExponent = v;
    else if(k == "uncertaintyMaxWeight") params.uncertaintyMaxWeight = v;
    else if(k == "useNoisePruning") params.useNoisePruning = v != 0;
    else if(k == "noisePruneUtilityScale") params.noisePruneUtilityScale = v;
    else if(k == "noisePruningCap") params.noisePruningCap = v;
    else { cerr << "unknown override " << k << endl; return 1; }
  }
  Rules rules;   // the rule subset of the loop
  rules.koRule = Rules::KO_SIMPLE; rules.scoringRule = Rules::SCORING_AREA; rules.taxRule = Rules::TAX_NONE;
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
  ConstSearchNodeChildrenReference children = root->getChildren((SearchNodeState)root->state.load());
  {
    std::ostringstream ss;   // makeSeed(search, 0) (search.cpp:24-36): the seed string of search thread 0's Rand
    ss << "searchfake" << "$searchThread$" << 0 << "$" << board.pos_hash << "$" << hist.moveHistory.size() << "$" << search->numSearchesBegun;
    cout << "threadseed " << ss.str() << endl;
  }
  cout << "rootweights " << Global::strprintf("%.17g %.17g", root->stats.weightSum.load(), root->stats.weightSqSum.load()) << endl;
  for(int i = 0; i < children.getCapacity(); i++) {
    const SearchChildPointer& cp = children[i];
    const SearchNode* child = cp.getIfAllocated();
    if(child == NULL) break;
    const Loc loc = cp.getMoveLoc();
    const int x = loc == Board::PASS_LOC ? -1 : Location::getX(loc, X), y = loc == Board::PASS_LOC ? -1 : Location::getY(loc, X);
    cout << "child " << x << " " << y << " " << cp.getEdgeVisits() << " " << Global::strprintf("%.17g", child->stats.utilityAvg.load()) << " "
         << Global::strprintf("%.17g %.17g", child->stats.weightSum.load(), child->stats.weightSqSum.load()) << endl;
  }
  delete search;
  delete nnEval;
  return 0;
}
