// Device-resident self-play playout loop (round-1 scope: see DESIGN.md §8 "device loop" for what is and is not
// reference-equivalent yet).  One warp per game; a "step" = one playout for every game:
//
//   spSelectKernel   (a) root move + tree reset when the visit budget is reached        play.cpp:1757-1936 (core only)
//                    (b) PUCT descent from the root on a register-resident bitboard      search.cpp:1189-1463,
//                        Board::playMoveAssumeLegal per edge (kgb_board.cuh)             searchexplorehelpers.cpp:22-54,265-643
//                    (c) leaf: liberty classes, legality, NN input row                   nninputs.cpp:2288-2731 (planes listed below)
//   NN forward       the CUDA-graph op list of the evaluator (kgb_api.cu), batch = number of games
//   spBackupKernel   (d) policy: legality mask + softmax; value: softmax -> white utility nneval.cpp:960-1051,1112-1215
//                    (e) backup along the path                                           searchupdatehelpers.cpp:11-81,139-360
//
// Tree layout (per game, per node, SoA):
//   by move position 0..X*Y (pass last): policy[pos] fp32 (-1 = illegal), childNode[pos] i32 (-1 = not expanded),
//                                        childVisits[pos] i32 (edge visits);
//   childOrder[k] = move position of the k-th child in CREATION order (the reference walks its children array in that order and
//                   breaks ties by it; sums over children are done sequentially in that order so doubles match);
//   node statistics as in NodeStats (searchnode.h:17-41): visits, weightSum, weightSqSum, utilityAvg, utilitySqAvg, plus the
//                   node's own evaluation utility (the reference keeps the NNOutput).
// Backup = the reference's recompute (searchupdatehelpers.cpp:139-360): every node on the path re-derives its statistics from
// its children (value weighting by the t-CDF of each child's z-score, :402-491) and its own evaluation.
//
// NN input planes written this round: 0 on-board, 1/2 own/opp stones, 3/4/5 liberties 1/2/3, 6 simple-ko ban and superko bans,
// 9-13 previous five move locations, 18/19 pass-alive + territory area (Benson, kgb_board.cuh); globals 0-4 pass history,
// 5 selfKomi/20, 8 multi-stone suicide, 14 pass would end the phase, 18 komi parity wave; ladder planes 14-17 (kgb_ladder.cuh).
// NOT written (stay 0, not reachable under the supported rule subset): encore planes 7/8/20/21.
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <memory>
#include <stdexcept>
#include <string>
#include <vector>

#include "../../include/kgb200.h"
#include "kgb_board.cuh"
#include "kgb_devrand.cuh"
#include "kgb_handle.h"
#include "kgb_history.cuh"
#include "kgb_ladder.cuh"
#include "kgb_scorevalue.h"
#include "kgb_rand.h"

namespace kgb {

static constexpr int SP_MAX_PLAYOUTS_PER_WAVE = 16;   // playouts a game may finish inside one wave without needing the evaluator
static constexpr int SP_MAX_INIT_MOVES = 512;   // policy-initialised opening moves kept per game (longer openings are cut there)
static constexpr int SP_LADDER_WARPS = 8;   // warps per game in the select kernel (ladder searches are dealt out to all of them)

struct SPDev {
  // configuration
  int X, Y, XY, policySize, numGames, maxVisits, maxNodes, maxDepth, maxMoves, earlyMoves;
  // per-game board size and rules (GameInitializer::createGameSharedUnsynchronized, program/play.cpp:330-650 draws them per game): the
  // evaluator's frame is X x Y (nnXLen x nnYLen), a game's board gX x gY <= the frame sits in its top-left corner, move positions are
  // y * X + x in the frame (NNPos::locToPos, nninputs.cpp:27-33) and plane 0 marks the board.  setup arrays are [game][4] = X, Y, koRule, multiSuicide.
  // search limits per move (getSearchLimitsThisMove / runBotWithLimits, program/play.cpp:1093-1300: cheap searches, reduced visits): the
  // visit budget of the current root and whether its root-only parameters are switched off (removeRootNoise: no Dirichlet noise, root
  // policy temperature 1, the root takes the tree's FPU parameters, no per-child visit floor, one root symmetry); next* = what the
  // following root gets, [game][2]: 0 = the game goes on, 1 = this move ends it and the slot's next game starts
  int *visitBudget, *nextBudget;
  uint8_t *plainRoot, *nextPlain;
  // policy-initialised openings (PlayUtils::initializeGameUsingPolicy, program/playutils.cpp:232-266): the first initMovesLeft moves of a game
  // are drawn from the net's raw policy ^ (1 / temperature) of the position (one evaluation per move, no search, never held for recording);
  // they are kept in initMoves for the game record.  nextInitMoves = the count for the slot's next game (the host draws it)
  double* rootRawEntropy;           // [game] entropy of the current root's policy as evaluated, before temperature and noise (NNRawStats::policyEntropy, play.cpp:890-914)
  int *initMovesLeft, *nextInitMoves, *initMoveCount;
  int16_t* initMoves;               // [game][SP_MAX_INIT_MOVES] move positions of the current game's opening
  double* policyInitTemperature;    // [1] in device memory (the wave's kernel arguments are frozen in its CUDA graph)
  int *gX, *gY, *gKoRule, *gMultiSuicide;   // [game] of the game in progress
  int *nextSetup, *lastSetup;               // [game][4]: of the slot's next game (kgb_selfplay_set_game_setup), of its last finished game
  double cpuctExploration, cpuctExplorationLog, cpuctExplorationBase, fpuReductionMax, rootFpuReductionMax;
  double cpuctUtilityStdevPrior, cpuctUtilityStdevPriorWeight, cpuctUtilityStdevScale;
  double fpuLossProp, rootFpuLossProp, fpuParentWeight, fpuParentWeightByVisitedPolicyPow, valueWeightExponent, rootDesiredPerChildVisitsCoeff;
  int fpuParentWeightByVisitedPolicy;
  // subtree value bias (search.cpp:913-922, searchupdatehelpers.cpp:26-36, 273-310; subtreevaluebiastable.cpp): per game, per move
  double subtreeValueBiasFactor, subtreeValueBiasWeightExponent;
  int biasTableSize;                // slots per game (power of two)
  unsigned long long* biasKey;      // [game][biasTableSize] 0 = empty
  double *biasDeltaSum, *biasWeightSum;   // [game][biasTableSize] SubtreeValueBiasEntry
  int* nodeBiasEntry;               // [game][maxNodes] slot or -1
  // full ko rules / game end (kgb_history.cuh): ko-hash history, pass situations, ever-occupied points, superko bans
  int histCap, pathCap;
  unsigned long long *gKo, *gPassB, *gPassW;   // [game][histCap]
  int *gKoLen, *gPassBLen, *gPassWLen;         // [game]
  uint32_t *gEverOcc, *rootBanned;             // [game][32]
  unsigned long long *pKo, *pPassB, *pPassW;   // [game][pathCap] the path part of the lists during a playout
  // graph search (search.cpp:875-936, game/graphhash.cpp): transposition table per game, cleared with the tree
  int useGraphSearch, graphSearchRepBound, holdAtMaxVisits;
  // evaluation cache (NNCacheTable, nneval.cpp:1273-1353; key = NNInputs::getHash, nninputs.cpp:869-943): direct mapped, shared by
  // all games of the GPU.  An entry holds what NNOutput holds for the search: post-processed policy, white win/loss/noResult,
  // white score mean / mean-square / lead, the two short-term errors (not the weight: it depends on the search's score centre),
  // plus the position's laddered stones (a function of the same position, needed by descendants).
  int cacheSize;                    // entries (power of two), 0 = off
  unsigned long long *cacheKey0, *cacheKey1;
  int* cacheLock;
  float* cachePolicy;               // [cacheSize][policySize]
  float* cacheVals;                 // [cacheSize][8]
  uint32_t* cacheLad;               // [cacheSize][32]
  unsigned long long *leafKey;      // [game][2] cache key of the current leaf
  unsigned long long *cacheHits, *cacheStores;
  // root policy temperature and Dirichlet noise (searchhelpers.cpp:78-215)
  // rootNumSymmetriesToSample (searchnnhelpers.cpp:95-101, nneval.cpp:811-838, nninputs.cpp:324-430): the root is evaluated under
  // several distinct symmetries, one per wave, and the post-processed outputs are averaged
  int rootNumSymmetries, fakeNN;    // fakeNN: 0 the evaluator, 1 the hash net, 2 the hash net with raw short-term error channels,
                                    // 3 the table net: every evaluation of game g returns the raw outputs in fakeTable,
                                    // 4 the wide hash net (same hash, wider output ranges)
  float* fakeTable;                 // [game][policySize + 3 + 6 + XY] raw policy logits, value, score-value and ownership (fakeNN 3 only)
  int* rootSymCount;                // [game] evaluations of the current root accumulated so far
  int* rootSymOrder;                // [game][8] the sampled symmetry order
  float* rootSymAcc;                // [game][8] sums of whiteWin, whiteLoss, noResult, whiteScoreMean, whiteScoreMeanSq, whiteLead,
                                    // shorttermWinlossError, shorttermScoreError (NNOutput(others), nninputs.cpp:327-363)
  int rootNoiseEnabled;
  double rootDirichletNoiseTotalConcentration, rootDirichletNoiseWeight, rootPolicyTemperature, rootPolicyTemperatureEarly, chosenMoveTemperatureHalflife;
  // root move choice (searchresults.cpp:24-330 play selection values, :573-598 getChosenMoveLoc, searchhelpers.cpp:12-76)
  int usePlaySelection, useLcbForSelection, useNonBuggyLcb;
  double lcbStdevs, minVisitPropForLCB, chosenMoveTemperature, chosenMoveTemperatureEarly, chosenMoveTemperatureOnlyBelowProb,
    chosenMoveSubtract, chosenMovePrune;
  DevRandState* nonSearchRand;      // [game] Search::nonSearchRand
  double* selScratch;               // [game][3][policySize] play selection values, lcb, radius
  DevRandState* searchRand;         // [game] the search thread's Rand
  double* noiseScratch;             // [game][policySize]
  int nodeTableSize;                // slots per game (power of two)
  unsigned long long *nodeTableKey0, *nodeTableKey1;   // [game][nodeTableSize]
  int* nodeTableNode;               // [game][nodeTableSize] node index or -1
  unsigned long long *nodePosH0, *nodePosH1, *nodeGH0, *nodeGH1;   // [game][maxNodes] Zobrist position hash and graph hash
  unsigned long long *rootPosH;     // [game][2]
  const ZobEntry* zob;              // Board::ZOBRIST_BOARD_HASH for this board size
  unsigned long long* instantPlayouts;   // playouts that ended on an edge catch-up or a cycle (no evaluation needed)
  double *nodeLastBiasDelta, *nodeLastBiasWeight;   // [game][maxNodes]
  const double* vwCdfTable;         // value-weighting t-CDF table [2000]
  double winLossUtilityFactor, noResultUtilityForWhite;
  // score utility (searchhelpers.cpp:272-279): static * SV(mean, stdev; 0, 2) + dynamic * SV(mean, stdev; recentScoreCenter, scale)
  double staticScoreUtilityFactor, dynamicScoreUtilityFactor, dynamicScoreCenterZeroWeight, dynamicScoreCenterScale, drawEquivalentWinsForWhite;
  double scoreMeanMultiplier, scoreStdevMultiplier;   // ModelPostProcessParams of the net
  const double* svTable;            // ScoreValue's expectedSVTable [842][421]
  double* recentScoreCenter;        // [game] Search::recentScoreCenter of the current root
  // evaluation weights (Search::computeWeightFromNNOutput, searchupdatehelpers.cpp:114-136): useUncertainty = the switch and a net that
  // reports short-term errors (model version >= 9, nneval.cpp:299); otherwise every evaluation has weight 1
  int useUncertainty, modelVersion;
  double uncertaintyCoeff, uncertaintyExponent, uncertaintyMaxWeight;
  double shorttermValueErrorMultiplier, shorttermScoreErrorMultiplier;   // ModelPostProcessParams of the net
  double* nodeNNWeight;             // [game][maxNodes] weight of the node's own evaluation (allocated when useUncertainty)
  // Search::pruneNoiseWeight (searchupdatehelpers.cpp:495-539) in every recompute
  int useNoisePruning;
  double noisePruneUtilityScale, noisePruningCap;
  float* leafTerminalScore;         // [game] finalWhiteMinusBlackScore of a terminal leaf
  const float* nnScore;             // [game][6] raw score head (whiteScoreMean, stdev pre-softplus, lead, ...)
  uint64_t seed;
  // root state [game]
  uint32_t *rootB, *rootW;          // [game][32]
  int *rootKo, *rootBlackToMove, *rootCapB, *rootCapW, *moveNum, *consecPasses;
  uint32_t *prevB, *prevW;          // [2][game][32]: boards 1 and 2 moves ago (BoardHistory::getRecentBoard), for ladder planes 15/16
  int* prevKo;                      // [2][game]
  int* leafNumHist;                 // [game] min(2, moves of history) at the current leaf
  uint32_t *leafB, *leafW, *leafCand;   // [game][32] leaf board and its 1-2 liberty stones, kept while its ladder searches run
  int* leafKo;                      // [game]
  int* ladPending;                  // [game] 1 = the leaf's ladder searches were cut off by ladderNodesPerWave; resume next wave
  int* leafValid;                   // [game] 1 = this wave produced a finished leaf (features complete) for the evaluator / backup
  int ladderNodesPerWave;           // per warp; 0 = unlimited
  int fixedSymmetryPlusOne;         // TEST ONLY (kgb_selfplay_config.debug_fixed_symmetry_plus_one)
  int maxPlayoutsPerWave;           // playouts a game may finish inside one select launch without needing the evaluator
  unsigned long long* stalledWaves; // game-waves that did not produce a leaf
  // Search::getEndingWhiteScoreBonus / isAllowedRootMove (searchhelpers.cpp:310-420): per-root data, filled when the root's evaluation is final
  double rootEndingBonusPoints; int rootPruneUselessMoves;
  const float* nnOwnership;         // [game][XY] raw ownership logits of the last wave (original orientation, mover's perspective)
  float* rootOwnAcc;                // [game][XY] sum over the root's evaluations of white's ownership (tanh, colour flipped): NNOutput averaging
  double* rootEndBonus;             // [game][policySize] ending score bonus of every root move, white's perspective (0 = none)
  uint32_t* rootAllowed;            // [game][32] root moves Search::isAllowedRootMove accepts (bit x of row y); the pass always is
  int* passStreak;                  // [game][2] consecutive passes most recently made by black / white (the opponent's last four moves were passes <=> >= 4)
  float* rootRow;                   // [game][XY*22 + 19]: the NN input row (fillRowV7, no symmetry) of the game's current root, kept when the root is evaluated
  long long* dbgCycles;             // [game][8] clock64 spans of the last select launch: whole block, root move + tree reset, warp 0 (descent + leaf features), ladder searches, descent, liberties + legality, area (Benson), feature-row writes
  uint32_t* ladderScratch;          // [game][SP_LADDER_WARPS][ladderScratchWordsPerWarp()]
  uint32_t* prevLad;                // [2][game][32]: laddered stones (plane 14) of those two boards = planes 15/16 at the root
  uint32_t* nodeLad;                // [game][maxNodes][32]: laddered stones of the node's own board, kept for its descendants
  unsigned long long* ladderCounters;   // [2] searches, search nodes
  int enableLadders;
  int* hist;                        // [game][5] last moves, most recent first: -1 none, -2 pass, else y*32+x
  // game recording (hold mode): a held game moves once the host has read its search and set its release flag; the root move and, when
  // it ended the game, the final position with its area stay readable until the slot's next move
  uint8_t* releaseFlag;             // [game]
  int* lastMove;                    // [game][4]: move position (policySize-1 = pass), 1 over | 2 no result | 4 move limit, its move number, games started
  float* lastScore;                 // [game] white minus black incl. komi of the game the last move ended
  uint32_t* finalBoard;             // [game][4][32]: black, white, black area, white area of that game's final position
  uint64_t* gameCounter;            // games started per slot (RNG stream)
  // tree [game][node]...
  int* nodeCount;                   // [game]
  int* nodeVisits;                  // [game][maxNodes]
  double *nodeWeightSum, *nodeWeightSqSum, *nodeUtilAvg, *nodeUtilSqAvg;   // [game][maxNodes] NodeStats (white's perspective)
  double* nodeNNUtil;               // [game][maxNodes] utility of the node's own evaluation (Search::getUtilityFromNN)
  // the other five moments of NodeStats (searchnode.h:17-41): winLossValueAvg, noResultValueAvg, scoreMeanAvg, scoreMeanSqAvg, leadAvg
  // (white's perspective) and the node's own evaluation of them; they feed targets and reports, not the selection
  double* nodeMoments;              // [game][maxNodes][5]
  double* nodeNNMoments;            // [game][maxNodes][5]
  double* leafMoments;              // [game][5] the current leaf's own values, set where its utility is computed
  double leadMultiplier;
  int* nodeNumChildren;             // [game][maxNodes]
  uint16_t* childOrder;             // [game][maxNodes][policySize] move position of the k-th created child
  int8_t* nodeTerminal;             // [game][maxNodes]   0 no, 1 yes
  float* policy;                    // [game][maxNodes][policySize]
  int* childNode;                   // same shape
  int* childVisits;                 // edge visits
  // per-playout scratch
  int *pathLen, *pathNode, *pathMove;   // [game], [game][maxDepth] x2
  int *leafNode, *leafTerminal, *leafBlackToMove;
  uint32_t* leafLegal;              // [game][32] row masks of legal points for the player to move at the leaf
  // statistics
  float *komiG, *nextKomi, *lastKomi;   // per game: komi of the game in progress, of the slot's next game, of its last finished game
  unsigned long long *totalVisits, *totalMoves, *gamesFinished, *blackWins, *nodesAllocated, *sumDepth;
  // evaluator buffers (owned by the kgb_handle)
  float *nnSpatial, *nnGlobal, *nnOptimism;
  int* nnSymmetry;
  const float *nnPolicy, *nnValue;
};

__device__ __forceinline__ int rootSyms(const SPDev& d, int g) { return d.plainRoot[g] ? 1 : d.rootNumSymmetries; }   // rootNumSymmetriesToSample of game g's current root

__device__ __forceinline__ uint64_t splitmix64(uint64_t x) {
  x += 0x9E3779B97F4A7C15ULL;
  x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ULL;
  x = (x ^ (x >> 27)) * 0x94D049BB133111EBULL;
  return x ^ (x >> 31);
}

__device__ __forceinline__ int posOf(int p, int X) { return (p >> 5) * X + (p & 31); }   // y*32+x -> y*X+x
__device__ __forceinline__ int pointOfPos(int pos, int X) { return ((pos / X) << 5) | (pos % X); }

__device__ __forceinline__ double warpSumD(double v) {
#pragma unroll
  for(int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(KGB_FULL, v, o);
  return v;
}

// Reset a node's per-move arrays (coalesced).
__device__ __forceinline__ void nodeInit(const SPDev& d, size_t nodeBase, int lane) {
  for(int i = lane; i < d.policySize; i += 32) {
    d.childNode[nodeBase + i] = -1;
    d.childVisits[nodeBase + i] = 0;
    d.policy[nodeBase + i] = -1.0f;
  }
}
// Fresh node: no visits, no children (one lane).
__device__ __forceinline__ void nodeStatsReset(const SPDev& d, size_t gn, bool terminal) {
  d.nodeVisits[gn] = 0; d.nodeWeightSum[gn] = 0.0; d.nodeWeightSqSum[gn] = 0.0; d.nodeUtilAvg[gn] = 0.0; d.nodeUtilSqAvg[gn] = 0.0;
  d.nodeNNUtil[gn] = 0.0; d.nodeNumChildren[gn] = 0; d.nodeTerminal[gn] = terminal ? 1 : 0;
  for(int i = 0; i < 5; i++) { d.nodeMoments[gn * 5 + i] = 0.0; d.nodeNNMoments[gn * 5 + i] = 0.0; }
  d.nodeBiasEntry[gn] = -1; d.nodeLastBiasDelta[gn] = 0.0; d.nodeLastBiasWeight[gn] = 0.0;
}
// Key of a SubtreeValueBiasTable entry (subtreevaluebiastable.cpp:70-88, localpattern.cpp:52-87): who moved, the move before,
// the move, the ko point and the 5x5 neighbourhood of the move on the board BEFORE it (colour and in-atari per on-board cell).
// The reference XORs Zobrist codes of exactly this information; any injective-enough hash of it defines the same classes.
__device__ unsigned long long biasEntryKey(const WarpBoard& bd, int X, int Y, bool moverBlack, int prevMove /*hist code*/, int p) {
  uint32_t lib1, lib2, lib3;
  boardLibertyClasses(bd, lib1, lib2, lib3);
  const int x = p & 31, y = p >> 5;
  unsigned long long lo = 0, hi = 0;
#pragma unroll
  for(int dy = -2; dy <= 2; dy++) {
    const int yy = y + dy;
    const int src = yy < 0 ? 0 : yy > 31 ? 31 : yy;
    const uint32_t rb = __shfl_sync(KGB_FULL, bd.b, src), rw = __shfl_sync(KGB_FULL, bd.w, src), ra = __shfl_sync(KGB_FULL, lib1, src);
#pragma unroll
    for(int dx = -2; dx <= 2; dx++) {
      const int xx = x + dx;
      unsigned long long code = 0;
      if(yy >= 0 && yy < Y && xx >= 0 && xx < X) {
        const uint32_t bit = 1u << xx;
        code = 8ull | ((rb & bit) ? 1ull : (rw & bit) ? 2ull : 0ull) | ((ra & bit) ? 4ull : 0ull);
      }
      const int cell = (dy + 2) * 5 + (dx + 2);
      if(cell < 16) lo |= code << (cell * 4); else hi |= code << ((cell - 16) * 4);
    }
  }
  hi |= (unsigned long long)(moverBlack ? 1 : 2) << 40;
  hi |= (unsigned long long)(unsigned)(prevMove + 2) << 42;      // -2 pass, else y*32+x (< 1024)
  hi |= (unsigned long long)(unsigned)p << 53;
  unsigned long long k = splitmix64(lo ^ splitmix64(hi ^ splitmix64((unsigned long long)(bd.ko + 1) * 0x9E3779B97F4A7C15ULL)));
  return k == 0 ? 1 : k;
}
__device__ int biasFindOrInsert(const SPDev& d, int g, unsigned long long key) {   // one lane
  const size_t tb = (size_t)g * d.biasTableSize;
  int slot = (int)(key & (unsigned long long)(d.biasTableSize - 1));
  while(true) {
    const unsigned long long k = d.biasKey[tb + slot];
    if(k == key) return slot;
    if(k == 0) { d.biasKey[tb + slot] = key; d.biasDeltaSum[tb + slot] = 0.0; d.biasWeightSum[tb + slot] = 0.0; return slot; }
    slot = (slot + 1) & (d.biasTableSize - 1);   // table is sized 2x the node pool: never full
  }
}
__device__ __forceinline__ void biasTableClear(const SPDev& d, int g, int lane) {
  const size_t tb = (size_t)g * d.biasTableSize;
  for(int i = lane; i < d.biasTableSize; i += 32) d.biasKey[tb + i] = 0;
}
// acc += v[0] + v[1] + ... + v[n-1] added one after the other in lane order (the order the reference adds its children in),
// for two quantities at once; every lane returns the same sums.  sh: 64 doubles of this warp's shared memory.
__device__ __forceinline__ void orderedAdd2(double a, double b, int n, double& accA, double& accB, double* sh, int lane) {
  sh[lane] = a; sh[32 + lane] = b;
  __syncwarp();
  for(int j = 0; j < n; j++) { accA += sh[j]; accB += sh[32 + j]; }
  __syncwarp();
}

// GraphHash::getStateHash (game/graphhash.cpp:4-24) for the rule subset: position, player to move, ko point, whether a pass
// ends the phase (passEnds: BoardHistory::passWouldEndPhase), game over, consecutive passes and the superko bans, which are part
// of the situation (boardhistory.cpp:1238-1244).  (Own mixing constants: only equality of hashes matters to the search.)
__device__ __forceinline__ void stateHashX(unsigned long long posH0, unsigned long long posH1, bool nextBlack, int ko, int passes, bool gameOver,
                                           bool passEnds, unsigned long long bannedHash, unsigned long long& s0, unsigned long long& s1) {
  s0 = posH0 ^ (nextBlack ? 0x8F1BBCDCA62C1D6BULL : 0x5A827999ED9EBA1FULL);
  s1 = posH1 ^ (nextBlack ? 0xC3A5C85C97CB3127ULL : 0xB492B66FBE98F273ULL);
  if(ko >= 0) { const unsigned long long k = splitmix64((unsigned long long)ko + 0x51ED27ULL); s0 ^= k; s1 ^= splitmix64(k); }
  // passEnds enters as two XORs, one on each side of the pass count: reordering them would change every key, and with the
  // keys which positions share an evaluation cache slot
  if(passes >= 1) { s0 ^= 0x9AE16A3B2F90404FULL; s1 ^= 0xCBF29CE484222325ULL; }
  if(gameOver) { s0 ^= 0x2545F4914F6CDD1DULL; s1 ^= 0x106689D45497FDB5ULL; }
  s0 += 2862933555777941757ULL * (unsigned long long)passes;
  s1 += 3202034522624059733ULL * (unsigned long long)passes;
  if(passEnds != (passes >= 1)) { s0 ^= 0x9AE16A3B2F90404FULL; s1 ^= 0xCBF29CE484222325ULL; }
  s0 ^= bannedHash; s1 ^= splitmix64(bannedHash + 0x1234567ULL) * (bannedHash != 0 ? 1ULL : 0ULL);
}
// ---- the lists of kgb_history.cuh for a game (appendable) and for a playout (game part read-only + path part)
__device__ __forceinline__ HistLists gameLists(const SPDev& d, int g) {
  HistLists L;
  L.gKo = nullptr; L.gKoLen = 0; L.gKoStart = 0; L.gPassB = nullptr; L.gPassBLen = 0; L.gPassW = nullptr; L.gPassWLen = 0;
  L.pKo = d.gKo + (size_t)g * d.histCap; L.pKoLen = d.gKoLen[g];
  L.pPassB = d.gPassB + (size_t)g * d.histCap; L.pPassBLen = d.gPassBLen[g];
  L.pPassW = d.gPassW + (size_t)g * d.histCap; L.pPassWLen = d.gPassWLen[g];
  return L;
}
__device__ __forceinline__ HistLists playoutLists(const SPDev& d, int g) {
  HistLists L;
  L.gKo = d.gKo + (size_t)g * d.histCap; L.gKoLen = d.gKoLen[g]; L.gKoStart = 0;
  L.gPassB = d.gPassB + (size_t)g * d.histCap; L.gPassBLen = d.gPassBLen[g];
  L.gPassW = d.gPassW + (size_t)g * d.histCap; L.gPassWLen = d.gPassWLen[g];
  L.pKo = d.pKo + (size_t)g * d.pathCap; L.pKoLen = 0;
  L.pPassB = d.pPassB + (size_t)g * d.pathCap; L.pPassBLen = 0;
  L.pPassW = d.pPassW + (size_t)g * d.pathCap; L.pPassWLen = 0;
  return L;
}
// A fresh game: the history starts with the initial situation (BoardHistory::clear).
__device__ __forceinline__ void gameHistReset(const SPDev& d, int g, int lane) {
  d.gEverOcc[g * 32 + lane] = 0; d.rootBanned[g * 32 + lane] = 0;
  if(lane == 0) { d.gKo[(size_t)g * d.histCap] = koHashOf(d.gKoRule[g], 0ULL, true); d.gKoLen[g] = 1; d.gPassBLen[g] = 0; d.gPassWLen[g] = 0; }
}
// One move of the GAME (root): board, Zobrist hash, pass count, the game's lists, bans and end flags.
__device__ void gameMakeMove(const SPDev& d, int g, WarpBoard& bd, int p, bool black, int lane, int& passes, bool& finished, bool& noResult) {
  if(lane == 0) d.passStreak[g * 2 + (black ? 0 : 1)] = p < 0 ? d.passStreak[g * 2 + (black ? 0 : 1)] + 1 : 0;
  HistLists L = gameLists(d, g);
  HistState st;
  st.passes = passes; st.finished = false; st.noResult = false; st.everOcc = d.gEverOcc[g * 32 + lane]; st.banned = 0;
  histMakeMove(bd, st, L, p, black, d.gKoRule[g], d.gMultiSuicide[g] != 0, d.zob, true);
  d.gEverOcc[g * 32 + lane] = st.everOcc; d.rootBanned[g * 32 + lane] = st.banned;
  __syncwarp();
  if(lane == 0) { d.gKoLen[g] = L.pKoLen; d.gPassBLen[g] = L.pPassBLen; d.gPassWLen[g] = L.pPassWLen; }
  __syncwarp();
  passes = st.passes; finished = st.finished; noResult = st.noResult;
}
// Board::simpleRepetitionBoundGt (board.cpp:2825-2888) on the board AFTER the move at p: stones of the chain at p plus all
// empty points of the regions its liberties belong to (or, if p is empty after a suicide, the empty region around p) > bound.
__device__ __forceinline__ bool simpleRepetitionBoundGt(const WarpBoard& bd, int p, int bound) {
  if(p < 0) return false;
  const uint32_t rm = bd.rowMask, pt = pointMask(p);
  const uint32_t empty = ~(bd.b | bd.w) & rm;
  const bool isB = __any_sync(KGB_FULL, (pt & bd.b) != 0), isW = __any_sync(KGB_FULL, (pt & bd.w) != 0);
  if(!isB && !isW) return warpCount(flood(pt, empty, rm)) > bound;
  const uint32_t chain = flood(pt, isB ? bd.b : bd.w, rm);
  const uint32_t region = flood(nbrs(chain, rm) & empty, empty, rm);
  return warpCount(chain) + warpCount(region) > bound;
}
// GraphHash::getGraphHash (game/graphhash.cpp:26-41): state hash alone when the last move cannot be part of a repetition,
// otherwise chained with the parent's graph hash (the node is then only shared by identical histories).
__device__ __forceinline__ void graphHashOfChild(unsigned long long pg0, unsigned long long pg1, unsigned long long s0, unsigned long long s1,
                                                 bool repetitionImpossible, unsigned long long& g0, unsigned long long& g1) {
  if(repetitionImpossible) { g0 = s0; g1 = s1; return; }
  g0 = splitmix64(pg0 ^ pg1);
  g1 = splitmix64(pg1 * 0x9FB21C651E98DF25ULL + 0x632BE59BD9B4E019ULL) + g0;
  g0 += s0; g1 += s1;
}
__device__ int nodeTableFind(const SPDev& d, int g, unsigned long long k0, unsigned long long k1, int& slotOut) {   // uniform
  const size_t tb = (size_t)g * d.nodeTableSize;
  int slot = (int)((k0 ^ (k1 >> 7)) & (unsigned long long)(d.nodeTableSize - 1));
  while(true) {
    const int n = d.nodeTableNode[tb + slot];
    if(n < 0) { slotOut = slot; return -1; }
    if(d.nodeTableKey0[tb + slot] == k0 && d.nodeTableKey1[tb + slot] == k1) { slotOut = slot; return n; }
    slot = (slot + 1) & (d.nodeTableSize - 1);
  }
}
__device__ __forceinline__ void nodeTableClear(const SPDev& d, int g, int lane) {
  const size_t tb = (size_t)g * d.nodeTableSize;
  for(int i = lane; i < d.nodeTableSize; i += 32) d.nodeTableNode[tb + i] = -1;
}
// The root node's hashes (after the root position changed): its position hash is tracked with the root board.
__device__ __forceinline__ void rootHashesInit(const SPDev& d, int g, int lane) {
  const size_t gb = (size_t)g * d.maxNodes;
  const unsigned long long h0 = d.rootPosH[g * 2], h1 = d.rootPosH[g * 2 + 1];
  WarpBoard bd;
  boardInit(bd, d.gX[g], d.gY[g]);
  bd.h0 = h0;
  HistLists L = playoutLists(d, g);
  HistState st;
  st.passes = d.consecPasses[g]; st.finished = false; st.noResult = false; st.everOcc = 0; st.banned = d.rootBanned[g * 32 + lane];
  const bool black = d.rootBlackToMove[g] != 0;
  unsigned long long s0, s1;
  stateHashX(h0, h1, black, d.rootKo[g], st.passes, false, histPassWouldEndPhase(bd, st, L, black, d.gKoRule[g]), pointSetHash(st.banned), s0, s1);
  if(lane == 0) { d.nodePosH0[gb] = h0; d.nodePosH1[gb] = h1; d.nodeGH0[gb] = s0; d.nodeGH1[gb] = s1; }
}
// The transposition table emptied and the root node's hashes set from the stored root position.
__device__ __forceinline__ void rootTableReset(const SPDev& d, int g, int lane) {
  nodeTableClear(d, g, lane);
  __syncwarp();
  rootHashesInit(d, g, lane);
  __syncwarp();
}
// After the root position changed: node 0 = the unevaluated root, every other node freed, every subtree value bias entry unused
// and dropped (search.cpp:860-861).
__device__ __forceinline__ void treeReset(const SPDev& d, int g, int lane) {
  const size_t gb = (size_t)g * d.maxNodes;
  if(lane == 0) { d.nodeCount[g] = 1; nodeStatsReset(d, gb, false); d.rootSymCount[g] = 0; }
  nodeInit(d, gb * d.policySize, lane);
  biasTableClear(d, g, lane);
  rootTableReset(d, g, lane);
}

__device__ __forceinline__ double rootChildUtilityWithBonus(const SPDev& d, int g, size_t gb, int c, int mv, double utilityAvg);
__device__ double scoreUtilityDiff(const SPDev& d, int g, double scoreMean, double scoreMeanSq, double delta, double center);
__device__ void computeRootExtras(const SPDev& d, int g, const WarpBoard& bd, bool rootBlack, bool haveOwnership, int numEvals, int lane);
// Search::getPlaySelectionValues for the root (searchresults.cpp:66-330; no human policy, no pass suppression, no ending
// bonus): values by child in creation order into psv[0..nc), their moves into moves[].  One thread.  Returns the child count.
__device__ int rootPlaySelectionValues(const SPDev& d, int g, double* psv, double* lcbBuf, double* radiusBuf) {
  const size_t gb = (size_t)g * d.maxNodes, nb = gb * d.policySize;
  const int nc = d.nodeNumChildren[gb];
  const bool rootWhite = d.rootBlackToMove[g] == 0;
  auto childWeightOf = [&](int k, int& mv, int& c, int& ev, int& cv) -> double {
    mv = (int)d.childOrder[nb + k]; c = d.childNode[nb + mv]; ev = d.childVisits[nb + mv]; cv = d.nodeVisits[gb + c];
    return d.nodeWeightSum[gb + c] * ((double)ev / (double)(cv > 1 ? cv : 1));
  };
  double totalChildWeight = 0.0;
  for(int k = 0; k < nc; k++) {
    int mv, c, ev, cv;
    const double w = childWeightOf(k, mv, c, ev, cv);
    totalChildWeight += w;
    psv[k] = d.policy[nb + mv] < 0 ? 0.0 : w;
  }
  // the most stably explored child: weight discounted by one visit, tiny prior term
  int nonLCBBestIdx = 0;
  double nonLCBBestChildWeight = -1e30, maxGoodness = -1e30;
  for(int k = 0; k < nc; k++) {
    const int mv = (int)d.childOrder[nb + k];
    const double edgeVisits = (double)d.childVisits[nb + mv];
    const double policyProb = d.policy[nb + mv];
    const double gdn = psv[k] * fmax(0.0, edgeVisits - 1.0) / fmax(1.0, edgeVisits) + 2.0 * policyProb;
    if(gdn > maxGoodness) { maxGoodness = gdn; nonLCBBestChildWeight = psv[k]; nonLCBBestIdx = k; }
  }
  if(nc > 0) {
    // children that got more visits than the final selection values justify are cut back to the weight PUCT would have wanted
    const int visits = d.nodeVisits[gb];
    const double weightSum = d.nodeWeightSum[gb], parentUtility = d.nodeUtilAvg[gb];
    double stdevFactor = 1.0;
    if(d.cpuctUtilityStdevScale != 0.0) {
      double utilitySqAvg = d.nodeUtilSqAvg[gb];
      const double variancePrior = d.cpuctUtilityStdevPrior * d.cpuctUtilityStdevPrior;
      double stdev;
      if(visits <= 0 || weightSum <= 1) stdev = d.cpuctUtilityStdevPrior;
      else {
        const double utilitySq = parentUtility * parentUtility;
        if(utilitySqAvg < utilitySq) utilitySqAvg = utilitySq;
        stdev = sqrt(fmax(0.0, ((utilitySq + variancePrior) * d.cpuctUtilityStdevPriorWeight + utilitySqAvg * weightSum) /
                                     (d.cpuctUtilityStdevPriorWeight + weightSum - 1.0) - utilitySq));
      }
      stdevFactor = 1.0 + d.cpuctUtilityStdevScale * (stdev / d.cpuctUtilityStdevPrior - 1.0);
    }
    const double cpuct = d.cpuctExploration + d.cpuctExplorationLog * log((totalChildWeight + d.cpuctExplorationBase) / d.cpuctExplorationBase);
    const double exploreScaling = cpuct * sqrt(totalChildWeight + 0.01) * stdevFactor;
    double bestValue;
    {
      int mv, c, ev, cv;
      const double w = childWeightOf(nonLCBBestIdx, mv, c, ev, cv);
      const float P = d.policy[nb + mv];
      // getExploreSelectionValueOfChild outside the search: a child without visits or weight would take the FPU value; the
      // most explored child always has both
      const double cu = rootChildUtilityWithBonus(d, g, gb, c, mv, d.nodeUtilAvg[gb + c]);
      bestValue = P < 0 ? -1e50 : exploreScaling * (double)P / (1.0 + w) + (rootWhite ? cu : -cu);
    }
    for(int k = 0; k < nc; k++) {
      if(k == nonLCBBestIdx) continue;
      int mv, c, ev, cv;
      const double w = childWeightOf(k, mv, c, ev, cv);
      double reduced = 0.0;
      if(!(cv <= 0 || w <= 0.0)) {
        const float P = d.policy[nb + mv];
        const double cu = rootChildUtilityWithBonus(d, g, gb, c, mv, d.nodeUtilAvg[gb + c]);
        double wanted = 0.0;                                               // getExploreSelectionValueInverse
        if(!(P < 0)) {
          const double valueComponent = rootWhite ? cu : -cu;
          const double exploreComponent = bestValue - valueComponent;
          if(exploreComponent <= 0) wanted = 1e100;
          else { wanted = exploreScaling * (double)P / exploreComponent - 1; if(wanted < 0) wanted = 0; }
        }
        reduced = w > wanted ? wanted : w;
      }
      psv[k] = ceil(reduced);
    }
  }
  if(d.useLcbForSelection && nc > 0) {
    // Search::getSelfUtilityLCBAndRadius (searchhelpers.cpp:555-604)
    const double utilityRangeRadius = d.winLossUtilityFactor + d.staticScoreUtilityFactor + d.dynamicScoreUtilityFactor;
    double bestLcb = -1e10; int bestLcbIndex = -1;
    for(int k = 0; k < nc; k++) {
      int mv, c, ev, cv;
      double weightSum = childWeightOf(k, mv, c, ev, cv);
      double weightSqSum = d.nodeWeightSqSum[gb + c] * ((double)ev / (double)(cv > 1 ? cv : 1));
      const double utilityAvg = d.nodeUtilAvg[gb + c];
      double utilitySqAvg = d.nodeUtilSqAvg[gb + c];
      radiusBuf[k] = 2.0 * utilityRangeRadius * d.lcbStdevs;
      lcbBuf[k] = -radiusBuf[k];
      if(!(cv <= 0 || weightSum <= 0.0 || weightSqSum <= 0.0)) {
        double ess = weightSum * weightSum / weightSqSum;
        const double priorWeight = weightSum / (ess * ess * ess);
        utilitySqAvg = fmax(utilitySqAvg, utilityAvg * utilityAvg + 1e-8);
        utilitySqAvg = (utilitySqAvg * weightSum + (utilitySqAvg + utilityRangeRadius * utilityRangeRadius) * priorWeight) / (weightSum + priorWeight);
        weightSum += priorWeight;
        weightSqSum += priorWeight * priorWeight;
        ess = weightSum * weightSum / weightSqSum;
        const double utilityWithBonus = rootChildUtilityWithBonus(d, g, gb, c, mv, utilityAvg);
        const double selfUtility = rootWhite ? utilityWithBonus : -utilityWithBonus;
        const double utilityVariance = utilitySqAvg - utilityAvg * utilityAvg;
        const double radius = sqrt(utilityVariance / ess) * d.lcbStdevs;
        lcbBuf[k] = selfUtility - radius;
        radiusBuf[k] = radius;
      }
      const double weight = psv[k];
      if(weight > 0 && weight >= d.minVisitPropForLCB * nonLCBBestChildWeight && lcbBuf[k] > bestLcb) { bestLcb = lcbBuf[k]; bestLcbIndex = k; }
    }
    if(d.useNonBuggyLcb ? (bestLcbIndex >= 0) : (bestLcbIndex > 0)) {
      double adjustedWeight = psv[bestLcbIndex];
      for(int k = 0; k < nc; k++) {
        if(k == bestLcbIndex) continue;
        const double excessValue = bestLcb - lcbBuf[k];
        if(excessValue < 0) continue;
        const double radius = radiusBuf[k];
        const double radiusFactor = (radius + excessValue) / (radius + 0.20 * excessValue);
        const double lbound = radiusFactor * radiusFactor * psv[k];
        if(lbound > adjustedWeight) adjustedWeight = lbound;
      }
      psv[bestLcbIndex] = adjustedWeight;
    }
  }
  if(nc == 0) return 0;
  double maxValue = 0.0;
  for(int k = 0; k < nc; k++) if(psv[k] > maxValue) maxValue = psv[k];
  if(maxValue <= 1e-50) {
    for(int k = 0; k < nc; k++) psv[k] = fmax(0.0, (double)d.policy[nb + (int)d.childOrder[nb + k]]);
    for(int k = 0; k < nc; k++) if(psv[k] > maxValue) maxValue = psv[k];
    if(maxValue <= 1e-50) return 0;
  }
  const double amountToSubtract = fmin(d.chosenMoveSubtract, maxValue / 64.0), amountToPrune = fmin(d.chosenMovePrune, maxValue / 64.0);
  for(int k = 0; k < nc; k++) {
    if(psv[k] < amountToPrune) psv[k] = 0.0;
    else { psv[k] -= amountToSubtract; if(psv[k] <= 0.0) psv[k] = 0.0; }
  }
  return nc;
}
// Search::chooseIndexWithTemperature (searchhelpers.cpp:12-76) with Rand::nextUInt(relProbs, n) (core/rand.h:222-243).  One thread.
__device__ int chooseIndexWithTemperature(DevRand& rand, const double* relativeProbs, int n, double temperature, double onlyBelowProb, double* processed) {
  double maxRelProb = 0.0, sumRelProb = 0.0;
  for(int i = 0; i < n; i++) { sumRelProb += fmax(0.0, relativeProbs[i]); if(relativeProbs[i] > maxRelProb) maxRelProb = relativeProbs[i]; }
  if(temperature <= 1.0e-4 && onlyBelowProb >= 1.0) {
    double bestProb = relativeProbs[0]; int bestIdx = 0;
    for(int i = 1; i < n; i++) if(relativeProbs[i] > bestProb) { bestProb = relativeProbs[i]; bestIdx = i; }
    return bestIdx;
  }
  const double logMaxRelProb = log(maxRelProb), logSumRelProb = log(sumRelProb), logOnlyBelowProb = log(fmax(1e-50, onlyBelowProb));
  double sum = 0.0;
  for(int i = 0; i < n; i++) {
    if(relativeProbs[i] <= 0.0) processed[i] = 0.0;
    else {
      const double logRelProb = log(relativeProbs[i]) - logMaxRelProb;
      const double logRelProbThreshold = fmin(0.0, logOnlyBelowProb + logSumRelProb - logMaxRelProb);
      const double newLogRelProb = logRelProb > logRelProbThreshold ? logRelProb : (logRelProb - logRelProbThreshold) / temperature + logRelProbThreshold;
      processed[i] = exp(newLogRelProb);
    }
    sum += processed[i];
  }
  double total = 0;
  for(int i = 0; i < n; i++) total += processed[i];
  const double dd = rand.nextDouble() * total;
  double run = 0.0;
  for(int i = 0; i < n; i++) { run += processed[i]; if(run > dd) return i; }
  return n - 1;
}
// Search::getChosenMoveLoc (searchresults.cpp:573-598): move position chosen for game g's root, or -1 if nothing can be chosen.
__device__ int rootChooseMove(const SPDev& d, int g) {
  double* psv = d.selScratch + (size_t)g * 3 * d.policySize;
  double* lcb = psv + d.policySize; double* radius = lcb + d.policySize;
  const int nc = rootPlaySelectionValues(d, g, psv, lcb, radius);
  if(nc <= 0) return -1;
  const double halflives = ((double)d.moveNum[g] / d.chosenMoveTemperatureHalflife) * 19.0 / sqrt((double)(d.gX[g] * d.gY[g]));
  const double temperature = d.chosenMoveTemperature + (d.chosenMoveTemperatureEarly - d.chosenMoveTemperature) * pow(0.5, halflives);
  DevRand rand;
  rand.s = d.nonSearchRand[g];
  const int k = chooseIndexWithTemperature(rand, psv, nc, temperature, d.chosenMoveTemperatureOnlyBelowProb, lcb /*reused as scratch*/);
  d.nonSearchRand[g] = rand.s;
  return (int)d.childOrder[(size_t)g * d.maxNodes * d.policySize + k];
}

// The game of slot g is over on board bd: score it (area scoring: komi - (black area - white area)), keep the final position and its
// area readable, count it, and start the slot's next game - empty board of the next game's size, its rules and komi (what the host
// handed over with kgb_selfplay_set_game_setup / set_komi), fresh history.  bd is the new game's empty board afterwards.
__device__ void gameOverStartNext(const SPDev& d, int g, WarpBoard& bd, bool noResult, int lane) {
  uint32_t areaB, areaW;
  boardCalculateArea(bd, true, true, true, d.gMultiSuicide[g] != 0, areaB, areaW);    // = the area boardAreaScoreBlackMinusWhite counts
  int diff = warpCount(areaB) - warpCount(areaW);
  float whiteScore = d.komiG[g] - (float)diff;
  uint32_t* fb = d.finalBoard + (size_t)g * 128;
  fb[lane] = bd.b; fb[32 + lane] = bd.w; fb[64 + lane] = areaB; fb[96 + lane] = areaW;
  if(lane == 0) d.lastScore[g] = whiteScore;
  if(lane == 0) {
    atomicAdd(d.gamesFinished, 1ULL);
    if(whiteScore < 0 && !noResult) atomicAdd(d.blackWins, 1ULL);
    d.gameCounter[g] += 1;
    d.lastKomi[g] = d.komiG[g];
    d.komiG[g] = d.nextKomi[g];          // the slot's next game (kgb_selfplay_set_komi)
    // ... and its board size and rules (kgb_selfplay_set_game_setup): what GameInitializer::createGame draws per game
    d.lastSetup[g * 4 + 0] = d.gX[g]; d.lastSetup[g * 4 + 1] = d.gY[g]; d.lastSetup[g * 4 + 2] = d.gKoRule[g]; d.lastSetup[g * 4 + 3] = d.gMultiSuicide[g];
    d.gX[g] = d.nextSetup[g * 4 + 0]; d.gY[g] = d.nextSetup[g * 4 + 1]; d.gKoRule[g] = d.nextSetup[g * 4 + 2]; d.gMultiSuicide[g] = d.nextSetup[g * 4 + 3];
    d.initMovesLeft[g] = d.nextInitMoves[g]; d.initMoveCount[g] = 0;       // the next game's policy-initialised opening
  }
  __syncwarp();
  boardInit(bd, d.gX[g], d.gY[g]);
  gameHistReset(d, g, lane);
  if(lane == 0) { d.passStreak[g * 2] = 0; d.passStreak[g * 2 + 1] = 0; }
}

// Game g's root board as stored; with withHash also its Zobrist hash (else 0, as boardInit leaves it).
__device__ __forceinline__ void rootBoardLoad(const SPDev& d, int g, int lane, WarpBoard& bd, bool withHash) {
  boardInit(bd, d.gX[g], d.gY[g]);
  bd.b = d.rootB[g * 32 + lane]; bd.w = d.rootW[g * 32 + lane];
  bd.ko = d.rootKo[g]; bd.capB = d.rootCapB[g]; bd.capW = d.rootCapW[g];
  if(withHash) { bd.h0 = d.rootPosH[g * 2]; bd.h1 = d.rootPosH[g * 2 + 1]; }
}
// A game's root position while one warp plays moves there: the board and the per-game scalars in registers.  The last five moves
// (hist) and the boards one and two moves ago (prevB/W/Ko, BoardHistory::getRecentBoard, for ladder planes 15/16) move along in
// memory, so that rootAdvance holds no more registers across gameMakeMove than the board before the move.
struct RootPos {
  WarpBoard bd;
  bool black;
  int moveNum, passes;
};
__device__ __forceinline__ void rootLoad(const SPDev& d, int g, int lane, RootPos& rp) {
  rootBoardLoad(d, g, lane, rp.bd, true);
  rp.black = d.rootBlackToMove[g] != 0;
  rp.moveNum = d.moveNum[g]; rp.passes = d.consecPasses[g];
}
__device__ __forceinline__ void rootStore(const SPDev& d, int g, int lane, const RootPos& rp) {
  d.rootB[g * 32 + lane] = rp.bd.b; d.rootW[g * 32 + lane] = rp.bd.w;
  if(lane == 0) {
    d.rootKo[g] = rp.bd.ko; d.rootCapB[g] = rp.bd.capB; d.rootCapW[g] = rp.bd.capW;
    d.rootPosH[g * 2] = rp.bd.h0; d.rootPosH[g * 2 + 1] = rp.bd.h1;
    d.rootBlackToMove[g] = rp.black ? 1 : 0; d.moveNum[g] = rp.moveNum; d.consecPasses[g] = rp.passes;
  }
}
// One move p (y*32+x, or -1 = pass) of the game at its root.
__device__ __forceinline__ void rootPlay(const SPDev& d, int g, int lane, RootPos& rp, int p, bool& finished, bool& noResult) {
  const uint32_t beforeB = rp.bd.b, beforeW = rp.bd.w; const int beforeKo = rp.bd.ko;
  gameMakeMove(d, g, rp.bd, p, rp.black, lane, rp.passes, finished, noResult);
  const int h = lane < 5 ? d.hist[g * 5 + lane] : -1;
  const int older = __shfl_up_sync(KGB_FULL, h, 1);
  if(lane < 5) d.hist[g * 5 + lane] = lane == 0 ? (p < 0 ? -2 : p) : older;
  const size_t G32 = (size_t)d.numGames * 32;
  d.prevB[G32 + g * 32 + lane] = d.prevB[g * 32 + lane]; d.prevW[G32 + g * 32 + lane] = d.prevW[g * 32 + lane];
  d.prevB[g * 32 + lane] = beforeB; d.prevW[g * 32 + lane] = beforeW;
  if(lane == 0) { d.prevKo[d.numGames + g] = d.prevKo[g]; d.prevKo[g] = beforeKo; }
  rp.black = !rp.black;
  rp.moveNum++;
}
// The root move record (lastMove): move position pos, end flags, the move's number, the game's index in its slot.
__device__ __forceinline__ void recordRootMove(const SPDev& d, int g, int lane, int pos, bool over, bool finished, bool noResult, int moveNum) {
  if(lane == 0) {
    d.lastMove[g * 4 + 0] = pos;
    d.lastMove[g * 4 + 1] = over ? (1 | (noResult ? 2 : 0) | (finished ? 0 : 4)) : 0;
    d.lastMove[g * 4 + 2] = moveNum;
    d.lastMove[g * 4 + 3] = (int)d.gameCounter[g];
  }
}
// The root move just played ended the game: the slot's next game starts from an empty root without history.
__device__ __forceinline__ void rootGameOver(const SPDev& d, int g, int lane, RootPos& rp, bool noResult) {
  gameOverStartNext(d, g, rp.bd, noResult, lane);
  rp.black = true; rp.moveNum = 0; rp.passes = 0;
  const size_t G32 = (size_t)d.numGames * 32;
  if(lane < 5) d.hist[g * 5 + lane] = -1;
  d.prevB[g * 32 + lane] = 0; d.prevW[g * 32 + lane] = 0; d.prevB[G32 + g * 32 + lane] = 0; d.prevW[G32 + g * 32 + lane] = 0;
  if(lane == 0) { d.prevKo[g] = -1; d.prevKo[d.numGames + g] = -1; }
}
// Laddered stones of the two previous boards (planes 15/16 at the root), searched again after moves the search did not make.
__device__ __forceinline__ void rootPrevLadders(const SPDev& d, int g, int lane) {
  if(!d.enableLadders) return;
  const size_t G32 = (size_t)d.numGames * 32;
  const LadderScratch sc = ladderScratchAt(d.ladderScratch + (size_t)g * SP_LADDER_WARPS * ladderScratchWordsPerWarp());
  __syncwarp();   // prevKo was written by lane 0
  WarpBoard pb;
  boardInit(pb, d.gX[g], d.gY[g]);
  uint32_t l1, l2, wB, wW;
  pb.b = d.prevB[g * 32 + lane]; pb.w = d.prevW[g * 32 + lane]; pb.ko = d.prevKo[g];
  boardLadders(pb, sc, d.gX[g], d.gY[g], l1, wB, wW);
  pb.b = d.prevB[G32 + g * 32 + lane]; pb.w = d.prevW[G32 + g * 32 + lane]; pb.ko = d.prevKo[d.numGames + g];
  boardLadders(pb, sc, d.gX[g], d.gY[g], l2, wB, wW);
  d.prevLad[g * 32 + lane] = l1; d.prevLad[G32 + g * 32 + lane] = l2;
}

// Choose and play the root move once the visit budget is spent; restart the game when it is over.
__device__ void rootAdvance(const SPDev& d, int g, int lane) {
  const size_t gb = (size_t)g * d.maxNodes;
  const size_t rootBase = gb * d.policySize;
  // visit counts of the root's children
  int best = -1, bestV = -1;
  long long total = 0;
  const bool early = d.moveNum[g] < d.earlyMoves;
  uint64_t r = splitmix64(d.seed ^ splitmix64(((uint64_t)g << 32) ^ (d.gameCounter[g] * 1315423911ULL) ^ (uint64_t)d.moveNum[g]));
  // pass 1: totals / argmax
  int myBest = -1, myBestV = -1;
  long long mySum = 0;
  for(int i = lane; i < d.policySize; i += 32) {
    int v = d.childVisits[rootBase + i];
    mySum += v;
    if(v > myBestV) { myBestV = v; myBest = i; }
  }
  for(int o = 16; o > 0; o >>= 1) {
    int ov = __shfl_xor_sync(KGB_FULL, myBestV, o), oi = __shfl_xor_sync(KGB_FULL, myBest, o);
    if(ov > myBestV || (ov == myBestV && oi < myBest)) { myBestV = ov; myBest = oi; }
    mySum += __shfl_xor_sync(KGB_FULL, mySum, o);
  }
  best = myBest; bestV = myBestV; total = mySum;
  if(early && total > 0) {
    // sample proportionally to visits (temperature 1): walk the cumulative distribution in position order
    long long target = (long long)(r % (uint64_t)total);
    long long run = 0;
    int chosen = best;
    bool found = false;
    for(int base = 0; base < d.policySize && !found; base += 32) {
      int i = base + lane;
      long long v = i < d.policySize ? d.childVisits[rootBase + i] : 0;
      long long incl = v;
      for(int o = 1; o < 32; o <<= 1) {
        long long t = __shfl_up_sync(KGB_FULL, incl, o);
        if(lane >= o) incl += t;
      }
      unsigned hit = __ballot_sync(KGB_FULL, v > 0 && run + incl > target);
      if(hit) { chosen = base + __ffs(hit) - 1; found = true; }
      run += __shfl_sync(KGB_FULL, incl, 31);
    }
    best = chosen;
  }
  if(d.usePlaySelection && d.initMovesLeft[g] <= 0) {
    int chosen = -1;
    if(lane == 0) chosen = rootChooseMove(d, g);
    chosen = __shfl_sync(KGB_FULL, chosen, 0);
    if(chosen >= 0) { best = chosen; bestV = 1; }
  }
  const bool initMove = d.initMovesLeft[g] > 0;
  if(initMove) {
    // PlayUtils::getGameInitializationMove (playutils.cpp:177-226): a legal move drawn in proportion to policy ^ (1 / temperature) of the
    // root's own evaluation (with probability 0.0002 uniformly), from the game's non-search generator
    int chosen = d.policySize - 1;
    if(lane == 0) {
      const float* pol = d.policy + rootBase;
      DevRand rand;
      rand.s = d.nonSearchRand[g];
      const double invT = 1.0 / d.policyInitTemperature[0];
      double sum = 0.0; int cnt = 0;
      for(int i = 0; i < d.policySize; i++) if(pol[i] > 0.0f) { sum += invT == 1.0 ? (double)pol[i] : pow((double)pol[i], invT); cnt++; }
      if(cnt > 0) {
        const bool uniform = rand.nextDouble() < 0.0002;
        double r = rand.nextDouble() * (uniform ? (double)cnt : sum), run = 0.0;
        for(int i = 0; i < d.policySize; i++) {
          if(!(pol[i] > 0.0f)) continue;
          run += uniform ? 1.0 : (invT == 1.0 ? (double)pol[i] : pow((double)pol[i], invT));
          chosen = i;
          if(run > r) break;
        }
      }
      d.nonSearchRand[g] = rand.s;
    }
    best = __shfl_sync(KGB_FULL, chosen, 0); bestV = 1;
  }
  if(bestV <= 0) best = d.policySize - 1;  // nothing searched (cannot happen with maxVisits >= 2): pass
  // play it on the root board
  RootPos rp;
  rootLoad(d, g, lane, rp);
  bool finished = false, noResult = false;
  rootPlay(d, g, lane, rp, best == d.policySize - 1 ? -1 : pointOfPos(best, d.X), finished, noResult);
  const bool over = finished || rp.moveNum >= d.maxMoves;
  recordRootMove(d, g, lane, best, over, finished, noResult, rp.moveNum - 1);
  if(over) rootGameOver(d, g, lane, rp, noResult);
  else {
    const size_t G32 = (size_t)d.numGames * 32;
    d.prevLad[G32 + g * 32 + lane] = d.prevLad[g * 32 + lane];
    d.prevLad[g * 32 + lane] = d.nodeLad[gb * 32 + lane];   // the old root was evaluated, so its ladders are known
  }
  rootStore(d, g, lane, rp);
  if(lane == 0) {
    atomicAdd(d.totalMoves, 1ULL);
    // the new root's search limits (kgb_selfplay_set_next_search_limits)
    d.visitBudget[g] = d.nextBudget[g * 2 + (over ? 1 : 0)];
    d.plainRoot[g] = d.nextPlain[g * 2 + (over ? 1 : 0)];
    if(initMove && !over) {
      const int k = d.initMoveCount[g];
      if(k < SP_MAX_INIT_MOVES) d.initMoves[(size_t)g * SP_MAX_INIT_MOVES + k] = (int16_t)best;
      d.initMoveCount[g] = k + 1;
      d.initMovesLeft[g] -= 1;
    }
    if(d.initMovesLeft[g] > 0) { d.visitBudget[g] = 1; d.plainRoot[g] = 1; }   // an opening root: one plain evaluation, then the policy draw
  }
  treeReset(d, g, lane);
}

__device__ void recomputeNodeStats(const SPDev& d, int g, int node, bool nodePlaWhite, double* sh, int lane);
__device__ void finishPlayout(const SPDev& d, int g, int node, double u, double w, bool terminal, bool leafBlack, int len, double* shSum, int lane);
__device__ __forceinline__ double evalWeight(const SPDev& d, int g, const float vals[8]);
__device__ double utilityFromEval(const SPDev& d, int g, int node, float whiteWin, float whiteLoss, float noResult, float whiteScoreMeanF,
                                  float whiteScoreMeanSqF, float whiteLeadF, int lane);
__device__ void maybeRootNoise(const SPDev& d, int g, int node, int lane);
__device__ bool cacheLookup(const SPDev& d, int g, int node, unsigned long long k0, unsigned long long k1, float vals[8], int lane);

// Warp 0 of a game's block: PUCT descent, leaf board, legality and every feature except the leaf's own ladder searches.
__device__ void spSelectWarp0(const SPDev& d, int g, int lane, uint32_t* shB, uint32_t* shW, uint32_t* shCand, int& shKo, int& shDoLadders,
                              double* shSum) {
  const size_t gb = (size_t)g * d.maxNodes;
  const size_t G32 = (size_t)d.numGames * 32;
  WarpBoard bd;
  bool black = true, terminal = false, gotLeaf = false;
  int h0 = -1, h1 = -1, h2 = -1, h3 = -1, h4 = -1, node = 0, depth = 0;
  uint32_t lad1 = 0, lad2 = 0;
  HistLists HL;                 // BoardHistory along the playout (kgb_history.cuh): the game's lists + the path part, and the
  HistState hst;                // pass count, end flags and bans of the current position
  bool bannedValid;             // hst.banned belongs to the current position
  const long long tW0 = clock64();
#ifdef KGB_PROFILE_DESCENT
  long long pfGather = 0, pfSelect = 0, pfMove = 0, pfEdge = 0, pfSteps = 0, pfT = clock64(), pfBackup = 0, pfAttempts = 0, pfAdvance = 0;
#endif
  // Under graph search a playout can end without reaching a new leaf (edge catch-up, cycle): it is backed up at once and the
  // next playout starts, so that the wave still delivers a leaf for the evaluator.
  for(int attempt = 0; attempt < d.maxPlayoutsPerWave && !gotLeaf; attempt++) {
  if(d.nodeVisits[gb] >= d.visitBudget[g]) {
    // hold mode (tests, game recording): keep the finished tree until the host has read it and released the game
    const bool released = d.releaseFlag[g] != 0;
    __syncwarp();
    if(d.holdAtMaxVisits && !released && d.initMovesLeft[g] <= 0) break;      // opening moves drawn from the policy are not recorded turns
    const long long tRA = clock64();
    rootAdvance(d, g, lane);
    if(lane == 0) { d.releaseFlag[g] = 0; d.dbgCycles[g * 8 + 1] = clock64() - tRA; }
#ifdef KGB_PROFILE_DESCENT
    { const long long t_ = clock64(); pfAdvance += t_ - pfT; pfT = t_; }
#endif
  }
  rootBoardLoad(d, g, lane, bd, true);   // the hash follows the whole path: ko hashes are taken from it
  const bool rootBlack = d.rootBlackToMove[g] != 0;
  black = rootBlack;
  h0 = d.hist[g * 5 + 0]; h1 = d.hist[g * 5 + 1]; h2 = d.hist[g * 5 + 2]; h3 = d.hist[g * 5 + 3]; h4 = d.hist[g * 5 + 4];
  // boards one and two moves ago (ladder planes 15/16): the root's recent boards, shifted as the descent plays moves.
  // Their laddered stones were computed when those positions were leaves themselves (a node's board is its child's
  // previous board), so only the leaf's own board ever needs a ladder search.
  lad1 = d.prevLad[g * 32 + lane]; lad2 = d.prevLad[G32 + g * 32 + lane];
  node = 0; depth = 0;
  terminal = false;
  HL = playoutLists(d, g);
  hst.passes = d.consecPasses[g]; hst.finished = false; hst.noResult = false;
  hst.everOcc = d.gEverOcc[g * 32 + lane]; hst.banned = d.rootBanned[g * 32 + lane];
  bannedValid = true;
  bool instant = false;   // this playout ended on an existing edge: back it up here, no leaf
#ifdef KGB_PROFILE_DESCENT   // build variant for tests/gpu_checks/descent_profile.py: where a descent step spends its cycles
  pfAttempts++;
#define PF(acc) do { const long long t_ = clock64(); acc += t_ - pfT; pfT = t_; } while(0)
#else
#define PF(acc) do {} while(0)
#endif
  while(true) {
    PF(pfEdge);
    const int visits = d.nodeVisits[gb + node];
    terminal = d.nodeTerminal[gb + node] != 0;
    if(visits == 0 || terminal || depth >= d.maxDepth - 1) break;
    const size_t nb = (gb + node) * d.policySize;
    const int nc = d.nodeNumChildren[gb + node];
    // ---- pass 1 over the children in creation order (searchexplorehelpers.cpp:338-364): visited policy mass, total child weight
    float P[12]; double CW[12], CU[12]; int CVis[12]; int MV[12];
    double massVisited = 0.0, totalW = 0.0;
#pragma unroll
    for(int ch = 0; ch < 12; ch++) {
      P[ch] = -1.0f; CW[ch] = 0.0; CU[ch] = 0.0; CVis[ch] = 0; MV[ch] = 0;
      if(ch * 32 < nc) {
        const int k = ch * 32 + lane;
        const bool in = k < nc;
        const int mv = in ? (int)d.childOrder[nb + k] : 0;
        MV[ch] = mv;
        const int c = in ? d.childNode[nb + mv] : 0;
        const int ev = in ? d.childVisits[nb + mv] : 0;
        const int cv = in ? d.nodeVisits[gb + c] : 0;
        const double cw = in ? d.nodeWeightSum[gb + c] : 0.0;
        const float p = in ? d.policy[nb + mv] : -1.0f;
        const double w = cw * ((double)ev / (double)(cv > 1 ? cv : 1));     // NodeStats::childWeight (searchnode.h:64-66)
        P[ch] = p; CW[ch] = w; CU[ch] = in ? d.nodeUtilAvg[gb + c] : 0.0; CVis[ch] = cv;
      }
    }
    // the gathers above carry no barrier, so the dependent loads (childOrder -> childNode -> child statistics) of all chunks are in
    // flight together; the ordered sums follow in the reference's order
#pragma unroll
    for(int ch = 0; ch < 12; ch++) {
      if(ch * 32 < nc) {
        const bool counts = ch * 32 + lane < nc && P[ch] >= 0.0f;
        const int n = nc - ch * 32 < 32 ? nc - ch * 32 : 32;
        orderedAdd2(counts ? (double)P[ch] : 0.0, counts ? CW[ch] : 0.0, n, massVisited, totalW, shSum, lane);
      }
    }
    PF(pfGather);
    // ---- FPU and exploration scaling (searchexplorehelpers.cpp:22-29, 265-321)
    const double parentUtility = d.nodeUtilAvg[gb + node];
    const bool isRoot = node == 0;
    double stdevFactor = 1.0;
    if(d.cpuctUtilityStdevScale != 0.0) {
      const double weightSum = d.nodeWeightSum[gb + node];
      double utilitySqAvg = d.nodeUtilSqAvg[gb + node];
      const double variancePrior = d.cpuctUtilityStdevPrior * d.cpuctUtilityStdevPrior;
      double stdev;
      if(visits <= 0 || weightSum <= 1) stdev = d.cpuctUtilityStdevPrior;
      else {
        const double utilitySq = parentUtility * parentUtility;
        if(utilitySqAvg < utilitySq) utilitySqAvg = utilitySq;
        stdev = sqrt(fmax(0.0, ((utilitySq + variancePrior) * d.cpuctUtilityStdevPriorWeight + utilitySqAvg * weightSum) /
                                     (d.cpuctUtilityStdevPriorWeight + weightSum - 1.0) - utilitySq));
      }
      stdevFactor = 1.0 + d.cpuctUtilityStdevScale * (stdev / d.cpuctUtilityStdevPrior - 1.0);
    }
    double parentUtilityForFPU = parentUtility;
    if(d.fpuParentWeightByVisitedPolicy) {
      const double pw = d.fpuParentWeightByVisitedPolicyPow;
      const double raised = pw == 1.0 ? massVisited : pw == 2.0 ? massVisited * massVisited : pow(massVisited, pw);
      const double avgWeight = fmin(1.0, raised);
      parentUtilityForFPU = avgWeight * parentUtility + (1.0 - avgWeight) * d.nodeNNUtil[gb + node];
    }
    else if(d.fpuParentWeight > 0.0) parentUtilityForFPU = d.fpuParentWeight * d.nodeNNUtil[gb + node] + (1.0 - d.fpuParentWeight) * parentUtility;
    double fpuValue;
    {
      const bool rootParams = isRoot && !d.plainRoot[g];      // a "plain" root searches like any other node (runBotWithLimits removeRootNoise)
      const double reduction = (rootParams ? d.rootFpuReductionMax : d.fpuReductionMax) * sqrt(massVisited);
      const double lossProp = rootParams ? d.rootFpuLossProp : d.fpuLossProp;
      const double utilityRadius = d.winLossUtilityFactor + d.staticScoreUtilityFactor + d.dynamicScoreUtilityFactor;
      fpuValue = black ? parentUtilityForFPU + reduction : parentUtilityForFPU - reduction;   // utilities are white's
      const double lossValue = black ? utilityRadius : -utilityRadius;
      fpuValue = fpuValue + (lossValue - fpuValue) * lossProp;
    }
    const double cpuct = d.cpuctExploration + d.cpuctExplorationLog * log((totalW + d.cpuctExplorationBase) / d.cpuctExplorationBase);
    const double exploreScaling = cpuct * sqrt(totalW + 0.01) * stdevFactor;
    // ---- pass 2: best existing child (first in creation order among equals, :452-486) ...
    double bestVal = -1e50; int bestK = -1;
#pragma unroll
    for(int ch = 0; ch < 12; ch++) {
      const int k = ch * 32 + lane;
      if(k >= nc) continue;
      double val = -1e50;                                           // POLICY_ILLEGAL_SELECTION_VALUE
      if(P[ch] >= 0.0f) {
        double cu = (CVis[ch] <= 0 || CW[ch] <= 0.0) ? fpuValue : CU[ch];
        if(isRoot && d.rootEndingBonusPoints != 0.0 && !(CVis[ch] <= 0 || CW[ch] <= 0.0)) {
          // rootChildUtilityWithBonus with the move kept from the gather: the bonus table (one line per game) is read directly, the
          // child's score moments only for the few moves that carry a bonus
          const double bonus = d.rootEndBonus[(size_t)g * d.policySize + MV[ch]];
          if(bonus != 0.0) {
            const double* cm = d.nodeMoments + (gb + d.childNode[nb + MV[ch]]) * 5;
            cu = cu + scoreUtilityDiff(d, g, cm[2], cm[3], bonus, d.recentScoreCenter[g]);
          }
        }
        val = exploreScaling * (double)P[ch] / (1.0 + CW[ch]) + (black ? -cu : cu);
        if(isRoot && !d.plainRoot[g] && d.rootDesiredPerChildVisitsCoeff > 0.0 && P[ch] > 0.0f &&
           CW[ch] < sqrt((double)P[ch] * totalW * d.rootDesiredPerChildVisitsCoeff)) val = 1e20;
      }
      if(val > bestVal) { bestVal = val; bestK = k; }
    }
#pragma unroll
    for(int o = 16; o > 0; o >>= 1) {
      double ov = __shfl_xor_sync(KGB_FULL, bestVal, o); int ok = __shfl_xor_sync(KGB_FULL, bestK, o);
      if(ok >= 0 && (bestK < 0 || ov > bestVal || (ov == bestVal && ok < bestK))) { bestVal = ov; bestK = ok; }
    }
    // ... and the unexpanded move with the largest prior (first in position order among equals, :548-590)
    float bestNewP = -1.0f; int bestNewIdx = -1;
    {
      // all loads first (two coalesced arrays, no branch between them), then the comparisons
      float PP[12]; int CN[12];
#pragma unroll
      for(int ch = 0; ch < 12; ch++) {
        const int i = ch * 32 + lane;
        const bool in = i < d.policySize;
        PP[ch] = in ? d.policy[nb + i] : -1.0f;
        CN[ch] = in ? d.childNode[nb + i] : 0;
      }
      if(isRoot && d.rootPruneUselessMoves) {     // Search::isAllowedRootMove: this lane's row of the allowed points, handed round by shuffle
        const uint32_t allowedMine = d.rootAllowed[g * 32 + lane];
#pragma unroll
        for(int ch = 0; ch < 12; ch++) {
          const int i = ch * 32 + lane;
          const int ic = i < d.XY ? i : 0;
          const uint32_t rowBits = __shfl_sync(KGB_FULL, allowedMine, ic / d.X);
          if(i < d.XY && !((rowBits >> (ic % d.X)) & 1u)) PP[ch] = -1.0f;
        }
      }
#pragma unroll
      for(int ch = 0; ch < 12; ch++) {
        const int i = ch * 32 + lane;
        if(PP[ch] >= 0.0f && CN[ch] < 0 && PP[ch] > bestNewP) { bestNewP = PP[ch]; bestNewIdx = i; }
      }
    }
#pragma unroll
    for(int o = 16; o > 0; o >>= 1) {
      float op = __shfl_xor_sync(KGB_FULL, bestNewP, o); int on = __shfl_xor_sync(KGB_FULL, bestNewIdx, o);
      if(on >= 0 && (bestNewIdx < 0 || op > bestNewP || (op == bestNewP && on < bestNewIdx))) { bestNewP = op; bestNewIdx = on; }
    }
    int move = bestK >= 0 ? (int)d.childOrder[nb + bestK] : -1;
    if(bestNewIdx >= 0) {
      const double newVal = exploreScaling * (double)bestNewP / (1.0 + 0.0) + (black ? -fpuValue : fpuValue);
      if(bestK < 0 || newVal > bestVal) move = bestNewIdx;
    }
    if(move < 0) break;  // no legal move at all (cannot happen: pass is always legal)
    PF(pfSelect);
#ifdef KGB_PROFILE_DESCENT
    pfSteps++;
#endif
    if(lane == 0) { d.pathNode[(size_t)g * d.maxDepth + depth] = node; d.pathMove[(size_t)g * d.maxDepth + depth] = move; }
    __syncwarp();
    // ---- graph search: an edge with fewer visits than its (shared) child catches up without descending (search.cpp:1468-1504)
    if(d.useGraphSearch && d.childNode[nb + move] >= 0 && d.childVisits[nb + move] < d.nodeVisits[gb + d.childNode[nb + move]]) { instant = true; break; }
    // ---- descend
    const bool isPass = move == d.policySize - 1;
    const int p = isPass ? -1 : pointOfPos(move, d.X);
    lad2 = lad1; lad1 = d.nodeLad[(gb + node) * 32 + lane];
    // a new child gets its subtree-value-bias entry from the position before the move (search.cpp:913-922): needs a previous
    // move in the history and a non-pass move
    unsigned long long biasKeyNew = 0;
    if(d.subtreeValueBiasFactor != 0.0 && d.childNode[nb + move] < 0 && !isPass && h0 != -1) biasKeyNew = biasEntryKey(bd, d.gX[g], d.gY[g], black, h0, p);
    int child = d.childNode[nb + move];
    const bool newEdge = child < 0;
    // BoardHistory::makeBoardMoveAssumeLegal along the path: pass situations, ko-hash history, game end by repetition rules
    histMakeMove(bd, hst, HL, p, black, d.gKoRule[g], d.gMultiSuicide[g] != 0, d.zob, false);
    bannedValid = false;
    if(newEdge && d.gKoRule[g] != KGB_KO_SIMPLE) {
      hst.banned = histSuperKoBanned(bd, HL, hst.everOcc, !black, d.gKoRule[g], d.gMultiSuicide[g] != 0, d.zob);
      bannedValid = true;
    }
    h4 = h3; h3 = h2; h2 = h1; h1 = h0; h0 = isPass ? -2 : p;
    black = !black;
    PF(pfMove);
    if(newEdge) {
      // Search::allocateOrFindNode (search.cpp:875-936): under graph search the child may already exist (transposition)
      unsigned long long cg0 = 0, cg1 = 0;
      int tableSlot = -1, found = -1;
      if(d.useGraphSearch) {
        unsigned long long s0, s1;
        stateHashX(bd.h0, bd.h1, black, bd.ko, hst.passes, hst.finished, histPassWouldEndPhase(bd, hst, HL, black, d.gKoRule[g]),
                   d.gKoRule[g] != KGB_KO_SIMPLE ? pointSetHash(hst.banned) : 0ULL, s0, s1);
        graphHashOfChild(d.nodeGH0[gb + node], d.nodeGH1[gb + node], s0, s1, simpleRepetitionBoundGt(bd, p, d.graphSearchRepBound), cg0, cg1);
        found = nodeTableFind(d, g, cg0, cg1, tableSlot);
      }
      if(found >= 0) child = found;
      else {
        child = d.nodeCount[g];
        if(child >= d.maxNodes) break;  // pool exhausted (sized maxVisits+2: cannot happen)
      }
      __syncwarp();
      if(lane == 0) {
        d.childNode[nb + move] = child;
        d.childOrder[nb + nc] = (uint16_t)move;
        d.nodeNumChildren[gb + node] = nc + 1;
        if(found < 0) {
          d.nodeCount[g] = child + 1;
          nodeStatsReset(d, gb + child, hst.finished);
          if(hst.noResult) d.nodeTerminal[gb + child] = 2;
          if(biasKeyNew != 0) d.nodeBiasEntry[gb + child] = biasFindOrInsert(d, g, biasKeyNew);
          d.nodePosH0[gb + child] = bd.h0; d.nodePosH1[gb + child] = bd.h1;
          if(d.useGraphSearch) {
            const size_t ts = (size_t)g * d.nodeTableSize + tableSlot;
            d.nodeTableKey0[ts] = cg0; d.nodeTableKey1[ts] = cg1; d.nodeTableNode[ts] = child;
            d.nodeGH0[gb + child] = cg0; d.nodeGH1[gb + child] = cg1;
          }
          atomicAdd(d.nodesAllocated, 1ULL);
        }
      }
      if(found < 0) nodeInit(d, (gb + child) * d.policySize, lane);
      __syncwarp();
      // a new edge onto an existing node starts with 0 visits against the node's n: it catches up right away instead of
      // descending (search.cpp:1382-1389, the same maybeCatchUpEdgeVisits as for existing edges)
      if(found >= 0 && d.nodeVisits[gb + found] > 0) { instant = true; break; }
    }
    depth++;
    if(d.useGraphSearch) {
      // a child that is already on this playout's path closes a cycle: count the edge and stop (search.cpp:1425-1443)
      bool onPath = false;
      for(int k = lane; k < depth; k += 32) onPath |= d.pathNode[(size_t)g * d.maxDepth + k] == child;
      if(__any_sync(KGB_FULL, onPath)) { depth--; instant = true; break; }
    }
    node = child;
  }
  if(instant) {
    // edge visit + updateStatsAfterPlayout for the node where the playout stopped and for every ancestor
    for(int k = depth; k >= 0; k--) {
      const int pn = d.pathNode[(size_t)g * d.maxDepth + k], mv = d.pathMove[(size_t)g * d.maxDepth + k];
      if(lane == 0) d.childVisits[(gb + pn) * d.policySize + mv] += 1;
      __syncwarp();
      const bool pnBlack = (k & 1) ? !rootBlack : rootBlack;
      recomputeNodeStats(d, g, pn, !pnBlack, shSum, lane);
      __syncwarp();
    }
    if(lane == 0) { atomicAdd(d.totalVisits, 1ULL); atomicAdd(d.instantPlayouts, 1ULL); }
    PF(pfBackup);
    continue;
  }
  if(d.cacheSize > 0 && d.nodeTerminal[gb + node] == 0 && d.nodeVisits[gb + node] == 0 && !(node == 0 && rootSyms(d, g) > 1)) {
    // NNEvaluator::evaluate's cache lookup (nneval.cpp:861-905): the key is the situation, not the history behind it
    unsigned long long k0, k1;
    stateHashX(d.nodePosH0[gb + node], d.nodePosH1[gb + node], black, bd.ko, hst.passes >= 1 ? 1 : 0, false, histPassWouldEndPhase(bd, hst, HL, black, d.gKoRule[g]),
               (d.gKoRule[g] != KGB_KO_SIMPLE && bannedValid) ? pointSetHash(hst.banned) : 0ULL, k0, k1);
    {
      // NNInputs::getHash (nninputs.cpp:869-943) = situation + rules + the mover's komi (boardhistory.cpp:1268-1274) + evaluation
      // options.  Komi varies from game to game inside one loop, so it is part of the key; scoring / tax rules, policy optimism and
      // playoutDoublingAdvantage are the same for every game of a loop (and the table belongs to the loop).
      const long long kd = (long long)((black ? -d.komiG[g] : d.komiG[g]) * 256.0f);
      // board size and the ko / suicide rules can differ from game to game too (kgb_selfplay_set_game_setup): the reference's hash starts
      // from a board hash that contains the size (Board::ZOBRIST_SIZE_X/Y_HASH) and mixes in Rules (ZOBRIST_KO_RULE_HASH, MULTI_STONE_SUICIDE_HASH)
      const unsigned long long setupBits = (unsigned long long)d.gX[g] | ((unsigned long long)d.gY[g] << 8) | ((unsigned long long)d.gKoRule[g] << 16) |
                                           ((unsigned long long)(d.gMultiSuicide[g] != 0) << 24);
      const unsigned long long kh = splitmix64((unsigned long long)kd + 0x6B6F6D69ULL) ^ splitmix64(setupBits * 0x9E3779B97F4A7C15ULL + 0x73657475ULL);
      k0 ^= kh; k1 ^= splitmix64(kh);
    }
    if(lane == 0) { d.leafKey[g * 2] = k0; d.leafKey[g * 2 + 1] = k1; }
    float vals[8];
    // a plain root (cheap search) is evaluated by the net even when the cache knows it: its input row is kept for the recorder; the key is
    // still set, so that the backup stores the fresh evaluation under it
    if(!(node == 0 && d.plainRoot[g]) && cacheLookup(d, g, node, k0, k1, vals, lane)) {
      if(node == 0 && (d.rootEndingBonusPoints != 0.0 || d.rootPruneUselessMoves))
        computeRootExtras(d, g, bd, black, false, 1, lane);     // a root served by the cache has no ownership map: allowed moves only
      maybeRootNoise(d, g, node, lane);
      const double u = utilityFromEval(d, g, node, vals[0], vals[1], vals[2], vals[3], vals[4], vals[5], lane);
      finishPlayout(d, g, node, u, evalWeight(d, g, vals), false, black, depth, shSum, lane);
      if(lane == 0) atomicAdd(d.cacheHits, 1ULL);
      PF(pfBackup);
      continue;
    }
  }
  PF(pfEdge);
  gotLeaf = true;
  }   // attempts
  if(!gotLeaf) {   // every playout of this wave ended on an existing edge: nothing for the evaluator
    if(lane == 0) { shDoLadders = 0; d.leafValid[g] = 0; atomicAdd(d.stalledWaves, 1ULL); }
    return;
  }
  terminal = d.nodeTerminal[gb + node] != 0;
  const long long tLeaf = clock64();

  // ---- leaf: liberties, legality, features
  uint32_t lib1, lib2, lib3;
  boardLibertyClasses(bd, lib1, lib2, lib3);
  uint32_t superKo = 0;
  if(d.gKoRule[g] != KGB_KO_SIMPLE) {
    if(!bannedValid) { hst.banned = histSuperKoBanned(bd, HL, hst.everOcc, black, d.gKoRule[g], d.gMultiSuicide[g] != 0, d.zob); bannedValid = true; }
    superKo = hst.banned;
  }
  const uint32_t legal = boardLegalMask(bd, black, d.gMultiSuicide[g] != 0, lib1) & ~superKo;    // BoardHistory::isLegal
  d.leafLegal[g * 32 + lane] = legal;
  if(lane == 0) {
    d.pathLen[g] = depth; d.leafNode[g] = node; d.leafTerminal[g] = (int)d.nodeTerminal[gb + node]; d.leafBlackToMove[g] = black ? 1 : 0;
    atomicAdd(d.sumDepth, (unsigned long long)depth);
  }
  if(terminal) {
    int diff = boardAreaScoreBlackMinusWhite(bd, d.gMultiSuicide[g] != 0);
    float whiteScore = d.komiG[g] - (float)diff;
    if(lane == 0) d.leafTerminalScore[g] = whiteScore;
  }
  const long long tLegal = clock64();
  // NN input row (NHWC [pos][22]) - zero fill, then the ones
  float* row = d.nnSpatial + (size_t)g * d.XY * 22;
  for(int i = lane; i < d.XY * 22; i += 32) row[i] = 0.0f;
  float* gl = d.nnGlobal + (size_t)g * 19;
  if(lane < 19) gl[lane] = 0.0f;
  __syncwarp();
  const uint32_t own = black ? bd.b : bd.w, opp = black ? bd.w : bd.b;
  // planes 18/19: pass-alive + territory area for area scoring without tax (nninputs.cpp:2375-2382, 2425-2436)
  uint32_t areaB, areaW;
  const long long tZero = clock64();
  boardCalculateArea(bd, true, true, true, d.gMultiSuicide[g] != 0, areaB, areaW);
  const long long tArea = clock64();
  const uint32_t areaOwn = black ? areaB : areaW, areaOpp = black ? areaW : areaB;
  // planes 14-17: ladders on the current board and on the boards 1 and 2 moves ago (nninputs.cpp:2547-2583).  15/16 come
  // from the ancestors' cached results; 14/17 are searched by the whole block after this function returns.
  const int numHist = (h0 == -1) ? 0 : (h1 == -1) ? 1 : 2;   // min(2, moves of history included)
  const bool doLadders = d.enableLadders && !terminal;
  if(!doLadders || numHist < 1) { lad1 = 0; lad2 = 0; }       // numHist 0: copies of plane 14, written with it
  else if(numHist < 2) lad2 = lad1;
  shB[lane] = bd.b; shW[lane] = bd.w; shCand[lane] = lib1 | lib2;
  d.leafB[g * 32 + lane] = bd.b; d.leafW[g * 32 + lane] = bd.w; d.leafCand[g * 32 + lane] = lib1 | lib2;
  if(lane == 0) { shKo = bd.ko; d.leafKo[g] = bd.ko; shDoLadders = doLadders ? 1 : 0; d.leafNumHist[g] = numHist; d.leafValid[g] = 1; }
  if(lane < d.gY[g]) {
    for(int x = 0; x < d.gX[g]; x++) {
      float* f = row + (size_t)(lane * d.X + x) * 22;
      const uint32_t bit = 1u << x;
      f[0] = 1.0f;
      if(superKo & bit) f[6] = 1.0f;                 // superko bans join the simple-ko point in plane 6 (nninputs.cpp:2342-2356)
      if(own & bit) f[1] = 1.0f; else if(opp & bit) f[2] = 1.0f;
      if(lib1 & bit) f[3] = 1.0f; else if(lib2 & bit) f[4] = 1.0f; else if(lib3 & bit) f[5] = 1.0f;
      if(areaOwn & bit) f[18] = 1.0f; else if(areaOpp & bit) f[19] = 1.0f;
      if(lad1 & bit) f[15] = 1.0f;
      if(lad2 & bit) f[16] = 1.0f;
    }
  }
  __syncwarp();
  const bool passEndsLeaf = histPassWouldEndPhase(bd, hst, HL, black, d.gKoRule[g]);
  if(lane == 0) {
    if(bd.ko >= 0) row[(size_t)posOf(bd.ko, d.X) * 22 + 6] = 1.0f;
    // history planes 9..13: the move k plies ago must have been made by the right colour, which alternation guarantees
    int hs[5] = {h0, h1, h2, h3, h4};
    for(int k = 0; k < 5; k++) {
      if(hs[k] == -1) break;                       // no more history (game start)
      if(hs[k] == -2) gl[k] = 1.0f;
      else row[(size_t)posOf(hs[k], d.X) * 22 + 9 + k] = 1.0f;
    }
    float selfKomi = black ? -d.komiG[g] : d.komiG[g];
    float bArea = (float)(d.gX[g] * d.gY[g]);
    selfKomi = fminf(fmaxf(selfKomi, -bArea - 20.0f), bArea + 20.0f);
    gl[5] = selfKomi / 20.0f;
    if(d.gMultiSuicide[g]) gl[8] = 1.0f;
    gl[14] = passEndsLeaf ? 1.0f : 0.0f;         // BoardHistory::passWouldEndPhase
    if(d.gKoRule[g] == KGB_KO_POSITIONAL || d.gKoRule[g] == KGB_KO_SPIGHT) { gl[6] = 1.0f; gl[7] = 0.5f; }   // ko rule (nninputs.cpp:2612-2621)
    else if(d.gKoRule[g] == KGB_KO_SITUATIONAL) { gl[6] = 1.0f; gl[7] = -0.5f; }
    // komi parity wave (nninputs.cpp:2696-2729)
    bool drawableKomisAreEven = ((d.gX[g] * d.gY[g]) % 2) == 0;
    float komiFloor = drawableKomisAreEven ? floorf(selfKomi / 2.0f) * 2.0f : floorf((selfKomi - 1.0f) / 2.0f) * 2.0f + 1.0f;
    float delta = fminf(fmaxf(selfKomi - komiFloor, 0.0f), 2.0f);
    gl[18] = delta < 0.5f ? delta : (delta < 1.5f ? 1.0f - delta : delta - 2.0f);
    int sym = (int)(splitmix64(d.seed ^ ((uint64_t)g << 40) ^ (d.gameCounter[g] << 28) ^ ((uint64_t)d.moveNum[g] << 14) ^
                               (uint64_t)d.nodeVisits[gb]) & 7);   // nneval.cpp:698-707: random symmetry per row
    if(d.fakeNN) sym = 0;                                          // the reference's evaluator without nnRandomize
    if(d.fixedSymmetryPlusOne > 0) sym = d.fixedSymmetryPlusOne - 1; // TEST ONLY: nnRandomize = false with a forced symmetry
    if(node == 0 && rootSyms(d, g) > 1 && d.nodeVisits[gb] == 0) {
      // NNEvaluator::averageMultipleSymmetries: a partial Fisher-Yates shuffle of 0..7 drawn from the search thread's generator
      // With a dynamic score utility Search::beginSearch first takes ONE ordinary evaluation of the root to centre it on
      // (computeRootNNEvaluation, search.cpp:1140-1147): evaluation 0 of the root is that one, the symmetric ones follow.
      const int lead = d.dynamicScoreUtilityFactor != 0.0 ? 1 : 0;
      int* order = d.rootSymOrder + g * 8;
      int cnt = d.rootSymCount[g] - lead;
      if(cnt == 0) {
        DevRand rand;
        rand.s = d.searchRand[g];
        for(int i = 0; i < 8; i++) order[i] = i;
        for(int i = 0; i < d.rootNumSymmetries; i++) {
          const uint32_t n = (uint32_t)(8 - i);
          uint32_t bits, val;
          do { bits = rand.nextUInt(); val = bits % n; } while((uint32_t)(bits - val + (n - 1)) < (uint32_t)(bits - val));   // Rand::nextUInt(n)
          const int j = i + (int)val, t = order[i];
          order[i] = order[j]; order[j] = t;
        }
        d.searchRand[g] = rand.s;
      }
      if(cnt >= 0) sym = order[cnt];
    }
    d.nnSymmetry[g] = sym;
    d.nnOptimism[g] = 0.0f;
    d.dbgCycles[g * 8 + 4] = tLeaf - tW0; d.dbgCycles[g * 8 + 5] = tLegal - tLeaf; d.dbgCycles[g * 8 + 6] = tArea - tZero;
    d.dbgCycles[g * 8 + 7] = (clock64() - tArea) + (tZero - tLegal);
#ifdef KGB_PROFILE_DESCENT   // slots 1 and 5-7 re-used: steps of the wave's last descent, gather + ordered sums, selection, move + history, new-edge work
    d.dbgCycles[g * 8 + 1] = (pfEdge << 16) | (pfAttempts << 10) | pfSteps; d.dbgCycles[g * 8 + 5] = pfGather; d.dbgCycles[g * 8 + 6] = pfSelect; d.dbgCycles[g * 8 + 7] = pfMove;
    d.dbgCycles[g * 8 + 4] = (pfBackup << 32) | (pfAdvance & 0xffffffffLL);      // replaces the descent total (= sum of the parts)
#endif
  }
}


// One block per game.  Warp 0 walks the tree, plays the moves and writes the features; the ladder searches of the leaf
// position (independent of each other, and by far the most expensive feature) are dealt out to all SP_LADDER_WARPS warps.
// With ladderNodesPerWave > 0 every warp stops after that many search moves: a game whose searches are unfinished delivers no
// leaf this wave (leafValid = 0: the evaluator's row for it is ignored, nothing is backed up) and carries on in the next one,
// so one deep ladder costs its own game a few waves instead of making all games wait.  Features are identical either way.
__global__ void __launch_bounds__(SP_LADDER_WARPS * 32, 2) spSelectKernel(const SPDev d) {
  const int g = blockIdx.x;
  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;
  __shared__ uint32_t shB[32], shW[32], shCand[32];
  __shared__ int shKo, shDoLadders, shFresh, shUnfinished;
  __shared__ double shSum[64];
  const long long tStart = clock64();
  long long tWarp0 = tStart;
  if(warp == 0) {
    if(d.ladPending[g]) {
      shB[lane] = d.leafB[g * 32 + lane]; shW[lane] = d.leafW[g * 32 + lane]; shCand[lane] = d.leafCand[g * 32 + lane];
      if(lane == 0) { shKo = d.leafKo[g]; shDoLadders = 1; shFresh = 0; }
    }
    else {
      spSelectWarp0(d, g, lane, shB, shW, shCand, shKo, shDoLadders, shSum);
      if(lane == 0) shFresh = 1;
    }
    if(lane == 0) shUnfinished = 0;
    tWarp0 = clock64();
  }
  __syncthreads();
  if(!shDoLadders) {
    if(warp == 0 && lane == 0) { d.dbgCycles[g * 8 + 0] = clock64() - tStart; d.dbgCycles[g * 8 + 2] = tWarp0 - tStart; d.dbgCycles[g * 8 + 3] = 0; }
    return;
  }
  const LadderScratch sc0 = ladderScratchAt(d.ladderScratch + (size_t)g * SP_LADDER_WARPS * ladderScratchWordsPerWarp());
  {
    WarpBoard bd;
    boardInit(bd, d.gX[g], d.gY[g]);
    bd.b = shB[lane]; bd.w = shW[lane]; bd.ko = shKo;
    LadderScratch sc = ladderScratchAt(d.ladderScratch + ((size_t)g * SP_LADDER_WARPS + warp) * ladderScratchWordsPerWarp());
    sc.counters = d.ladderCounters;
    int budget = d.ladderNodesPerWave > 0 ? d.ladderNodesPerWave : 0x7fffffff;
    const bool fresh = shFresh != 0;
    bool done = true;
    if(fresh || sc.st[LST_NEXT_ITEM] != 0x7fffffff) done = boardLaddersResumable(bd, shCand[lane], sc, d.gX[g], d.gY[g], warp, SP_LADDER_WARPS, budget, fresh);
    if(!done && lane == 0) atomicAdd(&shUnfinished, 1);
  }
  __syncthreads();
  if(warp == 0) {
    const long long tLad = clock64();
    if(lane == 0) { d.dbgCycles[g * 8 + 0] = tLad - tStart; d.dbgCycles[g * 8 + 2] = tWarp0 - tStart; d.dbgCycles[g * 8 + 3] = tLad - tWarp0; }
    if(shUnfinished != 0) {
      if(lane == 0) { d.ladPending[g] = 1; d.leafValid[g] = 0; atomicAdd(d.stalledWaves, 1ULL); }
      return;
    }
    uint32_t lad0 = 0, wB = 0, wW = 0;
    for(int w = 0; w < SP_LADDER_WARPS; w++) {
      const uint32_t* acc = sc0.accLad + (size_t)w * ladderScratchWordsPerWarp();   // accLad, accWB, accWW are consecutive
      lad0 |= acc[lane]; wB |= acc[32 + lane]; wW |= acc[64 + lane];
    }
    const uint32_t work17 = d.leafBlackToMove[g] ? wW : wB;   // working moves against the OPPONENT's 2-liberty chains
    const int node = d.leafNode[g];
    d.nodeLad[((size_t)g * d.maxNodes + node) * 32 + lane] = lad0;
    if(lane == 0) { d.ladPending[g] = 0; d.leafValid[g] = 1; }
    float* row = d.nnSpatial + (size_t)g * d.XY * 22;
    const int numHist = d.leafNumHist[g];
    if(lane < d.gY[g]) {
      for(int x = 0; x < d.gX[g]; x++) {
        float* f = row + (size_t)(lane * d.X + x) * 22;
        const uint32_t bit = 1u << x;
        if(lad0 & bit) {
          f[14] = 1.0f;
          if(numHist < 1) { f[15] = 1.0f; f[16] = 1.0f; }   // no earlier board: the reference reuses the current one
        }
        if(work17 & bit) f[17] = 1.0f;
      }
    }
  }
}

// Search::maybeAddPolicyNoiseAndTemp (searchhelpers.cpp:150-215) on the root's post-processed policy: temperature
// (interpolateEarly :541-545), then Dirichlet noise (addDirichletNoise / computeDirichletAlphaDistribution :78-147).
// One warp: every per-element expression (log / exp / pow, the divisions) is evaluated by the lanes in parallel, every sum is
// added in position order like the reference's loops (all lanes run the short loop over the staged values), and the gamma
// draws - one sequential stream of the reference's generator - are made by lane 0 without their final pow, which the lanes
// then apply in parallel (tests/test_gpu_board_selfplay.py::test_root_dirichlet_noise_matches_reference checks it against the
// reference's output).  r: [policySize], r2: [2 * policySize] doubles.
__device__ void rootPolicyTemperatureAndNoiseWarp(float* pol, int policySize, int X, int Y, int turnNumber, bool noise, double concentration,
                                                  double weight, double temperature, double temperatureEarly, double halflife, DevRandState* randState,
                                                  double* r, double* r2, int lane) {
  if(temperature != 1.0 || temperatureEarly != 1.0) {
    const double rawHalflives = (double)turnNumber / halflife;
    const double halflives = rawHalflives * 19.0 / sqrt((double)(X * Y));
    const double temp = temperature + (temperatureEarly - temperature) * pow(0.5, halflives);
    double maxValue = 0.0;
    for(int i = lane; i < policySize; i += 32) { const double prob = pol[i]; if(prob > maxValue) maxValue = prob; }
#pragma unroll
    for(int o = 16; o > 0; o >>= 1) maxValue = fmax(maxValue, __shfl_xor_sync(KGB_FULL, maxValue, o));
    const double logMaxValue = log(maxValue), invTemp = 1.0 / temp;
    for(int i = lane; i < policySize; i += 32)
      if(pol[i] > 0) pol[i] = (float)exp((log((double)pol[i]) - logMaxValue) * invTemp);
    __syncwarp();
    double sum = 0.0;
    for(int i = 0; i < policySize; i++) { const float p = pol[i]; if(p > 0) sum += p; }      // (a value that underflowed to 0 adds nothing either way)
    __syncwarp();
    for(int i = lane; i < policySize; i += 32)
      if(pol[i] >= 0) pol[i] = (float)(pol[i] / sum);
    __syncwarp();
  }
  if(!noise) return;
  int legalCount = 0;
  for(int i = lane; i < policySize; i += 32) if(pol[i] >= 0) legalCount++;
  legalCount = __reduce_add_sync(KGB_FULL, legalCount);
  // half of the alpha mass uniform, half shaped by the log policy (clipped at 0.01) above its mean
  for(int i = lane; i < policySize; i += 32)
    if(pol[i] >= 0) r[i] = log(fmin(0.01, (double)pol[i]) + 1e-20);
  __syncwarp();
  double logPolicySum = 0.0;
  for(int i = 0; i < policySize; i++) if(pol[i] >= 0) logPolicySum += r[i];
  const double logPolicyMean = logPolicySum / legalCount;
  __syncwarp();
  for(int i = lane; i < policySize; i += 32)
    if(pol[i] >= 0) r[i] = fmax(0.0, r[i] - logPolicyMean);
  __syncwarp();
  double alphaPropSum = 0.0;
  for(int i = 0; i < policySize; i++) if(pol[i] >= 0) alphaPropSum += r[i];
  const double uniformProb = 1.0 / legalCount;
  __syncwarp();
  for(int i = lane; i < policySize; i += 32)
    if(pol[i] >= 0) r[i] = alphaPropSum <= 0.0 ? uniformProb : 0.5 * (r[i] / alphaPropSum + uniformProb);
  __syncwarp();
  if(lane == 0) {
    DevRand rand;
    rand.s = *randState;
    for(int i = 0; i < policySize; i++) {
      if(pol[i] >= 0) { double u, inva; r[i] = rand.nextGammaCore(r[i] * concentration, u, inva); r2[i] = u; r2[policySize + i] = inva; }
      else { r[i] = 0.0; r2[i] = -1.0; }
    }
    *randState = rand.s;
  }
  __syncwarp();
  for(int i = lane; i < policySize; i += 32)
    if(r2[i] >= 0.0) r[i] = r[i] * pow(r2[i], r2[policySize + i]);
  __syncwarp();
  double rSum = 0.0;
  for(int i = 0; i < policySize; i++) if(pol[i] >= 0) rSum += r[i];
  __syncwarp();
  for(int i = lane; i < policySize; i += 32) {
    const double ri = r[i] / rSum;
    if(pol[i] >= 0) pol[i] = (float)(ri * weight + pol[i] * (1.0 - weight));
  }
  __syncwarp();
}

__global__ void playSelectionKernel(const SPDev d, int g, double* out /*[policySize] by move position*/) {
  if(threadIdx.x != 0 || blockIdx.x != 0) return;
  double* psv = d.selScratch + (size_t)g * 3 * d.policySize;
  for(int i = 0; i < d.policySize; i++) out[i] = -1.0;
  const int nc = rootPlaySelectionValues(d, g, psv, psv + d.policySize, psv + 2 * d.policySize);
  for(int k = 0; k < nc; k++) out[(int)d.childOrder[(size_t)g * d.maxNodes * d.policySize + k]] = psv[k];
}
__global__ void chooseIndexTestKernel(DevRandState* st, const double* probs, int n, double temperature, double onlyBelowProb, int count, int* out,
                                      double* scratch) {
  if(threadIdx.x != 0 || blockIdx.x != 0) return;
  DevRand rand;
  rand.s = *st;
  for(int i = 0; i < count; i++) out[i] = chooseIndexWithTemperature(rand, probs, n, temperature, onlyBelowProb, scratch);
}

__global__ void rootNoiseTestKernel(float* pol, int policySize, int X, int Y, int turnNumber, int noise, double concentration, double weight,
                                    double temperature, double temperatureEarly, double halflife, DevRandState* randState, double* scratch) {
  if(blockIdx.x == 0 && threadIdx.x < 32)
    rootPolicyTemperatureAndNoiseWarp(pol, policySize, X, Y, turnNumber, noise != 0, concentration, weight, temperature, temperatureEarly, halflife, randState, scratch,
                                      scratch + policySize, threadIdx.x);
}

// Search::recomputeNodeStats (searchupdatehelpers.cpp:167-360) for the parameter subset of the loop (no root noise subtraction:
// chosenMoveSubtract / chosenMovePrune are not applied during the search), one warp per node.  Noise pruning and the node's own
// evaluation weight (uncertainty) when switched on.
// Children are visited in creation order and every sum is accumulated in that order (orderedAdd2), like the reference's loops.
#ifdef KGB_PROFILE_DESCENT   // profiling build: cycles of the recompute's phases, accumulated per game (spBackupKernel zeroes the slots first)
#define RPF(slot) do { const long long t_ = clock64(); if(lane == 0) d.dbgCycles[g * 8 + (slot)] += t_ - rpT; rpT = t_; } while(0)
#else
#define RPF(slot) do {} while(0)
#endif
__device__ void recomputeNodeStats(const SPDev& d, int g, int node, bool nodePlaWhite, double* sh, int lane) {
#ifdef KGB_PROFILE_DESCENT
  long long rpT = clock64();
  if(lane == 0) d.dbgCycles[g * 8 + 1] += 1;
#endif
  const size_t gb = (size_t)g * d.maxNodes, gn = gb + node, nb = gn * d.policySize;
  const int nc = d.nodeNumChildren[gn];
  double WA[12], CU[12], CUSQ[12], CWS[12], CWSQ[12];   // weightAdjusted, child utilityAvg / utilitySqAvg / weightSum / weightSqSum
  int CI[12];                                             // the child's node index
  uint32_t GM[12];                                        // lanes holding a good child (noise pruning)
  double origTotal = 0.0, simpleValueSum = 0.0;
#pragma unroll
  for(int ch = 0; ch < 12; ch++) {
    WA[ch] = 0.0; CU[ch] = 0.0; CUSQ[ch] = 0.0; CWS[ch] = 1.0; CWSQ[ch] = 0.0; CI[ch] = 0; GM[ch] = 0;
    if(ch * 32 < nc) {
      const int k = ch * 32 + lane;
      const bool in = k < nc;
      const int mv = in ? (int)d.childOrder[nb + k] : 0;
      const int c = in ? d.childNode[nb + mv] : 0;
      CI[ch] = c;
      const int ev = in ? d.childVisits[nb + mv] : 0;
      const int cv = in ? d.nodeVisits[gb + c] : 0;
      const double cw = in ? d.nodeWeightSum[gb + c] : 0.0;
      const bool good = in && cv > 0 && cw > 0.0 && ev > 0;
      if(d.useNoisePruning) GM[ch] = __ballot_sync(KGB_FULL, good);
      if(good) {
        WA[ch] = cw * ((double)ev / (double)(cv > 1 ? cv : 1));
        CU[ch] = d.nodeUtilAvg[gb + c]; CUSQ[ch] = d.nodeUtilSqAvg[gb + c]; CWS[ch] = cw; CWSQ[ch] = d.nodeWeightSqSum[gb + c];
      }
    }
  }
  RPF(4);
  // (gathers first, without a barrier between the chunks: their dependent loads overlap; then the sums in the reference's order.
  // A child that is not `good` has WA = 0 and CU = 0, so its terms are exactly 0 as before.)
#pragma unroll
  for(int ch = 0; ch < 12; ch++) {
    if(ch * 32 < nc) {
      const double selfU = nodePlaWhite ? CU[ch] : -CU[ch];
      const int n = nc - ch * 32 < 32 ? nc - ch * 32 : 32;
      orderedAdd2(WA[ch], WA[ch] != 0.0 ? selfU * WA[ch] : 0.0, n, origTotal, simpleValueSum, sh, lane);
    }
  }
  double curTotal = origTotal;   // currentTotalChildWeight
  if(d.useNoisePruning && origTotal > 0.00001) {
    // pruneNoiseWeight (:495-539): one pass over the good children in creation order, each step depending on the sums before it.
    // Every lane runs the same pass on values broadcast from the lane that holds the child (warp-uniform), the owner keeps the result.
    // Its running sums are the ones downweightBadChildrenAndNormalizeWeight then takes (same terms, same order).
    int numGood = 0;
#pragma unroll
    for(int ch = 0; ch < 12; ch++) numGood += __popc(GM[ch]);
    if(numGood > 1) {
      const float* pol = d.policy + nb;   // the node's policy as the search sees it (noised at a noised root)
      double utilitySoFar = 0.0, weightSoFar = 0.0, policySoFar = 0.0;
#pragma unroll
      for(int ch = 0; ch < 12; ch++) {
        if(GM[ch] == 0) continue;
        const int k = ch * 32 + lane;
        const double rawPolicy = k < nc ? fmax(1e-30, (double)pol[d.childOrder[nb + k]]) : 0.0;
        const double selfU = nodePlaWhite ? CU[ch] : -CU[ch];
        for(uint32_t m = GM[ch]; m != 0; m &= m - 1) {
          const int j = __ffs(m) - 1;
          const double utility = __shfl_sync(KGB_FULL, selfU, j), oldWeight = __shfl_sync(KGB_FULL, WA[ch], j);
          const double p = __shfl_sync(KGB_FULL, rawPolicy, j);
          double newWeight = oldWeight;
          if(weightSoFar > 0 && policySoFar > 0) {
            const double utilityGap = utilitySoFar / weightSoFar - utility;
            if(utilityGap > 0) {
              const double lenientShare = 2.0 * (weightSoFar * p / policySoFar);
              if(oldWeight > lenientShare) {
                double weightToSubtract = (oldWeight - lenientShare) * (1.0 - exp(-utilityGap / d.noisePruneUtilityScale));
                if(weightToSubtract > d.noisePruningCap) weightToSubtract = d.noisePruningCap;
                newWeight = oldWeight - weightToSubtract;
                if(lane == j) WA[ch] = newWeight;
              }
            }
          }
          utilitySoFar += utility * newWeight;
          weightSoFar += newWeight;
          policySoFar += p;
        }
      }
      curTotal = weightSoFar;
      simpleValueSum = utilitySoFar;
    }
  }
  // downweightBadChildrenAndNormalizeWeight (:402-491) with nothing to subtract or prune
  if(d.valueWeightExponent != 0.0 && curTotal > 0.0) {
    const double simpleValue = simpleValueSum / curTotal;
    double totalNew = 0.0, unused = 0.0;
#pragma unroll
    for(int ch = 0; ch < 12; ch++) {
      if(ch * 32 < nc) {
        if(WA[ch] > 0.0) {
          const double selfU = nodePlaWhite ? CU[ch] : -CU[ch];
          const double precision = 1.5 * sqrt(WA[ch]);
          const double stdev = sqrt(0.00000001 + 1.0 / precision);
          const double z = (selfU - simpleValue) / stdev;
          const double p = vwCdf(d.vwCdfTable, z) + 0.0001;
          WA[ch] *= d.valueWeightExponent == 0.5 ? sqrt(p) : pow(p, d.valueWeightExponent);
        }
        const int n = nc - ch * 32 < 32 ? nc - ch * 32 : 32;
        orderedAdd2(WA[ch], 0.0, n, totalNew, unused, sh, lane);
      }
    }
    const double factor = curTotal / totalNew;
#pragma unroll
    for(int ch = 0; ch < 12; ch++) WA[ch] *= factor;
  }
  RPF(5);
  double utilitySum = 0.0, utilitySqSum = 0.0, weightSqSum = 0.0, unused = 0.0;
#pragma unroll
  for(int ch = 0; ch < 12; ch++) {
    if(ch * 32 < nc) {
      const double scaling = WA[ch] / CWS[ch];
      const int n = nc - ch * 32 < 32 ? nc - ch * 32 : 32;
      orderedAdd2(WA[ch] * CU[ch], WA[ch] * CUSQ[ch], n, utilitySum, utilitySqSum, sh, lane);
      orderedAdd2(scaling * scaling * CWSQ[ch], 0.0, n, weightSqSum, unused, sh, lane);
    }
  }
  // the other moments: sum of weightAdjusted * child average (searchupdatehelpers.cpp:246-251), same order.  Per pair of moments the
  // children's values are gathered first (loads of all chunks in flight together), then added in order.
  double mom[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
#pragma unroll
  for(int pair = 0; pair < 3; pair++) {
    double MA[12], MB[12];
#pragma unroll
    for(int ch = 0; ch < 12; ch++) {
      MA[ch] = 0.0; MB[ch] = 0.0;
      if(ch * 32 < nc) {
        const bool use = ch * 32 + lane < nc && WA[ch] > 0.0;
        const double* cm = d.nodeMoments + (gb + (use ? CI[ch] : 0)) * 5;
        if(use) { MA[ch] = WA[ch] * cm[2 * pair]; if(pair < 2) MB[ch] = WA[ch] * cm[2 * pair + 1]; }
      }
    }
#pragma unroll
    for(int ch = 0; ch < 12; ch++) {
      if(ch * 32 < nc) {
        const int n = nc - ch * 32 < 32 ? nc - ch * 32 : 32;
        orderedAdd2(MA[ch], MB[ch], n, mom[2 * pair], mom[2 * pair + 1], sh, lane);
      }
    }
  }
  RPF(6);
  double weightSum = curTotal;
  // the node's own evaluation, with its weight (1 unless uncertainty weighting applies)
  double utility = d.nodeNNUtil[gn];
  const double selfWeight = d.useUncertainty ? d.nodeNNWeight[gn] : 1.0;
  const int entry = d.subtreeValueBiasFactor != 0.0 ? d.nodeBiasEntry[gn] : -1;
  if(entry >= 0) {
    // searchupdatehelpers.cpp:273-310: the node reports how far its children's average is from its own evaluation to the entry
    // shared by all nodes reached by the same local move, and shifts its own evaluation by the entry's average observation
    const size_t te = (size_t)g * d.biasTableSize + entry;
    double newDelta, newWeight;
    if(curTotal > 1e-10) {
      const double utilityChildren = utilitySum / curTotal;
      const double biasWeight = pow(origTotal, d.subtreeValueBiasWeightExponent);
      const double biasDelta = (utilityChildren - utility) * biasWeight;
      newDelta = d.biasDeltaSum[te] + (biasDelta - d.nodeLastBiasDelta[gn]);
      newWeight = d.biasWeightSum[te] + (biasWeight - d.nodeLastBiasWeight[gn]);
      __syncwarp();
      if(lane == 0) { d.biasDeltaSum[te] = newDelta; d.biasWeightSum[te] = newWeight; d.nodeLastBiasDelta[gn] = biasDelta; d.nodeLastBiasWeight[gn] = biasWeight; }
    }
    else { newDelta = d.biasDeltaSum[te]; newWeight = d.biasWeightSum[te]; }
    if(newWeight > 0.001) utility += d.subtreeValueBiasFactor * newDelta / newWeight;
  }
  utilitySum += utility * selfWeight;
  utilitySqSum += utility * utility * selfWeight;
  weightSqSum += selfWeight * selfWeight;
  weightSum += selfWeight;
  __syncwarp();
  if(lane == 0) {
    for(int i = 0; i < 5; i++) d.nodeMoments[gn * 5 + i] = (mom[i] + d.nodeNNMoments[gn * 5 + i] * selfWeight) / weightSum;
    d.nodeUtilAvg[gn] = utilitySum / weightSum;
    d.nodeUtilSqAvg[gn] = utilitySqSum / weightSum;
    d.nodeWeightSqSum[gn] = weightSqSum;
    d.nodeWeightSum[gn] = weightSum;
    d.nodeVisits[gn] = d.nodeVisits[gn] + 1;
  }
  __syncwarp();
  RPF(7);
}

// Short-term errors of one evaluation from the raw score-value channels 4 and 5 (nneval.cpp:1161-1178, 1217-1226), by model version;
// -1 for nets below version 9, which have no such outputs.  Host and device share it (kgb_test_uncertainty_weight).
__host__ __device__ inline double spSoftPlus(double x) { return x > 40.0 ? x : log(1.0 + exp(x)); }
__host__ __device__ inline void shorttermErrors(int version, double valueMult, double scoreMult, double rawWinloss, double rawScore, float& winlossError,
                                                float& scoreError) {
  double wl, se;
  if(version >= 14) {
    const double a = spSoftPlus(rawWinloss * 0.5), b = spSoftPlus(rawScore * 0.5);
    wl = sqrt(a * a * valueMult);
    se = sqrt(b * b * scoreMult);
  }
  else if(version >= 10) { wl = sqrt(spSoftPlus(rawWinloss) * valueMult); se = sqrt(spSoftPlus(rawScore) * scoreMult); }
  else { wl = spSoftPlus(rawWinloss); se = spSoftPlus(rawScore) * 10.0; }
  winlossError = version >= 9 ? (float)wl : -1.0f;
  scoreError = version >= 9 ? (float)se : -1.0f;
}
// ScoreValue::whiteDScoreValueDScoreSmoothNoDrawAdjust (nninputs.cpp:64-69)
__host__ __device__ inline double dScoreValueDScore(double score, double center, double scale, double sqrtBoardArea) {
  const double adjustedScore = score - center;
  const double scaleFactor = scale * sqrtBoardArea;
  return scaleFactor / (scaleFactor * scaleFactor + adjustedScore * adjustedScore) * 0.63661977236758134308;
}
// Search::computeWeightFromNNOutput (searchupdatehelpers.cpp:114-136) with getApproxScoreUtilityDerivative (searchhelpers.cpp:296-301),
// for a search whose switch applies (useUncertainty and a net of version >= 9)
__host__ __device__ inline double uncertaintyWeight(double coeff, double exponent, double maxWeight, double winLossUtilityFactor, double staticFactor,
                                                   double dynamicFactor, double dynamicScale, double center, double sqrtBoardArea, float whiteScoreMean,
                                                   float winlossError, float scoreError) {
  const double scoreMean = (double)whiteScoreMean;
  const double derivative = dScoreValueDScore(scoreMean, 0.0, 2.0, sqrtBoardArea) * staticFactor +
                            dScoreValueDScore(scoreMean, center, dynamicScale, sqrtBoardArea) * dynamicFactor;
  const double uncertainty = winLossUtilityFactor * winlossError + derivative * scoreError;
  const double powered = exponent == 1.0 ? uncertainty : exponent == 0.5 ? sqrt(uncertainty) : pow(uncertainty, exponent);
  const double baseline = coeff / maxWeight;
  return coeff / (powered + baseline);
}
// Board::sqrtBoardArea (board.cpp:234-239) of game g
__device__ __forceinline__ double sqrtBoardAreaOf(const SPDev& d, int g) {
  return d.gX[g] == d.gY[g] ? (double)d.gX[g] : sqrt((double)(d.gX[g] * d.gY[g]));
}
// The weight of an evaluation of game g's search (vals: whiteScoreMean at 3, the two short-term errors at 6 and 7)
__device__ __forceinline__ double evalWeight(const SPDev& d, int g, const float vals[8]) {
  if(!d.useUncertainty) return 1.0;
  return uncertaintyWeight(d.uncertaintyCoeff, d.uncertaintyExponent, d.uncertaintyMaxWeight, d.winLossUtilityFactor, d.staticScoreUtilityFactor,
                           d.dynamicScoreUtilityFactor, d.dynamicScoreCenterScale, d.recentScoreCenter[g], sqrtBoardAreaOf(d, g), vals[3], vals[6], vals[7]);
}

// Search::getScoreUtility (searchhelpers.cpp:272-279)
__device__ double scoreUtilityOf(const SPDev& d, int g, double scoreMean, double scoreMeanSq, double center) {
  const double sqrtBoardArea = sqrt((double)(d.gX[g] * d.gY[g]));
  const double stdev = svScoreStdev(scoreMean, scoreMeanSq);
  double r = 0.0;
  if(d.staticScoreUtilityFactor != 0.0) r += svExpectedWhiteScoreValue(d.svTable, scoreMean, stdev, 0.0, 2.0, sqrtBoardArea) * d.staticScoreUtilityFactor;
  if(d.dynamicScoreUtilityFactor != 0.0)
    r += svExpectedWhiteScoreValue(d.svTable, scoreMean, stdev, center, d.dynamicScoreCenterScale, sqrtBoardArea) * d.dynamicScoreUtilityFactor;
  return r;
}
// Search::getScoreUtilityDiff (searchhelpers.cpp:281-293): what `delta` more points for white are worth at this child's score statistics
__device__ double scoreUtilityDiff(const SPDev& d, int g, double scoreMean, double scoreMeanSq, double delta, double center) {
  const double sqrtBoardArea = sqrt((double)(d.gX[g] * d.gY[g]));
  const double stdev = svScoreStdev(scoreMean, scoreMeanSq);
  const double staticDiff = svExpectedWhiteScoreValue(d.svTable, scoreMean + delta, stdev, 0.0, 2.0, sqrtBoardArea) -
                            svExpectedWhiteScoreValue(d.svTable, scoreMean, stdev, 0.0, 2.0, sqrtBoardArea);
  const double dynamicDiff = svExpectedWhiteScoreValue(d.svTable, scoreMean + delta, stdev, center, d.dynamicScoreCenterScale, sqrtBoardArea) -
                             svExpectedWhiteScoreValue(d.svTable, scoreMean, stdev, center, d.dynamicScoreCenterScale, sqrtBoardArea);
  return staticDiff * d.staticScoreUtilityFactor + dynamicDiff * d.dynamicScoreUtilityFactor;
}
// utility of root child c with the ending score bonus of its move folded in (getExploreSelectionValueOfChild, searchexplorehelpers.cpp:135-139)
__device__ __forceinline__ double rootChildUtilityWithBonus(const SPDev& d, int g, size_t gb, int c, int mv, double utilityAvg) {
  const double bonus = d.rootEndBonus[(size_t)g * d.policySize + mv];
  if(bonus == 0.0) return utilityAvg;
  const double* cm = d.nodeMoments + (gb + c) * 5;
  return utilityAvg + scoreUtilityDiff(d, g, cm[2], cm[3], bonus, d.recentScoreCenter[g]);
}
// Once the root's evaluation is final (one warp): which root moves are allowed (rootPruneUselessMoves) and the ending score bonus of every move.
// bd = the root position, rootBlack = the player to move, haveOwnership = d.rootOwnAcc holds the summed ownership of `numEvals` evaluations.
__device__ void computeRootExtras(const SPDev& d, int g, const WarpBoard& bd, bool rootBlack, bool haveOwnership, int numEvals, int lane) {
  const uint32_t rm = bd.rowMask;
  const uint32_t own = rootBlack ? bd.b : bd.w, opp = rootBlack ? bd.w : bd.b;
  const uint32_t empty = ~(bd.b | bd.w) & rm;
  uint32_t safeB = 0, safeW = 0;
  if(d.rootPruneUselessMoves || d.rootEndingBonusPoints != 0.0)
    boardCalculateArea(bd, false, false, false, d.gMultiSuicide[g] != 0, safeB, safeW);   // rootSafeArea: pass-alive groups and strictly safe territory (search.cpp:1111-1122)
  uint32_t allowed = 0xffffffffu;
  if(d.rootPruneUselessMoves && d.passStreak[g * 2 + (rootBlack ? 1 : 0)] >= 4) allowed = ~(safeB | safeW);
  d.rootAllowed[g * 32 + lane] = allowed;
  double* bonus = d.rootEndBonus + (size_t)g * d.policySize;
  for(int i = lane; i < d.policySize; i += 32) bonus[i] = 0.0;
  __syncwarp();
  if(d.rootEndingBonusPoints == 0.0 || !haveOwnership || bd.ko >= 0) return;   // area scoring, no button: nothing for the pass; nothing during a ko
  uint32_t lib1, lib2, lib3;
  boardLibertyClasses(bd, lib1, lib2, lib3);
  const uint32_t captures = nbrs(opp & lib1, rm) & empty;          // Board::wouldBeCapture
  const uint32_t touchesOpp = nbrs(opp, rm) & empty;               // Board::isAdjacentToPla(loc, opp)
  const uint32_t safeOwn = rootBlack ? safeB : safeW;
  // Board::isNonPassAliveSelfConnection: an empty point outside the player's own pass-alive area with a neighbouring own stone that
  // is in nobody's pass-alive area, whose own neighbours belong to at least two different chains (the chain picked first does not matter)
  uint32_t cand = empty & ~safeOwn & nbrs(own & ~(safeB | safeW), rm);
  uint32_t selfConn = 0;
  while(true) {
    const int p = firstPoint(cand);
    if(p < 0) break;
    const uint32_t pt = pointMask(p);
    cand &= ~pt;
    const uint32_t nb = nbrs(pt, rm) & own;
    const int q = firstPoint(nb);
    if(q < 0) continue;
    const uint32_t chain = flood(pointMask(q), own, rm);
    if(__any_sync(KGB_FULL, (nb & ~chain) != 0)) selfConn |= pt;
  }
  const float floatLen = (float)numEvals;
  const float* acc = d.rootOwnAcc + (size_t)g * d.XY;
  const double extreme = 0.95, tail = 0.05;
  if(lane < d.gY[g]) {
    for(int x = 0; x < d.gX[g]; x++) {
      const uint32_t bit = 1u << x;
      if(!(empty & bit)) continue;
      const int pos = lane * d.X + x;
      const float whiteOwn = numEvals > 1 ? acc[pos] / floatLen : acc[pos];
      const double plaOwnership = rootBlack ? -(double)whiteOwn : (double)whiteOwn;
      double extraRootPoints = 0.0;
      if(plaOwnership <= -extreme) {
        if(!(captures & bit)) extraRootPoints -= d.rootEndingBonusPoints * ((-extreme - plaOwnership) / tail);
      }
      else if(plaOwnership >= extreme) {
        if(!(touchesOpp & bit) && !(selfConn & bit)) extraRootPoints -= d.rootEndingBonusPoints * ((plaOwnership - extreme) / tail);
      }
      bonus[pos] = rootBlack ? -extraRootPoints : extraRootPoints;
    }
  }
  __syncwarp();
}
// Search::recentScoreCenter of a fresh root from the expected score of its first evaluation (Search::beginSearch, search.cpp:1148-1153).
__device__ __forceinline__ double rootScoreCenter(const SPDev& d, int g, double whiteScoreMean) {
  double c = whiteScoreMean * (1.0 - d.dynamicScoreCenterZeroWeight);
  const double cap = sqrt((double)(d.gX[g] * d.gY[g])) * d.dynamicScoreCenterScale;
  if(c > whiteScoreMean + cap) c = whiteScoreMean + cap;
  if(c < whiteScoreMean - cap) c = whiteScoreMean - cap;
  return c;
}
// Search::getUtilityFromNN (searchhelpers.cpp:304-307) from the NNOutput fields (floats, white's perspective); a fresh root
// first centres the dynamic score utility on its expected score (Search::beginSearch, search.cpp:1125-1154).
__device__ double utilityFromEval(const SPDev& d, int g, int node, float whiteWin, float whiteLoss, float noResult, float whiteScoreMeanF,
                                  float whiteScoreMeanSqF, float whiteLeadF, int lane) {
  const size_t gb = (size_t)g * d.maxNodes;
  if(lane == 0) {   // the evaluation's contribution to the NodeStats moments (searchupdatehelpers.cpp:83-112)
    d.leafMoments[g * 5 + 0] = (double)whiteWin - (double)whiteLoss; d.leafMoments[g * 5 + 1] = (double)noResult;
    d.leafMoments[g * 5 + 2] = (double)whiteScoreMeanF; d.leafMoments[g * 5 + 3] = (double)whiteScoreMeanSqF; d.leafMoments[g * 5 + 4] = (double)whiteLeadF;
  }
  __syncwarp();
  double u = ((double)whiteWin - (double)whiteLoss) * d.winLossUtilityFactor + (double)noResult * d.noResultUtilityForWhite;
  if(d.staticScoreUtilityFactor != 0.0 || d.dynamicScoreUtilityFactor != 0.0) {
    const double whiteScoreMean = (double)whiteScoreMeanF, whiteScoreMeanSq = (double)whiteScoreMeanSqF;
    if(node == 0 && d.nodeVisits[gb] == 0 && rootSyms(d, g) <= 1) {
      const double c = rootScoreCenter(d, g, whiteScoreMean);
      __syncwarp();
      if(lane == 0) d.recentScoreCenter[g] = c;
      __syncwarp();
    }
    u += scoreUtilityOf(d, g, whiteScoreMean, whiteScoreMeanSq, d.recentScoreCenter[g]);
  }
  return u;
}
// Root policy temperature + Dirichlet noise on the root's first evaluation (searchnnhelpers.cpp:61-173).
__device__ void maybeRootNoise(const SPDev& d, int g, int node, int lane) {
  const size_t gb = (size_t)g * d.maxNodes;
  if(node == 0 && d.nodeVisits[gb] == 0) {
    // what computeNNRawStats records of the net's own opinion (play.cpp:890-914): the policy entropy BEFORE temperature and noise
    const float* pol = d.policy + gb * d.policySize;
    double e = 0.0;
    for(int i = lane; i < d.policySize; i += 32) { const double p = (double)pol[i]; if(p > 1e-30) e -= p * log(p); }
    e = warpSumD(e);
    if(lane == 0) d.rootRawEntropy[g] = e;
  }
  if(node == 0 && d.nodeVisits[gb] == 0 && !d.plainRoot[g] && (d.rootNoiseEnabled || d.rootPolicyTemperature != 1.0 || d.rootPolicyTemperatureEarly != 1.0)) {
    __syncwarp();
    // the whole warp (the play-selection scratch is free while a root is being evaluated)
    rootPolicyTemperatureAndNoiseWarp(d.policy + gb * d.policySize, d.policySize, d.gX[g], d.gY[g], d.moveNum[g], d.rootNoiseEnabled != 0,
                                      d.rootDirichletNoiseTotalConcentration, d.rootDirichletNoiseWeight, d.rootPolicyTemperature,
                                      d.rootPolicyTemperatureEarly, d.chosenMoveTemperatureHalflife, d.searchRand + g, d.noiseScratch + (size_t)g * d.policySize,
                                      d.selScratch + (size_t)g * 3 * d.policySize, lane);
    __syncwarp();
  }
}
// The end of a playout whose leaf value is known: the leaf's own statistics (Search::addLeafValue, searchupdatehelpers.cpp:11-81,
// evaluation weight w), then edge visit + recomputeNodeStats for every node on the path (updateStatsAfterPlayout).
__device__ void finishPlayout(const SPDev& d, int g, int node, double u, double w, bool terminal, bool leafBlack, int len, double* shSum, int lane) {
  const size_t gb = (size_t)g * d.maxNodes, gl = gb + node;
  const int leafVisits = d.nodeVisits[gl];
  __syncwarp();
  if(terminal) {
    if(lane == 0) {
      const double oldW = d.nodeWeightSum[gl], newW = oldW + w;
      for(int i = 0; i < 5; i++) d.nodeMoments[gl * 5 + i] = (d.nodeMoments[gl * 5 + i] * oldW + d.leafMoments[g * 5 + i] * w) / newW;
      d.nodeUtilAvg[gl] = (d.nodeUtilAvg[gl] * oldW + u * w) / newW;
      d.nodeUtilSqAvg[gl] = (d.nodeUtilSqAvg[gl] * oldW + (u * u) * w) / newW;
      d.nodeWeightSqSum[gl] = d.nodeWeightSqSum[gl] + w * w;
      d.nodeWeightSum[gl] = newW;
      d.nodeVisits[gl] = leafVisits + 1;
    }
  }
  else if(leafVisits == 0) {
    if(lane == 0) {
      d.nodeNNUtil[gl] = u;
      if(d.useUncertainty) d.nodeNNWeight[gl] = w;
      for(int i = 0; i < 5; i++) { d.nodeNNMoments[gl * 5 + i] = d.leafMoments[g * 5 + i]; d.nodeMoments[gl * 5 + i] = d.leafMoments[g * 5 + i]; }
      const int entry = d.subtreeValueBiasFactor != 0.0 ? d.nodeBiasEntry[gl] : -1;
      if(entry >= 0) {   // searchupdatehelpers.cpp:26-36
        const size_t te = (size_t)g * d.biasTableSize + entry;
        const double ew = d.biasWeightSum[te];
        if(ew > 0.001) u += d.subtreeValueBiasFactor * d.biasDeltaSum[te] / ew;
      }
      d.nodeUtilAvg[gl] = u; d.nodeUtilSqAvg[gl] = u * u; d.nodeWeightSqSum[gl] = w * w; d.nodeWeightSum[gl] = w;
      d.nodeVisits[gl] = 1;
    }
  }
  else recomputeNodeStats(d, g, node, !leafBlack, shSum, lane);   // depth cap reached on an expanded node: one more visit, same evaluation
  __syncwarp();
  for(int k = len - 1; k >= 0; k--) {
    const int pn = d.pathNode[(size_t)g * d.maxDepth + k], mv = d.pathMove[(size_t)g * d.maxDepth + k];
    if(lane == 0) d.childVisits[(gb + pn) * d.policySize + mv] += 1;
    __syncwarp();
    const bool pnBlack = ((len - k) & 1) ? !leafBlack : leafBlack;   // players alternate along the path
    recomputeNodeStats(d, g, pn, !pnBlack, shSum, lane);
    __syncwarp();
  }
  if(lane == 0) atomicAdd(d.totalVisits, 1ULL);
}

// ---- evaluation cache -----------------------------------------------------------------------------------------------------
__device__ __forceinline__ size_t cacheSlotOf(const SPDev& d, unsigned long long k0, unsigned long long k1) {
  return (size_t)((k0 ^ (k1 * 0x9E3779B97F4A7C15ULL)) & (unsigned long long)(d.cacheSize - 1));
}
// Looks the leaf's key up; on a hit copies policy, values and laddered stones into the node (whole warp).  Writers hold the
// entry's lock while they change it and readers check key and lock before and after copying, so a torn entry is never used.
__device__ bool cacheLookup(const SPDev& d, int g, int node, unsigned long long k0, unsigned long long k1, float vals[8], int lane) {
  const size_t slot = cacheSlotOf(d, k0, k1);
  bool ok = false;
  if(lane == 0) ok = atomicAdd(&d.cacheLock[slot], 0) == 0 && __ldcg(d.cacheKey0 + slot) == k0 && __ldcg(d.cacheKey1 + slot) == k1;
  ok = __shfl_sync(KGB_FULL, ok ? 1 : 0, 0) != 0;
  if(!ok) return false;
  __threadfence();
  const size_t gb = (size_t)g * d.maxNodes, nb = (gb + node) * d.policySize;
  for(int i = lane; i < d.policySize; i += 32) d.policy[nb + i] = __ldcg(d.cachePolicy + slot * d.policySize + i);
  d.nodeLad[(gb + node) * 32 + lane] = __ldcg(d.cacheLad + slot * 32 + lane);
  float v = lane < 8 ? __ldcg(d.cacheVals + slot * 8 + lane) : 0.0f;
  __threadfence();
  if(lane == 0) ok = atomicAdd(&d.cacheLock[slot], 0) == 0 && __ldcg(d.cacheKey0 + slot) == k0 && __ldcg(d.cacheKey1 + slot) == k1;
  ok = __shfl_sync(KGB_FULL, ok ? 1 : 0, 0) != 0;
#pragma unroll
  for(int i = 0; i < 8; i++) vals[i] = __shfl_sync(KGB_FULL, v, i);
  return ok;
}
__device__ void cacheStore(const SPDev& d, int g, int node, unsigned long long k0, unsigned long long k1, const float vals[8], int lane) {
  const size_t slot = cacheSlotOf(d, k0, k1);
  bool mine = false;
  if(lane == 0) mine = atomicCAS(&d.cacheLock[slot], 0, 1) == 0;
  mine = __shfl_sync(KGB_FULL, mine ? 1 : 0, 0) != 0;
  if(!mine) return;   // somebody else is writing this entry: skip, it is only a cache
  if(lane == 0) { d.cacheKey0[slot] = 0; d.cacheKey1[slot] = 0; }
  __threadfence();
  const size_t gb = (size_t)g * d.maxNodes, nb = (gb + node) * d.policySize;
  for(int i = lane; i < d.policySize; i += 32) d.cachePolicy[slot * d.policySize + i] = d.policy[nb + i];
  d.cacheLad[slot * 32 + lane] = d.nodeLad[(gb + node) * 32 + lane];
  if(lane < 8) d.cacheVals[slot * 8 + lane] = vals[lane];
  __threadfence();
  __syncwarp();
  if(lane == 0) {
    d.cacheKey1[slot] = k1; d.cacheKey0[slot] = k0;
    __threadfence();
    atomicExch(&d.cacheLock[slot], 0);
    atomicAdd(d.cacheStores, 1ULL);
  }
}

__global__ void spBackupKernel(const SPDev d) {
  __shared__ double shSumAll[4][64];
  double* shSum = shSumAll[(threadIdx.x >> 5) & 3];
  const int g = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if(g >= d.numGames) return;
  if(!d.leafValid[g]) return;   // no leaf this wave (ladder searches still running, or every playout ended inside the select kernel)
#ifdef KGB_PROFILE_DESCENT
  const long long tBk0 = clock64();
  if(lane == 0) { d.dbgCycles[g * 8 + 1] = 0; d.dbgCycles[g * 8 + 4] = 0; d.dbgCycles[g * 8 + 5] = 0; d.dbgCycles[g * 8 + 6] = 0; d.dbgCycles[g * 8 + 7] = 0; }
  __syncwarp();
#endif
  const size_t gb = (size_t)g * d.maxNodes;
  const int node = d.leafNode[g];
  const bool terminal = d.leafTerminal[g] != 0;
  const bool leafBlack = d.leafBlackToMove[g] != 0;
  if(node == 0 && d.nodeVisits[gb] == 0) {
    // the leaf is the game's root: keep its input row for the recorder (TrainingWriteBuffers::addRow stores the root's fillRowV7 row,
    // trainingwrite.cpp:463-478).  Every evaluation of an unvisited root carries the same un-symmetrised row; it stays valid until
    // the next move replaces the root, whatever later waves write into the evaluator's input buffer.
    const int n = d.XY * 22;
    const float* src = d.nnSpatial + (size_t)g * n;
    float* dst = d.rootRow + (size_t)g * (n + 19);
    for(int i = lane; i < n; i += 32) dst[i] = src[i];
    if(lane < 19) dst[n + lane] = d.nnGlobal[(size_t)g * 19 + lane];
  }
  double u, weight = 1.0;
  if(terminal) weight = d.useUncertainty ? d.uncertaintyMaxWeight : 1.0;   // search.cpp:1210, 1220
  if(d.leafTerminal[g] == 2) {
    // search.cpp:1204-1212: a game ended without result (long cycle under simple ko)
    u = 1.0 * d.noResultUtilityForWhite + scoreUtilityOf(d, g, 0.0, 0.0, d.recentScoreCenter[g]);
    if(lane == 0) { d.leafMoments[g * 5 + 0] = 0.0; d.leafMoments[g * 5 + 1] = 1.0; d.leafMoments[g * 5 + 2] = 0.0; d.leafMoments[g * 5 + 3] = 0.0; d.leafMoments[g * 5 + 4] = 0.0; }
    __syncwarp();
  }
  else if(terminal) {
    // search.cpp:1213-1222: the game result as a leaf value (area scoring: no "no result")
    const double score = (double)d.leafTerminalScore[g];
    const double whiteWins = score > 0 ? 1.0 : score < 0 ? 0.0 : d.drawEquivalentWinsForWhite;       // ScoreValue::whiteWinsOfWinner
    const double winLoss = 2.0 * whiteWins - 1.0;
    const bool integral = score == floor(score);
    // BoardHistory::whiteKomiAdjustmentForDraws folds the draw value into integer results; whiteScoreMeanSqOfScoreGridded
    const double scoreMean = score + (integral ? (double)(float)(d.drawEquivalentWinsForWhite - 0.5) : 0.0);
    double scoreMeanSq = score * score;
    if(integral) {
      const double lo = (score - 0.5) * (score - 0.5), hi = (score + 0.5) * (score + 0.5);
      scoreMeanSq = lo + (hi - lo) * d.drawEquivalentWinsForWhite;
    }
    u = winLoss * d.winLossUtilityFactor + scoreUtilityOf(d, g, scoreMean, scoreMeanSq, d.recentScoreCenter[g]);
    if(lane == 0) {   // search.cpp:1213-1222: winLoss, no "no result", score, its square, lead = score
      d.leafMoments[g * 5 + 0] = winLoss; d.leafMoments[g * 5 + 1] = 0.0; d.leafMoments[g * 5 + 2] = scoreMean;
      d.leafMoments[g * 5 + 3] = scoreMeanSq; d.leafMoments[g * 5 + 4] = scoreMean;
    }
    __syncwarp();
  }
  else {
    // ---- policy: legality mask + softmax (nneval.cpp:960-1051)
    const float* logits = d.nnPolicy + (size_t)g * d.policySize;
    const uint32_t legalRow = d.leafLegal[g * 32 + lane];
    float v[12]; bool ok[12];
    float mx = -1e25f;
#pragma unroll
    for(int k = 0; k < 12; k++) {
      int i = k * 32 + lane;
      ok[k] = false; v[k] = -1e30f;
      const int ic = i < d.XY ? i : d.XY - 1;                       // every lane takes part in the shuffle
      const uint32_t rowBits = __shfl_sync(KGB_FULL, legalRow, ic / d.X);
      if(i < d.policySize) {
        const bool legal = (i == d.policySize - 1) ? true : (((rowBits >> (ic % d.X)) & 1u) != 0);
        ok[k] = legal;
        if(legal) v[k] = logits[i];
        mx = fmaxf(mx, v[k]);
      }
    }
#pragma unroll
    for(int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(KGB_FULL, mx, o));
    float sum = 0.0f;
#pragma unroll
    for(int k = 0; k < 12; k++) { v[k] = ok[k] ? expf(v[k] - mx) : 0.0f; sum += v[k]; }
#pragma unroll
    for(int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(KGB_FULL, sum, o);
    const size_t nb = (gb + node) * d.policySize;
    const bool multiSymRoot = node == 0 && rootSyms(d, g) > 1 && d.nodeVisits[gb] == 0;
    const int symLead = d.dynamicScoreUtilityFactor != 0.0 ? 1 : 0;           // evaluation 0 only centres the dynamic score utility
    const int symCount = multiSymRoot ? d.rootSymCount[g] - symLead : 0;
#pragma unroll
    for(int k = 0; k < 12; k++) {
      int i = k * 32 + lane;
      if(i < d.policySize) {
        const float pk = ok[k] ? v[k] / sum : -1.0f;
        d.policy[nb + i] = symCount > 0 ? d.policy[nb + i] + pk : pk;     // NNOutput(others): float sums in evaluation order
      }
    }
    // ---- value: softmax(win, loss, noResult) from the mover's perspective -> white's (nneval.cpp:1112-1215); NNOutput stores the
    // results as float and the search widens them again (searchupdatehelpers.cpp:87-88) - the same rounding happens here
    const float* val = d.nnValue + (size_t)g * 3;
    double wl = val[0], ll = val[1], nl = val[2];
    double m = fmax(fmax(wl, ll), nl);
    if(d.gKoRule[g] != KGB_KO_SIMPLE) { nl -= 100000.0; m = fmax(fmax(wl, ll), nl); }   // nneval.cpp:1136-1147: no "no result" under superko
    double w = exp(wl - m), l = exp(ll - m), n = exp(nl - m);
    if(d.gKoRule[g] != KGB_KO_SIMPLE) n = 0.0;
    double s = w + l + n;
    w /= s; l /= s; n /= s;
    const float wf = (float)w, lf = (float)l, nf = (float)n;
    // score head (nneval.cpp:1150-1160, 1200-1215): mean * 20, softplus(stdev) * 20, both scaled by P(result)
    const float* sc = d.nnScore + (size_t)g * 6;
    double scoreMean = (double)sc[0] * d.scoreMeanMultiplier;
    const double pre = (double)sc[1];
    const double stdev = (pre > 40.0 ? pre : log(1.0 + exp(pre))) * d.scoreStdevMultiplier;
    double scoreMeanSq = scoreMean * scoreMean + stdev * stdev;
    scoreMean = scoreMean * (1.0 - n);
    scoreMeanSq = scoreMeanSq * (1.0 - n);
    const double lead = (double)sc[2] * d.leadMultiplier * (1.0 - n);
    float vals[8];
    vals[0] = leafBlack ? lf : wf; vals[1] = leafBlack ? wf : lf; vals[2] = nf;
    vals[3] = leafBlack ? -(float)scoreMean : (float)scoreMean; vals[4] = (float)scoreMeanSq; vals[5] = leafBlack ? -(float)lead : (float)lead;
    vals[6] = 0.0f; vals[7] = 0.0f;
    if(d.useUncertainty)   // channels 4 and 5: no colour flip
      shorttermErrors(d.modelVersion, d.shorttermValueErrorMultiplier, d.shorttermScoreErrorMultiplier, (double)sc[4], (double)sc[5], vals[6], vals[7]);
    __syncwarp();
    const bool freshRoot = node == 0 && d.nodeVisits[gb] == 0;
    const bool wantRootExtras = freshRoot && (d.rootEndingBonusPoints != 0.0 || d.rootPruneUselessMoves);
    if(wantRootExtras && d.rootEndingBonusPoints != 0.0 && symCount >= 0) {
      // NNOutput::whiteOwnerMap of this evaluation (nneval.cpp:1233-1250: tanh, flipped to white's perspective), summed like NNOutput(others)
      const float* raw = d.nnOwnership + (size_t)g * d.XY;
      float* oacc = d.rootOwnAcc + (size_t)g * d.XY;
      for(int i = lane; i < d.XY; i += 32) {
        const float o = leafBlack ? -tanhf(raw[i]) : tanhf(raw[i]);
        oacc[i] = symCount > 0 ? oacc[i] + o : o;
      }
      __syncwarp();
    }
    if(multiSymRoot) {
      if(symCount < 0) {
        // the centring evaluation: recentScoreCenter from its expected score (search.cpp:1148-1153), nothing else is kept
        const double c = rootScoreCenter(d, g, (double)vals[3]);
        if(lane == 0) { d.recentScoreCenter[g] = c; d.rootSymCount[g] = 1; atomicAdd(d.stalledWaves, 1ULL); }   // a wave without a playout
        return;
      }
      float* acc = d.rootSymAcc + g * 8;
      if(lane < 8) acc[lane] = symCount > 0 ? acc[lane] + vals[lane] : vals[lane];
      __syncwarp();
      if(symCount + 1 < d.rootNumSymmetries) {
        if(lane == 0) { d.rootSymCount[g] = symCount + symLead + 1; atomicAdd(d.stalledWaves, 1ULL); }   // the root stays unvisited: next wave, next symmetry
        return;
      }
      const float floatLen = (float)d.rootNumSymmetries;
      for(int i = lane; i < d.policySize; i += 32) d.policy[nb + i] = d.policy[nb + i] / floatLen;
#pragma unroll
      for(int i = 0; i < 8; i++) vals[i] = acc[i] / floatLen;
      if(lane == 0) d.rootSymCount[g] = 0;
      __syncwarp();
    }
    else if(d.cacheSize > 0) cacheStore(d, g, node, d.leafKey[g * 2], d.leafKey[g * 2 + 1], vals, lane);   // before any root noise: the raw evaluation
    if(wantRootExtras) {
      WarpBoard rb;
      rootBoardLoad(d, g, lane, rb, false);
      computeRootExtras(d, g, rb, leafBlack, true, multiSymRoot ? d.rootNumSymmetries : 1, lane);
    }
    maybeRootNoise(d, g, node, lane);
    u = utilityFromEval(d, g, node, vals[0], vals[1], vals[2], vals[3], vals[4], vals[5], lane);
    weight = evalWeight(d, g, vals);   // after utilityFromEval: a fresh root's score centre is set there
  }
  __syncwarp();
#ifdef KGB_PROFILE_DESCENT
  const long long tBk1 = clock64();
#endif
  finishPlayout(d, g, node, u, weight, terminal, leafBlack, d.pathLen[g], shSum, lane);
#ifdef KGB_PROFILE_DESCENT
  if(lane == 0) { d.dbgCycles[g * 8 + 0] = clock64() - tBk0; d.dbgCycles[g * 8 + 2] = tBk1 - tBk0; d.dbgCycles[g * 8 + 3] = d.pathLen[g]; }   // whole warp, before the path update, path length
#endif
}

// ------------------------------------------------------------------------------------------------------------
// TEST SUPPORT: deterministic fake net (identical to the one oracle/ref_driver.cpp gives the reference Search, so tree
// parity can be checked against the reference without any real net) and root-position setup.
// ------------------------------------------------------------------------------------------------------------
__global__ void spFakeNNKernel(const SPDev d, float* policyOut, float* valueOut, float* scoreOut, float* ownershipOut) {
  const int g = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if(g >= d.numGames) return;
  if(d.fakeNN == 3) {   // the table net: the outputs the host chose for this game (kgb_selfplay_debug_set_raw_outputs), whatever the position
    const float* t = d.fakeTable + (size_t)g * (d.policySize + 9 + d.XY);
    for(int i = lane; i < d.policySize; i += 32) policyOut[(size_t)g * d.policySize + i] = t[i];
    if(lane < 3) valueOut[g * 3 + lane] = t[d.policySize + lane];
    if(lane < 6) scoreOut[g * 6 + lane] = t[d.policySize + 3 + lane];
    if(ownershipOut != nullptr)
      for(int i = lane; i < d.XY; i += 32) ownershipOut[(size_t)g * d.XY + i] = t[d.policySize + 9 + i];
    return;
  }
  const float* row = d.nnSpatial + (size_t)g * d.XY * 22;
  uint64_t h = 0;
  for(int pos = lane; pos < d.XY; pos += 32) {
    int s = row[pos * 22 + 1] != 0.0f ? 1 : row[pos * 22 + 2] != 0.0f ? 2 : 0;
    if(s) h += splitmix64((uint64_t)pos * 4 + s);
  }
#pragma unroll
  for(int o = 16; o > 0; o >>= 1) h += __shfl_xor_sync(KGB_FULL, h, o);
  if(d.nnGlobal[(size_t)g * 19 + 5] < 0.0f) h ^= 0xABCDEFULL;
  if(d.nnSymmetry[g] != 0) h ^= splitmix64(0x5151ULL + (uint64_t)d.nnSymmetry[g]);   // outputs differ per symmetry, in the original orientation
  const bool wide = d.fakeNN == 4;   // oracle/ref_driver.cpp with KGREF_FAKE_WIDE=1: the same hash, outputs over wider ranges
  for(int i = lane; i < d.policySize; i += 32) {
    uint32_t u = (uint32_t)(splitmix64(h + (uint64_t)(i + 1) * 0x9E3779B97F4A7C15ULL) >> 48);
    float logit = wide ? (float)u * (3.0f / 4096.0f) - 24.0f : (float)u * (1.0f / 8192.0f) - 4.0f;
    if(wide && (u & 15u) == 0u) logit -= 96.0f;   // one point in 16 far below the rest: its exp underflows to 0 in float
    if(i == d.policySize - 1) logit -= 3.0f;
    policyOut[(size_t)g * d.policySize + i] = logit;
  }
  if(ownershipOut != nullptr)   // raw ownership logits in [-4,4) per point, mover's perspective (oracle/ref_driver.cpp's fake net)
    for(int i = lane; i < d.XY; i += 32)
      ownershipOut[(size_t)g * d.XY + i] = (float)(uint32_t)(splitmix64(h + (uint64_t)(i + 1) * 0xD1B54A32D192ED03ULL) >> 48) * (1.0f / 8192.0f) - 4.0f;
  if(lane == 0 && wide) {   // win, loss and no result from [-6,6), stdev pre-softplus from [-8,56), mean and lead from [-3,3)
    valueOut[g * 3 + 0] = (float)(uint32_t)(splitmix64(h ^ 0x1111ULL) >> 48) * (3.0f / 16384.0f) - 6.0f;
    valueOut[g * 3 + 1] = (float)(uint32_t)(splitmix64(h ^ 0x2222ULL) >> 48) * (3.0f / 16384.0f) - 6.0f;
    valueOut[g * 3 + 2] = (float)(uint32_t)(splitmix64(h ^ 0x8888ULL) >> 48) * (3.0f / 16384.0f) - 6.0f;
    scoreOut[g * 6 + 0] = (float)(uint32_t)(splitmix64(h ^ 0x3333ULL) >> 48) * (3.0f / 32768.0f) - 3.0f;
    scoreOut[g * 6 + 1] = (float)(uint32_t)(splitmix64(h ^ 0x4444ULL) >> 48) * (1.0f / 1024.0f) - 8.0f;
    scoreOut[g * 6 + 2] = (float)(uint32_t)(splitmix64(h ^ 0x5555ULL) >> 48) * (3.0f / 32768.0f) - 3.0f;
    scoreOut[g * 6 + 3] = 0.0f; scoreOut[g * 6 + 4] = 0.0f; scoreOut[g * 6 + 5] = 0.0f;
  }
  else if(lane == 0) {
    valueOut[g * 3 + 0] = (float)(uint32_t)(splitmix64(h ^ 0x1111ULL) >> 48) * (1.0f / 8192.0f) - 4.0f;
    valueOut[g * 3 + 1] = (float)(uint32_t)(splitmix64(h ^ 0x2222ULL) >> 48) * (1.0f / 8192.0f) - 4.0f;
    valueOut[g * 3 + 2] = -30.0f;
    scoreOut[g * 6 + 0] = (float)(uint32_t)(splitmix64(h ^ 0x3333ULL) >> 48) * (1.0f / 32768.0f) - 1.0f;
    scoreOut[g * 6 + 1] = (float)(uint32_t)(splitmix64(h ^ 0x4444ULL) >> 48) * (1.0f / 16384.0f) - 2.0f;
    scoreOut[g * 6 + 2] = (float)(uint32_t)(splitmix64(h ^ 0x5555ULL) >> 48) * (1.0f / 32768.0f) - 1.0f;
    scoreOut[g * 6 + 3] = 0.0f; scoreOut[g * 6 + 4] = 0.0f; scoreOut[g * 6 + 5] = 0.0f;
    if(d.fakeNN == 2) {   // the variant with raw short-term error channels in [-2,2) (tests/cpp/uncertainty_search_driver.cpp gives the reference Search the same net)
      scoreOut[g * 6 + 4] = (float)(uint32_t)(splitmix64(h ^ 0x6666ULL) >> 48) * (1.0f / 16384.0f) - 2.0f;
      scoreOut[g * 6 + 5] = (float)(uint32_t)(splitmix64(h ^ 0x7777ULL) >> 48) * (1.0f / 16384.0f) - 2.0f;
    }
  }
}

// Apply a move list (x, y, or -1,-1 = pass; colours alternate from the current player) to every game's root.
__global__ void spPlayMovesKernel(const SPDev d, const int8_t* moves, int numMoves, int onlyGame, int endGames) {
  const int g = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if(g >= d.numGames || (onlyGame >= 0 && g != onlyGame)) return;
  RootPos rp;
  rootLoad(d, g, lane, rp);
  for(int m = 0; m < numMoves; m++) {
    const int p = moves[m * 2] < 0 ? -1 : (moves[m * 2 + 1] * 32 + moves[m * 2]);
    bool fin, nores;
    rootPlay(d, g, lane, rp, p, fin, nores);
    if(endGames && (fin || rp.moveNum >= d.maxMoves)) {
      // a move of the list ended the game (match play mirrors the opponent's moves into this loop, kgb_selfplay_play_moves_game): the same
      // game-over handling as when the loop's own move ends it - result kept readable, next game started; further moves go to that game
      recordRootMove(d, g, lane, p < 0 ? d.policySize - 1 : posOf(p, d.X), true, fin, nores, rp.moveNum - 1);
      __syncwarp();
      rootGameOver(d, g, lane, rp, nores);
    }
  }
  rootStore(d, g, lane, rp);
  rootPrevLadders(d, g, lane);
  if(lane == 0) { d.ladPending[g] = 0; d.leafValid[g] = 0; }
  treeReset(d, g, lane);
}

// Desynchronise the games: every game's root is advanced by its own random number (0..maxLen) of uniformly random legal
// non-pass moves (its own generator).  Bench / test support: a steady-state self-play server holds games at all stages, and
// SURVEY.md §8d asks for positions "from random legal play-outs" for the kernel-level measurements.
__global__ void spRandomOpeningsKernel(const SPDev d, int maxLen) {
  const int g = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if(g >= d.numGames) return;
  RootPos rp;
  rootLoad(d, g, lane, rp);
  rp.passes = 0;   // every move counts passes from 0 and the game's end is ignored; no move is a pass, so the count stays 0
  DevRand rand;
  if(lane == 0) rand.s = d.nonSearchRand[g];
  unsigned len = 0;
  if(lane == 0) len = maxLen > 0 ? rand.nextUInt() % (unsigned)(maxLen + 1) : 0;
  len = __shfl_sync(KGB_FULL, len, 0);
  for(unsigned m = 0; m < len; m++) {
    uint32_t l1, l2, l3;
    boardLibertyClasses(rp.bd, l1, l2, l3);
    const uint32_t legal = boardLegalMask(rp.bd, rp.black, d.gMultiSuicide[g] != 0, l1) & ~d.rootBanned[g * 32 + lane];
    const int n = warpCount(legal);
    if(n == 0) break;
    unsigned r = 0;
    if(lane == 0) r = rand.nextUInt() % (unsigned)n;
    r = __shfl_sync(KGB_FULL, r, 0);
    // the r-th legal point in row-major order
    int mine = __popc(legal), incl = mine;
    for(int o = 1; o < 32; o <<= 1) { int t = __shfl_up_sync(KGB_FULL, incl, o); if(lane >= o) incl += t; }
    const int before = incl - mine;
    int p = -1;
    if((int)r >= before && (int)r < incl) {
      uint32_t bits = legal;
      for(int k = (int)r - before; k > 0; k--) bits &= bits - 1;
      p = lane * 32 + (__ffs(bits) - 1);
    }
    const unsigned who = __ballot_sync(KGB_FULL, p >= 0);
    p = __shfl_sync(KGB_FULL, p, __ffs(who) - 1);
    bool fin, nores;
    rootPlay(d, g, lane, rp, p, fin, nores);
  }
  rootStore(d, g, lane, rp);
  rootPrevLadders(d, g, lane);
  if(lane == 0) { d.nonSearchRand[g] = rand.s; d.ladPending[g] = 0; d.leafValid[g] = 0; }
  treeReset(d, g, lane);
}

__global__ void spInitRootsKernel(const SPDev d) {
  const int g = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if(g >= d.numGames) return;
  gameHistReset(d, g, lane);
  rootTableReset(d, g, lane);
}

// ------------------------------------------------------------------------------------------------------------
// Board test kernel: replays move streams (parity tests against the reference Board fixtures)
// ------------------------------------------------------------------------------------------------------------
__global__ void boardReplayKernel(int X, int Y, int numBoards, int numMoves, int multiSuicide, const int8_t* moves /*[b][m][3]: x,y,pla(1=black,2=white)*/,
                                  uint8_t* colors /*[b][m][Y*X]*/, int8_t* ko /*[b][m][2]*/, int16_t* caps /*[b][m][2]*/,
                                  uint8_t* libClass /*[b][m][Y*X] 0..3 (0 = >3 or empty)*/, uint8_t* legalNext /*[b][m][Y*X]*/,
                                  const ZobEntry* zob, unsigned long long sizeH0, unsigned long long sizeH1, unsigned long long* posHash /*[b][m][2]*/,
                                  uint8_t* area /*[b][m][Y*X] Board::calculateArea, all flags on*/) {
  const int bidx = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if(bidx >= numBoards) return;
  WarpBoard bd;
  boardInit(bd, X, Y);
  bd.h0 = sizeH0; bd.h1 = sizeH1;
  for(int m = 0; m < numMoves; m++) {
    const int8_t* mv = moves + ((size_t)bidx * numMoves + m) * 3;
    const bool black = mv[2] == 1;
    const int p = mv[0] < 0 ? -1 : (mv[1] * 32 + mv[0]);
    boardPlay(bd, p, black, zob);
    uint32_t l1, l2, l3;
    boardLibertyClasses(bd, l1, l2, l3);
    uint32_t legal = boardLegalMask(bd, !black, multiSuicide != 0, l1);
    uint32_t aB, aW;
    boardCalculateArea(bd, true, true, true, multiSuicide != 0, aB, aW);
    const size_t o = ((size_t)bidx * numMoves + m) * X * Y;
    if(lane < Y)
      for(int x = 0; x < X; x++) {
        uint32_t bit = 1u << x;
        colors[o + lane * X + x] = (bd.b & bit) ? 1 : (bd.w & bit) ? 2 : 0;
        libClass[o + lane * X + x] = (l1 & bit) ? 1 : (l2 & bit) ? 2 : (l3 & bit) ? 3 : 0;
        legalNext[o + lane * X + x] = (legal & bit) ? 1 : 0;
        area[o + lane * X + x] = (aB & bit) ? 1 : (aW & bit) ? 2 : 0;
      }
    if(lane == 0) {
      size_t q = (size_t)bidx * numMoves + m;
      ko[q * 2] = bd.ko < 0 ? -1 : (int8_t)(bd.ko & 31);
      ko[q * 2 + 1] = bd.ko < 0 ? -1 : (int8_t)(bd.ko >> 5);
      caps[q * 2] = (int16_t)bd.capB; caps[q * 2 + 1] = (int16_t)bd.capW;
      posHash[q * 2] = bd.h0; posHash[q * 2 + 1] = bd.h1;
    }
  }
}

// Test kernel for Board::simpleRepetitionBoundGt: one board, a move stream (x, y, pla 1/2), flag after every move.
__global__ void repBoundKernel(int X, int Y, int numMoves, int bound, const int8_t* moves, uint8_t* out) {
  const int lane = threadIdx.x & 31;
  if(blockIdx.x != 0 || threadIdx.x >= 32) return;
  WarpBoard bd;
  boardInit(bd, X, Y);
  for(int m = 0; m < numMoves; m++) {
    const int p = moves[m * 3] < 0 ? -1 : (moves[m * 3 + 1] * 32 + moves[m * 3]);
    boardPlay(bd, p, moves[m * 3 + 2] == 1);
    const bool r = simpleRepetitionBoundGt(bd, p, bound);
    if(lane == 0) out[m] = r ? 1 : 0;
  }
}

// Rules test kernel: replays games through histMakeMove (parity tests against the reference BoardHistory fixtures).
__global__ void historyReplayKernel(int X, int Y, int koRule, int multiSuicide, int numGames, int maxMoves, const int8_t* moves /*[g][m][2]*/,
                                    const ZobEntry* zob, unsigned long long* lists /*[g][3][maxMoves+2]*/, uint8_t* flags /*[g][m]*/,
                                    uint8_t* legal /*[g][m][Y*X]*/, uint8_t* banned /*[g][m][Y*X]*/) {
  const int g = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if(g >= numGames) return;
  WarpBoard bd;
  boardInit(bd, X, Y);
  const int cap = maxMoves + 2;
  HistLists L;
  L.gKo = nullptr; L.gKoLen = 0; L.gKoStart = 0; L.gPassB = nullptr; L.gPassBLen = 0; L.gPassW = nullptr; L.gPassWLen = 0;
  L.pKo = lists + (size_t)g * 3 * cap; L.pPassB = L.pKo + cap; L.pPassW = L.pKo + 2 * cap;
  L.pKoLen = 0; L.pPassBLen = 0; L.pPassWLen = 0;
  HistState st;
  st.passes = 0; st.finished = false; st.noResult = false; st.everOcc = 0; st.banned = 0;
  // BoardHistory::clear: the history starts with the initial situation
  if(lane == 0) L.pKo[0] = koHashOf(koRule, bd.h0, true);
  L.pKoLen = 1;
  __syncwarp();
  bool black = true;
  for(int m = 0; m < maxMoves; m++) {
    const int8_t* mv = moves + ((size_t)g * maxMoves + m) * 2;
    if(mv[0] == -2) break;
    const int p = mv[0] < 0 ? -1 : (mv[1] * 32 + mv[0]);
    histMakeMove(bd, st, L, p, black, koRule, multiSuicide != 0, zob);
    black = !black;
    uint32_t l1, l2, l3;
    boardLibertyClasses(bd, l1, l2, l3);
    const uint32_t lg = boardLegalMask(bd, black, multiSuicide != 0, l1) & ~st.banned;
    const bool pwe = histPassWouldEndPhase(bd, st, L, black, koRule);
    const size_t o = ((size_t)g * maxMoves + m) * X * Y;
    if(lane < Y)
      for(int x = 0; x < X; x++) { legal[o + lane * X + x] = (lg >> x) & 1; banned[o + lane * X + x] = (st.banned >> x) & 1; }
    if(lane == 0) flags[(size_t)g * maxMoves + m] = (st.finished ? 1 : 0) | (st.noResult ? 2 : 0) | (pwe ? 4 : 0);
  }
}

// Board size and ko / suicide rules per game (GameInitializer::createGameSharedUnsynchronized, program/play.cpp:330-650: bSizes /
// bSizeRelProbs, koRules, multiStoneSuicideLegals drawn per game).  setup[numGames][4] = X, Y, ko rule, multi-stone suicide: taken by each slot's
// NEXT game; with alsoCurrent also by the game in progress, which must not have started (no move played, root not searched) - its history
// restarts under the new rules.
__global__ void spApplySetupKernel(const SPDev d, int* refused) {
  const int g = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if(g >= d.numGames) return;
  const size_t gb = (size_t)g * d.maxNodes;
  if(d.moveNum[g] != 0 || d.nodeVisits[gb] != 0 || d.rootSymCount[g] != 0 || d.ladPending[g] != 0) { if(lane == 0) atomicAdd(refused, 1); return; }
  __syncwarp();
  if(lane == 0) { d.gX[g] = d.nextSetup[g * 4 + 0]; d.gY[g] = d.nextSetup[g * 4 + 1]; d.gKoRule[g] = d.nextSetup[g * 4 + 2]; d.gMultiSuicide[g] = d.nextSetup[g * 4 + 3]; }
  __syncwarp();
  gameHistReset(d, g, lane);
  __syncwarp();
  rootHashesInit(d, g, lane);
}

// Search limits of the roots to come (getSearchLimitsThisMove, program/play.cpp:1093-1223: cheap searches, reduced visits).  visits[numGames][2],
// plain[numGames][2] (may be NULL = all 0): index 0 applies to the root after the slot's next move when the game goes on, index 1 when that
// move ends the game (first root of the slot's next game).  alsoCurrent: index 0 also replaces the limits of the current roots, which
// must not have been searched yet.
__global__ void spApplyLimitsKernel(const SPDev d, int* refused) {
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if(g >= d.numGames) return;
  if(d.nodeVisits[(size_t)g * d.maxNodes] != 0 || d.rootSymCount[g] != 0) { atomicAdd(refused, 1); return; }
  d.visitBudget[g] = d.nextBudget[g * 2]; d.plainRoot[g] = d.nextPlain[g * 2];
}

// Policy-initialised openings (PlaySettings::initGamesWithPolicy / policyInitAreaProp / policyInitAreaTemperature; playutils.cpp:232-266): moves[numGames] =
// how many opening moves each slot's NEXT game draws from the raw policy before its first searched move (the host draws the count: floor of an
// exponential with mean area * policyInitAreaProp).  alsoCurrent: the games in progress take them too; they must not have started.
__global__ void spApplyPolicyInitKernel(const SPDev d, int* refused) {
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if(g >= d.numGames) return;
  if(d.moveNum[g] != 0 || d.nodeVisits[(size_t)g * d.maxNodes] != 0 || d.rootSymCount[g] != 0) { atomicAdd(refused, 1); return; }
  d.initMovesLeft[g] = d.nextInitMoves[g]; d.initMoveCount[g] = 0;
  if(d.initMovesLeft[g] > 0) { d.visitBudget[g] = 1; d.plainRoot[g] = 1; }
}

}  // namespace kgb

// ------------------------------------------------------------------------------------------------------------
// Host side
// ------------------------------------------------------------------------------------------------------------
using namespace kgb;

namespace {

// Device scratch of one call, freed on every way out of it
template <class T>
struct Scratch {
  T* p = nullptr;
  explicit Scratch(size_t count) { CK(cudaMalloc(&p, count * sizeof(T))); }
  ~Scratch() { cudaFree(p); }
  Scratch(const Scratch&) = delete;
  Scratch& operator=(const Scratch&) = delete;
};

// The device twin of the reference's Rand seeded from `seed`
DevRandState devRandState(const std::string& seed) {
  RefRand rr(seed);
  DevRandState st;
  memset(&st, 0, sizeof(st));
  uint64_t a[16], idx, pcg;
  rr.exportState(a, idx, pcg);
  for(int i = 0; i < 16; i++) st.a[i] = a[i];
  st.aIdx = idx; st.pcg = pcg;
  return st;
}

}  // namespace

// One device loop on an evaluator handle.  Every transfer and launch of the loop goes on the handle's stream, which orders it
// against the waves (the stream is non-blocking: the legacy default stream would not).
struct kgb_selfplay {
  kgb_handle* h = nullptr;
  SPDev d;
  std::vector<void*> allocs;
  int* refused = nullptr;      // games an apply kernel had to leave unchanged
  cudaGraphExec_t stepGraph = nullptr;

  ~kgb_selfplay() {
    if(stepGraph) cudaGraphExecDestroy(stepGraph);
    for(void* p : allocs) cudaFree(p);
  }
  template <class T> T* alloc(size_t count) {
    void* p = nullptr;
    CK(cudaMalloc(&p, count * sizeof(T)));
    allocs.push_back(p);
    fill((T*)p, 0, count);
    return (T*)p;
  }
  // counts are in elements of the device array
  template <class T> void upload(T* dst, const void* src, size_t count) {
    CK(cudaMemcpyAsync(dst, src, count * sizeof(T), cudaMemcpyHostToDevice, h->stream));
  }
  template <class T> void download(void* dst, const T* src, size_t count) {
    CK(cudaMemcpyAsync(dst, src, count * sizeof(T), cudaMemcpyDeviceToHost, h->stream));
    sync();
  }
  template <class T> void fill(T* dst, int byte, size_t count) { CK(cudaMemsetAsync(dst, byte, count * sizeof(T), h->stream)); }
  void sync() { CK(cudaStreamSynchronize(h->stream)); }
  // What every entry point does first: make the loop's device current and, with `drain`, wait for the waves queued on its stream
  void enter(bool drain = true) {
    CK(cudaSetDevice(h->device));
    if(drain) sync();
  }
  void checkGame(int g) const {
    if(g < 0 || g >= d.numGames) throw std::invalid_argument("selfplay: game index out of range");
  }

  void launchSelect() {
    spSelectKernel<<<d.numGames, SP_LADDER_WARPS * 32, 0, h->stream>>>(d);
    CK(cudaGetLastError());
  }
  void launchBackup() {
    int threads = 128, warpsPerBlock = threads / 32;
    spBackupKernel<<<(d.numGames + warpsPerBlock - 1) / warpsPerBlock, threads, 0, h->stream>>>(d);
    CK(cudaGetLastError());
  }
  // One wave: select a leaf per game, evaluate the leaves (debug_fake_nn: a stand-in for the net), back up
  void stepLaunches() {
    launchSelect();
    if(d.fakeNN) {
      int threads = 128, warpsPerBlock = threads / 32;
      spFakeNNKernel<<<(d.numGames + warpsPerBlock - 1) / warpsPerBlock, threads, 0, h->stream>>>(d, h->dPolicy, h->dValue, h->dScore, h->dOwnership);
      CK(cudaGetLastError());
    }
    else for(auto& op : h->ops) op(d.numGames, h->stream);
    launchBackup();
  }

  // The values of each slot's NEXT game have been uploaded; with alsoCurrent `kernel` also gives them to the games in progress.
  // Games that have already started are left unchanged and reported as "selfplay: <count><refusal>".  threadsPerGame: 32 for a
  // kernel that runs a warp per game, 1 for a thread per game.
  void applyNext(bool alsoCurrent, void (*kernel)(const SPDev, int*), int threadsPerGame, const char* refusal) {
    if(alsoCurrent) {
      fill(refused, 0, 1);
      kernel<<<(d.numGames * threadsPerGame + 127) / 128, 128, 0, h->stream>>>(d, refused);
      CK(cudaGetLastError());
      int n = 0;
      download(&n, refused, 1);
      if(n != 0) throw std::invalid_argument("selfplay: " + std::to_string(n) + refusal);
    }
    sync();
  }

  void playMoves(const int8_t* movesXY, int numMoves, int onlyGame) {
    if(onlyGame >= d.numGames) throw std::invalid_argument("selfplay: game index out of range");
    {   // every move must lie on the board of every game it is played on (a game's board can be smaller than the evaluator's frame)
      std::vector<int> gx((size_t)d.numGames), gy((size_t)d.numGames);
      download(gx.data(), d.gX, gx.size());
      download(gy.data(), d.gY, gy.size());
      for(int g = 0; g < d.numGames; g++) {
        if(onlyGame >= 0 && g != onlyGame) continue;
        for(int m = 0; m < numMoves; m++)
          if(movesXY[2 * m] >= 0 && (movesXY[2 * m] >= gx[g] || movesXY[2 * m + 1] < 0 || movesXY[2 * m + 1] >= gy[g]))
            throw std::invalid_argument("selfplay: move " + std::to_string(m) + " is off the board of game " + std::to_string(g));
      }
    }
    Scratch<int8_t> dm((size_t)numMoves * 2);
    upload(dm.p, movesXY, (size_t)numMoves * 2);
    int threads = 128, warpsPerBlock = threads / 32;
    spPlayMovesKernel<<<(d.numGames + warpsPerBlock - 1) / warpsPerBlock, threads, 0, h->stream>>>(d, dm.p, numMoves, onlyGame, onlyGame >= 0 ? 1 : 0);
    CK(cudaGetLastError());
    sync();
  }
};

static void initLoop(kgb_selfplay* sp, const kgb_selfplay_config& c) {
  const kgb_handle& hd = *sp->h;
  const int X = hd.L.X, Y = hd.L.Y;
  if(X > 19 || Y > 19 || X < 2 || Y < 2) throw std::invalid_argument("selfplay: board sizes 2..19 only");
  if(c.num_games < 1 || c.max_visits < 2) throw std::invalid_argument("selfplay: num_games >= 1 and max_visits >= 2 required");
  SPDev& d = sp->d;
  memset(&d, 0, sizeof(d));
  d.X = X; d.Y = Y; d.XY = X * Y; d.policySize = X * Y + 1;
  if(d.policySize > 12 * 32) throw std::invalid_argument("selfplay: policy size too large");
  d.numGames = c.num_games; d.maxVisits = c.max_visits; d.maxNodes = c.max_visits + 2;
  d.maxDepth = std::min(c.max_visits + 2, 512);
  d.maxMoves = c.max_moves > 0 ? c.max_moves : 2 * X * Y;
  d.earlyMoves = c.early_temperature_moves;
  {
    std::vector<float> k((size_t)c.num_games, (float)c.komi);
    d.komiG = sp->alloc<float>(c.num_games); d.nextKomi = sp->alloc<float>(c.num_games); d.lastKomi = sp->alloc<float>(c.num_games);
    for(float* dst : {d.komiG, d.nextKomi, d.lastKomi}) sp->upload(dst, k.data(), k.size());
  }
  {   // every game starts with the frame as its board and the configuration's rules (kgb_selfplay_set_game_setup changes that per game)
    if(c.ko_rule < 0 || c.ko_rule > 3) throw std::invalid_argument("selfplay: ko_rule must be 0 (simple), 1 (positional), 2 (situational) or 3 (spight)");
    const int G = c.num_games;
    d.gX = sp->alloc<int>(G); d.gY = sp->alloc<int>(G); d.gKoRule = sp->alloc<int>(G); d.gMultiSuicide = sp->alloc<int>(G);
    d.nextSetup = sp->alloc<int>((size_t)G * 4); d.lastSetup = sp->alloc<int>((size_t)G * 4);
    const int vals[4] = {X, Y, c.ko_rule, c.multi_stone_suicide_legal ? 1 : 0};
    int* const dst[4] = {d.gX, d.gY, d.gKoRule, d.gMultiSuicide};
    std::vector<int> one((size_t)G), four((size_t)G * 4);
    for(int k = 0; k < 4; k++) {
      std::fill(one.begin(), one.end(), vals[k]);
      sp->upload(dst[k], one.data(), one.size());
      for(int g = 0; g < G; g++) four[(size_t)g * 4 + k] = vals[k];
    }
    sp->upload(d.nextSetup, four.data(), four.size());
    sp->upload(d.lastSetup, four.data(), four.size());
    // every root gets the full budget and its root parameters unless the host says otherwise (kgb_selfplay_set_next_search_limits)
    d.visitBudget = sp->alloc<int>(G); d.nextBudget = sp->alloc<int>((size_t)G * 2);
    d.plainRoot = sp->alloc<uint8_t>(G); d.nextPlain = sp->alloc<uint8_t>((size_t)G * 2);
    d.rootRawEntropy = sp->alloc<double>(G);
    d.initMovesLeft = sp->alloc<int>(G); d.nextInitMoves = sp->alloc<int>(G); d.initMoveCount = sp->alloc<int>(G);
    d.initMoves = sp->alloc<int16_t>((size_t)G * SP_MAX_INIT_MOVES);
    d.policyInitTemperature = sp->alloc<double>(1);
    { const double one = 1.0; sp->upload(d.policyInitTemperature, &one, 1); }
    std::vector<int> full((size_t)G * 2, c.max_visits);
    sp->upload(d.visitBudget, full.data(), G);
    sp->upload(d.nextBudget, full.data(), (size_t)G * 2);
  }
  d.cpuctExploration = c.cpuct_exploration; d.cpuctExplorationLog = c.cpuct_exploration_log; d.cpuctExplorationBase = c.cpuct_exploration_base;
  d.fpuReductionMax = c.fpu_reduction_max; d.rootFpuReductionMax = c.root_fpu_reduction_max;
  d.cpuctUtilityStdevPrior = c.cpuct_utility_stdev_prior; d.cpuctUtilityStdevPriorWeight = c.cpuct_utility_stdev_prior_weight;
  d.cpuctUtilityStdevScale = c.cpuct_utility_stdev_scale;
  if(d.cpuctUtilityStdevScale != 0.0 && !(d.cpuctUtilityStdevPrior > 0.0)) throw std::invalid_argument("selfplay: cpuct_utility_stdev_prior must be > 0");
  d.fpuLossProp = c.fpu_loss_prop; d.rootFpuLossProp = c.root_fpu_loss_prop; d.fpuParentWeight = c.fpu_parent_weight;
  d.fpuParentWeightByVisitedPolicy = c.fpu_parent_weight_by_visited_policy;
  d.fpuParentWeightByVisitedPolicyPow = c.fpu_parent_weight_by_visited_policy_pow;
  d.subtreeValueBiasFactor = c.subtree_value_bias_factor; d.subtreeValueBiasWeightExponent = c.subtree_value_bias_weight_exponent;
  d.valueWeightExponent = c.value_weight_exponent; d.rootDesiredPerChildVisitsCoeff = c.root_desired_per_child_visits_coeff;
  if(c.max_visits + 2 > 65535) throw std::invalid_argument("selfplay: max_visits above 65533 not supported");
  d.winLossUtilityFactor = c.win_loss_utility_factor; d.noResultUtilityForWhite = c.no_result_utility_for_white;
  d.staticScoreUtilityFactor = c.static_score_utility_factor; d.dynamicScoreUtilityFactor = c.dynamic_score_utility_factor;
  d.dynamicScoreCenterZeroWeight = c.dynamic_score_center_zero_weight; d.dynamicScoreCenterScale = c.dynamic_score_center_scale;
  d.drawEquivalentWinsForWhite = c.draw_equivalent_wins_for_white;
  if(d.dynamicScoreUtilityFactor != 0.0 && !(d.dynamicScoreCenterScale > 0.0)) throw std::invalid_argument("selfplay: dynamic_score_center_scale must be > 0");
  d.scoreMeanMultiplier = hd.model->scoreMeanMultiplier; d.scoreStdevMultiplier = hd.model->scoreStdevMultiplier; d.leadMultiplier = hd.model->leadMultiplier;
  d.seed = c.seed;
  const size_t G = d.numGames, N = d.maxNodes, PS = d.policySize;
  d.rootB = sp->alloc<uint32_t>(G * 32); d.rootW = sp->alloc<uint32_t>(G * 32);
  d.rootKo = sp->alloc<int>(G); d.rootBlackToMove = sp->alloc<int>(G); d.rootCapB = sp->alloc<int>(G); d.rootCapW = sp->alloc<int>(G);
  d.moveNum = sp->alloc<int>(G); d.consecPasses = sp->alloc<int>(G); d.hist = sp->alloc<int>(G * 5);
  d.gameCounter = sp->alloc<uint64_t>(G);
  d.releaseFlag = sp->alloc<uint8_t>(G); d.lastMove = sp->alloc<int>(G * 4); d.lastScore = sp->alloc<float>(G); d.finalBoard = sp->alloc<uint32_t>(G * 128);
  d.prevB = sp->alloc<uint32_t>(2 * G * 32); d.prevW = sp->alloc<uint32_t>(2 * G * 32); d.prevKo = sp->alloc<int>(2 * G);
  d.enableLadders = c.disable_ladder_features ? 0 : 1;
  d.ladderScratch = sp->alloc<uint32_t>(G * SP_LADDER_WARPS * ladderScratchWordsPerWarp());
  d.prevLad = sp->alloc<uint32_t>(2 * G * 32); d.nodeLad = sp->alloc<uint32_t>(G * (size_t)(c.max_visits + 2) * 32);
  d.leafNumHist = sp->alloc<int>(G);
  d.leafB = sp->alloc<uint32_t>(G * 32); d.leafW = sp->alloc<uint32_t>(G * 32); d.leafCand = sp->alloc<uint32_t>(G * 32);
  d.leafKo = sp->alloc<int>(G); d.ladPending = sp->alloc<int>(G); d.leafValid = sp->alloc<int>(G);
  d.ladderNodesPerWave = c.ladder_nodes_per_wave > 0 ? c.ladder_nodes_per_wave : 0;
  d.fixedSymmetryPlusOne = (c.debug_fixed_symmetry_plus_one >= 1 && c.debug_fixed_symmetry_plus_one <= 8) ? c.debug_fixed_symmetry_plus_one : 0;
  d.maxPlayoutsPerWave = c.max_playouts_per_wave > 0 ? c.max_playouts_per_wave : SP_MAX_PLAYOUTS_PER_WAVE;
  { std::vector<int> kos2(2 * G, -1); sp->upload(d.prevKo, kos2.data(), 2 * G); }
  d.nodeCount = sp->alloc<int>(G); d.nodeVisits = sp->alloc<int>(G * N); 
  d.nodeWeightSum = sp->alloc<double>(G * N); d.nodeWeightSqSum = sp->alloc<double>(G * N); d.nodeUtilAvg = sp->alloc<double>(G * N);
  d.nodeUtilSqAvg = sp->alloc<double>(G * N); d.nodeNNUtil = sp->alloc<double>(G * N); d.nodeNumChildren = sp->alloc<int>(G * N);
  d.childOrder = sp->alloc<uint16_t>(G * N * PS);
  d.nodeMoments = sp->alloc<double>(G * N * 5); d.nodeNNMoments = sp->alloc<double>(G * N * 5); d.leafMoments = sp->alloc<double>(G * 5);
  d.histCap = (d.maxMoves > 1024 ? d.maxMoves : 1024) + 16;   // also holds openings given by kgb_selfplay_play_moves (up to 1024 moves)
  d.pathCap = d.maxDepth + 8;
  d.gKo = sp->alloc<unsigned long long>(G * d.histCap); d.gPassB = sp->alloc<unsigned long long>(G * d.histCap); d.gPassW = sp->alloc<unsigned long long>(G * d.histCap);
  d.gKoLen = sp->alloc<int>(G); d.gPassBLen = sp->alloc<int>(G); d.gPassWLen = sp->alloc<int>(G);
  d.gEverOcc = sp->alloc<uint32_t>(G * 32); d.rootBanned = sp->alloc<uint32_t>(G * 32);
  d.pKo = sp->alloc<unsigned long long>(G * d.pathCap); d.pPassB = sp->alloc<unsigned long long>(G * d.pathCap); d.pPassW = sp->alloc<unsigned long long>(G * d.pathCap);
  d.holdAtMaxVisits = c.debug_hold_at_max_visits ? 1 : 0;
  if(c.debug_fake_nn < 0 || c.debug_fake_nn > 4) throw std::invalid_argument("selfplay: debug_fake_nn must be 0 to 4");
  d.fakeNN = c.debug_fake_nn;
  d.fakeTable = d.fakeNN == 3 ? sp->alloc<float>(G * (PS + 9 + (size_t)X * Y)) : nullptr;
  d.rootNumSymmetries = c.root_num_symmetries_to_sample > 1 ? (c.root_num_symmetries_to_sample > 8 ? 8 : c.root_num_symmetries_to_sample) : 1;
  d.rootSymCount = sp->alloc<int>(G); d.rootSymOrder = sp->alloc<int>(G * 8); d.rootSymAcc = sp->alloc<float>(G * 8);
  d.rootNoiseEnabled = c.root_noise_enabled ? 1 : 0;
  d.rootDirichletNoiseTotalConcentration = c.root_dirichlet_noise_total_concentration; d.rootDirichletNoiseWeight = c.root_dirichlet_noise_weight;
  d.rootPolicyTemperature = c.root_policy_temperature == 0.0 ? 1.0 : c.root_policy_temperature;                 // 0 = unset
  d.rootPolicyTemperatureEarly = c.root_policy_temperature_early == 0.0 ? 1.0 : c.root_policy_temperature_early;
  d.chosenMoveTemperatureHalflife = c.chosen_move_temperature_halflife == 0.0 ? 19.0 : c.chosen_move_temperature_halflife;
  d.noiseScratch = sp->alloc<double>(G * PS);
  d.selScratch = sp->alloc<double>(G * 3 * PS);
  d.usePlaySelection = c.use_play_selection ? 1 : 0; d.useLcbForSelection = c.use_lcb_for_selection ? 1 : 0; d.useNonBuggyLcb = c.use_non_buggy_lcb ? 1 : 0;
  d.lcbStdevs = c.lcb_stdevs; d.minVisitPropForLCB = c.min_visit_prop_for_lcb;
  d.chosenMoveTemperature = c.chosen_move_temperature; d.chosenMoveTemperatureEarly = c.chosen_move_temperature_early;
  d.chosenMoveTemperatureOnlyBelowProb = c.chosen_move_temperature_only_below_prob == 0.0 ? 1.0 : c.chosen_move_temperature_only_below_prob;
  d.chosenMoveSubtract = c.chosen_move_subtract; d.chosenMovePrune = c.chosen_move_prune;
  {
    // one generator per game, seeded like the reference's Rand from a string (the reference reseeds its search thread's
    // generator for every search from strings the device cannot hash; here the stream simply continues from move to move)
    std::vector<DevRandState> st(G);
    const std::string prefix = "kgb200$seed" + std::to_string(c.seed) + "$game";
    for(size_t g2 = 0; g2 < G; g2++) st[g2] = devRandState(prefix + std::to_string(g2) + "$searchThread");
    d.searchRand = sp->alloc<DevRandState>(G);
    sp->upload(d.searchRand, st.data(), G);
    for(size_t g2 = 0; g2 < G; g2++) st[g2] = devRandState(prefix + std::to_string(g2) + "$nonSearchRand");
    d.nonSearchRand = sp->alloc<DevRandState>(G);
    sp->upload(d.nonSearchRand, st.data(), G);
  }
  d.cacheSize = 0;
  if(c.nn_cache_size_power_of_two > 0) {
    if(c.nn_cache_size_power_of_two > 26) throw std::invalid_argument("selfplay: nn_cache_size_power_of_two above 26 not supported");
    d.cacheSize = 1 << c.nn_cache_size_power_of_two;
    const size_t S = (size_t)d.cacheSize;
    d.cacheKey0 = sp->alloc<unsigned long long>(S); d.cacheKey1 = sp->alloc<unsigned long long>(S); d.cacheLock = sp->alloc<int>(S);
    d.cachePolicy = sp->alloc<float>(S * PS); d.cacheVals = sp->alloc<float>(S * 8); d.cacheLad = sp->alloc<uint32_t>(S * 32);
  }
  d.leafKey = sp->alloc<unsigned long long>(G * 2);
  d.useGraphSearch = c.use_graph_search ? 1 : 0; d.graphSearchRepBound = c.graph_search_rep_bound;
  d.nodeTableSize = 64;
  while(d.nodeTableSize < 2 * (int)N) d.nodeTableSize *= 2;
  d.nodeTableKey0 = sp->alloc<unsigned long long>(G * d.nodeTableSize); d.nodeTableKey1 = sp->alloc<unsigned long long>(G * d.nodeTableSize);
  d.nodeTableNode = sp->alloc<int>(G * d.nodeTableSize);
  d.nodePosH0 = sp->alloc<unsigned long long>(G * N); d.nodePosH1 = sp->alloc<unsigned long long>(G * N);
  d.nodeGH0 = sp->alloc<unsigned long long>(G * N); d.nodeGH1 = sp->alloc<unsigned long long>(G * N);
  d.rootPosH = sp->alloc<unsigned long long>(G * 2);
  {
    const ZobristTables zt = makeZobristTables(X, Y);
    static_assert(sizeof(ZobEntry) == sizeof(Hash128), "layout");
    ZobEntry* dz = sp->alloc<ZobEntry>(zt.board.size());
    sp->upload(dz, zt.board.data(), zt.board.size());
    d.zob = dz;
  }
  d.biasTableSize = 64;
  while(d.biasTableSize < 2 * (int)N) d.biasTableSize *= 2;
  d.biasKey = sp->alloc<unsigned long long>(G * d.biasTableSize); d.biasDeltaSum = sp->alloc<double>(G * d.biasTableSize);
  d.biasWeightSum = sp->alloc<double>(G * d.biasTableSize);
  d.nodeBiasEntry = sp->alloc<int>(G * N); d.nodeLastBiasDelta = sp->alloc<double>(G * N); d.nodeLastBiasWeight = sp->alloc<double>(G * N);
  d.nodeTerminal = sp->alloc<int8_t>(G * N);
  d.policy = sp->alloc<float>(G * N * PS); d.childNode = sp->alloc<int>(G * N * PS); d.childVisits = sp->alloc<int>(G * N * PS);
  d.pathLen = sp->alloc<int>(G); d.pathNode = sp->alloc<int>(G * d.maxDepth); d.pathMove = sp->alloc<int>(G * d.maxDepth);
  d.leafNode = sp->alloc<int>(G); d.leafTerminal = sp->alloc<int>(G); d.leafBlackToMove = sp->alloc<int>(G);
  d.leafLegal = sp->alloc<uint32_t>(G * 32);
  unsigned long long* stats = sp->alloc<unsigned long long>(16);
  d.totalVisits = stats; d.totalMoves = stats + 1; d.gamesFinished = stats + 2; d.blackWins = stats + 3; d.nodesAllocated = stats + 4;
  d.rootEndingBonusPoints = c.root_ending_bonus_points; d.rootPruneUselessMoves = c.root_prune_useless_moves != 0 ? 1 : 0;
  d.nnOwnership = hd.dOwnership;
  d.rootOwnAcc = sp->alloc<float>(G * (size_t)X * Y); d.rootEndBonus = sp->alloc<double>(G * PS); d.rootAllowed = sp->alloc<uint32_t>(G * 32);
  d.passStreak = sp->alloc<int>(G * 2);
  sp->fill(d.rootAllowed, 0xff, G * 32);
  d.dbgCycles = sp->alloc<long long>(G * 8);
  d.rootRow = sp->alloc<float>(G * ((size_t)X * Y * 22 + 19));
  d.sumDepth = stats + 5; d.ladderCounters = stats + 6; d.stalledWaves = stats + 8; d.instantPlayouts = stats + 9; d.cacheHits = stats + 10; d.cacheStores = stats + 11;
  d.nnSpatial = hd.dSpatial; d.nnGlobal = hd.dGlobal; d.nnOptimism = hd.dOptimism; d.nnSymmetry = hd.dSymmetry;
  d.nnPolicy = hd.dPolicy; d.nnValue = hd.dValue; d.nnScore = hd.dScore;
  {
    const std::vector<double> table = makeExpectedSVTable();
    double* dt = sp->alloc<double>(table.size());
    sp->upload(dt, table.data(), table.size());
    d.svTable = dt;
    const std::vector<double> cdf = makeValueWeightCdfTable();
    double* dc = sp->alloc<double>(cdf.size());
    sp->upload(dc, cdf.data(), cdf.size());
    d.vwCdfTable = dc;
  }
  d.recentScoreCenter = sp->alloc<double>(G); d.leafTerminalScore = sp->alloc<float>(G);
  d.modelVersion = hd.model->version;
  d.shorttermValueErrorMultiplier = hd.model->shorttermValueErrorMultiplier; d.shorttermScoreErrorMultiplier = hd.model->shorttermScoreErrorMultiplier;
  d.useUncertainty = (c.use_uncertainty && d.modelVersion >= 9) ? 1 : 0;   // NNEvaluator::supportsShorttermError (nneval.cpp:299-301)
  d.uncertaintyCoeff = c.uncertainty_coeff; d.uncertaintyExponent = c.uncertainty_exponent; d.uncertaintyMaxWeight = c.uncertainty_max_weight;
  if(c.use_uncertainty && !(c.uncertainty_coeff > 0.0 && c.uncertainty_max_weight > 0.0))
    throw std::invalid_argument("selfplay: use_uncertainty needs uncertainty_coeff > 0 and uncertainty_max_weight > 0");
  d.nodeNNWeight = d.useUncertainty ? sp->alloc<double>(G * N) : nullptr;
  d.useNoisePruning = c.use_noise_pruning ? 1 : 0;
  d.noisePruneUtilityScale = c.noise_prune_utility_scale; d.noisePruningCap = c.noise_pruning_cap;
  if(d.useNoisePruning && !(c.noise_prune_utility_scale > 0.0)) throw std::invalid_argument("selfplay: use_noise_pruning needs noise_prune_utility_scale > 0");
  sp->refused = sp->alloc<int>(1);
  // initial state: empty boards, black to move, history empty, one unevaluated root node per game
  std::vector<int> ones(G, 1), minus(G * 5, -1), kos(G, -1);
  sp->upload(d.rootBlackToMove, ones.data(), G);
  sp->upload(d.nodeCount, ones.data(), G);
  sp->upload(d.hist, minus.data(), G * 5);
  sp->upload(d.rootKo, kos.data(), G);
  sp->fill(d.childNode, 0xff, G * N * PS);
  spInitRootsKernel<<<(unsigned)((G * 32 + 127) / 128), 128, 0, hd.stream>>>(d);
  CK(cudaGetLastError());
  sp->sync();
}

// ------------------------------------------------------------------------------------------------------------
// C ABI of the loop
// ------------------------------------------------------------------------------------------------------------
extern "C" {

KGB_API int kgb_selfplay_create(kgb_handle* handle, const kgb_selfplay_config* config, kgb_selfplay** out) {
  return guarded([&] {
    if(!handle || !config || !out) throw std::invalid_argument("kgb_selfplay_create: NULL argument");
    if(config->num_games > handle->maxBatch) throw std::invalid_argument("kgb_selfplay_create: num_games exceeds the handle's max_batch_size");
    if(!handle->nhwc) throw std::invalid_argument("kgb_selfplay_create: the handle must be created with inputs_nhwc = 1");
    if(handle->model->numInputChannels != 22 || handle->model->numInputGlobalChannels != 19)
      throw std::invalid_argument("kgb_selfplay_create: the device loop writes V7 features (22 spatial, 19 global)");
    if(handle->model->numInputMetaChannels > 0)
      throw std::invalid_argument("kgb_selfplay_create: SGF-metadata nets need a metadata row per evaluation; the self-play loop has none");
    CK(cudaSetDevice(handle->device));
    std::unique_ptr<kgb_selfplay> sp(new kgb_selfplay());
    sp->h = handle;
    initLoop(sp.get(), *config);
    *out = sp.release();
  });
}

KGB_API void kgb_selfplay_free(kgb_selfplay* sp) { delete sp; }

KGB_API int kgb_selfplay_run(kgb_selfplay* sp, int steps) {
  return guarded([&] {
    if(!sp || steps < 0) throw std::invalid_argument("kgb_selfplay_run: bad argument");
    sp->enter(false);
    if(!sp->stepGraph) sp->stepGraph = captureGraph(sp->h->stream, [&] { sp->stepLaunches(); });
    for(int i = 0; i < steps; i++) CK(cudaGraphLaunch(sp->stepGraph, sp->h->stream));
  });
}

KGB_API int kgb_selfplay_set_search_rand(kgb_selfplay* sp, const char* seed_string) {
  return guarded([&] {
    if(!sp || !seed_string) throw std::invalid_argument("kgb_selfplay_set_search_rand: NULL argument");
    sp->enter();
    const std::vector<DevRandState> all(sp->d.numGames, devRandState(seed_string));
    sp->upload(sp->d.searchRand, all.data(), all.size());
    sp->sync();
  });
}

KGB_API int kgb_selfplay_random_openings(kgb_selfplay* sp, int max_moves) {
  return guarded([&] {
    if(!sp || max_moves < 0) throw std::invalid_argument("kgb_selfplay_random_openings: bad argument");
    sp->enter(false);
    spRandomOpeningsKernel<<<(sp->d.numGames * 32 + 127) / 128, 128, 0, sp->h->stream>>>(sp->d, max_moves);
    CK(cudaGetLastError());
    sp->sync();
  });
}

KGB_API int kgb_selfplay_get_stats(kgb_selfplay* sp, kgb_selfplay_stats* out) {
  return guarded([&] {
    if(!sp || !out) throw std::invalid_argument("kgb_selfplay_get_stats: NULL argument");
    sp->enter();
    unsigned long long h[16];
    sp->download(h, sp->d.totalVisits, 16);
    out->total_visits = h[0]; out->total_moves = h[1]; out->games_finished = h[2]; out->black_wins = h[3];
    out->nodes_allocated = h[4]; out->sum_leaf_depth = h[5]; out->ladder_searches = h[6]; out->ladder_nodes = h[7];
    out->stalled_waves = h[8]; out->instant_playouts = h[9]; out->nn_cache_hits = h[10]; out->nn_cache_stores = h[11];
  });
}

KGB_API int kgb_selfplay_get_game(kgb_selfplay* sp, int game, uint8_t* colors, int32_t* info) {
  return guarded([&] {
    if(!sp || !colors || !info) throw std::invalid_argument("kgb_selfplay_get_game: NULL argument");
    sp->enter();
    const SPDev& d = sp->d;
    const int g = game;
    sp->checkGame(g);
    uint32_t b[32], w[32];
    sp->download(b, d.rootB + (size_t)g * 32, 32);
    sp->download(w, d.rootW + (size_t)g * 32, 32);
    for(int y = 0; y < d.Y; y++)
      for(int x = 0; x < d.X; x++) colors[y * d.X + x] = (b[y] >> x) & 1 ? 1 : (w[y] >> x) & 1 ? 2 : 0;
    sp->download(&info[0], d.moveNum + g, 1);
    sp->download(&info[1], d.rootBlackToMove + g, 1);
    sp->download(&info[2], d.rootKo + g, 1);
    sp->download(&info[3], d.rootCapB + g, 1);
    sp->download(&info[4], d.rootCapW + g, 1);
    sp->download(&info[5], d.nodeVisits + (size_t)g * d.maxNodes, 1);
  });
}

KGB_API int kgb_selfplay_get_root_children(kgb_selfplay* sp, int game, int32_t* visits, float* policy, double* util_sum) {
  return guarded([&] {
    if(!sp || !visits || !policy || !util_sum) throw std::invalid_argument("kgb_selfplay_get_root_children: NULL argument");
    sp->enter();
    const SPDev& d = sp->d;
    sp->checkGame(game);
    const size_t nb = (size_t)game * d.maxNodes * d.policySize;
    sp->download(visits, d.childVisits + nb, d.policySize);
    sp->download(policy, d.policy + nb, d.policySize);
    std::vector<int> child(d.policySize);
    std::vector<double> avg(d.maxNodes);
    sp->download(child.data(), d.childNode + nb, d.policySize);
    sp->download(avg.data(), d.nodeUtilAvg + (size_t)game * d.maxNodes, d.maxNodes);
    for(int i = 0; i < d.policySize; i++) util_sum[i] = child[i] >= 0 ? avg[child[i]] : 0.0;
  });
}

KGB_API int kgb_selfplay_get_root_weights(kgb_selfplay* sp, int game, double* child_weights, double* root_weights) {
  return guarded([&] {
    if(!sp || !child_weights || !root_weights) throw std::invalid_argument("kgb_selfplay_get_root_weights: NULL argument");
    sp->enter();
    const SPDev& d = sp->d;
    sp->checkGame(game);
    std::vector<int> child(d.policySize);
    std::vector<double> ws(d.maxNodes), wsq(d.maxNodes);
    sp->download(child.data(), d.childNode + (size_t)game * d.maxNodes * d.policySize, d.policySize);
    sp->download(ws.data(), d.nodeWeightSum + (size_t)game * d.maxNodes, d.maxNodes);
    sp->download(wsq.data(), d.nodeWeightSqSum + (size_t)game * d.maxNodes, d.maxNodes);
    for(int i = 0; i < d.policySize; i++) {
      child_weights[i * 2] = child[i] >= 0 ? ws[child[i]] : 0.0;
      child_weights[i * 2 + 1] = child[i] >= 0 ? wsq[child[i]] : 0.0;
    }
    root_weights[0] = ws[0]; root_weights[1] = wsq[0];
  });
}

KGB_API int kgb_selfplay_get_root_utility(kgb_selfplay* sp, int game, double* utility) {
  return guarded([&] {
    if(!sp || !utility) throw std::invalid_argument("kgb_selfplay_get_root_utility: NULL argument");
    sp->enter();
    const SPDev& d = sp->d;
    sp->checkGame(game);
    sp->download(utility, d.nodeNNUtil + (size_t)game * d.maxNodes, 1);
    sp->download(utility + 1, d.nodeUtilAvg + (size_t)game * d.maxNodes, 1);
  });
}

KGB_API int kgb_selfplay_debug_set_raw_outputs(kgb_selfplay* sp, int game, const float* policy, const float* value, const float* score,
                                               const float* ownership) {
  return guarded([&] {
    if(!sp || !policy || !value || !score || !ownership) throw std::invalid_argument("kgb_selfplay_debug_set_raw_outputs: NULL argument");
    sp->enter();
    const SPDev& d = sp->d;
    sp->checkGame(game);
    if(d.fakeNN != 3) throw std::invalid_argument("kgb_selfplay_debug_set_raw_outputs: the loop was not created with debug_fake_nn = 3");
    const size_t stride = (size_t)d.policySize + 9 + d.XY;
    float* t = d.fakeTable + (size_t)game * stride;
    sp->upload(t, policy, d.policySize);
    sp->upload(t + d.policySize, value, 3);
    sp->upload(t + d.policySize + 3, score, 6);
    sp->upload(t + d.policySize + 9, ownership, d.XY);
    sp->sync();
  });
}

KGB_API int kgb_test_uncertainty_weight(int n, const int32_t* model_version, const double* raw, const double* params, double* out) {
  return guarded([&] {
    if(n < 0 || !model_version || !raw || !params || !out) throw std::invalid_argument("kgb_test_uncertainty_weight: bad argument");
    for(int i = 0; i < n; i++) {
      const double* r = raw + (size_t)i * 2;
      const double* p = params + (size_t)i * 12;
      float wl, se;
      shorttermErrors(model_version[i], p[0], p[1], r[0], r[1], wl, se);
      out[i * 3] = wl; out[i * 3 + 1] = se;
      out[i * 3 + 2] = uncertaintyWeight(p[2], p[3], p[4], p[5], p[6], p[7], p[8], p[9], p[10], (float)p[11], wl, se);
    }
  });
}

KGB_API int kgb_selfplay_get_root_value_stats(kgb_selfplay* sp, int game, double* child_stats, double* root_stats) {
  return guarded([&] {
    if(!sp || !child_stats || !root_stats) throw std::invalid_argument("kgb_selfplay_get_root_value_stats: NULL argument");
    sp->enter();
    const SPDev& d = sp->d;
    sp->checkGame(game);
    std::vector<int> child(d.policySize);
    std::vector<double> mom((size_t)d.maxNodes * 5);
    sp->download(child.data(), d.childNode + (size_t)game * d.maxNodes * d.policySize, d.policySize);
    sp->download(mom.data(), d.nodeMoments + (size_t)game * d.maxNodes * 5, mom.size());
    for(int i = 0; i < d.policySize; i++)
      for(int k = 0; k < 5; k++) child_stats[i * 5 + k] = child[i] >= 0 ? mom[(size_t)child[i] * 5 + k] : 0.0;
    for(int k = 0; k < 5; k++) root_stats[k] = mom[k];
  });
}

// Komi per game (GameInitializer draws one per game: program/play.cpp:330-420 komiMean / komiStdev / ...).  `komi[numGames]` becomes
// the komi of each slot's NEXT game; with also_current_games it also replaces the komi of the game in progress (meant for games that
// have not started searching).
KGB_API int kgb_selfplay_set_komi(kgb_selfplay* sp, const float* komi, int also_current_games) {
  return guarded([&] {
    if(!sp || !komi) throw std::invalid_argument("kgb_selfplay_set_komi: NULL argument");
    sp->enter();
    const SPDev& d = sp->d;
    for(int g = 0; g < d.numGames; g++)
      if(!(komi[g] >= -150.0f && komi[g] <= 150.0f) || komi[g] * 2.0f != floorf(komi[g] * 2.0f))
        throw std::invalid_argument("selfplay: komi must be a multiple of 0.5 in [-150, 150] (Rules::komiIsIntOrHalfInt)");
    sp->upload(d.nextKomi, komi, d.numGames);
    if(also_current_games) sp->upload(d.komiG, komi, d.numGames);
    sp->sync();
  });
}

KGB_API int kgb_selfplay_set_game_setup(kgb_selfplay* sp, const int32_t* setup, int also_current_games) {
  return guarded([&] {
    if(!sp || !setup) throw std::invalid_argument("kgb_selfplay_set_game_setup: NULL argument");
    sp->enter();
    const SPDev& d = sp->d;
    for(int g = 0; g < d.numGames; g++) {
      const int* q = setup + (size_t)g * 4;
      if(q[0] < 2 || q[0] > d.X || q[1] < 2 || q[1] > d.Y) throw std::invalid_argument("selfplay: a game's board must be at least 2x2 and fit the evaluator's frame");
      if(q[2] < 0 || q[2] > 3) throw std::invalid_argument("selfplay: ko_rule must be 0 (simple), 1 (positional), 2 (situational) or 3 (spight)");
      if(q[3] != 0 && q[3] != 1) throw std::invalid_argument("selfplay: multi_stone_suicide_legal must be 0 or 1");
    }
    sp->upload(d.nextSetup, setup, (size_t)d.numGames * 4);
    sp->applyNext(also_current_games != 0, spApplySetupKernel, 32, " game(s) in progress have already started; their setup was left unchanged");
  });
}

KGB_API int kgb_selfplay_set_next_search_limits(kgb_selfplay* sp, const int32_t* visits, const uint8_t* plain_root, int also_current_roots) {
  return guarded([&] {
    if(!sp || !visits) throw std::invalid_argument("kgb_selfplay_set_next_search_limits: NULL argument");
    sp->enter();
    const SPDev& d = sp->d;
    for(int i = 0; i < d.numGames * 2; i++)
      if(visits[i] < 2 || visits[i] > d.maxVisits) throw std::invalid_argument("selfplay: a visit budget must lie between 2 and max_visits");
    sp->upload(d.nextBudget, visits, (size_t)d.numGames * 2);
    if(plain_root) sp->upload(d.nextPlain, plain_root, (size_t)d.numGames * 2);
    else sp->fill(d.nextPlain, 0, (size_t)d.numGames * 2);
    sp->applyNext(also_current_roots != 0, spApplyLimitsKernel, 1, " root(s) have already been searched; their limits were left unchanged");
  });
}

KGB_API int kgb_selfplay_get_search_limits(kgb_selfplay* sp, int32_t* visits, uint8_t* plain_root) {
  return guarded([&] {
    if(!sp) throw std::invalid_argument("kgb_selfplay_get_search_limits: NULL argument");
    sp->enter();
    if(visits) sp->download(visits, sp->d.visitBudget, sp->d.numGames);
    if(plain_root) sp->download(plain_root, sp->d.plainRoot, sp->d.numGames);
  });
}

KGB_API int kgb_selfplay_set_policy_init(kgb_selfplay* sp, const int32_t* num_moves, double temperature, int also_current_games) {
  return guarded([&] {
    if(!sp || !num_moves) throw std::invalid_argument("kgb_selfplay_set_policy_init: NULL argument");
    sp->enter();
    const SPDev& d = sp->d;
    if(!(temperature > 0.0 && temperature < 10.0)) throw std::invalid_argument("selfplay: policy init temperature must lie in (0, 10)");
    for(int g = 0; g < d.numGames; g++)
      if(num_moves[g] < 0) throw std::invalid_argument("selfplay: negative number of opening moves");
    sp->upload(d.policyInitTemperature, &temperature, 1);
    sp->upload(d.nextInitMoves, num_moves, d.numGames);
    sp->applyNext(also_current_games != 0, spApplyPolicyInitKernel, 1, " game(s) in progress have already started; their openings were left unchanged");
  });
}

// moves_left[numGames]: opening moves still to be drawn (> 0 = the slot is not a recorded turn yet); count / moves[numGames][max_moves]: the
// opening played so far in the current game (move positions, pass = policy size - 1).  Any pointer may be NULL.
KGB_API int kgb_selfplay_get_policy_init(kgb_selfplay* sp, int32_t* moves_left, int32_t* count, int16_t* moves, int max_moves) {
  return guarded([&] {
    if(!sp) throw std::invalid_argument("kgb_selfplay_get_policy_init: NULL argument");
    sp->enter();
    const SPDev& d = sp->d;
    if(moves_left) sp->download(moves_left, d.initMovesLeft, d.numGames);
    if(count) sp->download(count, d.initMoveCount, d.numGames);
    if(moves) {
      if(max_moves < 1 || max_moves > SP_MAX_INIT_MOVES) throw std::invalid_argument("selfplay: max_moves must lie in 1..512");
      CK(cudaMemcpy2DAsync(moves, (size_t)max_moves * sizeof(int16_t), d.initMoves, (size_t)SP_MAX_INIT_MOVES * sizeof(int16_t),
                           (size_t)max_moves * sizeof(int16_t), (size_t)d.numGames, cudaMemcpyDeviceToHost, sp->h->stream));
      sp->sync();
    }
  });
}

KGB_API int kgb_selfplay_get_nn_symmetries(kgb_selfplay* sp, int32_t* symmetries) {
  return guarded([&] {
    if(!sp || !symmetries) throw std::invalid_argument("kgb_selfplay_get_nn_symmetries: NULL argument");
    sp->enter();
    sp->download(symmetries, sp->d.nnSymmetry, sp->d.numGames);
  });
}

KGB_API int kgb_selfplay_get_root_raw_policy_entropy(kgb_selfplay* sp, double* entropy) {
  return guarded([&] {
    if(!sp || !entropy) throw std::invalid_argument("kgb_selfplay_get_root_raw_policy_entropy: NULL argument");
    sp->enter();
    sp->download(entropy, sp->d.rootRawEntropy, sp->d.numGames);
  });
}

KGB_API int kgb_selfplay_get_game_setup(kgb_selfplay* sp, int32_t* current, int32_t* last_finished) {
  return guarded([&] {
    if(!sp) throw std::invalid_argument("kgb_selfplay_get_game_setup: NULL argument");
    sp->enter();
    const SPDev& d = sp->d;
    if(current) {
      std::vector<int> a((size_t)d.numGames);
      int* const src[4] = {d.gX, d.gY, d.gKoRule, d.gMultiSuicide};
      for(int k = 0; k < 4; k++) {
        sp->download(a.data(), src[k], a.size());
        for(int g = 0; g < d.numGames; g++) current[(size_t)g * 4 + k] = a[g];
      }
    }
    if(last_finished) sp->download(last_finished, d.lastSetup, (size_t)d.numGames * 4);
  });
}

KGB_API int kgb_selfplay_get_komi(kgb_selfplay* sp, float* current, float* last_finished) {
  return guarded([&] {
    if(!sp) throw std::invalid_argument("kgb_selfplay_get_komi: NULL argument");
    sp->enter();
    if(current) sp->download(current, sp->d.komiG, sp->d.numGames);
    if(last_finished) sp->download(last_finished, sp->d.lastKomi, sp->d.numGames);
  });
}

KGB_API int kgb_selfplay_get_leaf_cache_key(kgb_selfplay* sp, int game, uint64_t* key2) {
  return guarded([&] {
    if(!sp || !key2) throw std::invalid_argument("kgb_selfplay_get_leaf_cache_key: NULL argument");
    sp->enter();
    sp->checkGame(game);
    sp->download(key2, sp->d.leafKey + (size_t)game * 2, 2);
  });
}

// After a weight swap (kgb_handle_commit_weights) the cached outputs belong to the previous net: the reference gets the same effect by
// giving every NNEvaluator its own NNCacheTable (nneval.cpp:129-130).  Ordered on the wave stream.
KGB_API int kgb_selfplay_clear_nn_cache(kgb_selfplay* sp) {
  return guarded([&] {
    if(!sp) throw std::invalid_argument("kgb_selfplay_clear_nn_cache: NULL argument");
    sp->enter(false);
    if(sp->d.cacheSize <= 0) return;
    sp->fill(sp->d.cacheKey0, 0, sp->d.cacheSize);
    sp->fill(sp->d.cacheKey1, 0, sp->d.cacheSize);
  });
}

// ---- game recording support (hold mode) ------------------------------------------------------------------------------------------
KGB_API int kgb_selfplay_release(kgb_selfplay* sp, const uint8_t* games_mask /*[numGames] or NULL = all*/) {
  return guarded([&] {
    if(!sp) throw std::invalid_argument("kgb_selfplay_release: NULL argument");
    sp->enter();
    if(games_mask) sp->upload(sp->d.releaseFlag, games_mask, sp->d.numGames);
    else sp->fill(sp->d.releaseFlag, 1, sp->d.numGames);
    sp->sync();
  });
}

KGB_API int kgb_selfplay_get_root_visits(kgb_selfplay* sp, int32_t* visits /*[numGames]*/) {
  return guarded([&] {
    if(!sp || !visits) throw std::invalid_argument("kgb_selfplay_get_root_visits: NULL argument");
    sp->enter();
    const SPDev& d = sp->d;
    CK(cudaMemcpy2DAsync(visits, sizeof(int), d.nodeVisits, (size_t)d.maxNodes * sizeof(int), sizeof(int), d.numGames, cudaMemcpyDeviceToHost,
                         sp->h->stream));
    sp->sync();
  });
}

// Visits of the root's child NODES by move position (0 where there is no child; under graph search a node's visits can exceed its
// edge's) and the root's own evaluation: winLoss, noResult, scoreMean, scoreMeanSq, lead (white's perspective).
KGB_API int kgb_selfplay_get_root_extra(kgb_selfplay* sp, int game, int32_t* child_node_visits, double* root_nn_stats) {
  return guarded([&] {
    if(!sp || !child_node_visits || !root_nn_stats) throw std::invalid_argument("kgb_selfplay_get_root_extra: NULL argument");
    sp->enter();
    const SPDev& d = sp->d;
    sp->checkGame(game);
    std::vector<int> child(d.policySize), nv(d.maxNodes);
    sp->download(child.data(), d.childNode + (size_t)game * d.maxNodes * d.policySize, d.policySize);
    sp->download(nv.data(), d.nodeVisits + (size_t)game * d.maxNodes, d.maxNodes);
    for(int i = 0; i < d.policySize; i++) child_node_visits[i] = child[i] >= 0 ? nv[child[i]] : 0;
    sp->download(root_nn_stats, d.nodeNNMoments + (size_t)game * d.maxNodes * 5, 5);
  });
}

// The last root move of game slot g: info[4] = move position (X*Y = pass), flags (1 it ended the game | 2 without result | 4 by the
// move limit), the move number it was played at, the slot's game index; when it ended the game also the final score (white minus
// black, komi included), the final position and its area (0 none, 1 black, 2 white).
KGB_API int kgb_selfplay_get_last_move(kgb_selfplay* sp, int game, int32_t* info, float* final_score, uint8_t* final_colors, uint8_t* final_area) {
  return guarded([&] {
    if(!sp || !info || !final_score || !final_colors || !final_area) throw std::invalid_argument("kgb_selfplay_get_last_move: NULL argument");
    sp->enter();
    const SPDev& d = sp->d;
    sp->checkGame(game);
    sp->download(info, d.lastMove + (size_t)game * 4, 4);
    sp->download(final_score, d.lastScore + game, 1);
    uint32_t fb[128];
    sp->download(fb, d.finalBoard + (size_t)game * 128, 128);
    for(int y = 0; y < d.Y; y++)
      for(int x = 0; x < d.X; x++) {
        final_colors[y * d.X + x] = (fb[y] >> x) & 1 ? 1 : (fb[32 + y] >> x) & 1 ? 2 : 0;
        final_area[y * d.X + x] = (fb[64 + y] >> x) & 1 ? 1 : (fb[96 + y] >> x) & 1 ? 2 : 0;
      }
  });
}

KGB_API int kgb_selfplay_get_nn_row(kgb_selfplay* sp, int game, float* spatial, float* global) {
  return guarded([&] {
    if(!sp || !spatial || !global || game < 0 || game >= sp->d.numGames) throw std::invalid_argument("kgb_selfplay_get_nn_row: bad argument");
    sp->enter();
    const size_t XY = (size_t)sp->h->L.X * sp->h->L.Y;
    sp->download(spatial, sp->h->dSpatial + (size_t)game * XY * 22, XY * 22);
    sp->download(global, sp->h->dGlobal + (size_t)game * 19, 19);
  });
}

KGB_API int kgb_selfplay_get_root_row(kgb_selfplay* sp, int game, float* spatial, float* global) {
  return guarded([&] {
    if(!sp || !spatial || !global || game < 0 || game >= sp->d.numGames) throw std::invalid_argument("kgb_selfplay_get_root_row: bad argument");
    sp->enter();
    const size_t n = (size_t)sp->d.XY * 22;
    sp->download(spatial, sp->d.rootRow + (size_t)game * (n + 19), n);
    sp->download(global, sp->d.rootRow + (size_t)game * (n + 19) + n, 19);
  });
}

KGB_API int kgb_selfplay_get_leaf_path(kgb_selfplay* sp, int game, int32_t* moves_xy, int32_t max_len, int32_t* len_out, int32_t* valid_out) {
  return guarded([&] {
    if(!sp || !moves_xy || !len_out || !valid_out || max_len < 0) throw std::invalid_argument("kgb_selfplay_get_leaf_path: bad argument");
    sp->enter();
    const SPDev& d = sp->d;
    sp->checkGame(game);
    int len = 0;
    sp->download(&len, d.pathLen + game, 1);
    sp->download(valid_out, d.leafValid + game, 1);
    std::vector<int> mv(len > 0 ? len : 1);
    if(len > 0) sp->download(mv.data(), d.pathMove + (size_t)game * d.maxDepth, len);
    for(int i = 0; i < len && i < max_len; i++) {
      const bool pass = mv[i] == d.policySize - 1;
      moves_xy[2 * i] = pass ? -1 : mv[i] % d.X; moves_xy[2 * i + 1] = pass ? -1 : mv[i] / d.X;
    }
    *len_out = len;
  });
}

KGB_API int kgb_selfplay_play_moves(kgb_selfplay* sp, const int8_t* moves_xy, int num_moves) {
  return guarded([&] {
    if(!sp || (!moves_xy && num_moves > 0) || num_moves < 0) throw std::invalid_argument("kgb_selfplay_play_moves: bad argument");
    sp->enter(false);
    sp->playMoves(moves_xy, num_moves, -1);
  });
}

KGB_API int kgb_selfplay_play_moves_game(kgb_selfplay* sp, int game, const int8_t* moves_xy, int num_moves) {
  return guarded([&] {
    if(!sp || game < 0 || (!moves_xy && num_moves > 0) || num_moves < 0) throw std::invalid_argument("kgb_selfplay_play_moves_game: bad argument");
    sp->enter();
    sp->playMoves(moves_xy, num_moves, game);
  });
}

KGB_API int kgb_selfplay_get_play_selection_values(kgb_selfplay* sp, int game, double* values) {
  return guarded([&] {
    if(!sp || !values) throw std::invalid_argument("kgb_selfplay_get_play_selection_values: NULL argument");
    sp->enter();
    sp->checkGame(game);
    Scratch<double> out(sp->d.policySize);
    playSelectionKernel<<<1, 32, 0, sp->h->stream>>>(sp->d, game, out.p);
    CK(cudaGetLastError());
    sp->download(values, out.p, sp->d.policySize);
  });
}

KGB_API int kgb_selfplay_time_tree_kernels(kgb_selfplay* sp, int iters, float* ms_select, float* ms_backup) {
  return guarded([&] {
    if(!sp || iters < 1 || !ms_select || !ms_backup) throw std::invalid_argument("kgb_selfplay_time_tree_kernels: bad argument");
    sp->enter();
    cudaStream_t s = sp->h->stream;
    cudaEvent_t e0, e1, e2;
    CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1)); CK(cudaEventCreate(&e2));
    float accS = 0.f, accB = 0.f;
    for(int i = 0; i < iters; i++) {   // the evaluator outputs of the last wave are reused: the trees keep growing normally
      CK(cudaEventRecord(e0, s));
      sp->launchSelect();
      CK(cudaEventRecord(e1, s));
      sp->launchBackup();
      CK(cudaEventRecord(e2, s));
      sp->sync();
      float a = 0.f, b = 0.f;
      CK(cudaEventElapsedTime(&a, e0, e1)); CK(cudaEventElapsedTime(&b, e1, e2));
      accS += a; accB += b;
    }
    cudaEventDestroy(e0); cudaEventDestroy(e1); cudaEventDestroy(e2);
    *ms_select = accS / iters; *ms_backup = accB / iters;
  });
}

KGB_API int kgb_selfplay_debug_cycles(kgb_selfplay* sp, int64_t* cycles /*[numGames][8]*/, int clear) {
  return guarded([&] {
    if(!sp || !cycles) throw std::invalid_argument("kgb_selfplay_debug_cycles: NULL argument");
    sp->enter();
    sp->download(cycles, sp->d.dbgCycles, (size_t)sp->d.numGames * 8);
    if(clear) {
      sp->fill(sp->d.dbgCycles, 0, (size_t)sp->d.numGames * 8);
      sp->sync();
    }
  });
}

KGB_API int kgb_selfplay_launches_per_step(const kgb_selfplay* sp) { return sp ? sp->h->launchesPerForward + 2 : 0; }

// ---- test hooks of the loop's device code: no handle, so on the default stream -------------------------------------------------
KGB_API int kgb_test_choose_index_with_temperature(const char* seed_string, const double* relative_probs, int n, double temperature,
                                                   double only_below_prob, int count, int32_t* chosen) {
  return guarded([&] {
    if(!seed_string || !relative_probs || !chosen || n < 1 || count < 1) throw std::invalid_argument("kgb_test_choose_index_with_temperature: bad argument");
    const DevRandState st = devRandState(seed_string);
    Scratch<DevRandState> ds(1);
    Scratch<double> dp(n), dscr(n);
    Scratch<int> dout(count);
    CK(cudaMemcpy(ds.p, &st, sizeof(st), cudaMemcpyHostToDevice));
    CK(cudaMemcpy(dp.p, relative_probs, n * sizeof(double), cudaMemcpyHostToDevice));
    chooseIndexTestKernel<<<1, 32>>>(ds.p, dp.p, n, temperature, only_below_prob, count, dout.p, dscr.p);
    CK(cudaGetLastError());
    CK(cudaDeviceSynchronize());
    CK(cudaMemcpy(chosen, dout.p, count * sizeof(int), cudaMemcpyDeviceToHost));
  });
}

KGB_API int kgb_test_history_replay(int x_len, int y_len, int ko_rule, int multi_stone_suicide_legal, int num_games, int max_moves, const int8_t* moves_xy,
                                    uint8_t* flags, uint8_t* legal_next, uint8_t* super_ko_banned) {
  return guarded([&] {
    if(!moves_xy || !flags || !legal_next || !super_ko_banned || num_games < 1 || max_moves < 1 || ko_rule < 0 || ko_rule > 3)
      throw std::invalid_argument("kgb_test_history_replay: bad argument");
    const int X = x_len, Y = y_len;
    if(X > 19 || Y > 19 || X < 2 || Y < 2) throw std::invalid_argument("history replay: board sizes 2..19 only");
    const size_t nm = (size_t)num_games * max_moves, cells = nm * X * Y;
    const ZobristTables zt = makeZobristTables(X, Y);
    Scratch<int8_t> dMoves(nm * 2);
    Scratch<uint8_t> dFlags(nm), dLegal(cells), dBanned(cells);
    Scratch<unsigned long long> dLists((size_t)num_games * 3 * (max_moves + 2));
    Scratch<ZobEntry> dZob(zt.board.size());
    CK(cudaMemcpy(dMoves.p, moves_xy, nm * 2, cudaMemcpyHostToDevice));
    CK(cudaMemcpy(dZob.p, zt.board.data(), zt.board.size() * sizeof(ZobEntry), cudaMemcpyHostToDevice));
    CK(cudaMemset(dFlags.p, 0, nm)); CK(cudaMemset(dLegal.p, 0, cells)); CK(cudaMemset(dBanned.p, 0, cells));
    historyReplayKernel<<<(num_games * 32 + 127) / 128, 128>>>(X, Y, ko_rule, multi_stone_suicide_legal, num_games, max_moves, dMoves.p, dZob.p,
                                                               dLists.p, dFlags.p, dLegal.p, dBanned.p);
    CK(cudaGetLastError());
    CK(cudaDeviceSynchronize());
    CK(cudaMemcpy(flags, dFlags.p, nm, cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(legal_next, dLegal.p, cells, cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(super_ko_banned, dBanned.p, cells, cudaMemcpyDeviceToHost));
  });
}

KGB_API int kgb_test_repetition_bound(int x_len, int y_len, int num_moves, int bound, const int8_t* moves_xyp, uint8_t* out) {
  return guarded([&] {
    if(!moves_xyp || !out || num_moves < 1) throw std::invalid_argument("kgb_test_repetition_bound: bad argument");
    Scratch<int8_t> dm((size_t)num_moves * 3);
    Scratch<uint8_t> dout(num_moves);
    CK(cudaMemcpy(dm.p, moves_xyp, (size_t)num_moves * 3, cudaMemcpyHostToDevice));
    repBoundKernel<<<1, 32>>>(x_len, y_len, num_moves, bound, dm.p, dout.p);
    CK(cudaGetLastError());
    CK(cudaDeviceSynchronize());
    CK(cudaMemcpy(out, dout.p, num_moves, cudaMemcpyDeviceToHost));
  });
}

KGB_API int kgb_test_root_policy_noise(const char* seed_string, int x_len, int y_len, int policy_size, int turn_number, int noise_enabled,
                                       double concentration, double weight, double temperature, double temperature_early, double halflife,
                                       const float* policy_in, float* policy_out) {
  return guarded([&] {
    if(!seed_string || !policy_in || !policy_out || policy_size < 1 || policy_size > 362) throw std::invalid_argument("kgb_test_root_policy_noise: bad argument");
    const DevRandState st = devRandState(seed_string);
    Scratch<float> dp(policy_size);
    Scratch<DevRandState> ds(1);
    Scratch<double> dr(3 * (size_t)policy_size);
    CK(cudaMemcpy(dp.p, policy_in, policy_size * sizeof(float), cudaMemcpyHostToDevice));
    CK(cudaMemcpy(ds.p, &st, sizeof(st), cudaMemcpyHostToDevice));
    rootNoiseTestKernel<<<1, 32>>>(dp.p, policy_size, x_len, y_len, turn_number, noise_enabled, concentration, weight, temperature, temperature_early,
                                   halflife, ds.p, dr.p);
    CK(cudaGetLastError());
    CK(cudaDeviceSynchronize());
    CK(cudaMemcpy(policy_out, dp.p, policy_size * sizeof(float), cudaMemcpyDeviceToHost));
  });
}

KGB_API int kgb_test_board_replay(int x_size, int y_size, int num_boards, int num_moves, int multi_stone_suicide_legal, const int8_t* moves,
                                  uint8_t* colors, int8_t* ko, int16_t* caps, uint8_t* lib_class, uint8_t* legal_next, uint64_t* pos_hash, uint8_t* area) {
  return guarded([&] {
    if(!moves || !colors || !ko || !caps || !lib_class || !legal_next || !pos_hash || !area || num_boards < 1 || num_moves < 1)
      throw std::invalid_argument("kgb_test_board_replay: bad argument");
    int count = 0;
    if(cudaGetDeviceCount(&count) != cudaSuccess || count == 0) throw CudaFailure("libkgb200: no CUDA device is visible");
    const int X = x_size, Y = y_size;
    if(X > 19 || Y > 19 || X < 2 || Y < 2) throw std::invalid_argument("board replay: board sizes 2..19 only");
    const size_t nm = (size_t)num_boards * num_moves, cells = nm * X * Y;
    const ZobristTables zt = makeZobristTables(X, Y);
    static_assert(sizeof(ZobEntry) == sizeof(Hash128), "layout");
    Scratch<int8_t> dMoves(nm * 3), dKo(nm * 2);
    Scratch<int16_t> dCaps(nm * 2);
    Scratch<uint8_t> dColors(cells), dLib(cells), dLegal(cells), dArea(cells);
    Scratch<ZobEntry> dZob(zt.board.size());
    Scratch<unsigned long long> dHash(nm * 2);
    CK(cudaMemcpy(dMoves.p, moves, nm * 3, cudaMemcpyHostToDevice));
    CK(cudaMemcpy(dZob.p, zt.board.data(), zt.board.size() * sizeof(ZobEntry), cudaMemcpyHostToDevice));
    int threads = 128;
    boardReplayKernel<<<(num_boards * 32 + threads - 1) / threads, threads>>>(X, Y, num_boards, num_moves, multi_stone_suicide_legal, dMoves.p, dColors.p,
                                                                               dKo.p, dCaps.p, dLib.p, dLegal.p, dZob.p, zt.sizeHash.h0, zt.sizeHash.h1,
                                                                               dHash.p, dArea.p);
    CK(cudaGetLastError());
    CK(cudaDeviceSynchronize());
    CK(cudaMemcpy(pos_hash, dHash.p, nm * 2 * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(area, dArea.p, cells, cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(colors, dColors.p, cells, cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(lib_class, dLib.p, cells, cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(legal_next, dLegal.p, cells, cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(ko, dKo.p, nm * 2, cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(caps, dCaps.p, nm * 2 * sizeof(int16_t), cudaMemcpyDeviceToHost));
  });
}

}  // extern "C"
