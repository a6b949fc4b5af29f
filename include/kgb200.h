/* kgb200.h - C ABI of the H100-native KataGo NN-evaluator backend (libkgb200.so).
 *
 * Drop-in boundary: the reference selects ONE translation unit defining `namespace NeuralNet`
 * (cpp/neuralnet/nninterface.h:32-182) at link time.  A maintainer adds `neuralnet/b200backend.cpp`
 * (integration/b200backend.cpp in this repository; see INTEGRATION.md) whose functions forward 1:1 to the entry
 * points below.  Plain pointers and sizes only; no exceptions, no C++ or torch types cross this boundary; every
 * function returns KGB_OK (0) or a negative status with the message available from kgb_last_error().
 * Buffers passed to kgb_forward are HOST memory owned by the caller (the reference's NNResultBuf / NNOutput arrays);
 * host<->device copies happen inside the call, exactly like cudabackend.cpp:3714-3782.
 */
#ifndef KGB200_H_
#define KGB200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(__GNUC__)
#define KGB_API __attribute__((visibility("default")))
#else
#define KGB_API
#endif

#define KGB_OK 0
#define KGB_ERR_INVALID (-1)   /* bad argument / unsupported model */
#define KGB_ERR_IO (-2)        /* model file could not be read / sha256 mismatch */
#define KGB_ERR_CUDA (-3)      /* CUDA runtime or driver failure, or no sm_90 device */

typedef struct kgb_model kgb_model;     /* replaces LoadedModel     (nninterface.h:27, eigenbackend.cpp:94-107) */
typedef struct kgb_context kgb_context; /* replaces ComputeContext  (nninterface.h:17) */
typedef struct kgb_handle kgb_handle;   /* replaces ComputeHandle   (nninterface.h:21) - one per server thread, not thread-safe */

/* Subset of ModelDesc (cpp/neuralnet/desc.h:508-571) that NNEvaluator reads through getModelDesc(). */
typedef struct kgb_model_info {
  char name[128];
  char sha256[65];
  int32_t model_version;
  int32_t num_input_channels;
  int32_t num_input_global_channels;
  int32_t num_policy_channels;
  int32_t num_value_channels;
  int32_t num_score_value_channels;
  int32_t num_ownership_channels;
  int32_t trunk_num_channels;
  int32_t num_blocks;
  int32_t prefer_pass_alive_under_suicide_rules;
  float td_score_multiplier;
  float score_mean_multiplier;
  float score_stdev_multiplier;
  float lead_multiplier;
  float variance_time_multiplier;
  float shortterm_value_error_multiplier;
  float shortterm_score_error_multiplier;
  int64_t conv_macs_per_position; /* direct-convolution MACs per board point (ModelDesc::iterConvLayers, desc.cpp:2643) */
  int32_t num_input_meta_channels; /* 192 for an SGF-metadata (human SL) net, which needs kgb_forward_meta; 0 otherwise */
} kgb_model_info;

/* NeuralNet::globalInitialize / globalCleanup (nninterface.h:34-36). */
KGB_API int kgb_global_init(void);
KGB_API int kgb_global_cleanup(void);
/* Message of the last failure on the calling thread ("" if none). */
KGB_API const char* kgb_last_error(void);
/* NeuralNet::printDevices (nninterface.h:39): number of CUDA devices and, per device, name/compute capability. */
KGB_API int kgb_device_count(int* count);
KGB_API int kgb_device_name(int device, char* buf, int buf_len, int* cc_major, int* cc_minor);

/* NeuralNet::loadModelFile / freeLoadedModel / getModelDesc (nninterface.h:43-46).
 * expected_sha256 may be NULL or "" to skip verification. */
KGB_API int kgb_model_load_file(const char* path, const char* expected_sha256, kgb_model** out);
KGB_API void kgb_model_free(kgb_model* model);
KGB_API int kgb_model_get_info(const kgb_model* model, kgb_model_info* out);

/* NeuralNet::createComputeContext / freeComputeContext (nninterface.h:50-65).
 * fp16_mode: 0 = "fp32-equivalent" (3-term split-fp16 on the tensor pipe, fp32 streams), 1 = fp16 operands with fp32
 * accumulation, -1 = auto (fp16). */
KGB_API int kgb_context_create(const int* gpu_idxs, int num_gpu_idxs, int nn_x_len, int nn_y_len, int fp16_mode,
                       const kgb_model* model, kgb_context** out);
KGB_API void kgb_context_free(kgb_context* ctx);

/* NeuralNet::createComputeHandle / freeComputeHandle / isUsingFP16 (nninterface.h:76-94).
 * gpu_idx == -1 selects the context's first device (or device 0).  inputs_nhwc selects the layout of `spatial`
 * in kgb_forward: 1 = [n][Y][X][C], 0 = [n][C][Y][X]. */
KGB_API int kgb_handle_create(kgb_context* ctx, const kgb_model* model, int max_batch_size, int require_exact_nn_len,
                      int inputs_nhwc, int gpu_idx, kgb_handle** out);
KGB_API void kgb_handle_free(kgb_handle* handle);
KGB_API int kgb_handle_is_fp16(const kgb_handle* handle);

/* NeuralNet::getOutput (nninterface.h:117-123).  For each of the n rows:
 *   spatial        [n][num_input_channels * X * Y]   NNResultBuf::rowSpatialBuf (fillRowV7 output, no symmetry applied)
 *   global         [n][num_input_global_channels]    NNResultBuf::rowGlobalBuf
 *   symmetry       [n] in 0..7                       NNResultBuf::symmetry (applied to inputs, inverted on outputs)
 *   policy_optimism[n]                               NNResultBuf::policyOptimism
 * Outputs (raw logits; NNEvaluator does the softmax/tanh post-processing, nneval.cpp:960-1249):
 *   policy         [n][X*Y + 1]  NNOutput::policyProbs (pass last)
 *   value          [n][3]        whiteWinProb, whiteLossProb, whiteNoResultProb
 *   score_value    [n][6]        whiteScoreMean, whiteScoreMeanSq, whiteLead, varTimeLeft, shorttermWinlossError,
 *                                shorttermScoreError (filled by model version as eigenbackend.cpp:2583-2626)
 *   ownership      [n][X*Y] or NULL (NNOutput::whiteOwnerMap)
 */
KGB_API int kgb_forward(kgb_handle* handle, int n, const float* spatial, const float* global, const int32_t* symmetry,
                const float* policy_optimism, float* policy, float* value, float* score_value, float* ownership);

/* Same computation with every buffer already resident in this handle's device memory (used by the device-resident
 * self-play loop and by bench.py's HBM-resident timing).  Pointers are device pointers; the call is asynchronous on the
 * handle's stream - use kgb_handle_sync() before reading results from another stream. */
KGB_API int kgb_forward_device(kgb_handle* handle, int n, const float* d_spatial, const float* d_global, const int32_t* d_symmetry,
                       const float* d_policy_optimism, float* d_policy, float* d_value, float* d_score_value,
                       float* d_ownership);
/* The same two entry points for an SGF-metadata (human SL) net (kgb_model_info.num_input_meta_channels = 192), with one more input:
 *   meta           [n][192]   NNResultBuf::rowMetaBuf (SGFMetadata::fillMetadataRow output)
 * The net's metadata encoder (three fully connected layers) turns each row into a per-image bias of the initial convolution, added
 * to the global inputs' one (eigenbackend.cpp:1927-1932).  kgb_forward / kgb_forward_device on such a net, and these two on a net
 * without an encoder, are KGB_ERR_INVALID. */
KGB_API int kgb_forward_meta(kgb_handle* handle, int n, const float* spatial, const float* global, const float* meta, const int32_t* symmetry,
                             const float* policy_optimism, float* policy, float* value, float* score_value, float* ownership);
KGB_API int kgb_forward_device_meta(kgb_handle* handle, int n, const float* d_spatial, const float* d_global, const float* d_meta,
                                    const int32_t* d_symmetry, const float* d_policy_optimism, float* d_policy, float* d_value,
                                    float* d_score_value, float* d_ownership);
KGB_API int kgb_handle_sync(kgb_handle* handle);
/* cudaStream_t of the handle (as an integer) so a torch/CUDA caller can order its own work against it. */
KGB_API uint64_t kgb_handle_stream(kgb_handle* handle);
/* Number of kernel launches one kgb_forward of batch n issues (for bench.py's gpu_launches accounting); a metadata net's encoder adds 3. */
KGB_API int kgb_handle_launches_per_forward(const kgb_handle* handle);
/* The row layout the last forward or self-play wave on the handle used (waits for the handle's stream): the rows and 128-row
 * tiles every convolution ran over, and the number of segments (board widths).  Each image takes (h+pad)*(w+pad) rows for the
 * bounding box w x h of its mask, so a batch of small boards takes fewer rows than n*(nnYLen+pad)*(nnXLen+pad).  All zero
 * before the first forward. */
KGB_API int kgb_handle_get_layout_stats(kgb_handle* handle, int64_t* rows, int64_t* m_tiles, int64_t* segments);

/* New weights into a live handle.  The reference polls its models directory and builds a fresh NNEvaluator for every new net
 * (command/selfplay.cpp:142-231 loadLatestNeuralNetIntoManager, :336-352 the polling thread; dataio/loadmodel.cpp:58
 * findLatestModel); games switch over between moves (switchNetsMidGame, program/play.cpp maybeGetNewNet).  Here the handle keeps
 * its graphs and buffers and only the weight arena changes:
 *   kgb_handle_stage_weights   packs `model` (same architecture as the handle's, else an error) for this handle's kernels and
 *                              copies it to a shadow arena on a side stream - evaluation continues meanwhile
 *   kgb_handle_commit_weights  orders "shadow -> live" on the handle's stream: every forward pass / self-play wave enqueued
 *                              afterwards runs the new net, none sees a mixture
 * Between GPUs of one node (one process per GPU) the packed arena travels by ncclBroadcast straight between device memories,
 * so only one rank reads and packs the model file:
 *   kgb_nccl_unique_id                   on one rank; the 128 bytes reach the others by any side channel (torch.distributed, MPI, a file)
 *   kgb_handle_comm_init                 on every rank, once per handle
 *   kgb_handle_broadcast_staged_weights  on every rank; the root must have staged; *ms_out = the collective's device time
 * followed by kgb_handle_commit_weights on every rank.  NCCL is bound at run time (libnccl.so.2, or KGB_NCCL_LIB). */
KGB_API int kgb_handle_weights_bytes(const kgb_handle* handle, uint64_t* bytes);
KGB_API int kgb_handle_stage_weights(kgb_handle* handle, const kgb_model* model);
KGB_API int kgb_handle_commit_weights(kgb_handle* handle);
/* Blocks the host until the staging copy (or a received broadcast) has landed in the shadow arena; not needed before a commit
 * (ordered on the device), useful before a barrier that lines the ranks up for a timed broadcast. */
KGB_API int kgb_handle_wait_staged(kgb_handle* handle);
KGB_API int kgb_nccl_unique_id(void* id_out_128_bytes);
KGB_API int kgb_handle_comm_init(kgb_handle* handle, const void* id_128_bytes, int rank, int num_ranks);
KGB_API int kgb_handle_broadcast_staged_weights(kgb_handle* handle, int root, float* ms_out);

/* FOR TESTING: NeuralNet::testEvaluateConv (nninterface.h:134-143).  weights in the model-file order
 * [ky][kx][in_c][out_c]; input/output [n][Y][X][C] (NHWC) fp32.  use_fp16 selects the operand mode as in
 * kgb_context_create.  Returns KGB_OK and fills output[n*Y*X*out_c]. */
KGB_API int kgb_test_conv(int ky, int kx, int in_c, int out_c, const float* weights, int n, int nn_x_len, int nn_y_len, int use_fp16,
                  const float* input, float* output);

/* ---------------------------------------------------------------------------------------------------------------
 * Boundary 2 (SURVEY.md §8b): device-resident self-play slots.  Boards, MCTS node pools and NN rows stay in HBM; one
 * kgb_selfplay_run(steps) call performs `steps` playout waves (select+featurize -> NN forward -> backup, one visit per
 * game per wave) without returning to the host.  Replaces, for the supported rule/parameter subset (DESIGN.md §8),
 * Search::runWholeSearch/playoutDescend (search.cpp:473,1189), selectBestChildToDescend (searchexplorehelpers.cpp:324),
 * NNEvaluator::evaluate's featurize/post-process halves (nneval.cpp:861-1262) and the per-move core of Play::runGame
 * (play.cpp:1757-1936).  Parameters are the reference's SearchParams names (search/searchparams.h). */
typedef struct kgb_selfplay kgb_selfplay;

typedef struct kgb_selfplay_config {
  int32_t num_games;                 /* concurrent games (= NN batch per wave); <= the handle's max_batch_size */
  int32_t max_visits;                /* maxVisits: visits per move on a cleared tree */
  int32_t max_moves;                 /* game length cap (0 = 2*X*Y) */
  int32_t multi_stone_suicide_legal; /* Rules::multiStoneSuicideLegal */
  int32_t early_temperature_moves;   /* moves chosen proportionally to visits (chosenMoveTemperatureEarly = 1), then argmax */
  float komi;
  double cpuct_exploration;          /* cpuctExploration       (default 1.0) */
  double cpuct_exploration_log;      /* cpuctExplorationLog    (0.45 in selfplay cfgs) */
  double cpuct_exploration_base;     /* cpuctExplorationBase   (500) */
  double fpu_reduction_max;          /* fpuReductionMax        (0.2) */
  double root_fpu_reduction_max;     /* rootFpuReductionMax    (0.1 in selfplay cfgs) */
  double win_loss_utility_factor;    /* winLossUtilityFactor   (1.0) */
  double no_result_utility_for_white;
  uint64_t seed;
  int32_t debug_fake_nn;             /* TEST ONLY: replace the evaluator by the deterministic hash net of oracle/ref_driver.cpp; 1 = short-term
                                        error channels 0 (its default), 2 = hash-derived raw values there (tests/cpp/uncertainty_search_driver.cpp),
                                        3 = the table net: each game's evaluations return the raw outputs set by kgb_selfplay_debug_set_raw_outputs,
                                        4 = the wide hash net of oracle/ref_driver.cpp (KGREF_FAKE_WIDE=1): the same hash, wider output ranges */
  int32_t disable_ladder_features;   /* 1 = leave NN input planes 14-17 zero (timing experiments only) */
  int32_t ladder_nodes_per_wave;     /* > 0: each of a game's 8 ladder-reader warps plays at most this many search moves per wave;
                                        a game whose searches are unfinished skips the wave (no visit) and resumes in the next.
                                        0 = run every search to the end inside the wave.  Features are identical either way. */
  int32_t max_playouts_per_wave;     /* a playout that ends without needing the evaluator (evaluation-cache hit, graph-search edge catch-up,
                                        cycle) is backed up inside the select kernel and the game starts its next playout in the same wave,
                                        up to this many (0 = 16).  The launch lasts as long as its slowest game, so a small bound (2-3) caps
                                        the tail: a game that uses it up delivers no leaf this wave and carries on in the next.  The sequence
                                        of playouts of a game, hence every result, is the same for every bound. */
  /* Score utility (Search::getScoreUtility, searchhelpers.cpp:272-279; selfplay8mainb18.cfg: 0.05, 0.30, 0.25, 0.50).
   * Both factors 0 = win/loss utility only. */
  double static_score_utility_factor;
  double dynamic_score_utility_factor;
  double dynamic_score_center_zero_weight;
  double dynamic_score_center_scale;
  double draw_equivalent_wins_for_white;   /* 0.5 in every stock config; used for integer komi results */
  /* More SearchParams of the selection / backup formulas (search/searchparams.h), by their cfg names.  All 0 = the plain
   * PUCT + visit-weighted average of the first fixtures. */
  double value_weight_exponent;                   /* valueWeightExponent (0.5): t-CDF value weighting in the backup */
  int32_t fpu_parent_weight_by_visited_policy;    /* fpuParentWeightByVisitedPolicy */
  int32_t debug_fixed_symmetry_plus_one;          /* TEST ONLY: k + 1 = evaluate every row under symmetry k (the reference's nnRandomize = false with
                                                     nnForcedSymmetry / default symmetry k, nneval.cpp:698-707); 0 = a random symmetry per row */
  double fpu_parent_weight_by_visited_policy_pow; /* fpuParentWeightByVisitedPolicyPow */
  double fpu_parent_weight;                       /* fpuParentWeight */
  double fpu_loss_prop;                           /* fpuLossProp */
  double root_fpu_loss_prop;                      /* rootFpuLossProp */
  double cpuct_utility_stdev_prior;               /* cpuctUtilityStdevPrior (0.25) */
  double cpuct_utility_stdev_prior_weight;        /* cpuctUtilityStdevPriorWeight (1.0) */
  double cpuct_utility_stdev_scale;               /* cpuctUtilityStdevScale (0 = off) */
  double root_desired_per_child_visits_coeff;     /* rootDesiredPerChildVisitsCoeff */
  double subtree_value_bias_factor;               /* subtreeValueBiasFactor (0.30 in selfplay8mainb18.cfg; 0 = off) */
  double subtree_value_bias_weight_exponent;      /* subtreeValueBiasWeightExponent (0.8) */
  int32_t use_graph_search;                       /* useGraphSearch: transpositions share a node (search.cpp:875-936) */
  int32_t graph_search_rep_bound;                 /* graphSearchRepBound (11) */
  int32_t debug_hold_at_max_visits;               /* hold mode: a game whose root has max_visits visits idles until kgb_selfplay_release (tests; game recording) */
  int32_t root_noise_enabled;                     /* rootNoiseEnabled: Dirichlet noise on the root policy */
  double root_dirichlet_noise_total_concentration;/* rootDirichletNoiseTotalConcentration (10.83) */
  double root_dirichlet_noise_weight;             /* rootDirichletNoiseWeight (0.25) */
  double root_policy_temperature;                 /* rootPolicyTemperature (0 = unset = 1.0) */
  double root_policy_temperature_early;           /* rootPolicyTemperatureEarly (0 = unset = 1.0) */
  double chosen_move_temperature_halflife;        /* chosenMoveTemperatureHalflife (0 = unset = 19): also the half-life of the early root temperature */
  /* Root move choice like Search::getChosenMoveLoc (play selection values, LCB, temperature).  use_play_selection = 0 keeps the
   * simple rule: proportional to visits for the first early_temperature_moves moves, then the most visited. */
  int32_t use_play_selection;
  int32_t use_lcb_for_selection;                  /* useLcbForSelection */
  int32_t use_non_buggy_lcb;                      /* useNonBuggyLcb */
  int32_t root_prune_useless_moves;               /* rootPruneUselessMoves: when the opponent's last four moves were passes, the root never plays
                                                     inside either player's pass-alive area (Search::isAllowedRootMove, searchhelpers.cpp:310-342) */
  double lcb_stdevs;                              /* lcbStdevs (5.0) */
  double min_visit_prop_for_lcb;                  /* minVisitPropForLCB (0.15) */
  double chosen_move_temperature;                 /* chosenMoveTemperature (0.15) */
  double chosen_move_temperature_early;           /* chosenMoveTemperatureEarly (0.75) */
  double chosen_move_temperature_only_below_prob; /* chosenMoveTemperatureOnlyBelowProb (0 = unset = 1.0) */
  double chosen_move_subtract;                    /* chosenMoveSubtract (0) */
  double chosen_move_prune;                       /* chosenMovePrune (1) */
  int32_t nn_cache_size_power_of_two;             /* nnCacheSizePowerOfTwo: evaluation cache shared by the games of this GPU (0 = off) */
  int32_t root_num_symmetries_to_sample;          /* rootNumSymmetriesToSample (4): the root is evaluated under that many symmetries, one per wave */
  int32_t ko_rule;                                /* Rules::koRule: 0 simple, 1 positional superko, 2 situational superko, 3 spight (area scoring) */
  double root_ending_bonus_points;                /* rootEndingBonusPoints (0.5 in the stock configs): at the root, moves into territory the net's
                                                     ownership head is sure about (|ownership| >= 0.95) lose up to this many points of score
                                                     utility unless they capture / touch the opponent / connect groups that are not pass-alive
                                                     (Search::getEndingWhiteScoreBonus, searchhelpers.cpp:351-420; area scoring).  Needs the
                                                     root to be evaluated by the net (root_num_symmetries_to_sample >= 2 or the cache off). */
  /* Uncertainty-weighted evaluations (Search::computeWeightFromNNOutput, searchupdatehelpers.cpp:114-136; on in the stock gatekeeper
   * configs and under katago match, off in self-play).  With a net of model version >= 9 each evaluation enters the search with weight
   * coeff / ((winLossUtilityFactor * shorttermWinlossError + dScoreUtility/dScore * shorttermScoreError)^exponent + coeff / max_weight)
   * instead of 1, and terminal positions with max_weight.  Nets below version 9 report no short-term error: weight 1.  0 = off. */
  int32_t use_uncertainty;                        /* useUncertainty */
  double uncertainty_coeff;                       /* uncertaintyCoeff (0.25) */
  double uncertainty_exponent;                    /* uncertaintyExponent (1.0; 1.0 and 0.5 are exact, other values use pow) */
  double uncertainty_max_weight;                  /* uncertaintyMaxWeight (8.0) */
  /* Noise pruning (Search::pruneNoiseWeight, searchupdatehelpers.cpp:495-539): in every backup, a child whose utility is below the
   * average of the children before it (creation order) loses weight beyond twice its policy share of theirs.  0 = off. */
  int32_t use_noise_pruning;                      /* useNoisePruning */
  double noise_prune_utility_scale;               /* noisePruneUtilityScale (0.15) */
  double noise_pruning_cap;                       /* noisePruningCap (1e50) */
} kgb_selfplay_config;

typedef struct kgb_selfplay_stats {
  uint64_t total_visits;     /* playouts completed (sum over games of root visits) */
  uint64_t total_moves;      /* root moves played */
  uint64_t games_finished;
  uint64_t black_wins;
  uint64_t nodes_allocated;
  uint64_t sum_leaf_depth;   /* sum over playouts of the leaf depth */
  uint64_t ladder_searches;  /* ladder searches run for feature planes 14-17 */
  uint64_t ladder_nodes;     /* moves played inside those searches */
  uint64_t stalled_waves;    /* game-waves that finished no playout: ladder searches still running (ladder_nodes_per_wave), every
                                playout of the wave ended on an existing edge, or one of the root's extra symmetric evaluations */
  uint64_t instant_playouts; /* graph search: playouts that ended on an edge catch-up or a cycle and needed no evaluation */
  uint64_t nn_cache_hits;    /* playouts whose leaf evaluation came from the evaluation cache */
  uint64_t nn_cache_stores;
} kgb_selfplay_stats;

/* ScoreValue::expectedWhiteScoreValue (neuralnet/nninputs.cpp:160-192) on the host, with the table the device loop uploads:
 * n independent lookups.  Test hook for the score-utility table (SURVEY.md row a21). */
KGB_API int kgb_expected_white_score_value(int n, const double* mean, const double* stdev, const double* center, const double* scale,
                                           const double* sqrt_board_area, double* out);
/* The first n 32-bit outputs of the reference's Rand(seed_string) as the library's host generator produces them (core/rand.h:149-152,
 * core/rand.cpp:279-320).  Test hook (row a25): the reference's own self-test vector for "abc" (core/rand.cpp:386-415) pins it. */
KGB_API int kgb_rand_uint32_stream(const char* seed_string, int n, uint32_t* out);
/* The value-weighting CDF table the device loop uploads (Search's DistributionTable over tdistcdf(z, 3), search.cpp:131-137):
 * n must be 2000.  Test hook (row a20). */
KGB_API int kgb_value_weight_cdf_table(double* out, int n);
/* Search::getPlaySelectionValues of game g's root (searchresults.cpp:66-330), indexed by move position (-1 = no child):
 * the weights the root move is drawn from (reduced weights, LCB bonus, subtract / prune applied). */
KGB_API int kgb_selfplay_get_play_selection_values(kgb_selfplay* sp, int game, double* values);
/* TEST HOOK: `count` consecutive draws of Search::chooseIndexWithTemperature (searchhelpers.cpp:12-76) from the device Rand
 * seeded with seed_string. */
KGB_API int kgb_test_choose_index_with_temperature(const char* seed_string, const double* relative_probs, int n, double temperature,
                                                   double only_below_prob, int count, int32_t* chosen);
/* TEST HOOK (row a23): Board::simpleRepetitionBoundGt(move, bound) after every move of a stream (x, y, player 1 black / 2 white; x < 0 pass)
 * - the predicate that decides whether a graph-search node may be shared between histories (game/board.cpp:2853-2888). */
KGB_API int kgb_test_repetition_bound(int x_len, int y_len, int num_moves, int bound, const int8_t* moves_xyp, uint8_t* out);
/* TEST HOOK (row a3): replay num_games games (moves_xy [game][max_moves][2]: x,y; -1,-1 pass; -2 = end of that game; black first) through
 * the device ko rules (ko_rule 0 simple, 1 positional, 2 situational, 3 spight; area scoring).  Per move: flags (1 game over, 2 no result,
 * 4 a pass by the next player would end the phase), legality of every point for the next player (incl. ko and superko bans), and
 * the superko-banned points - BoardHistory::makeBoardMoveAssumeLegal / isLegal / passWouldEndPhase (game/boardhistory.cpp). */
KGB_API int kgb_test_history_replay(int x_len, int y_len, int ko_rule, int multi_stone_suicide_legal, int num_games, int max_moves, const int8_t* moves_xy,
                                    uint8_t* flags, uint8_t* legal_next, uint8_t* super_ko_banned);
/* TEST HOOK (rows a22/a25): the device loop's root-policy temperature + Dirichlet noise on a given policy (-1 = illegal), with the
 * device Rand initialised from seed_string like the reference's Rand(seed_string): the counterpart of
 * Search::maybeAddPolicyNoiseAndTemp / addDirichletNoise (searchhelpers.cpp:78-215). */
KGB_API int kgb_test_root_policy_noise(const char* seed_string, int x_len, int y_len, int policy_size, int turn_number, int noise_enabled,
                                       double concentration, double weight, double temperature, double temperature_early, double halflife,
                                       const float* policy_in, float* policy_out);
KGB_API int kgb_selfplay_create(kgb_handle* handle, const kgb_selfplay_config* config, kgb_selfplay** out);
KGB_API void kgb_selfplay_free(kgb_selfplay* sp);
/* Enqueue `steps` playout waves on the handle's stream (asynchronous; kgb_handle_sync() to wait). */
KGB_API int kgb_selfplay_run(kgb_selfplay* sp, int steps);
KGB_API int kgb_selfplay_get_stats(kgb_selfplay* sp, kgb_selfplay_stats* out);
/* Root position of game g: colors[Y*X] (0 empty, 1 black, 2 white); info[6] = move number, black-to-move, ko point
 * (y*32+x or -1), black stones captured, white stones captured, root visits. */
KGB_API int kgb_selfplay_get_game(kgb_selfplay* sp, int game, uint8_t* colors, int32_t* info);
/* Root children of game g, indexed by move position 0..X*Y (pass last): edge visit counts, NN policy (-1 illegal), and each
 * child's utilityAvg (white's perspective; 0 where there is no child). */
KGB_API int kgb_selfplay_get_root_children(kgb_selfplay* sp, int game, int32_t* visits, float* policy, double* utility_avg);
/* NodeStats moments (searchnode.h:17-41; white's perspective) of game g's root and of its children by move position:
 * winLossValueAvg, noResultValueAvg, scoreMeanAvg, scoreMeanSqAvg, leadAvg.  child_stats[(X*Y+1)*5] (0 where no child), root_stats[5]. */
KGB_API int kgb_selfplay_get_root_value_stats(kgb_selfplay* sp, int game, double* child_stats, double* root_stats);
/* NodeStats weightSum and weightSqSum of game g's root (root_weights[2]) and of its children by move position
 * (child_weights[(X*Y+1)*2], 0 where there is no child): 1 per evaluation unless uncertainty weighting or noise pruning acts. */
KGB_API int kgb_selfplay_get_root_weights(kgb_selfplay* sp, int game, double* child_weights, double* root_weights);
/* Game g's root utility (white's perspective): utility[0] = the utility of its own evaluation (Search::getUtilityFromNN),
 * utility[1] = NodeStats utilityAvg. */
KGB_API int kgb_selfplay_get_root_utility(kgb_selfplay* sp, int game, double* utility);
/* TEST ONLY (debug_fake_nn = 3): the raw net outputs every later evaluation of game g returns, in the evaluator's frame and from the
 * mover's perspective as the net gives them: policy logits [X*Y+1] (pass last), value logits [3] (win, loss, no result),
 * score-value channels [6] (mean, stdev before softplus, lead, variance of time left, short-term value and score errors before
 * softplus), ownership logits [X*Y]. */
KGB_API int kgb_selfplay_debug_set_raw_outputs(kgb_selfplay* sp, int game, const float* policy, const float* value, const float* score,
                                               const float* ownership);
/* TEST HOOK (row a20): the device loop's short-term error post-processing and evaluation weight on the host, n independent cases.
 * raw[n][2] = score-value channels 4 and 5 as the net outputs them; params[n][12] = shortterm value / score error multipliers,
 * uncertaintyCoeff, uncertaintyExponent, uncertaintyMaxWeight, winLossUtilityFactor, staticScoreUtilityFactor,
 * dynamicScoreUtilityFactor, dynamicScoreCenterScale, recentScoreCenter, sqrtBoardArea, whiteScoreMean.  out[n][3] =
 * shorttermWinlossError, shorttermScoreError (float as NNOutput keeps them; -1 below version 9) and the weight the search would use
 * with useUncertainty on and a net that supports short-term errors. */
KGB_API int kgb_test_uncertainty_weight(int n, const int32_t* model_version, const double* raw, const double* params, double* out);
/* Game recording (SURVEY.md §8f row 2; replaces the bookkeeping around the search in Play::runGame, program/play.cpp:1757-1936).
 * With kgb_selfplay_config.debug_hold_at_max_visits = 1 a game whose search reached max_visits idles until it is released; the
 * host reads the finished search (getters above and below), releases, and the next wave lets the device choose and play the move
 * as usual.  games_mask[num_games] (1 = release) or NULL = all.  A released game holds again at its next finished search. */
KGB_API int kgb_selfplay_release(kgb_selfplay* sp, const uint8_t* games_mask);
/* Komi per game.  The reference's GameInitializer draws a komi for every game (program/play.cpp:330-420: komiMean, komiStdev,
 * komiBigStdevProb, komiAuto ...); here the host draws and the device applies: komi[num_games] (multiples of 0.5) becomes the komi of
 * each slot's NEXT game, taken when the slot's game in progress ends; also_current_games != 0 replaces the komi of the games in
 * progress too (for games that have not begun to search).  kgb_selfplay_get_komi: komi of the game in progress and of the slot's
 * last finished game (either pointer may be NULL).  The evaluation cache keys on the mover's komi (NNInputs::getHash,
 * neuralnet/nninputs.cpp:869-943 via BoardHistory::getSituationRulesAndKoHash), so games of different komi never share an entry. */
KGB_API int kgb_selfplay_set_komi(kgb_selfplay* sp, const float* komi, int also_current_games);
KGB_API int kgb_selfplay_get_komi(kgb_selfplay* sp, float* current, float* last_finished);
/* Board size and ko / suicide rules per game.  The reference's GameInitializer draws them for every game (program/play.cpp:330-650:
 * bSizes / bSizeRelProbs, koRules, multiStoneSuicideLegals; BASELINE config 4 "mixed 9/13/19 board sizes"); here the host draws and the
 * device applies, like the komi.  setup[num_games][4] = board X, board Y (2..the context's nn_x_len / nn_y_len), ko rule (0-3 as in
 * kgb_selfplay_config.ko_rule), multi-stone suicide legal (0/1).  A game's board occupies the top-left corner of the evaluator's frame:
 * move positions stay y * nn_x_len + x (NNPos::locToPos, neuralnet/nninputs.cpp:27-33), input plane 0 marks the board and the conv
 * trunk masks everything outside it (nneval.cpp:874-883 does the same with nnXLen > board size).  The values become each slot's NEXT
 * game's; also_current_games != 0 applies them to the games in progress too, which must not have started (no move, no visit) -
 * KGB_ERR_INVALID otherwise, nothing changed for those.
 * kgb_selfplay_get_game_setup: setup of the game in progress and of the slot's last finished game (either pointer may be NULL).
 * The evaluation cache keys on board size and rules as NNInputs::getHash does, so such games never share an entry. */
KGB_API int kgb_selfplay_set_game_setup(kgb_selfplay* sp, const int32_t* setup, int also_current_games);
KGB_API int kgb_selfplay_get_game_setup(kgb_selfplay* sp, int32_t* current, int32_t* last_finished);
/* Search limits per move.  Play::runGame gives every move its own limits (getSearchLimitsThisMove / runBotWithLimits, program/play.cpp:
 * 1093-1300): a "cheap search" (cheapSearchProb, cheapSearchVisits) or a visit count reduced in decided positions (reduceVisits), and for
 * cheap searches that are not recorded the root-only parameters off (no Dirichlet noise, root policy temperature 1, the tree's FPU
 * parameters at the root, no per-child visit floor, a single root symmetry).  Here the host draws (katago_b200/game_recorder.py) and the
 * device applies: visits[num_games][2] in [2, max_visits] and plain_root[num_games][2] (NULL = all 0) are taken by the root that follows
 * the slot's NEXT move - entry 0 if the game goes on, entry 1 if that move ends the game (first root of the slot's next game);
 * also_current_roots != 0 applies entry 0 to the current roots too, which must not have been searched yet (KGB_ERR_INVALID otherwise).
 * A game is held / moves when its root's visits reach ITS budget: kgb_selfplay_get_search_limits returns the current roots' budgets and
 * flags (either pointer may be NULL).  Deviation: the reference keeps the previous tree for unrecorded cheap searches, this loop always
 * starts a move on a cleared tree. */
KGB_API int kgb_selfplay_set_next_search_limits(kgb_selfplay* sp, const int32_t* visits, const uint8_t* plain_root, int also_current_roots);
KGB_API int kgb_selfplay_get_search_limits(kgb_selfplay* sp, int32_t* visits, uint8_t* plain_root);
/* Policy-initialised openings (PlaySettings::initGamesWithPolicy, policyInitAreaProp, policyInitAreaTemperature; PlayUtils::initializeGameUsingPolicy,
 * program/playutils.cpp:232-266, called from Play::runGame, play.cpp:1675-1700): the first num_moves[g] moves of slot g's NEXT game are drawn
 * from the net's own policy ^ (1 / temperature) of each position - one plain evaluation per move, no search, no noise; a slot in its opening is
 * never held for recording (the moves belong to the game's start history, not to its training turns).  The host draws the count (floor of an
 * exponential with mean board area * policyInitAreaProp).  also_current_games != 0: the games in progress take them too; they must not have
 * started (KGB_ERR_INVALID otherwise).  kgb_selfplay_get_policy_init: moves_left[num_games] (> 0 = still in its opening), count[num_games] and
 * moves[num_games][max_moves] = the opening of the game in progress (move positions, pass = nn_x_len * nn_y_len; max_moves <= 512); any
 * pointer may be NULL.  Not restated: the separately noised komi during the opening and the komi compensation after it
 * (compensateAfterPolicyInitProb needs searches before the game). */
KGB_API int kgb_selfplay_set_policy_init(kgb_selfplay* sp, const int32_t* num_moves, double temperature, int also_current_games);
KGB_API int kgb_selfplay_get_policy_init(kgb_selfplay* sp, int32_t* moves_left, int32_t* count, int16_t* moves, int max_moves);
/* FOR TESTING: the evaluation-cache key (the loop's NNInputs::getHash) of the leaf that slot `game` sent to the evaluator in the
 * last wave; only meaningful with nn_cache_size_power_of_two > 0. */
KGB_API int kgb_selfplay_get_leaf_cache_key(kgb_selfplay* sp, int game, uint64_t* key2);
/* Empties the loop's evaluation cache, ordered on the handle's stream: call it with kgb_handle_commit_weights - cached outputs
 * belong to the previous net (the reference gives every NNEvaluator its own NNCacheTable, nneval.cpp:129-130). */
KGB_API int kgb_selfplay_clear_nn_cache(kgb_selfplay* sp);
/* Root visits of every game (visits[num_games]): a game is held when its entry has reached max_visits. */
KGB_API int kgb_selfplay_get_root_visits(kgb_selfplay* sp, int32_t* visits);
/* What extractQValueTargets / computeNNRawStats (play.cpp:859-914) read besides the NodeStats: visits of the root's child NODES by
 * move position (0 = no child), and the root's own evaluation root_nn_stats[5] = winLoss, noResult, scoreMean, scoreMeanSq, lead (white). */
KGB_API int kgb_selfplay_get_root_extra(kgb_selfplay* sp, int game, int32_t* child_node_visits, double* root_nn_stats);
/* symmetries[num_games]: the symmetry (0-7) under which each game's row of the LAST wave was evaluated.  The wave is the loop's batcher (row a9:
 * one row per game, NNEvaluator::serve's batching replaced by the fixed wave); like the reference with nnRandomize = true every row draws its
 * own symmetry (nneval.cpp:698-707) - here from splitmix64 of (seed, game, game index, move, root visits) - except for a root's sampled
 * symmetries (root_num_symmetries_to_sample) and debug_fixed_symmetry. */
KGB_API int kgb_selfplay_get_nn_symmetries(kgb_selfplay* sp, int32_t* symmetries);
/* entropy[num_games]: the entropy of every current root's policy as the net gave it (averaged over the root's symmetric evaluations), BEFORE the
 * root policy temperature and the Dirichlet noise - NNRawStats::policyEntropy of computeNNRawStats (program/play.cpp:890-914; training global 59).
 * The reference takes it from a fresh single-symmetry evaluation of the root; here it is the root's own evaluation. */
KGB_API int kgb_selfplay_get_root_raw_policy_entropy(kgb_selfplay* sp, double* entropy);
/* The last root move of slot `game`: info[4] = move position (X*Y = pass), flags (1 = it ended the game | 2 = without result | 4 = by
 * the move limit), the move number it was played at, the slot's game index.  If it ended the game: final_score = white minus black
 * with komi, final_colors[Y*X] and final_area[Y*X] (0 none, 1 black, 2 white; Board::calculateArea with every flag on, which under
 * area scoring without tax is both the ownership and the full area of FinishedGameData). */
KGB_API int kgb_selfplay_get_last_move(kgb_selfplay* sp, int game, int32_t* info, float* final_score, uint8_t* final_colors, uint8_t* final_area);
/* The NN input row (NHWC [X*Y][22] + 19 globals) the last wave wrote for game g - what NNInputs::fillRowV7 would produce
 * for that leaf (planes listed in DESIGN.md §8; used by the feature parity tests). */
KGB_API int kgb_selfplay_get_nn_row(kgb_selfplay* sp, int game, float* spatial, float* global);
/* The NN input row (NNInputs::fillRowV7, NHWC, no symmetry) of the game's CURRENT ROOT, kept on the device from the wave that evaluated
 * the root until the next move: what TrainingWriteBuffers::addRow stores for the turn (dataio/trainingwrite.cpp:463-478).  Valid once the
 * root has been evaluated by the net (always, when root_num_symmetries_to_sample >= 2 or the evaluation cache is off). */
KGB_API int kgb_selfplay_get_root_row(kgb_selfplay* sp, int game, float* spatial, float* global);
/* The moves from the root to the leaf the last wave selected for game g (x,y pairs, -1,-1 = pass; at most max_len pairs are
 * written, *len_out is the full length) and whether that wave delivered a finished leaf (see ladder_nodes_per_wave). */
KGB_API int kgb_selfplay_get_leaf_path(kgb_selfplay* sp, int game, int32_t* moves_xy, int32_t max_len, int32_t* len_out, int32_t* valid_out);
/* Re-seed every game's search-thread generator like the reference's Rand(seed_string) (tests: reproduce a reference search whose
 * SearchThread seed string is known). */
KGB_API int kgb_selfplay_set_search_rand(kgb_selfplay* sp, const char* seed_string);
/* Desynchronise the games (bench / test support): every game plays its own random number (0..max_moves) of uniformly random
 * legal non-pass moves from its current root and clears its tree - positions "from random legal play-outs" (SURVEY.md §8d). */
KGB_API int kgb_selfplay_random_openings(kgb_selfplay* sp, int max_moves);
/* Play a fixed move list on EVERY game's root (x,y pairs, -1,-1 = pass; colours alternate) and clear the trees. */
KGB_API int kgb_selfplay_play_moves(kgb_selfplay* sp, const int8_t* moves_xy, int num_moves);
/* The same for one game only (games of different board sizes need different lists; match play mirrors the opponent's moves into the
 * other net's loop).  A move off the game's board is KGB_ERR_INVALID.  Unlike kgb_selfplay_play_moves, a move that ends the game - by
 * the rules or by max_moves - is treated like the loop's own: result readable with kgb_selfplay_get_last_move, the slot's next game
 * starts (next setup and komi), later moves of the list go to that game. */
KGB_API int kgb_selfplay_play_moves_game(kgb_selfplay* sp, int game, const int8_t* moves_xy, int num_moves);
/* Timing hook for bench.py's tree/board roofline entry: runs `iters` waves of ONLY the select(+board+featurize) and backup
 * kernels (evaluator outputs of the last wave are reused) and returns their CUDA-event averages per launch. */
KGB_API int kgb_selfplay_time_tree_kernels(kgb_selfplay* sp, int iters, float* ms_select, float* ms_backup);
/* Profiling aid: SM-clock spans of every game's block in the LAST select launch, cycles[game][8] = whole block, root move + tree reset
 * (only in waves where the game's visit budget was spent), warp 0 (descent + leaf features), ladder searches, then warp 0 split into
 * descent, liberties + legality, area (Benson), feature-row writes.  The launch lasts as
 * long as its slowest block; this shows which games those are and what they were doing.  clear != 0 zeroes the buffer afterwards. */
KGB_API int kgb_selfplay_debug_cycles(kgb_selfplay* sp, int64_t* cycles, int clear);
/* Kernel launches per playout wave (evaluator launches + 2). */
KGB_API int kgb_selfplay_launches_per_step(const kgb_selfplay* sp);

/* Zobrist data of the reference Board (game/board.cpp:151-216, Rand seeded "Board::initHash()"), regenerated by the backend's
 * own Rand restatement: board_hash[y][x][colour (0 black, 1 white)][2 x u64] and the empty-board hash size_hash[2]. */
KGB_API int kgb_zobrist_tables(int x_size, int y_size, uint64_t* board_hash, uint64_t* size_hash);

/* FOR TESTING (rows a1/a2): replay move streams on the device board.  moves[b][m] = {x, y (or -1,-1 = pass), pla (1 black,
 * 2 white)}; after every move returns stones, simple-ko point {x,y or -1,-1}, capture counters {black stones captured,
 * white stones captured}, liberty class of every stone (1,2,3, 0 = more / empty), Board::isLegal of every point for
 * the NEXT player, Board::pos_hash {hash0, hash1}, and Board::calculateArea (all flags on; 0 none, 1 black, 2 white). */
KGB_API int kgb_test_board_replay(int x_size, int y_size, int num_boards, int num_moves, int multi_stone_suicide_legal, const int8_t* moves,
                          uint8_t* colors, int8_t* ko, int16_t* caps, uint8_t* lib_class, uint8_t* legal_next, uint64_t* pos_hash, uint8_t* area);

/* Kernel-level timing hook for bench.py's roofline object: runs ONE convolution layer (random weights / inputs resident in HBM)
 * `iters` times on a stream after `warmup` launches and returns the CUDA-event average per launch.  epilogue_kind chooses the
 * production epilogue: 0 = fp32 raw output only (heads / gpool conv), 1 = BN + mish + mask -> fp16 (first conv of a residual unit),
 * 2 = + residual stream read and rewritten in place (second conv of a unit, a nested block's post conv), 3 = raw stream + activated
 * operand (a nested block's pre conv), 4 = kind 2 with an fp32 residual stream also in fp16 mode (the trunk's block exit with
 * KGB_STREAM_FP32=trunk; in fp32-equivalent mode every stream is fp32).  `rotate` >= 1 independent input / output buffer sets are
 * cycled through so that the timed loop's working set exceeds L2. */
KGB_API int kgb_bench_conv_ex(int ky, int kx, int in_c, int out_c, int n, int nn_x_len, int nn_y_len, int use_fp16, int epilogue_kind, int rotate,
                      int warmup, int iters, float* ms_per_launch);
/* Test hook for the fused epilogues (kinds 1-4 above) of one convolution layer: NHWC input [n][y][x][in_c], optional NHWC residual
 * [n][y][x][out_c], per-channel BN scale / bias (NULL = 1 / 0), activation (0 identity, 1 relu, 2 mish, 3 silu); returns the raw stream after
 * the launch (kinds 2-4) and the activated fp16 operand, both NHWC [n][y][x][out_c] as floats.  Also checks that every pad row of the
 * activated operand was written as zero (reference semantics: the conv's zero padding, eigenbackend.cpp:448-701). */
KGB_API int kgb_test_conv_epilogue(int ky, int kx, int in_c, int out_c, const float* weights, int n, int nn_x_len, int nn_y_len, int use_fp16,
                           int epilogue_kind, const float* input, const float* residual_in, const float* bn_scale, const float* bn_bias,
                           int activation, float* raw_out, float* act_out);
/* Test hook that reaches every input of the fused epilogue (kinds 0-4 above; kgb_test_conv and kgb_test_conv_epilogue are its
 * narrower forms).  Beyond kgb_test_conv_epilogue's arguments:
 *   board_xy [n][2] {X_i, Y_i}, or NULL for the whole frame: the mask is 1 on image i's top-left X_i x Y_i board and 0 elsewhere, as
 *     the self-play loop places smaller boards.  The input may be nonzero off the board; only the mask zeroes those outputs.
 *   ncbias [n][out_c] or NULL: a per-image bias added before the residual, as the initial conv adds the global-input bias.  The
 *     kernel applies it in every kind; tests/test_gpu_conv_fp64.py checks it in kind 3, the initial conv's, only.
 *   residual_in is fp32; an fp16 stream holds it rounded to nearest.  activation 0 identity, 1 relu, 2 mish, 3 silu.
 * Outputs, NHWC [n][y][x][out_c] as floats: raw_out (kind 0 and kinds 2-4), act_hi_out (kinds 1-4) and, in split mode, act_lo_out
 * (kinds 1-4), the activated operand's two fp16 halves as the next layer reads them.  The hook fails if any output is nonzero in a
 * row the mask zeroes, or in the padded channels out_c..cout_p of any row. */
KGB_API int kgb_test_conv_ex(int ky, int kx, int in_c, int out_c, const float* weights, int n, int nn_x_len, int nn_y_len, int use_fp16,
                             int epilogue_kind, const float* input, const int32_t* board_xy, const float* ncbias, const float* residual_in,
                             const float* bn_scale, const float* bn_bias, int activation, float* raw_out, float* act_hi_out,
                             float* act_lo_out);
/* Test hook for the fused nested-block boundary (DESIGN.md §4): a block's exit 1x1 (inner_c -> trunk_c, + the trunk stream) and
 * the next block's entry 1x1 (trunk_c -> inner_c, mish at both ends) on inputs and weights drawn from `seed`, run once as one fused
 * launch and once as two launches.  board_xy [n][2] or NULL as in kgb_test_conv_ex; the trunk stream is fp32 when trunk_fp32, the
 * inner one when inner_fp32 (which needs trunk_fp32, as KGB_STREAM_FP32=all).  out[0..2]: elements of the trunk stream, the inner
 * stream and the inner operand whose bits differ between the two; out[3..5]: nonzero elements of the fused outputs in masked rows
 * or padded channels.  Fails when the fused kernel does not take the shape. */
KGB_API int kgb_test_conv_boundary(int inner_c, int trunk_c, int n, int nn_x_len, int nn_y_len, const int32_t* board_xy, int trunk_fp32,
                                   int inner_fp32, uint32_t seed, int64_t* out);
/* Plan mode of the layer hooks.  The rows are planned on the device as a forward plans them (launchPlanRows, then launchPackInput):
 * image i's mask is 1 on the top-left board_xy[i] of the frame ({0, 0}: an empty mask) and 0 elsewhere, moved by symmetry[i] (NULL:
 * all 0); ragged 1 lays each board out at its own box, ragged 0 every image at the full frame.  Row buffers are sized for the largest
 * plan of n images.  Every input but `input` (given before the symmetry, zero off the board, as fillRowV7 writes it) and every
 * output is NHWC in the coordinates after the symmetry.  Rows of the operand at or past the plan's end hold a finite sentinel (fp16
 * 1024), as a larger earlier forward can leave them; rows of the outputs there are filled with all-ones bytes (NaN) before the launch.
 * The hook fails if an output row past the plan's end was written, or if any channel of a row below it that is not a board position
 * (pad rows and columns, gap rows, the tail up to 128 rows), or a padded channel of any row, is not exactly zero.  layout_stats [3]
 * (rows, 128-row tiles, segments) and plan_out [n][5] (box x0, y0, w, h and first row; -1 for an empty mask), either may be NULL. */
KGB_API int kgb_test_conv_plan(int ky, int kx, int in_c, int out_c, const float* weights, int n, int nn_x_len, int nn_y_len, int use_fp16,
                               int epilogue_kind, const float* input, const int32_t* board_xy, const int32_t* symmetry, int ragged,
                               const float* ncbias, const float* residual_in, const float* bn_scale, const float* bn_bias, int activation,
                               float* raw_out, float* act_hi_out, float* act_lo_out, int64_t* layout_stats, int32_t* plan_out);
/* kgb_test_conv_boundary under a plan made as for kgb_test_conv_plan, every buffer's rows past the plan's end NaN.  out [12]:
 * out[0..5] as kgb_test_conv_boundary over the rows below the plan's end; out[6..8] NaN elements of the fused outputs there;
 * out[9..11] bytes past the plan's end that either path changed.  layout_stats [3] or NULL. */
KGB_API int kgb_test_conv_boundary_plan(int inner_c, int trunk_c, int n, int nn_x_len, int nn_y_len, const int32_t* board_xy,
                                        const int32_t* symmetry, int ragged, int trunk_fp32, int inner_fp32, uint32_t seed, int64_t* out,
                                        int64_t* layout_stats);
/* Test hook of the evaluator's fp32 kernels: one launch of kernel `which` on caller-given fp32 tensors, in a frame of
 * nn_x_len x nn_y_len with `pad` (1 or 2).  Kernels that read rows run under a plan made as for kgb_test_conv_plan (board_xy,
 * symmetry, ragged; layout_stats and plan_out as there); their row inputs are NHWC [n][y][x][C] after the symmetry and are placed
 * in the rows of the board positions, every other element of the row buffer NaN.  Outputs the kernel does not write hold NaN.
 *   0 pack     iparams {C, split, nhwc}; inputs {spatial [n][C][y][x] or [n][y][x][C], channel 0 the mask}, planned from the
 *              spatial itself (board_xy unused); outputs {hi [n][y][x][C], lo (split) or NULL, mask sums [n], mask [n][y][x]}, after
 *              the symmetry.  Fails if a row that is not a board position, or a padded channel, is not zero.
 *   1 gpool    iparams {C, act, valueHead, rawFp32, c0, ldr}; inputs {raw (stored as fp16 when !rawFp32), bn scale [C], bias [C]};
 *              outputs {pooled [n][3C]}.
 *   2 biasAct  iparams {C, act, split, rawFp32}; inputs {raw, ncbias [n][C] or NULL, scale, bias}; outputs {hi, lo (split) or NULL}
 *              NHWC after the symmetry.  Fails as pack does, or if a row past the plan's end was written.
 *   3 matMulNC iparams {cin, cout, act, ldi, ldo}; inputs {in [n][ldi], W [cin][cout], bias [cout] or NULL}; outputs {[n][ldo]}.
 *   4 policy   iparams {C, act, cp2, c0, ldr}; inputs {raw, g1bias [n][C], scale, bias, Wp2 [C][cp2], optimism [n] or NULL};
 *              outputs {policy [n][x*y+1]}.
 *   5 ownership iparams {C, act, c0, ldr}; inputs {raw, scale, bias, Wown [C]}; outputs {ownership [n][x*y]}.
 *   6 finalize iparams {cp2, numSV, version, ldp}; inputs {pass logits [n][ldp], optimism [n] or NULL, value [n][3], score values
 *              [n][numSV]}; outputs {policy [n][x*y+1], value [n][3], score [n][6]}. */
KGB_API int kgb_test_head_kernel(int which, int n, int nn_x_len, int nn_y_len, int pad, const int32_t* board_xy, const int32_t* symmetry,
                                 int ragged, const int32_t* iparams, int num_iparams, const float* const* inputs, int num_inputs,
                                 float* const* outputs, int num_outputs, int64_t* layout_stats, int32_t* plan_out);
/* Timing hook of the same boundary (whole boards): ms per boundary, fused (one launch) or not (two launches), cycling through
 * `rotate` buffer sets. */
KGB_API int kgb_bench_conv_boundary(int inner_c, int trunk_c, int n, int nn_x_len, int nn_y_len, int trunk_fp32, int inner_fp32, int fused,
                                    int rotate, int warmup, int iters, float* ms_per_boundary);

#ifdef __cplusplus
}
#endif
#endif /* KGB200_H_ */
