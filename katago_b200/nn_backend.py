"""Host-side mirror of the reference's backend interface `namespace NeuralNet` (cpp/neuralnet/nninterface.h:32-182)
over the C ABI of libkgb200.so (include/kgb200.h).  Same names, argument meaning and error behaviour as the
reference: failures raise (StringError there, KGBError here); there is NO CPU fallback - a missing library or a
missing sm_90 device is an error.

    model  = NeuralNet.loadModelFile(path, expectedSha256)          # nninterface.h:43
    ctx    = NeuralNet.createComputeContext([0], nnXLen, nnYLen, useFP16Mode, model)   # :50
    handle = NeuralNet.createComputeHandle(ctx, model, maxBatchSize, requireExactNNLen, inputsUseNHWC, gpuIdx)  # :76
    out    = NeuralNet.getOutput(handle, spatial, global_, symmetry, policyOptimism)   # :117
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Optional, Sequence

import numpy as np


class KGBError(RuntimeError):
    pass


class _ModelInfo(C.Structure):
    _fields_ = [
        ("name", C.c_char * 128), ("sha256", C.c_char * 65),
        ("model_version", C.c_int32), ("num_input_channels", C.c_int32), ("num_input_global_channels", C.c_int32),
        ("num_policy_channels", C.c_int32), ("num_value_channels", C.c_int32), ("num_score_value_channels", C.c_int32),
        ("num_ownership_channels", C.c_int32), ("trunk_num_channels", C.c_int32), ("num_blocks", C.c_int32),
        ("prefer_pass_alive_under_suicide_rules", C.c_int32),
        ("td_score_multiplier", C.c_float), ("score_mean_multiplier", C.c_float), ("score_stdev_multiplier", C.c_float),
        ("lead_multiplier", C.c_float), ("variance_time_multiplier", C.c_float),
        ("shortterm_value_error_multiplier", C.c_float), ("shortterm_score_error_multiplier", C.c_float),
        ("conv_macs_per_position", C.c_int64), ("num_input_meta_channels", C.c_int32),
    ]


class SelfplayConfig(C.Structure):
    """kgb_selfplay_config: the reference's SearchParams / rules names (search/searchparams.h, game/rules.h)."""
    _fields_ = [
        ("num_games", C.c_int32), ("max_visits", C.c_int32), ("max_moves", C.c_int32), ("multi_stone_suicide_legal", C.c_int32),
        ("early_temperature_moves", C.c_int32), ("komi", C.c_float),
        ("cpuct_exploration", C.c_double), ("cpuct_exploration_log", C.c_double), ("cpuct_exploration_base", C.c_double),
        ("fpu_reduction_max", C.c_double), ("root_fpu_reduction_max", C.c_double), ("win_loss_utility_factor", C.c_double),
        ("no_result_utility_for_white", C.c_double), ("seed", C.c_uint64), ("debug_fake_nn", C.c_int32), ("disable_ladder_features", C.c_int32),
        ("ladder_nodes_per_wave", C.c_int32), ("max_playouts_per_wave", C.c_int32),
        ("static_score_utility_factor", C.c_double), ("dynamic_score_utility_factor", C.c_double),
        ("dynamic_score_center_zero_weight", C.c_double), ("dynamic_score_center_scale", C.c_double),
        ("draw_equivalent_wins_for_white", C.c_double),
        ("value_weight_exponent", C.c_double), ("fpu_parent_weight_by_visited_policy", C.c_int32), ("debug_fixed_symmetry_plus_one", C.c_int32),
        ("fpu_parent_weight_by_visited_policy_pow", C.c_double), ("fpu_parent_weight", C.c_double), ("fpu_loss_prop", C.c_double),
        ("root_fpu_loss_prop", C.c_double), ("cpuct_utility_stdev_prior", C.c_double), ("cpuct_utility_stdev_prior_weight", C.c_double),
        ("cpuct_utility_stdev_scale", C.c_double), ("root_desired_per_child_visits_coeff", C.c_double),
        ("subtree_value_bias_factor", C.c_double), ("subtree_value_bias_weight_exponent", C.c_double),
        ("use_graph_search", C.c_int32), ("graph_search_rep_bound", C.c_int32),
        ("debug_hold_at_max_visits", C.c_int32), ("root_noise_enabled", C.c_int32),
        ("root_dirichlet_noise_total_concentration", C.c_double), ("root_dirichlet_noise_weight", C.c_double),
        ("root_policy_temperature", C.c_double), ("root_policy_temperature_early", C.c_double),
        ("chosen_move_temperature_halflife", C.c_double),
        ("use_play_selection", C.c_int32), ("use_lcb_for_selection", C.c_int32), ("use_non_buggy_lcb", C.c_int32), ("root_prune_useless_moves", C.c_int32),
        ("lcb_stdevs", C.c_double), ("min_visit_prop_for_lcb", C.c_double), ("chosen_move_temperature", C.c_double),
        ("chosen_move_temperature_early", C.c_double), ("chosen_move_temperature_only_below_prob", C.c_double),
        ("chosen_move_subtract", C.c_double), ("chosen_move_prune", C.c_double),
        ("nn_cache_size_power_of_two", C.c_int32), ("root_num_symmetries_to_sample", C.c_int32),
        ("ko_rule", C.c_int32), ("root_ending_bonus_points", C.c_double),
        ("use_uncertainty", C.c_int32), ("uncertainty_coeff", C.c_double), ("uncertainty_exponent", C.c_double),
        ("uncertainty_max_weight", C.c_double), ("use_noise_pruning", C.c_int32), ("noise_prune_utility_scale", C.c_double),
        ("noise_pruning_cap", C.c_double),
    ]


class SelfplayStats(C.Structure):
    _fields_ = [("total_visits", C.c_uint64), ("total_moves", C.c_uint64), ("games_finished", C.c_uint64), ("black_wins", C.c_uint64),
                ("nodes_allocated", C.c_uint64), ("sum_leaf_depth", C.c_uint64), ("ladder_searches", C.c_uint64), ("ladder_nodes", C.c_uint64), ("stalled_waves", C.c_uint64), ("instant_playouts", C.c_uint64), ("nn_cache_hits", C.c_uint64),
                ("nn_cache_stores", C.c_uint64)]


# Every symbol include/kgb200.h declares (tests/test_abi.py checks the library exports all of them).
ABI_SYMBOLS = [
    "kgb_global_init", "kgb_global_cleanup", "kgb_last_error", "kgb_device_count", "kgb_device_name",
    "kgb_model_load_file", "kgb_model_free", "kgb_model_get_info", "kgb_context_create", "kgb_context_free",
    "kgb_handle_create", "kgb_handle_free", "kgb_handle_is_fp16", "kgb_forward", "kgb_forward_device", "kgb_test_forward_serial", "kgb_conv_chain_error", "kgb_forward_meta", "kgb_forward_device_meta", "kgb_handle_sync",
    "kgb_handle_stream", "kgb_handle_launches_per_forward", "kgb_handle_chained_launches_per_forward", "kgb_handle_epilogue_wg_launches_per_forward", "kgb_handle_pair_epilogue_wg_launches_per_forward", "kgb_handle_get_layout_stats", "kgb_test_conv", "kgb_bench_conv_ex", "kgb_test_conv_epilogue",
    "kgb_test_conv_ex", "kgb_test_conv_boundary", "kgb_bench_conv_boundary", "kgb_test_conv_plan", "kgb_test_conv_boundary_plan",
    "kgb_test_conv_boundary_ex", "kgb_test_last_conv_kernel", "kgb_test_head_kernel",
    "kgb_selfplay_create", "kgb_selfplay_free", "kgb_selfplay_run", "kgb_selfplay_get_stats", "kgb_selfplay_get_game",
    "kgb_selfplay_get_root_children", "kgb_selfplay_launches_per_step", "kgb_selfplay_play_moves", "kgb_selfplay_time_tree_kernels", "kgb_zobrist_tables", "kgb_selfplay_get_nn_row", "kgb_selfplay_get_root_row", "kgb_test_board_replay", "kgb_selfplay_get_leaf_path", "kgb_expected_white_score_value", "kgb_value_weight_cdf_table", "kgb_rand_uint32_stream", "kgb_test_root_policy_noise", "kgb_test_history_replay", "kgb_test_repetition_bound", "kgb_selfplay_get_play_selection_values", "kgb_selfplay_random_openings", "kgb_selfplay_set_search_rand", "kgb_selfplay_get_root_value_stats", "kgb_test_choose_index_with_temperature",
    "kgb_handle_weights_bytes", "kgb_handle_stage_weights", "kgb_handle_commit_weights", "kgb_handle_wait_staged", "kgb_nccl_unique_id", "kgb_handle_comm_init",
    "kgb_handle_broadcast_staged_weights", "kgb_selfplay_clear_nn_cache", "kgb_selfplay_set_komi", "kgb_selfplay_get_komi", "kgb_selfplay_get_leaf_cache_key",
    "kgb_selfplay_debug_cycles", "kgb_selfplay_release", "kgb_selfplay_get_root_visits", "kgb_selfplay_get_root_extra", "kgb_selfplay_get_last_move",
    "kgb_selfplay_set_game_setup", "kgb_selfplay_get_game_setup", "kgb_selfplay_play_moves_game",
    "kgb_selfplay_set_next_search_limits", "kgb_selfplay_get_search_limits", "kgb_selfplay_set_policy_init", "kgb_selfplay_get_policy_init",
    "kgb_selfplay_get_root_raw_policy_entropy", "kgb_selfplay_get_nn_symmetries", "kgb_selfplay_get_root_weights", "kgb_test_uncertainty_weight",
    "kgb_selfplay_get_root_utility", "kgb_selfplay_debug_set_raw_outputs",
]

_lib = None


def library_path() -> str:
    return os.path.join(os.path.dirname(os.path.abspath(__file__)), "libkgb200.so")


def load_library():
    """dlopen the in-tree libkgb200.so; raises KGBError (never falls back) if it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    path = library_path()
    if not os.path.exists(path):
        raise KGBError(f"{path} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
                       "(katago_b200/csrc/build.sh). There is no CPU fallback.")
    lib = C.CDLL(path)
    P, I, F = C.c_void_p, C.c_int, C.POINTER(C.c_float)
    lib.kgb_last_error.restype = C.c_char_p
    lib.kgb_device_count.argtypes = [C.POINTER(I)]
    lib.kgb_device_name.argtypes = [I, C.c_char_p, I, C.POINTER(I), C.POINTER(I)]
    lib.kgb_model_load_file.argtypes = [C.c_char_p, C.c_char_p, C.POINTER(P)]
    lib.kgb_model_free.argtypes = [P]
    lib.kgb_model_free.restype = None
    lib.kgb_model_get_info.argtypes = [P, C.POINTER(_ModelInfo)]
    lib.kgb_context_create.argtypes = [C.POINTER(I), I, I, I, I, P, C.POINTER(P)]
    lib.kgb_context_free.argtypes = [P]
    lib.kgb_context_free.restype = None
    lib.kgb_handle_create.argtypes = [P, P, I, I, I, I, C.POINTER(P)]
    lib.kgb_handle_free.argtypes = [P]
    lib.kgb_handle_free.restype = None
    lib.kgb_handle_is_fp16.argtypes = [P]
    lib.kgb_handle_weights_bytes.argtypes = [P, C.POINTER(C.c_uint64)]
    lib.kgb_handle_stage_weights.argtypes = [P, P]
    lib.kgb_handle_commit_weights.argtypes = [P]
    lib.kgb_handle_wait_staged.argtypes = [P]
    lib.kgb_nccl_unique_id.argtypes = [P]
    lib.kgb_handle_comm_init.argtypes = [P, P, I, I]
    lib.kgb_handle_broadcast_staged_weights.argtypes = [P, I, C.POINTER(C.c_float)]
    lib.kgb_selfplay_clear_nn_cache.argtypes = [P]
    lib.kgb_selfplay_set_komi.argtypes = [P, P, I]
    lib.kgb_selfplay_get_komi.argtypes = [P, P, P]
    lib.kgb_selfplay_set_game_setup.argtypes = [P, P, I]
    lib.kgb_selfplay_get_game_setup.argtypes = [P, P, P]
    lib.kgb_selfplay_play_moves_game.argtypes = [P, I, P, I]
    lib.kgb_selfplay_set_next_search_limits.argtypes = [P, P, P, I]
    lib.kgb_selfplay_get_search_limits.argtypes = [P, P, P]
    lib.kgb_selfplay_set_policy_init.argtypes = [P, P, C.c_double, I]
    lib.kgb_selfplay_get_policy_init.argtypes = [P, P, P, P, I]
    lib.kgb_selfplay_get_root_raw_policy_entropy.argtypes = [P, P]
    lib.kgb_selfplay_get_nn_symmetries.argtypes = [P, P]
    lib.kgb_selfplay_get_leaf_cache_key.argtypes = [P, I, P]
    lib.kgb_forward.argtypes = [P, I, P, P, P, P, P, P, P, P]
    lib.kgb_forward_device.argtypes = [P, I, P, P, P, P, P, P, P, P]
    lib.kgb_test_forward_serial.argtypes = [P, I, P, P, P, P, P, P, P, P]
    lib.kgb_conv_chain_error.argtypes = [P]
    lib.kgb_forward_meta.argtypes = [P, I, P, P, P, P, P, P, P, P, P]
    lib.kgb_forward_device_meta.argtypes = [P, I, P, P, P, P, P, P, P, P, P]
    lib.kgb_handle_sync.argtypes = [P]
    lib.kgb_handle_stream.argtypes = [P]
    lib.kgb_handle_stream.restype = C.c_uint64
    lib.kgb_handle_launches_per_forward.argtypes = [P]
    lib.kgb_handle_chained_launches_per_forward.argtypes = [P]
    lib.kgb_handle_epilogue_wg_launches_per_forward.argtypes = [P]
    lib.kgb_handle_pair_epilogue_wg_launches_per_forward.argtypes = [P]
    lib.kgb_handle_get_layout_stats.argtypes = [P, P, P, P]
    lib.kgb_test_conv.argtypes = [I, I, I, I, P, I, I, I, I, P, P]
    lib.kgb_bench_conv_ex.argtypes = [I, I, I, I, I, I, I, I, I, I, I, I, F]
    lib.kgb_test_conv_epilogue.argtypes = [I, I, I, I, P, I, I, I, I, I, P, P, P, P, I, P, P]
    lib.kgb_test_conv_ex.argtypes = [I, I, I, I, P, I, I, I, I, I, P, P, P, P, P, P, I, P, P, P]
    lib.kgb_test_conv_plan.argtypes = [I, I, I, I, P, I, I, I, I, I, P, P, P, I, P, P, P, P, I, P, P, P, P, P]
    lib.kgb_test_conv_boundary_plan.argtypes = [I, I, I, I, I, P, P, I, I, I, C.c_uint32, P, P]
    lib.kgb_test_conv_boundary_ex.argtypes = [I, I, I, I, I, P, P, P, P, P, P, P, P, P, P, I, I, I, I, P, P, P, P]
    lib.kgb_test_last_conv_kernel.argtypes = [C.POINTER(I)]
    lib.kgb_test_head_kernel.argtypes = [I, I, I, I, I, P, P, I, P, I, P, I, P, I, P, P]
    lib.kgb_selfplay_create.argtypes = [P, C.POINTER(SelfplayConfig), C.POINTER(P)]
    lib.kgb_selfplay_free.argtypes = [P]
    lib.kgb_selfplay_free.restype = None
    lib.kgb_selfplay_run.argtypes = [P, I]
    lib.kgb_selfplay_get_stats.argtypes = [P, C.POINTER(SelfplayStats)]
    lib.kgb_selfplay_get_game.argtypes = [P, I, P, P]
    lib.kgb_selfplay_get_root_children.argtypes = [P, I, P, P, P]
    lib.kgb_selfplay_launches_per_step.argtypes = [P]
    lib.kgb_selfplay_play_moves.argtypes = [P, P, I]
    lib.kgb_selfplay_random_openings.argtypes = [P, I]
    lib.kgb_selfplay_get_root_value_stats.argtypes = [P, I, P, P]
    lib.kgb_selfplay_get_root_weights.argtypes = [P, I, P, P]
    lib.kgb_selfplay_get_root_utility.argtypes = [P, I, P]
    lib.kgb_selfplay_debug_set_raw_outputs.argtypes = [P, I, P, P, P, P]
    lib.kgb_test_uncertainty_weight.argtypes = [I, P, P, P, P]
    lib.kgb_selfplay_release.argtypes = [P, P]
    lib.kgb_selfplay_get_root_visits.argtypes = [P, P]
    lib.kgb_selfplay_get_root_extra.argtypes = [P, I, P, P]
    lib.kgb_selfplay_get_last_move.argtypes = [P, I, P, P, P, P]
    lib.kgb_selfplay_set_search_rand.argtypes = [P, C.c_char_p]
    lib.kgb_selfplay_time_tree_kernels.argtypes = [P, I, F, F]
    lib.kgb_selfplay_debug_cycles.argtypes = [P, P, I]
    lib.kgb_zobrist_tables.argtypes = [I, I, P, P]
    lib.kgb_selfplay_get_nn_row.argtypes = [P, I, P, P]
    lib.kgb_selfplay_get_root_row.argtypes = [P, I, P, P]
    lib.kgb_expected_white_score_value.argtypes = [I, P, P, P, P, P, P]
    lib.kgb_value_weight_cdf_table.argtypes = [P, I]
    lib.kgb_rand_uint32_stream.argtypes = [C.c_char_p, I, P]
    lib.kgb_test_repetition_bound.argtypes = [I, I, I, I, P, P]
    lib.kgb_test_history_replay.argtypes = [I, I, I, I, I, I, P, P, P, P]
    lib.kgb_selfplay_get_play_selection_values.argtypes = [P, I, P]
    lib.kgb_test_choose_index_with_temperature.argtypes = [C.c_char_p, P, I, C.c_double, C.c_double, I, P]
    lib.kgb_test_root_policy_noise.argtypes = [C.c_char_p, I, I, I, I, I, C.c_double, C.c_double, C.c_double, C.c_double, C.c_double, P, P]
    lib.kgb_selfplay_get_leaf_path.argtypes = [P, I, P, I, C.POINTER(C.c_int32), C.POINTER(C.c_int32)]
    lib.kgb_test_board_replay.argtypes = [I, I, I, I, I, P, P, P, P, P, P, P, P]
    _lib = lib
    return lib


def _check(rc: int):
    if rc != 0:
        raise KGBError(load_library().kgb_last_error().decode("utf-8", "replace"))


class LoadedModel:
    """LoadedModel (nninterface.h:27).  `.desc` mirrors the ModelDesc fields NNEvaluator reads."""

    def __init__(self, file: str, expectedSha256: str = ""):
        lib = load_library()
        self._p = C.c_void_p()
        _check(lib.kgb_model_load_file(file.encode(), (expectedSha256 or "").encode(), C.byref(self._p)))
        info = _ModelInfo()
        _check(lib.kgb_model_get_info(self._p, C.byref(info)))
        self.desc = {k: (getattr(info, k).decode() if isinstance(getattr(info, k), bytes) else getattr(info, k))
                     for k, _ in _ModelInfo._fields_}

    def free(self):
        if self._p:
            load_library().kgb_model_free(self._p)
            self._p = C.c_void_p()

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


class ComputeContext:
    def __init__(self, gpuIdxs: Sequence[int], nnXLen: int, nnYLen: int, useFP16Mode, loadedModel: LoadedModel):
        lib = load_library()
        arr = (C.c_int * max(1, len(gpuIdxs)))(*gpuIdxs)
        fp16 = {True: 1, False: 0, None: -1, "auto": -1, "true": 1, "false": 0}.get(useFP16Mode, useFP16Mode)
        self._p = C.c_void_p()
        self.nnXLen, self.nnYLen, self.model = nnXLen, nnYLen, loadedModel
        _check(lib.kgb_context_create(arr, len(gpuIdxs), nnXLen, nnYLen, int(fp16), loadedModel._p, C.byref(self._p)))

    def free(self):
        if self._p:
            load_library().kgb_context_free(self._p)
            self._p = C.c_void_p()

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


class ComputeHandle:
    def __init__(self, context: ComputeContext, loadedModel: LoadedModel, maxBatchSize: int, requireExactNNLen: bool,
                 inputsUseNHWC: bool, gpuIdxForThisThread: int = -1):
        lib = load_library()
        self._p = C.c_void_p()
        self.context, self.model = context, loadedModel
        self.maxBatchSize, self.inputsUseNHWC = maxBatchSize, inputsUseNHWC
        _check(lib.kgb_handle_create(context._p, loadedModel._p, maxBatchSize, int(requireExactNNLen), int(inputsUseNHWC),
                                     gpuIdxForThisThread, C.byref(self._p)))

    @property
    def launches_per_forward(self) -> int:
        return load_library().kgb_handle_launches_per_forward(self._p)

    def layout_stats(self) -> dict:
        """The row layout of the last forward or self-play wave on this handle (waits for its stream): rows and 128-row tiles
        the convolutions ran over, and segments (board widths)."""
        v = [C.c_int64() for _ in range(3)]
        _check(load_library().kgb_handle_get_layout_stats(self._p, *(C.byref(x) for x in v)))
        return dict(zip(("rows", "m_tiles", "segments"), (int(x.value) for x in v)))

    @property
    def stream(self) -> int:
        return load_library().kgb_handle_stream(self._p)

    def sync(self):
        _check(load_library().kgb_handle_sync(self._p))

    # ---- new weights into the live handle (kgb200.h: kgb_handle_stage_weights ...) ----
    @property
    def weights_bytes(self) -> int:
        n = C.c_uint64()
        _check(load_library().kgb_handle_weights_bytes(self._p, C.byref(n)))
        return int(n.value)

    def stage_weights(self, loadedModel: LoadedModel):
        """Pack another net of the same architecture into the shadow arena (evaluation continues meanwhile)."""
        _check(load_library().kgb_handle_stage_weights(self._p, loadedModel._p))

    def wait_staged(self):
        _check(load_library().kgb_handle_wait_staged(self._p))

    def commit_weights(self):
        """Every forward pass / wave enqueued after this call runs the staged (or received) net."""
        _check(load_library().kgb_handle_commit_weights(self._p))

    def comm_init(self, unique_id: bytes, rank: int, num_ranks: int):
        if len(unique_id) != 128:
            raise ValueError("comm_init: the NCCL unique id is 128 bytes")
        buf = C.create_string_buffer(unique_id, 128)
        _check(load_library().kgb_handle_comm_init(self._p, C.cast(buf, C.c_void_p), rank, num_ranks))

    def broadcast_staged_weights(self, root: int = 0) -> float:
        """ncclBroadcast of the packed weight arena from `root`'s shadow arena into every rank's; returns the device time in ms."""
        ms = C.c_float()
        _check(load_library().kgb_handle_broadcast_staged_weights(self._p, root, C.byref(ms)))
        return float(ms.value)

    def free(self):
        if self._p:
            load_library().kgb_handle_free(self._p)
            self._p = C.c_void_p()

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


def nccl_unique_id() -> bytes:
    """ncclGetUniqueId through the library (one rank calls it; the bytes reach the others by any side channel)."""
    buf = C.create_string_buffer(128)
    _check(load_library().kgb_nccl_unique_id(C.cast(buf, C.c_void_p)))
    return buf.raw


def _f32(a):
    return np.ascontiguousarray(a, dtype=np.float32)


class NeuralNet:
    """Static functions named as in `namespace NeuralNet`."""

    @staticmethod
    def globalInitialize():
        _check(load_library().kgb_global_init())

    @staticmethod
    def globalCleanup():
        _check(load_library().kgb_global_cleanup())

    @staticmethod
    def printDevices():
        lib = load_library()
        n = C.c_int(0)
        _check(lib.kgb_device_count(C.byref(n)))
        out = []
        for i in range(n.value):
            buf = C.create_string_buffer(256)
            ma, mi = C.c_int(0), C.c_int(0)
            _check(lib.kgb_device_name(i, buf, 256, C.byref(ma), C.byref(mi)))
            out.append((i, buf.value.decode(), ma.value, mi.value))
            print(f"Found CUDA device {i}: {buf.value.decode()} (sm_{ma.value}{mi.value})")
        return out

    @staticmethod
    def loadModelFile(file: str, expectedSha256: str = "") -> LoadedModel:
        return LoadedModel(file, expectedSha256)

    @staticmethod
    def freeLoadedModel(m: LoadedModel):
        m.free()

    @staticmethod
    def getModelDesc(m: LoadedModel) -> dict:
        return m.desc

    @staticmethod
    def createComputeContext(gpuIdxs, nnXLen, nnYLen, useFP16Mode, loadedModel) -> ComputeContext:
        return ComputeContext(gpuIdxs, nnXLen, nnYLen, useFP16Mode, loadedModel)

    @staticmethod
    def freeComputeContext(c: ComputeContext):
        c.free()

    @staticmethod
    def createComputeHandle(context, loadedModel, maxBatchSize, requireExactNNLen, inputsUseNHWC, gpuIdxForThisThread=-1,
                            serverThreadIdx=0) -> ComputeHandle:
        return ComputeHandle(context, loadedModel, maxBatchSize, requireExactNNLen, inputsUseNHWC, gpuIdxForThisThread)

    @staticmethod
    def freeComputeHandle(h: ComputeHandle):
        h.free()

    @staticmethod
    def isUsingFP16(h: ComputeHandle) -> bool:
        return bool(load_library().kgb_handle_is_fp16(h._p))

    @staticmethod
    def getOutput(handle: ComputeHandle, spatial, global_, symmetry=None, policyOptimism=None, includeOwnerMap=True, meta=None) -> dict:
        """spatial [n, C*X*Y] (layout per inputsUseNHWC), global_ [n, G] -> dict(policy [n,X*Y+1], value [n,3],
        score_value [n,6], ownership [n,X*Y] or None); raw logits as NeuralNet::getOutput writes into NNOutput.  meta [n, 192]:
        the SGF-metadata rows (SGFMetadata::fillMetadataRow) an SGF-metadata net needs, and only such a net takes."""
        lib = load_library()
        sp, gl = _f32(spatial), _f32(global_)
        n = sp.shape[0]
        xy = handle.context.nnXLen * handle.context.nnYLen
        d = handle.model.desc
        if sp.size != n * d["num_input_channels"] * xy or gl.size != n * d["num_input_global_channels"]:
            raise KGBError("getOutput: input buffer sizes do not match the model / nnXLen*nnYLen")
        sym = np.zeros(n, np.int32) if symmetry is None else np.ascontiguousarray(symmetry, dtype=np.int32)
        opt = np.zeros(n, np.float32) if policyOptimism is None else _f32(policyOptimism)
        policy = np.empty((n, xy + 1), np.float32)
        value = np.empty((n, 3), np.float32)
        score = np.empty((n, 6), np.float32)
        own = np.empty((n, xy), np.float32) if includeOwnerMap else None
        outs = (policy.ctypes.data, value.ctypes.data, score.ctypes.data, own.ctypes.data if own is not None else None)
        if meta is None:
            _check(lib.kgb_forward(handle._p, n, sp.ctypes.data, gl.ctypes.data, sym.ctypes.data, opt.ctypes.data, *outs))
        else:
            mt = _f32(meta)
            if mt.size != n * 192:
                raise KGBError("getOutput: meta must hold 192 floats per row")
            _check(lib.kgb_forward_meta(handle._p, n, sp.ctypes.data, gl.ctypes.data, mt.ctypes.data, sym.ctypes.data, opt.ctypes.data, *outs))
        return dict(policy=policy, value=value, score_value=score, ownership=own)

    @staticmethod
    def testEvaluateConv(convYSize, convXSize, inChannels, outChannels, weights, batchSize, nnXLen, nnYLen, useFP16, inputBuffer):
        """NeuralNet::testEvaluateConv (nninterface.h:134-143), NHWC; weights in model-file order [ky][kx][ic][oc]."""
        lib = load_library()
        w, x = _f32(weights), _f32(inputBuffer)
        out = np.empty((batchSize, nnYLen, nnXLen, outChannels), np.float32)
        _check(lib.kgb_test_conv(convYSize, convXSize, inChannels, outChannels, w.ctypes.data, batchSize, nnXLen, nnYLen,
                                 int(bool(useFP16)), x.ctypes.data, out.ctypes.data))
        return out


def test_conv_epilogue(ky, kx, in_c, out_c, weights, n, nn_x_len, nn_y_len, use_fp16, kind, x, residual=None, bn_scale=None, bn_bias=None,
                       activation=2):
    """One convolution launch with a production epilogue (include/kgb200.h kgb_test_conv_epilogue): kind 1 = BN + act + mask -> fp16
    operand, 2 = + residual stream updated in place, 3 = raw stream + operand, 4 = kind 2 with an fp32 residual stream in fp16 mode
    too.  Returns (raw or None, act), NHWC."""
    if kind not in (1, 2, 3, 4):
        raise ValueError(f"test_conv_epilogue: epilogue kind {kind} is not 1-4")
    lib = load_library()
    w, xx = _f32(weights), _f32(x)
    raw = np.zeros((n, nn_y_len, nn_x_len, out_c), np.float32)
    act = np.zeros((n, nn_y_len, nn_x_len, out_c), np.float32)
    res = _f32(residual) if residual is not None else None
    sc = _f32(bn_scale) if bn_scale is not None else None
    bi = _f32(bn_bias) if bn_bias is not None else None
    _check(lib.kgb_test_conv_epilogue(ky, kx, in_c, out_c, w.ctypes.data, n, nn_x_len, nn_y_len, int(bool(use_fp16)), kind, xx.ctypes.data,
                                      res.ctypes.data if res is not None else None, sc.ctypes.data if sc is not None else None,
                                      bi.ctypes.data if bi is not None else None, activation, raw.ctypes.data, act.ctypes.data))
    return (raw if kind >= 2 else None), act


def test_conv_ex(ky, kx, in_c, out_c, weights, n, nn_x_len, nn_y_len, use_fp16, kind, x, board_xy=None, ncbias=None, residual=None,
                 bn_scale=None, bn_bias=None, activation=2):
    """One convolution launch with every epilogue input (include/kgb200.h kgb_test_conv_ex): kinds 0-4 as in test_conv_epilogue, 5 and
    6 = kinds 2 and 4 without the raw output; board_xy [n][2] = (X_i, Y_i) boards in the top-left of the frame (None = the whole frame),
    ncbias [n][out_c], residual in fp32, activation 0-3.  Returns (raw or None, act hi or None, act lo or None), NHWC; lo only in split
    mode."""
    if kind not in (0, 1, 2, 3, 4, 5, 6):
        raise ValueError(f"test_conv_ex: epilogue kind {kind} is not 0-6")
    lib = load_library()
    shape = (n, nn_y_len, nn_x_len, out_c)
    w, xx = _f32(weights), _f32(x)
    raw = np.zeros(shape, np.float32) if kind in (0, 2, 3, 4) else None
    hi = np.zeros(shape, np.float32) if kind != 0 else None
    lo = np.zeros(shape, np.float32) if kind != 0 and not use_fp16 else None
    bxy = np.ascontiguousarray(board_xy, dtype=np.int32) if board_xy is not None else None
    opt = [_f32(a) if a is not None else None for a in (ncbias, residual, bn_scale, bn_bias)]
    ptr = lambda a: a.ctypes.data if a is not None else None
    _check(lib.kgb_test_conv_ex(ky, kx, in_c, out_c, w.ctypes.data, n, nn_x_len, nn_y_len, int(bool(use_fp16)), kind, xx.ctypes.data,
                                ptr(bxy), *[ptr(a) for a in opt], activation, ptr(raw), ptr(hi), ptr(lo)))
    return raw, hi, lo


def test_conv_plan(ky, kx, in_c, out_c, weights, n, nn_x_len, nn_y_len, use_fp16, kind, x, board_xy, symmetry, ragged, ncbias=None,
                   residual=None, bn_scale=None, bn_bias=None, activation=2):
    """test_conv_ex under a row plan made on the device (include/kgb200.h kgb_test_conv_plan): boards board_xy [n][2] ((0, 0): an empty
    mask) moved by symmetry [n], ragged or at the full frame.  x is given before the symmetry and must be zero off the board; residual,
    ncbias and the outputs are after it.  Returns (raw, hi, lo, layout stats dict, plan int32 [n][5] = box x0, y0, w, h, first row)."""
    lib = load_library()
    shape = (n, nn_y_len, nn_x_len, out_c)
    w, xx = _f32(weights), _f32(x)
    raw = np.zeros(shape, np.float32) if kind in (0, 2, 3, 4) else None
    hi = np.zeros(shape, np.float32) if kind != 0 else None
    lo = np.zeros(shape, np.float32) if kind != 0 and not use_fp16 else None
    bxy = np.ascontiguousarray(board_xy, dtype=np.int32)
    sym = np.ascontiguousarray(symmetry, dtype=np.int32)
    opt = [_f32(a) if a is not None else None for a in (ncbias, residual, bn_scale, bn_bias)]
    stats = np.zeros(3, np.int64)
    plan = np.zeros((n, 5), np.int32)
    ptr = lambda a: a.ctypes.data if a is not None else None
    _check(lib.kgb_test_conv_plan(ky, kx, in_c, out_c, w.ctypes.data, n, nn_x_len, nn_y_len, int(bool(use_fp16)), kind, xx.ctypes.data,
                                  bxy.ctypes.data, sym.ctypes.data, int(bool(ragged)), *[ptr(a) for a in opt], activation, ptr(raw), ptr(hi),
                                  ptr(lo), stats.ctypes.data, plan.ctypes.data))
    return raw, hi, lo, dict(rows=int(stats[0]), m_tiles=int(stats[1]), segments=int(stats[2])), plan


def test_conv_boundary_ex(inner_c, trunk_c, n, nn_x_len, nn_y_len, inner_a, exit_w, trunk_s, trunk_scale, trunk_bias, entry_w, inner_scale,
                          inner_bias, board_xy=None, symmetry=None, ragged=None, trunk_fp32=False, inner_fp32=False, fused=True):
    """The fused block boundary on caller data (include/kgb200.h kgb_test_conv_boundary_ex): inner_a [n][y][x][inner_c], exit_w
    [inner_c][trunk_c], trunk_s [n][y][x][trunk_c], entry_w [trunk_c][inner_c], BN constants per channel.  ragged None is the frame
    layout, else plan mode with board_xy moved by symmetry.  Returns (trunk stream, inner stream, inner operand), NHWC float32, and
    the layout stats dict in plan mode (else None)."""
    lib = load_library()
    arrs = [_f32(a) for a in (inner_a, exit_w, trunk_s, trunk_scale, trunk_bias, entry_w, inner_scale, inner_bias)]
    s_out = np.zeros((n, nn_y_len, nn_x_len, trunk_c), np.float32)
    i_out = np.zeros((n, nn_y_len, nn_x_len, inner_c), np.float32)
    a_out = np.zeros((n, nn_y_len, nn_x_len, inner_c), np.float32)
    bxy = np.ascontiguousarray(board_xy, dtype=np.int32) if board_xy is not None else None
    sym = np.ascontiguousarray(symmetry, dtype=np.int32) if symmetry is not None else None
    stats = np.zeros(3, np.int64)
    ptr = lambda a: a.ctypes.data if a is not None else None
    _check(lib.kgb_test_conv_boundary_ex(inner_c, trunk_c, n, nn_x_len, nn_y_len, *[a.ctypes.data for a in arrs], ptr(bxy), ptr(sym),
                                         -1 if ragged is None else int(bool(ragged)), int(bool(trunk_fp32)), int(bool(inner_fp32)),
                                         int(bool(fused)), s_out.ctypes.data, i_out.ctypes.data, a_out.ctypes.data, stats.ctypes.data))
    layout = None if ragged is None else dict(rows=int(stats[0]), m_tiles=int(stats[1]), segments=int(stats[2]))
    return s_out, i_out, a_out, layout


CONV_KERNELS = ("kgb_conv_wg_kernel", "kgb_conv_wg_epi_kernel", "kgb_conv_pair_kernel", "kgb_conv_pair_epi_kernel")


def test_last_conv_kernel():
    """The kernel the last convolution test hook launched (include/kgb200.h kgb_test_last_conv_kernel), by name (CONV_KERNELS)."""
    lib = load_library()
    k = C.c_int(-1)
    _check(lib.kgb_test_last_conv_kernel(C.byref(k)))
    return CONV_KERNELS[k.value]


HEAD_KERNELS = {"pack": 0, "gpool": 1, "bias_act": 2, "matmul": 3, "policy": 4, "ownership": 5, "finalize": 6}


def test_head_kernel(which, n, nn_x_len, nn_y_len, iparams, inputs, output_shapes, board_xy=None, symmetry=None, ragged=True, pad=1):
    """One launch of an fp32 evaluator kernel (include/kgb200.h kgb_test_head_kernel).  inputs: arrays or None, in the hook's order;
    output_shapes: a shape per output, or None for an output not asked for.  Returns (outputs, layout stats dict or None, plan)."""
    lib = load_library()
    ins = [None if a is None else _f32(a) for a in inputs]
    outs = [None if s is None else np.zeros(s, np.float32) for s in output_shapes]
    in_ptrs = (C.c_void_p * len(ins))(*[None if a is None else a.ctypes.data for a in ins])
    out_ptrs = (C.c_void_p * len(outs))(*[None if a is None else a.ctypes.data for a in outs])
    ip = np.ascontiguousarray(iparams, dtype=np.int32)
    bxy = None if board_xy is None else np.ascontiguousarray(board_xy, dtype=np.int32)
    sym = None if symmetry is None else np.ascontiguousarray(symmetry, dtype=np.int32)
    stats = np.zeros(3, np.int64)
    plan = np.zeros((n, 5), np.int32)
    ptr = lambda a: a.ctypes.data if a is not None else None
    _check(lib.kgb_test_head_kernel(HEAD_KERNELS[which], n, nn_x_len, nn_y_len, pad, ptr(bxy), ptr(sym), int(bool(ragged)), ip.ctypes.data, len(ip),
                                    C.cast(in_ptrs, C.c_void_p), len(ins), C.cast(out_ptrs, C.c_void_p), len(outs), stats.ctypes.data,
                                    plan.ctypes.data))
    planned = which not in ("matmul", "finalize")
    return outs, (dict(rows=int(stats[0]), m_tiles=int(stats[1]), segments=int(stats[2])) if planned else None), plan


def zobrist_tables(x_size: int, y_size: int):
    """(board_hash uint64 [Y, X, 2 colours, 2], size_hash uint64 [2]) - the reference's Zobrist data (Board::initHash)."""
    lib = load_library()
    bh = np.zeros((y_size, x_size, 2, 2), np.uint64)
    sh = np.zeros(2, np.uint64)
    _check(lib.kgb_zobrist_tables(x_size, y_size, bh.ctypes.data, sh.ctypes.data))
    return bh, sh


def root_policy_noise(seed_string, x, y, policy, turn_number=0, noise=True, concentration=10.83, weight=0.25, temperature=1.0,
                      temperature_early=1.0, halflife=19.0):
    """The device loop's root temperature + Dirichlet noise on `policy` (-1 = illegal), Rand seeded from seed_string (GPU)."""
    pin = np.ascontiguousarray(policy, np.float32); out = np.zeros_like(pin)
    _check(load_library().kgb_test_root_policy_noise(seed_string.encode(), x, y, pin.size, turn_number, int(noise), concentration, weight,
                                                     temperature, temperature_early, halflife, pin.ctypes.data, out.ctypes.data))
    return out


def choose_index_with_temperature(seed_string, relative_probs, temperature, only_below_prob=1.0, count=1):
    p = np.ascontiguousarray(relative_probs, np.float64); out = np.zeros(count, np.int32)
    _check(load_library().kgb_test_choose_index_with_temperature(seed_string.encode(), p.ctypes.data, p.size, temperature, only_below_prob, count,
                                                                 out.ctypes.data))
    return out


def repetition_bound(x, y, moves_xyp, bound=11):
    mv = np.ascontiguousarray(moves_xyp, np.int8); out = np.zeros(len(mv), np.uint8)
    _check(load_library().kgb_test_repetition_bound(x, y, len(mv), bound, mv.ctypes.data, out.ctypes.data))
    return out


def history_replay(x, y, ko_rule, multi_stone_suicide_legal, moves):
    """moves [games, max_moves, 2] int8 (x, y; -1 pass; -2 end).  Returns flags [g, m], legal_next [g, m, y*x], banned [g, m, y*x] (GPU)."""
    mv = np.ascontiguousarray(moves, np.int8)
    g, m = mv.shape[:2]
    flags = np.zeros((g, m), np.uint8); legal = np.zeros((g, m, x * y), np.uint8); banned = np.zeros((g, m, x * y), np.uint8)
    _check(load_library().kgb_test_history_replay(x, y, ko_rule, int(multi_stone_suicide_legal), g, m, mv.ctypes.data, flags.ctypes.data,
                                                  legal.ctypes.data, banned.ctypes.data))
    return flags, legal, banned


def rand_uint32_stream(seed_string: str, n: int):
    out = np.zeros(n, np.uint32)
    _check(load_library().kgb_rand_uint32_stream(seed_string.encode(), n, out.ctypes.data))
    return out


def value_weight_cdf_table():
    out = np.zeros(2000, np.float64)
    _check(load_library().kgb_value_weight_cdf_table(out.ctypes.data, 2000))
    return out


def expected_white_score_value(mean, stdev, center, scale, sqrt_board_area):
    """ScoreValue::expectedWhiteScoreValue for arrays of arguments (host-side lookup in the table the device loop uses)."""
    a = [np.ascontiguousarray(np.broadcast_to(np.asarray(v, np.float64), np.shape(mean))) for v in (mean, stdev, center, scale, sqrt_board_area)]
    out = np.zeros(a[0].shape, np.float64)
    _check(load_library().kgb_expected_white_score_value(out.size, *[v.ctypes.data for v in a], out.ctypes.data))
    return out


def uncertainty_weight(model_version, raw_winloss, raw_score, value_error_multiplier=0.25, score_error_multiplier=30.0, coeff=0.25,
                       exponent=1.0, max_weight=8.0, win_loss_utility_factor=1.0, static_score_utility_factor=0.0,
                       dynamic_score_utility_factor=0.0, dynamic_score_center_scale=1.0, center=0.0, sqrt_board_area=19.0,
                       white_score_mean=0.0):
    """kgb_test_uncertainty_weight for arrays of arguments: (shorttermWinlossError, shorttermScoreError, weight), the short-term
    error post-processing of the net's raw channels 4 and 5 and Search::computeWeightFromNNOutput as the device loop does them."""
    ver = np.ascontiguousarray(np.asarray(model_version, np.int32).reshape(-1))
    n = ver.size
    col = lambda v: np.broadcast_to(np.asarray(v, np.float64).reshape(-1), (n,))
    raw = np.ascontiguousarray(np.stack([col(raw_winloss), col(raw_score)], axis=1))
    params = np.ascontiguousarray(np.stack([col(v) for v in (value_error_multiplier, score_error_multiplier, coeff, exponent, max_weight,
                                                             win_loss_utility_factor, static_score_utility_factor, dynamic_score_utility_factor,
                                                             dynamic_score_center_scale, center, sqrt_board_area, white_score_mean)], axis=1))
    out = np.zeros((n, 3), np.float64)
    _check(load_library().kgb_test_uncertainty_weight(n, ver.ctypes.data, raw.ctypes.data, params.ctypes.data, out.ctypes.data))
    return out[:, 0], out[:, 1], out[:, 2]


def board_replay(x_size: int, y_size: int, moves, multi_stone_suicide_legal: bool):
    """kgb_test_board_replay: moves int8 [boards, m, 3] = (x, y, pla) with (-1,-1) = pass, pla 1 black / 2 white.
    Returns dict(colors [b,m,Y,X], ko [b,m,2], caps [b,m,2], lib_class [b,m,Y,X], legal_next [b,m,Y,X])."""
    lib = load_library()
    mv = np.ascontiguousarray(moves, dtype=np.int8)
    nb, nm = mv.shape[0], mv.shape[1]
    colors = np.zeros((nb, nm, y_size, x_size), np.uint8)
    libc = np.zeros_like(colors); legal = np.zeros_like(colors)
    ko = np.zeros((nb, nm, 2), np.int8); caps = np.zeros((nb, nm, 2), np.int16)
    pos_hash = np.zeros((nb, nm, 2), np.uint64)
    area = np.zeros_like(colors)
    _check(lib.kgb_test_board_replay(x_size, y_size, nb, nm, int(bool(multi_stone_suicide_legal)), mv.ctypes.data, colors.ctypes.data,
                                     ko.ctypes.data, caps.ctypes.data, libc.ctypes.data, legal.ctypes.data, pos_hash.ctypes.data,
                                     area.ctypes.data))
    return dict(colors=colors, ko=ko, caps=caps, lib_class=libc, legal_next=legal, pos_hash=pos_hash, area=area)


class SelfPlay:
    """Device-resident self-play slots on one ComputeHandle (include/kgb200.h "Boundary 2")."""

    def __init__(self, handle: ComputeHandle, num_games: int, max_visits: int, komi: float = 7.5, max_moves: int = 0,
                 multi_stone_suicide_legal: bool = True, early_temperature_moves: int = 30, cpuct_exploration: float = 1.0,
                 cpuct_exploration_log: float = 0.45, cpuct_exploration_base: float = 500.0, fpu_reduction_max: float = 0.2,
                 root_fpu_reduction_max: float = 0.1, win_loss_utility_factor: float = 1.0, no_result_utility_for_white: float = 0.0,
                 seed: int = 0, debug_fake_nn: int = 0, disable_ladder_features: bool = False, ladder_nodes_per_wave: int = 0, max_playouts_per_wave: int = 0,
                 static_score_utility_factor: float = 0.0, dynamic_score_utility_factor: float = 0.0,
                 dynamic_score_center_zero_weight: float = 0.0, dynamic_score_center_scale: float = 1.0,
                 draw_equivalent_wins_for_white: float = 0.5, value_weight_exponent: float = 0.0,
                 fpu_parent_weight_by_visited_policy: bool = False, fpu_parent_weight_by_visited_policy_pow: float = 1.0,
                 fpu_parent_weight: float = 0.0, fpu_loss_prop: float = 0.0, root_fpu_loss_prop: float = 0.0,
                 cpuct_utility_stdev_prior: float = 0.25, cpuct_utility_stdev_prior_weight: float = 1.0,
                 cpuct_utility_stdev_scale: float = 0.0, root_desired_per_child_visits_coeff: float = 0.0,
                 subtree_value_bias_factor: float = 0.0, subtree_value_bias_weight_exponent: float = 0.5,
                 use_graph_search: bool = False, graph_search_rep_bound: int = 11, debug_hold_at_max_visits: bool = False,
                 root_noise_enabled: bool = False, root_dirichlet_noise_total_concentration: float = 10.83,
                 root_dirichlet_noise_weight: float = 0.25, root_policy_temperature: float = 1.0,
                 root_policy_temperature_early: float = 1.0, chosen_move_temperature_halflife: float = 19.0,
                 use_play_selection: bool = False, use_lcb_for_selection: bool = False, use_non_buggy_lcb: bool = False,
                 lcb_stdevs: float = 4.0, min_visit_prop_for_lcb: float = 0.05, chosen_move_temperature: float = 0.0,
                 chosen_move_temperature_early: float = 0.0, chosen_move_temperature_only_below_prob: float = 1.0,
                 chosen_move_subtract: float = 0.0, chosen_move_prune: float = 1.0, nn_cache_size_power_of_two: int = 0, root_num_symmetries_to_sample: int = 1,
                 ko_rule: int = 0, full_history_rules: bool = True, debug_fixed_symmetry: int = -1,
                 root_ending_bonus_points: float = 0.0, root_prune_useless_moves: bool = False,
                 use_uncertainty: bool = False, uncertainty_coeff: float = 0.25, uncertainty_exponent: float = 1.0,
                 uncertainty_max_weight: float = 8.0, use_noise_pruning: bool = False, noise_prune_utility_scale: float = 0.15,
                 noise_pruning_cap: float = 1e50):
        # The loop always plays BoardHistory's game-end rules.  full_history_rules stays a keyword because bench.py passes it;
        # False is refused rather than silently ignored.
        if not full_history_rules:
            raise ValueError("SelfPlay: the loop always plays the full game-end rules; full_history_rules=False is not supported")
        lib = load_library()
        self.handle = handle
        self.cfg = SelfplayConfig(num_games, max_visits, max_moves, int(multi_stone_suicide_legal), early_temperature_moves, komi,
                                  cpuct_exploration, cpuct_exploration_log, cpuct_exploration_base, fpu_reduction_max,
                                  root_fpu_reduction_max, win_loss_utility_factor, no_result_utility_for_white, seed, int(debug_fake_nn), int(disable_ladder_features),
                                  int(ladder_nodes_per_wave), int(max_playouts_per_wave), static_score_utility_factor, dynamic_score_utility_factor,
                                  dynamic_score_center_zero_weight, dynamic_score_center_scale, draw_equivalent_wins_for_white,
                                  value_weight_exponent, int(fpu_parent_weight_by_visited_policy), int(debug_fixed_symmetry) + 1, fpu_parent_weight_by_visited_policy_pow,
                                  fpu_parent_weight, fpu_loss_prop, root_fpu_loss_prop, cpuct_utility_stdev_prior,
                                  cpuct_utility_stdev_prior_weight, cpuct_utility_stdev_scale, root_desired_per_child_visits_coeff,
                                  subtree_value_bias_factor, subtree_value_bias_weight_exponent, int(use_graph_search),
                                  int(graph_search_rep_bound), int(debug_hold_at_max_visits), int(root_noise_enabled),
                                  root_dirichlet_noise_total_concentration, root_dirichlet_noise_weight, root_policy_temperature,
                                  root_policy_temperature_early, chosen_move_temperature_halflife,
                                  int(use_play_selection), int(use_lcb_for_selection), int(use_non_buggy_lcb), int(root_prune_useless_moves), lcb_stdevs, min_visit_prop_for_lcb,
                                  chosen_move_temperature, chosen_move_temperature_early, chosen_move_temperature_only_below_prob,
                                  chosen_move_subtract, chosen_move_prune, int(nn_cache_size_power_of_two), int(root_num_symmetries_to_sample),
                                  int(ko_rule), float(root_ending_bonus_points),
                                  int(use_uncertainty), float(uncertainty_coeff), float(uncertainty_exponent), float(uncertainty_max_weight),
                                  int(use_noise_pruning), float(noise_prune_utility_scale), float(noise_pruning_cap))
        self._p = C.c_void_p()
        _check(lib.kgb_selfplay_create(handle._p, C.byref(self.cfg), C.byref(self._p)))
        self.x, self.y = handle.context.nnXLen, handle.context.nnYLen
        self.num_games, self.max_visits = int(num_games), int(max_visits)

    def run(self, steps: int):
        _check(load_library().kgb_selfplay_run(self._p, steps))

    def set_search_rand(self, seed_string: str):
        """Every game's search-thread generator := Rand(seed_string) (tests)."""
        _check(load_library().kgb_selfplay_set_search_rand(self._p, seed_string.encode()))

    def random_openings(self, max_moves: int):
        """Every game plays its own random number (0..max_moves) of uniformly random legal moves; trees cleared."""
        _check(load_library().kgb_selfplay_random_openings(self._p, max_moves))

    def play_moves(self, moves_xy):
        """moves_xy: iterable of (x, y) or None for pass; applied to every game's root, trees cleared."""
        arr = np.array([(-1, -1) if m is None else (m[0], m[1]) for m in moves_xy], dtype=np.int8).reshape(-1, 2)
        _check(load_library().kgb_selfplay_play_moves(self._p, arr.ctypes.data if len(arr) else None, len(arr)))

    def play_moves_game(self, g: int, moves_xy):
        """The same for game g only (games of different board sizes need different lists)."""
        arr = np.array([(-1, -1) if m is None else (m[0], m[1]) for m in moves_xy], dtype=np.int8).reshape(-1, 2)
        _check(load_library().kgb_selfplay_play_moves_game(self._p, g, arr.ctypes.data if len(arr) else None, len(arr)))

    def nn_row(self, g: int):
        """(spatial [X*Y, 22], global [19]) written by the last wave for game g."""
        sp = np.zeros((self.x * self.y, 22), np.float32); gl = np.zeros(19, np.float32)
        _check(load_library().kgb_selfplay_get_nn_row(self._p, g, sp.ctypes.data, gl.ctypes.data))
        return sp, gl

    def root_row(self, g: int):
        """(spatial [X*Y, 22], global [19]): the fillRowV7 row of game g's current root, kept on the device since the wave that
        evaluated it (kgb_selfplay_get_root_row)."""
        sp = np.zeros((self.x * self.y, 22), np.float32); gl = np.zeros(19, np.float32)
        _check(load_library().kgb_selfplay_get_root_row(self._p, g, sp.ctypes.data, gl.ctypes.data))
        return sp, gl

    def leaf_path(self, g: int, max_len: int = 512):
        """(moves, valid): the (x, y) / None moves from the root to game g's leaf of the last wave; valid = that wave delivered it."""
        mv = np.zeros((max_len, 2), np.int32); n = C.c_int32(0); v = C.c_int32(0)
        _check(load_library().kgb_selfplay_get_leaf_path(self._p, g, mv.ctypes.data, max_len, C.byref(n), C.byref(v)))
        return [None if m[0] < 0 else (int(m[0]), int(m[1])) for m in mv[:min(n.value, max_len)]], bool(v.value)

    def stats(self) -> dict:
        s = SelfplayStats()
        _check(load_library().kgb_selfplay_get_stats(self._p, C.byref(s)))
        return {k: int(getattr(s, k)) for k, _ in SelfplayStats._fields_}

    def game(self, g: int):
        colors = np.zeros((self.y, self.x), np.uint8)
        info = np.zeros(6, np.int32)
        _check(load_library().kgb_selfplay_get_game(self._p, g, colors.ctypes.data, info.ctypes.data))
        return colors, dict(move_num=int(info[0]), black_to_move=bool(info[1]), ko=int(info[2]), cap_b=int(info[3]), cap_w=int(info[4]),
                            root_visits=int(info[5]))

    def root_value_stats(self, g: int):
        """(children [X*Y+1, 5], root [5]): winLossValueAvg, noResultValueAvg, scoreMeanAvg, scoreMeanSqAvg, leadAvg."""
        ch = np.zeros((self.x * self.y + 1, 5), np.float64); rt = np.zeros(5, np.float64)
        _check(load_library().kgb_selfplay_get_root_value_stats(self._p, g, ch.ctypes.data, rt.ctypes.data))
        return ch, rt

    def root_utility(self, g: int):
        """(utility of the root's own evaluation, NodeStats utilityAvg) of game g, white's perspective."""
        out = np.zeros(2, np.float64)
        _check(load_library().kgb_selfplay_get_root_utility(self._p, g, out.ctypes.data))
        return float(out[0]), float(out[1])

    def debug_set_raw_outputs(self, g: int, policy, value, score, ownership=None):
        """debug_fake_nn = 3: every later evaluation of game g returns these raw net outputs (frame-indexed policy logits [X*Y+1],
        value logits [3], score-value channels [6], ownership logits [X*Y]; mover's perspective)."""
        n = self.x * self.y
        arrs = [np.ascontiguousarray(a, np.float32).reshape(-1) for a in (policy, value, score, np.zeros(n) if ownership is None else ownership)]
        if [a.size for a in arrs] != [n + 1, 3, 6, n]:
            raise ValueError(f"raw outputs of sizes {[a.size for a in arrs]}, want {[n + 1, 3, 6, n]}")
        _check(load_library().kgb_selfplay_debug_set_raw_outputs(self._p, g, *(a.ctypes.data for a in arrs)))

    def root_weights(self, g: int):
        """(children [X*Y+1, 2], root [2]): NodeStats weightSum and weightSqSum of game g's root children and root."""
        ch = np.zeros((self.x * self.y + 1, 2), np.float64); rt = np.zeros(2, np.float64)
        _check(load_library().kgb_selfplay_get_root_weights(self._p, g, ch.ctypes.data, rt.ctypes.data))
        return ch, rt

    # ---- game recording (hold mode, kgb200.h) ----
    def release(self, mask=None):
        """Let held games (all, or those with mask[g] != 0) choose and play their move in the next wave."""
        if mask is None:
            _check(load_library().kgb_selfplay_release(self._p, None))
        else:
            m = np.ascontiguousarray(mask, np.uint8)
            if m.shape != (self.num_games,):
                raise ValueError("release: mask must have one entry per game")
            _check(load_library().kgb_selfplay_release(self._p, m.ctypes.data))

    def set_komi(self, komi, also_current_games: bool = False):
        """komi[num_games] for each slot's next game (and, optionally, for the games in progress)."""
        k = np.ascontiguousarray(np.broadcast_to(np.asarray(komi, np.float32), (self.num_games,)))
        _check(load_library().kgb_selfplay_set_komi(self._p, k.ctypes.data, int(also_current_games)))

    def set_game_setup(self, setup, also_current_games: bool = False):
        """setup[num_games][4] = board X, board Y, ko rule (0-3), multi-stone suicide legal, for each slot's next game (and, optionally,
        the games in progress that have not started): what GameInitializer draws per game (program/play.cpp:330-650)."""
        a = np.ascontiguousarray(np.broadcast_to(np.asarray(setup, np.int32), (self.num_games, 4)))
        _check(load_library().kgb_selfplay_set_game_setup(self._p, a.ctypes.data, int(also_current_games)))

    def set_next_search_limits(self, visits, plain_root=None, also_current_roots: bool = False):
        """visits[num_games][2], plain_root[num_games][2]: limits of the root after each slot's next move ([:, 0] the game goes on,
        [:, 1] the move ends it) - cheap searches / reduced visits of Play::runGame (kgb_selfplay_set_next_search_limits)."""
        v = np.ascontiguousarray(np.broadcast_to(np.asarray(visits, np.int32), (self.num_games, 2)))
        p = None if plain_root is None else np.ascontiguousarray(np.broadcast_to(np.asarray(plain_root, np.uint8), (self.num_games, 2)))
        _check(load_library().kgb_selfplay_set_next_search_limits(self._p, v.ctypes.data, None if p is None else p.ctypes.data, int(also_current_roots)))

    def search_limits(self):
        """(visit budget [num_games], plain-root flag [num_games]) of the current roots: a game holds / moves at ITS budget."""
        v = np.zeros(self.num_games, np.int32); p = np.zeros(self.num_games, np.uint8)
        _check(load_library().kgb_selfplay_get_search_limits(self._p, v.ctypes.data, p.ctypes.data))
        return v, p

    def set_policy_init(self, num_moves, temperature: float = 1.0, also_current_games: bool = False):
        """num_moves[num_games]: opening moves the slot's next game draws from the net's raw policy before its first search
        (PlayUtils::initializeGameUsingPolicy; kgb_selfplay_set_policy_init)."""
        a = np.ascontiguousarray(np.broadcast_to(np.asarray(num_moves, np.int32), (self.num_games,)))
        _check(load_library().kgb_selfplay_set_policy_init(self._p, a.ctypes.data, float(temperature), int(also_current_games)))

    def policy_init(self, max_moves: int = 0):
        """(moves_left [num_games], count [num_games], moves) - moves: per game the list of (x, y) / (-1, -1) opening moves played so far (only
        when max_moves > 0)."""
        left = np.zeros(self.num_games, np.int32); cnt = np.zeros(self.num_games, np.int32)
        mv = np.zeros((self.num_games, max_moves), np.int16) if max_moves > 0 else None
        _check(load_library().kgb_selfplay_get_policy_init(self._p, left.ctypes.data, cnt.ctypes.data, None if mv is None else mv.ctypes.data, max_moves))
        moves = None
        if mv is not None:
            n = self.x * self.y
            moves = [[(-1, -1) if int(p) == n else (int(p) % self.x, int(p) // self.x) for p in mv[g, :min(int(cnt[g]), max_moves)]] for g in range(self.num_games)]
        return left, cnt, moves

    def nn_symmetries(self):
        """Symmetry (0-7) of every game's row in the last wave (kgb_selfplay_get_nn_symmetries)."""
        a = np.zeros(self.num_games, np.int32)
        _check(load_library().kgb_selfplay_get_nn_symmetries(self._p, a.ctypes.data))
        return a

    def root_raw_policy_entropy(self):
        """Entropy of every root's policy before temperature and noise (NNRawStats::policyEntropy)."""
        e = np.zeros(self.num_games, np.float64)
        _check(load_library().kgb_selfplay_get_root_raw_policy_entropy(self._p, e.ctypes.data))
        return e

    def game_setups(self):
        """(setup [num_games, 4] of the games in progress, of each slot's last finished game)."""
        cur = np.zeros((self.num_games, 4), np.int32); last = np.zeros((self.num_games, 4), np.int32)
        _check(load_library().kgb_selfplay_get_game_setup(self._p, cur.ctypes.data, last.ctypes.data))
        return cur, last

    def komi_values(self):
        """(komi of the games in progress, komi of each slot's last finished game)."""
        cur = np.zeros(self.num_games, np.float32); last = np.zeros(self.num_games, np.float32)
        _check(load_library().kgb_selfplay_get_komi(self._p, cur.ctypes.data, last.ctypes.data))
        return cur, last

    def leaf_cache_key(self, g: int):
        k = np.zeros(2, np.uint64)
        _check(load_library().kgb_selfplay_get_leaf_cache_key(self._p, g, k.ctypes.data))
        return int(k[0]), int(k[1])

    def clear_nn_cache(self):
        """With ComputeHandle.commit_weights: the cached outputs belong to the previous net."""
        _check(load_library().kgb_selfplay_clear_nn_cache(self._p))

    def root_visits(self):
        out = np.zeros(self.num_games, np.int32)
        _check(load_library().kgb_selfplay_get_root_visits(self._p, out.ctypes.data))
        return out

    def root_extra(self, g: int):
        """Visits of the root's child nodes by move position and the root's own evaluation (winLoss, noResult, scoreMean, scoreMeanSq, lead)."""
        nv = np.zeros(self.x * self.y + 1, np.int32); nn = np.zeros(5, np.float64)
        _check(load_library().kgb_selfplay_get_root_extra(self._p, g, nv.ctypes.data, nn.ctypes.data))
        return dict(child_node_visits=nv, root_nn_moments=nn)

    def last_move(self, g: int):
        info = np.zeros(4, np.int32); score = np.zeros(1, np.float32)
        colors = np.zeros((self.y, self.x), np.uint8); area = np.zeros((self.y, self.x), np.uint8)
        _check(load_library().kgb_selfplay_get_last_move(self._p, g, info.ctypes.data, score.ctypes.data, colors.ctypes.data, area.ctypes.data))
        pos = int(info[0])
        return dict(pos=pos, xy=(-1, -1) if pos == self.x * self.y else (pos % self.x, pos // self.x), game_over=bool(info[1] & 1),
                    no_result=bool(info[1] & 2), hit_move_limit=bool(info[1] & 4), move_num=int(info[2]), game_index=int(info[3]),
                    final_white_minus_black_score=float(score[0]), final_colors=colors, final_area=area)

    def play_selection_values(self, g: int):
        """Search::getPlaySelectionValues of the root by move position (-1 = no child)."""
        out = np.zeros(self.x * self.y + 1, np.float64)
        _check(load_library().kgb_selfplay_get_play_selection_values(self._p, g, out.ctypes.data))
        return out

    def root_children(self, g: int):
        n = self.x * self.y + 1
        visits = np.zeros(n, np.int32); policy = np.zeros(n, np.float32); util = np.zeros(n, np.float64)
        _check(load_library().kgb_selfplay_get_root_children(self._p, g, visits.ctypes.data, policy.ctypes.data, util.ctypes.data))
        return visits, policy, util

    def debug_cycles(self, clear: bool = True):
        """int64 [games, 8]: SM-clock spans of every game's block in the last select launch (whole, root move + reset, warp 0, ladders,
        descent, liberties + legality, area, feature-row writes)."""
        out = np.zeros((self.num_games, 8), np.int64)
        _check(load_library().kgb_selfplay_debug_cycles(self._p, out.ctypes.data, int(clear)))
        return out

    def time_tree_kernels(self, iters: int = 20):
        """(ms_select, ms_backup): CUDA-event averages of the two tree kernels alone (evaluator skipped)."""
        a, b = C.c_float(0), C.c_float(0)
        _check(load_library().kgb_selfplay_time_tree_kernels(self._p, iters, C.byref(a), C.byref(b)))
        return a.value, b.value

    @property
    def launches_per_step(self) -> int:
        return load_library().kgb_selfplay_launches_per_step(self._p)

    def free(self):
        if self._p:
            load_library().kgb_selfplay_free(self._p)
            self._p = C.c_void_p()

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass
