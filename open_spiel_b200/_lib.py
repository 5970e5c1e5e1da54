"""ctypes loader for libb2s.so (the C ABI declared in include/b2s.h).

The library is built in-tree by open_spiel_b200/csrc/Makefile (see __graft_entry__.build()).  There is
no fallback: if the shared object is missing this module raises, and every compute entry point of the
library itself fails when no CUDA device is present.
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
# B2S_LIBRARY: another build of the same C ABI (A/B kernel measurements); still a CUDA library, not a fallback
SO_PATH = os.environ.get("B2S_LIBRARY") or os.path.join(_HERE, "libb2s.so")


class B2SError(RuntimeError):
    """Mirror of pyspiel.SpielError (python/pybind11/pyspiel.cc:831-837)."""


class Params(C.Structure):
    _fields_ = [
        ("rows", C.c_int32), ("columns", C.c_int32), ("x_in_row", C.c_int32),
        ("egocentric_obs_tensor", C.c_int32), ("board_size", C.c_int32), ("swap", C.c_int32),
        ("plain_obs_tensor", C.c_int32), ("handicap", C.c_int32), ("max_game_length", C.c_int32),
        ("players", C.c_int32), ("starting_player", C.c_int32), ("reserved", C.c_int32 * 5),
        ("komi", C.c_double), ("reserved_d", C.c_double * 3),
    ]


class GameInfo(C.Structure):
    _fields_ = [
        ("game_id", C.c_int32), ("num_players", C.c_int32), ("num_distinct_actions", C.c_int32),
        ("max_game_length", C.c_int32), ("max_chance_outcomes", C.c_int32),
        ("observation_tensor_size", C.c_int32), ("information_state_tensor_size", C.c_int32),
        ("mask_words", C.c_int32), ("state_bytes", C.c_int32), ("history_bytes", C.c_int32),
        ("min_utility", C.c_double), ("max_utility", C.c_double),
        ("obs_shape", C.c_int32 * 4), ("reserved", C.c_int32 * 4),
    ]


class MctsConfig(C.Structure):
    _fields_ = [("max_simulations", C.c_int32), ("n_rollouts", C.c_int32), ("solve", C.c_int32),
                ("child_selection_policy", C.c_int32), ("uct_c", C.c_double), ("seed", C.c_uint64),
                ("tree_index_offset", C.c_int64), ("max_nodes_total", C.c_int64), ("max_nodes_per_tree", C.c_int64),
                ("max_wall_clock_time", C.c_double), ("gc_runs_d", C.c_void_p)]


class TrajectoryOut(C.Structure):
    _fields_ = [("observations", C.c_void_p), ("legal_mask", C.c_void_p), ("actions", C.c_void_p),
                ("player_ids", C.c_void_p), ("valid", C.c_void_p), ("next_is_terminal", C.c_void_p),
                ("rewards", C.c_void_p), ("lengths", C.c_void_p)]


class CfrInfo(C.Structure):
    _fields_ = [("num_nodes", C.c_int32), ("num_levels", C.c_int32), ("num_infosets", C.c_int32),
                ("num_entries", C.c_int32), ("key_floats", C.c_int32), ("iteration", C.c_int32),
                ("chance_nodes", C.c_int32), ("decision_nodes", C.c_int32), ("terminal_nodes", C.c_int32),
                ("reserved", C.c_int32 * 3)]


# name -> (restype, argtypes); the complete export list of include/b2s.h
_VP, _I64, _I32, _U64 = C.c_void_p, C.c_int64, C.c_int32, C.c_uint64
SIGNATURES = {
    "b2s_game_id": (C.c_int, [C.c_char_p]),
    "b2s_params_default": (None, [C.POINTER(Params)]),
    "b2s_game_info_get": (C.c_int, [C.c_int, C.POINTER(Params), C.POINTER(GameInfo)]),
    "b2s_batch_create": (C.c_int, [C.c_int, C.POINTER(Params), _I64, C.c_int, C.POINTER(_VP)]),
    "b2s_batch_destroy": (None, [_VP]),
    "b2s_batch_info": (C.c_int, [_VP, C.POINTER(GameInfo)]),
    "b2s_batch_capacity": (_I64, [_VP]),
    "b2s_reset": (C.c_int, [_VP, _I64, _VP]),
    "b2s_apply_actions": (C.c_int, [_VP, _VP, _I64, _VP]),
    "b2s_legal_mask": (C.c_int, [_VP, _VP, _I64, _VP]),
    "b2s_legal_list": (C.c_int, [_VP, _VP, _VP, _I32, _I64, _VP]),
    "b2s_status": (C.c_int, [_VP, _VP, _VP, _VP, _I64, _VP]),
    "b2s_observation": (C.c_int, [_VP, C.c_int, _VP, _I64, _VP]),
    "b2s_information_state": (C.c_int, [_VP, C.c_int, _VP, _I64, _VP]),
    "b2s_step_fused": (C.c_int, [_VP, _VP, _VP, _VP, _VP, _I64, _VP]),
    "b2s_step_fused_host": (C.c_int, [_VP, _VP, _VP, _VP, _VP, _I64]),
    "b2s_step_fused_host_compact": (C.c_int, [_VP, _VP, C.c_int, _VP, _VP, _I64]),
    "b2s_bind_host_to_device": (C.c_int, [C.c_int, C.POINTER(C.c_int)]),
    "b2s_error_count": (C.c_int, [_VP, C.POINTER(_I64), C.POINTER(_I64), _VP]),
    "b2s_state_get": (C.c_int, [_VP, _I64, _VP, C.c_size_t]),
    "b2s_state_set": (C.c_int, [_VP, _I64, _VP, C.c_size_t]),
    "b2s_broadcast_state": (C.c_int, [_VP, _I64, _I64, _VP, _I64, _VP]),
    "b2s_copy_states": (C.c_int, [_VP, _I64, _VP, _I64, _I64, _VP]),
    "b2s_rollout": (C.c_int, [_VP, _U64, _I64, _I64, _VP, _VP, _VP]),
    "b2s_record_trajectories": (C.c_int, [_VP, _U64, _I64, _I64, C.c_int32, C.POINTER(TrajectoryOut), _VP]),
    "b2s_mcts_search": (C.c_int, [_VP, _I64, C.POINTER(MctsConfig), _VP, _VP, _VP, _VP, _VP, _VP]),
    "b2s_mcts_nodes_used": (C.c_int, [_VP, C.POINTER(_I64)]),
    "b2s_gather_states": (C.c_int, [_VP, _VP, _VP, _I64, _VP]),
    "b2s_cfr_create": (C.c_int, [C.c_int, C.POINTER(Params), C.c_int, C.c_int, C.POINTER(_VP)]),
    "b2s_cfr_destroy": (None, [_VP]),
    "b2s_cfr_iterate": (C.c_int, [_VP, C.c_int, _VP]),
    "b2s_cfr_info_get": (C.c_int, [_VP, C.POINTER(CfrInfo)]),
    "b2s_cfr_export": (C.c_int, [_VP, _VP, _VP, _VP, _VP, _VP, _VP, _VP, _VP]),
    "b2s_cfr_import": (C.c_int, [_VP, _VP, _VP, _VP, C.c_int, _VP]),
    "b2s_cfr_best_response": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]),
    "b2s_cfr_nash_conv": (C.c_int, [_VP, C.c_int, C.POINTER(C.c_double), C.POINTER(C.c_double), _VP]),
    "b2s_cfr_tables": (C.c_int, [_VP, C.POINTER(_VP), C.POINTER(_VP), C.POINTER(_VP)]),
    "b2s_cfr_traverse_shard": (C.c_int, [_VP, C.c_int, C.c_int, C.c_int, C.c_int, _VP]),
    "b2s_cfr_apply_deltas": (C.c_int, [_VP, _VP]),
    "b2s_cfr_delta_buffer": (C.c_int, [_VP, C.POINTER(_VP)]),
    "b2s_cfr_delta_count": (C.c_int, [_VP, C.POINTER(_I64)]),
    "b2s_nccl_unique_id": (C.c_int, [_VP]),
    "b2s_cfr_comm_init": (C.c_int, [_VP, _VP, C.c_int, C.c_int]),
    "b2s_cfr_comm_adopt": (C.c_int, [_VP, _VP, C.c_int, C.c_int]),
    "b2s_cfr_iterate_sharded": (C.c_int, [_VP, C.c_int, _VP]),
    "b2s_cfr_allreduce_probe": (C.c_int, [_VP, C.c_int, C.POINTER(C.c_double)]),
    "b2s_mccfr_external_iterate": (C.c_int, [_VP, C.c_int, C.c_int, _U64, _VP]),
    "b2s_mccfr_external_iterate_ex": (C.c_int, [_VP, C.c_int, C.c_int, _U64, C.c_int, _VP]),
    "b2s_mccfr_outcome_iterate": (C.c_int, [_VP, C.c_int, C.c_int, _U64, C.c_double, _VP]),
    "b2s_mccfr_traverse_lanes": (C.c_int, [_VP, C.c_int, C.c_int, _U64, C.c_int, C.c_int, _VP, _VP]),
    "b2s_mccfr_apply_partials": (C.c_int, [_VP, C.c_int, _VP, _VP]),
    "b2s_cfr_set_iteration": (C.c_int, [_VP, C.c_int]),
    "b2s_host_alloc": (C.c_int, [C.POINTER(_VP), C.c_size_t]),
    "b2s_host_free": (None, [_VP]),
    "b2s_device_alloc": (C.c_int, [C.c_int, C.POINTER(_VP), C.c_size_t]),
    "b2s_device_free": (None, [C.c_int, _VP]),
    "b2s_memcpy_h2d": (C.c_int, [C.c_int, _VP, _VP, C.c_size_t, _VP]),
    "b2s_memcpy_d2h": (C.c_int, [C.c_int, _VP, _VP, C.c_size_t, _VP]),
    "b2s_stream_synchronize": (C.c_int, [C.c_int, _VP]),
    "b2s_device_count": (C.c_int, []),
    "b2s_launch_count": (_I64, []),
    "b2s_host_graph_launches": (_I64, []),
    "b2s_host_zero_copy_steps": (_I64, []),
    "b2s_last_error": (C.c_char_p, []),
    "b2s_version": (C.c_char_p, []),
}

_lib = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(SO_PATH):
            raise B2SError(
                "libb2s.so not built (%s): run `python -c 'import __graft_entry__ as g; g.build()'` "
                "or `make -C open_spiel_b200/csrc`. There is no CPU fallback." % SO_PATH)
        L = C.CDLL(SO_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(L, name)       # AttributeError if the .so does not export a declared symbol
            fn.restype = res
            fn.argtypes = args
        _lib = L
    return _lib


def check(rc):
    if rc != 0:
        raise B2SError(lib().b2s_last_error().decode())
