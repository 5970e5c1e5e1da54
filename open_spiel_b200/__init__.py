"""open_spiel_b200 — H100-native batched game simulation + search behind OpenSpiel's State/Game API.

Host-side mirror of the reference's Python surface for the hot path (python/pybind11/pyspiel.cc:355-476,
720-735): load_game, Game.new_initial_state, State.{apply_action, legal_actions, ...}, plus the batched
extension (Game.new_batch -> BatchedState) that the kernels exist for.  All compute goes through the
C ABI in include/b2s.h (libb2s.so); torch is used only for device buffers and streams.
"""
from ._lib import B2SError as SpielError  # noqa: F401
from .spiel import (BatchedState, BatchedTrajectory, CFRSolver, ChildSelectionPolicy, ExternalSamplingMCCFRSolver, OutcomeSamplingMCCFRSolver, Game, MCTSBot, RandomRolloutEvaluator, State, load_game, bind_host_to_device, mcts_nodes_used,
                    mcts_search, registered_names)  # noqa: F401
