"""The oracle side of tests/test_gpu_bench_loops.py: one job per sampled tree, lane, episode or solver run, mapped over
a process pool.  The module imports neither torch nor the device library, so the pool's spawned workers start quickly
and never touch the GPU.  Every job builds its own oracle game: ctypes handles do not cross processes."""
import multiprocessing
import os

from oracle_lib import OracleGame, OracleMCCFR, OracleOSMCCFR, oracle_mcts, oracle_record_trajectory


def pool():
    """A pool of spawned workers, one per CPU this process may run on (leave the result in a `with`)."""
    return multiprocessing.get_context("spawn").Pool(len(os.sched_getaffinity(0)))


def mcts_tree(job):
    """oracle_mcts from the initial state of `game` with tree index `tree` (bench.py's searches: uct_c 2, one rollout,
    solve)."""
    game, sims, seed, tree = job
    return oracle_mcts(OracleGame(game).new_initial_state(), 2.0, sims, 1, True, seed, tree_index=tree)


def rollout_lane(job):
    """b2s_rollout of lane `lane` (lane_offset included) replayed on the oracle: uniform over the legal actions by
    rejection from the candidate list on the lane's Philox words (test_gpu_parity_games.py).  Returns (plies, returns)."""
    from philox_ref import philox_uniform
    game, seed, lane = job
    st = OracleGame(game).new_initial_state()
    ply = 0
    while not st.is_terminal():
        la, cand = st.legal_actions(), st.rollout_candidates()
        retry = 0
        while True:
            a = cand[philox_uniform(seed, lane, ply + 4096 * retry, len(cand))]
            if a in la:
                break
            retry += 1
        st.apply_action(a)
        ply += 1
    return ply, st.returns()


def trajectory(job):
    """oracle_record_trajectory of lane `lane` from the initial state."""
    game, seed, lane, T = job
    return oracle_record_trajectory(OracleGame(game).new_initial_state(), seed, lane, T)


def mccfr_tables(job):
    """The oracle's tables after each of `steps` (cumulative iteration counts reached by running steps[i] more).
    kind: "es" (external sampling, simple averaging), "es_full" (full averaging) or "os" (outcome sampling, epsilon 0.6)."""
    kind, game, K, seed, steps = job
    og = OracleGame(game)
    if kind == "os":
        s = OracleOSMCCFR(og, seed=seed, rng_mode=1, trajectories_per_update=K)
    else:
        s = OracleMCCFR(og, seed=seed, rng_mode=1, traversals_per_update=K, full_average=kind == "es_full")
    out = []
    for n in steps:
        s.iterate(n)
        out.append(s.table())
    return out
