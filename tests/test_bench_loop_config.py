"""bench.py still makes the loop calls tests/test_gpu_bench_loops.py restates: sizes, seeds, arena size and warm-up calls.
When the bench changes, this fails instead of the loop tests quietly checking a configuration the bench no longer runs."""
import os
import re

import test_gpu_bench_loops as loops

BENCH = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "bench.py")


def source():
    with open(BENCH) as f:
        return re.sub(r"[ \t]+", " ", f.read())


def test_restated_bench_calls_are_still_in_bench():
    src = source()
    expected = [
        # MCTS lines: warm-up on the same roots, then the timed search; deep arena of 240,000 nodes per tree
        'go = b2.Game("go", {"board_size": 9}, device=local)',
        "b2.mcts_search(roots, %d, seed=%d, tree_index_offset=rank * trees, max_nodes_total=nodes)" % (
            loops.MCTS_WARMUP_SIMS, loops.MCTS_SEED),
        "out = b2.mcts_search(roots, sims, uct_c=2.0, n_rollouts=1, solve=True, seed=%d, tree_index_offset=rank * trees," % (
            loops.MCTS_SEED),
        'loops["mcts_go9x9"] = mcts_line(%d, %d)' % (loops.MCTS_TREES, loops.MCTS_SIMS),
        'loops["mcts_go9x9_deep"] = mcts_line(args.deep_trees, args.deep_sims, nodes=args.deep_trees * %d)' % (
            loops.DEEP_NODES_PER_TREE),
        'ap.add_argument("--deep-trees", type=int, default=%d,' % loops.DEEP_TREES,
        'ap.add_argument("--deep-sims", type=int, default=%d,' % loops.DEEP_SIMS,
        # breakthrough rollouts: warm-up, reset, full rollout
        'bt = b2.Game("breakthrough", device=local)',
        "games = 1 << %d" % (loops.ROLLOUT_GAMES.bit_length() - 1),
        "bb.rollout(seed=%d, lane_offset=rank * games, n=%d)\n bb.reset()" % (loops.ROLLOUT_SEED, loops.ROLLOUT_WARMUP),
        "rets_r, plies_r = bb.rollout(seed=%d, lane_offset=rank * games)" % loops.ROLLOUT_SEED,
        # CFR: plain CFRSolver, warm-up then the configured iteration count
        'leduc = b2.Game("leduc_poker", device=local)',
        "solver = b2.CFRSolver(leduc)\n solver.evaluate_and_update_policy(%d)" % loops.CFR_WARMUP,
        'ap.add_argument("--cfr-iters", type=int, default=%d,' % loops.CFR_ITERS,
        "solver.evaluate_and_update_policy(iters)",
        '"exploitability": solver.exploitability()',
        # external-sampling MCCFR
        "mc = b2.ExternalSamplingMCCFRSolver(leduc, seed=%d + rank, traversals_per_update=%d)" % (loops.MCCFR_SEED, loops.MCCFR_K),
        "mc.run_iteration(%d)" % loops.MCCFR_WARMUP,
        "mc.run_iteration(%d)" % loops.MCCFR_ITERS,
        # connect_four trajectories: warm-up recording, reset, recording
        'c4 = b2.Game("connect_four", device=local)',
        "eps = 1 << %d" % (loops.EPISODES.bit_length() - 1),
        "tb.record_trajectories(seed=1, lane_offset=rank * eps)\n tb.reset()",
        "tr = tb.record_trajectories(seed=2, lane_offset=rank * eps)",
    ]
    missing = [e for e in expected if e not in src]
    assert not missing, "bench.py no longer makes these calls; update tests/test_gpu_bench_loops.py: %s" % missing
