"""CPU: pins the oracle's MCTS with a deterministic Evaluator (oracle/algorithms/mcts_eval.cc) to the UNMODIFIED reference's
MCTSBot (algorithms/mcts.cc, built by oracle/ref_build.mk) driven by the same test evaluator (oracle/ref_glue/ref_mcts_eval.cc,
built by oracle/ref_eval.mk).  On the reference's own random streams — std::shuffle of the new children and,
with dirichlet_alpha > 0, std::gamma_distribution draws on the bot's std::mt19937 — the restatement must reproduce the search
BIT FOR BIT: the root's children in the same (shuffled) order, their visit counts, their total rewards as exact doubles,
BestChild and the root's visit count.  The device search (b2s_mcts_eval_*) is compared with the same oracle code on the
Philox stream (tests/test_gpu_mcts_eval.py, tests/test_mcts_eval_host.py)."""
import random

import pytest

from mcts_eval_lib import oracle_mcts_eval, ref_eval_available, ref_mcts_eval, ref_sizeof_search_node
from oracle_lib import OracleGame

pytestmark = pytest.mark.skipif(not ref_eval_available(), reason="oracle/_ref/libspiel_ref_mcts_eval.so not built")

CASES = [
    # game, prefix plies, simulations, solve, PUCT, dirichlet_alpha, seed
    ("tic_tac_toe", 0, 500, True, False, 0.0, 1),
    ("tic_tac_toe", 2, 400, False, True, 0.0, 3),
    ("tic_tac_toe", 1, 300, True, True, 0.3, 4),
    ("connect_four", 0, 600, True, False, 0.0, 42),
    ("connect_four", 9, 400, False, True, 0.0, 5),
    ("connect_four", 4, 500, True, True, 1.0, 6),
    ("breakthrough(rows=6,columns=6)", 4, 200, True, True, 0.0, 11),
    ("hex(board_size=5)", 3, 300, True, False, 0.0, 2),
    ("hex(board_size=5)", 1, 300, False, True, 0.5, 8),
    ("go(board_size=5)", 6, 200, True, True, 0.0, 9),
    ("go(board_size=5)", 2, 200, False, True, 0.03, 10),
    ("go(board_size=9)", 10, 80, True, False, 0.0, 13),
    ("othello", 20, 200, True, True, 0.0, 21),
    ("othello", 54, 400, True, False, 0.0, 22),
    ("othello", 10, 200, False, True, 0.3, 27),
    ("mnk(m=5,n=5,k=4)", 6, 200, True, True, 0.0, 23),
    ("y(board_size=5)", 4, 300, True, True, 0.0, 24),
    ("havannah(board_size=3)", 4, 300, True, False, 0.0, 25),
    ("havannah(board_size=4,swap=True)", 10, 200, False, True, 0.3, 26),
]


def _roots(gs, prefix, seed):
    """The root after up to `prefix` random non-terminal plies; returns (oracle state, history)."""
    rng = random.Random(seed)
    st = OracleGame(gs).new_initial_state()
    hist = []
    for _ in range(prefix):
        a = rng.choice(st.legal_actions())
        nxt = st.clone()
        nxt.apply_action(a)
        if nxt.is_terminal():
            break
        st.apply_action(a)
        hist.append(a)
    return st, hist


def _assert_same(mine, ref):
    assert [c[0] for c in mine["children"]] == [c[0] for c in ref["children"]]          # same shuffled child order
    assert [c[1] for c in mine["children"]] == [c[1] for c in ref["children"]]          # visit counts
    assert [c[2] for c in mine["children"]] == [c[2] for c in ref["children"]]          # total rewards, exact doubles
    assert mine["best_action"] == ref["best_action"]
    assert mine["root_visits"] == ref["root_visits"]


@pytest.mark.parametrize("gs,prefix,sims,solve,puct,alpha,seed", CASES, ids=["%s-%d-%s%s" % (c[0], c[2], "puct" if c[4] else "uct",
                                                                                            "-noise" if c[5] else "") for c in CASES])
def test_oracle_evaluated_mcts_equals_reference_mctsbot_bitwise(gs, prefix, sims, solve, puct, alpha, seed):
    os_, hist = _roots(gs, prefix, seed)
    eps = 0.25 if alpha > 0 else 0.0
    ref = ref_mcts_eval(gs, hist, os_.game.num_distinct_actions, 2.0, sims, solve, seed, puct=puct, dirichlet_alpha=alpha,
                        dirichlet_epsilon=eps)
    mine = oracle_mcts_eval(os_, 2.0, sims, solve, seed, puct=puct, reference_rng=True, dirichlet_alpha=alpha, dirichlet_epsilon=eps)
    _assert_same(mine, ref)
    if alpha > 0:        # the noise changes the search
        plain = oracle_mcts_eval(os_, 2.0, sims, solve, seed, puct=puct, reference_rng=True)
        assert [c[:3] for c in plain["children"]] != [c[:3] for c in mine["children"]]


GC_CASES = [("connect_four", 16000, True, 3), ("hex(board_size=4)", 9000, False, 5)]


@pytest.mark.parametrize("gs,sims,puct,seed", GC_CASES)
def test_oracle_evaluated_garbage_collection_equals_reference_bitwise(gs, sims, puct, seed):
    """max_memory_mb = 1: the tree is collected several times; the reference's Prior is asked again at every re-expansion,
    which the oracle does as well (and the device through a prior-only request)."""
    os_ = OracleGame(gs).new_initial_state()
    max_nodes = (1 << 20) // ref_sizeof_search_node() + 1
    ref = ref_mcts_eval(gs, [], os_.game.num_distinct_actions, 2.0, sims, False, seed, puct=puct, max_memory_mb=1)
    mine = oracle_mcts_eval(os_, 2.0, sims, False, seed, puct=puct, reference_rng=True, max_nodes=max_nodes)
    assert mine["gc_runs"] >= 2, mine["gc_runs"]
    _assert_same(mine, ref)
