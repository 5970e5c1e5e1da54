"""GPU: the device searches past one block of trees.

Tree i of a search depends only on (seed, i + tree_index_offset, root), so tree i of a large search must equal a one-tree
search of the same root with tree_index_offset = i.  The one-tree runs go through the few-trees instantiation that
test_gpu_mcts.py / test_gpu_mcts_eval.py pin to the oracle; two trees per case are also compared with the oracle directly.

- mcts_search with 100,003 trees: at n >= 100,000 the rollout search launches its register-capped instantiation (DESIGN §4b
  lists its spills for the wide go core), which no smaller test reaches.
- mcts_search_evaluated with 300 trees: three blocks of the caller-evaluated search."""
import math

import numpy as np
import pytest
import torch

import open_spiel_b200 as b2
from open_spiel_b200 import _lib
from mcts_eval_lib import evaluate_leaves, oracle_mcts_eval
from oracle_lib import oracle_mcts
from test_gpu_mcts import make_roots

pytestmark = pytest.mark.gpu

SEED = 0x5EED5


def gather(game, roots, which):
    """A batch whose lane i holds lane which[i] of `roots` (b2s_gather_states)."""
    b = game.new_batch(len(which))
    idx = torch.from_numpy(np.asarray(which, dtype=np.int64)).cuda()
    _lib.check(_lib.lib().b2s_gather_states(b._h, roots._h, idx.data_ptr(), len(which), b._stream()))
    assert b.error_count()[0] == 0
    return b


def sampled_trees(n, count, seed):
    edges = {0, 1, 127, 128, 129, 255, 256, n // 2, n - 1}
    if n > 100000:
        edges |= {99999, 100000, n - 2}
    rng = np.random.RandomState(seed)
    extra = rng.choice(n, size=count, replace=False).tolist()
    return sorted(edges | set(extra[:max(0, count - len(edges))]))


def host(out, t):
    return {k: out[k][t].cpu().numpy() for k in ("visits", "total_reward", "outcome_p0", "best_action", "sims_run")}


def assert_same_tree(big, one, what):
    np.testing.assert_array_equal(big["visits"], one["visits"], err_msg=what)
    np.testing.assert_array_equal(big["total_reward"].view(np.int64), one["total_reward"].view(np.int64), err_msg=what)
    np.testing.assert_array_equal(np.isnan(big["outcome_p0"]), np.isnan(one["outcome_p0"]), err_msg=what)
    np.testing.assert_array_equal(np.nan_to_num(big["outcome_p0"]), np.nan_to_num(one["outcome_p0"]), err_msg=what)
    assert big["best_action"] == one["best_action"] and big["sims_run"] == one["sims_run"], what


def assert_matches_oracle(dev, o, what):
    assert dev["sims_run"] == o["sims_run"] and dev["best_action"] == o["best_action"], what
    assert int(dev["visits"].sum()) == sum(v for _, v, _, _ in o["children"]), what
    for a, v, r, oc in o["children"]:
        assert dev["visits"][a] == v and dev["total_reward"][a] == r, (what, a)
        assert (math.isnan(oc) and math.isnan(dev["outcome_p0"][a])) or dev["outcome_p0"][a] == oc, (what, a)


# game, roots' random prefix plies, simulations
MANY = [("connect_four", 10, 32), ("go(board_size=9)", 30, 20), ("go(board_size=13)", 60, 12)]


@pytest.mark.parametrize("gs,prefix,sims", MANY, ids=[c[0] for c in MANY])
def test_hundred_thousand_trees_equal_one_tree_searches(gs, prefix, sims):
    n = 100003
    game, roots, states = make_roots(gs, 8, prefix, seed=sum(map(ord, gs)) % 1000)
    assert not any(st.is_terminal() for st in states)
    root_of = np.random.RandomState(1).randint(0, 8, size=n)
    big = gather(game, roots, root_of)
    out = b2.mcts_search(big, sims, uct_c=2.0, n_rollouts=1, solve=True, seed=SEED)
    assert big.error_count()[0] == 0
    assert bool((out["sims_run"] >= 1).all())
    for t in sampled_trees(n, 48, seed=2):
        one = gather(game, roots, [root_of[t]])
        o = b2.mcts_search(one, sims, uct_c=2.0, n_rollouts=1, solve=True, seed=SEED, tree_index_offset=t)
        assert one.error_count()[0] == 0
        assert_same_tree(host(out, t), host(o, 0), "%s tree %d" % (gs, t))
    for t in (128, n - 1):
        o = oracle_mcts(states[root_of[t]], 2.0, sims, 1, True, SEED, tree_index=t)
        assert_matches_oracle(host(out, t), o, "%s tree %d vs oracle" % (gs, t))


EVALUATED = [("connect_four", 10, 60), ("go(board_size=9)", 30, 40)]


@pytest.mark.parametrize("gs,prefix,sims", EVALUATED, ids=[c[0] for c in EVALUATED])
def test_evaluated_search_across_blocks_equals_one_tree_searches(gs, prefix, sims):
    n = 300
    game, roots, states = make_roots(gs, 8, prefix, seed=sum(map(ord, gs)) % 1000 + 1)
    root_of = np.random.RandomState(3).randint(0, 8, size=n)
    big = gather(game, roots, root_of)
    kw = dict(uct_c=2.0, solve=True, seed=SEED, child_selection_policy=b2.ChildSelectionPolicy.PUCT)
    out = b2.mcts_search_evaluated(big, evaluate_leaves, sims, **kw)
    assert out["failed_trees"] == 0 and big.error_count()[0] == 0
    for t in sampled_trees(n, 40, seed=4):
        one = gather(game, roots, [root_of[t]])
        o = b2.mcts_search_evaluated(one, evaluate_leaves, sims, tree_index_offset=t, **kw)
        assert o["failed_trees"] == 0
        assert_same_tree(host(out, t), host(o, 0), "%s tree %d" % (gs, t))
    for t in (128, n - 1):
        o = oracle_mcts_eval(states[root_of[t]], 2.0, sims, True, SEED, tree_index=t, puct=True)
        assert_matches_oracle(host(out, t), o, "%s tree %d vs oracle" % (gs, t))
