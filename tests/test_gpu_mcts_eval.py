"""GPU: the caller-evaluated device MCTS (b2s_mcts_eval_*, mcts_search_evaluated) with the test evaluator written in torch
from the leaves batch's observation tensor and legal mask, vs the oracle's MCTS with the same evaluator on the Philox stream
(oracle/algorithms/mcts_eval.cc; pinned to the unmodified reference's MCTSBot by test_mcts_eval_oracle_vs_reference.py): root child
visit counts, total rewards (exact doubles), proven outcomes, BestChild, simulations run and collections must be identical for
every tree.  Plus the protocol's invariants and its argument checks."""
import math

import numpy as np
import pytest
import torch

import open_spiel_b200 as b2
from open_spiel_b200 import _lib
from mcts_eval_lib import dirichlet_rows, evaluate_leaves, oracle_mcts_eval
from test_gpu_mcts import CASES as ROLLOUT_CASES, make_roots

pytestmark = pytest.mark.gpu

SEED, OFFSET = 0xC0FFEE, 17

# game, trees, prefix plies, sims, solve, PUCT, node budget (MCTSBot::max_nodes_), dirichlet alpha
CASES = [(gs, n, prefix, sims, solve, False, 0, 0.0) for gs, n, prefix, sims, _, solve in ROLLOUT_CASES] + [
    ("tic_tac_toe", 48, 4, 300, True, True, 0, 0.0),
    ("connect_four", 32, 10, 300, True, True, 0, 0.0),
    ("breakthrough(rows=6,columns=6)", 16, 8, 150, False, True, 0, 0.0),
    ("go(board_size=5)", 24, 8, 150, True, True, 0, 0.0),
    ("othello", 16, 20, 150, True, True, 0, 0.0),
    ("havannah(board_size=4,swap=True)", 16, 8, 150, False, True, 0, 0.0),
    # the root's Dirichlet noise, drawn per tree over its legal actions; the oracle is given the same noise
    ("tic_tac_toe", 32, 2, 300, True, True, 0, 0.3),
    ("connect_four", 32, 6, 300, False, True, 0, 1.0),
    ("hex(board_size=5)", 16, 4, 200, True, False, 0, 0.5),
    ("go(board_size=5)", 16, 6, 150, True, True, 0, 0.03),
    ("y(board_size=5)", 16, 4, 200, True, True, 0, 0.3),
    # node budget: collections free children and cached priors; freed nodes ask again for their prior
    ("connect_four", 16, 6, 3000, False, True, 300, 0.0),
    ("tic_tac_toe", 16, 2, 1500, True, False, 120, 0.3),
    ("hex(board_size=4)", 12, 2, 2500, True, True, 400, 0.0),
    ("go(board_size=5)", 8, 6, 1200, True, False, 600, 0.0),
    ("othello", 8, 10, 1200, False, True, 300, 0.0),
    # mid-game go roots on tiny boards: positional superko decides many descents, so the leaves must carry the root's history
    ("go(board_size=2)", 32, 12, 200, True, True, 0, 0.0),
    ("go(board_size=3)", 32, 14, 300, False, True, 0, 0.0),
    ("go(board_size=3)", 16, 8, 1500, True, False, 200, 0.0),
]


def run_device(gs, n, prefix, sims, solve, puct, budget, alpha):
    game, batch, states = make_roots(gs, n, prefix, seed=sum(map(ord, gs)) % 1000)
    noise = dirichlet_rows([st.legal_actions() for st in states], game.num_distinct_actions(), alpha, seed=7) if alpha > 0 else None
    out = b2.mcts_search_evaluated(batch, evaluate_leaves, sims, uct_c=2.0, solve=solve, seed=SEED, tree_index_offset=OFFSET,
                                   child_selection_policy=b2.ChildSelectionPolicy.PUCT if puct else b2.ChildSelectionPolicy.UCT,
                                   max_nodes_per_tree=budget,
                                   root_noise=torch.from_numpy(noise).cuda() if noise is not None else None,
                                   dirichlet_epsilon=0.25 if alpha > 0 else 0.0)
    return game, batch, states, noise, out


@pytest.mark.parametrize("gs,n,prefix,sims,solve,puct,budget,alpha", CASES,
                         ids=["%s-%d%s%s%s" % (c[0], c[3], "-puct" if c[5] else "", "-gc" if c[6] else "", "-noise" if c[7] else "")
                              for c in CASES])
def test_device_evaluated_mcts_equals_oracle(gs, n, prefix, sims, solve, puct, budget, alpha):
    game, batch, states, noise, out = run_device(gs, n, prefix, sims, solve, puct, budget, alpha)
    visits, reward = out["visits"].cpu().numpy(), out["total_reward"].cpu().numpy()
    outcome, best, ran = out["outcome_p0"].cpu().numpy(), out["best_action"].cpu().numpy(), out["sims_run"].cpu().numpy()
    gcs, asks = out["gc_runs"].cpu().numpy(), out["prior_requests"].cpu().numpy()
    collections = 0
    for i, st in enumerate(states):
        o = oracle_mcts_eval(st, 2.0, sims, solve, SEED, tree_index=i + OFFSET, puct=puct, max_nodes=budget or 1,
                             root_noise=noise[i] if noise is not None else None, dirichlet_epsilon=0.25 if alpha > 0 else 0.0)
        assert ran[i] == o["sims_run"], (gs, i)
        assert gcs[i] == o["gc_runs"], (gs, i)
        collections += o["gc_runs"]
        assert int(visits[i].sum()) == sum(v for _, v, _, _ in o["children"])
        for a, v, r, oc in o["children"]:
            assert visits[i, a] == v, (gs, i, a)
            assert reward[i, a] == r, (gs, i, a, reward[i, a], r)            # exact double equality
            assert (math.isnan(oc) and math.isnan(outcome[i, a])) or outcome[i, a] == oc, (gs, i, a)
        illegal = sorted(set(range(game.num_distinct_actions())) - {a for a, _, _, _ in o["children"]})
        assert not visits[i, illegal].any()
        assert best[i] == o["best_action"], (gs, i)
    # one request per tree and round: at most one Evaluate per simulation plus the prior-only re-expansions
    assert out["rounds"] <= int((ran + asks).max())
    if budget:
        assert collections >= n
    else:
        assert int(asks.sum()) == 0
    assert out["failed_trees"] == 0 and batch.error_count()[0] == 0


def test_evaluated_root_invariants_many_trees():
    """Every tree: child visits sum to sims_run - 1 (the first simulation evaluates the root), reruns are reproducible, the
    number of rounds is bounded by simulations plus re-expansions, no tree fails, each step is one kernel launch."""
    game = b2.load_game("connect_four")
    n, sims = 4096, 64
    batch = game.new_batch(n)
    out = b2.mcts_search_evaluated(batch, evaluate_leaves, sims, solve=False, seed=5,
                                   child_selection_policy=b2.ChildSelectionPolicy.PUCT)
    assert bool((out["visits"].sum(dim=1) == out["sims_run"] - 1).all())
    assert bool((out["sims_run"] == sims).all())
    assert out["rounds"] <= int((out["sims_run"] + out["prior_requests"]).max())
    assert out["failed_trees"] == 0
    out2 = b2.mcts_search_evaluated(batch, evaluate_leaves, sims, solve=False, seed=5,
                                    child_selection_policy=b2.ChildSelectionPolicy.PUCT)
    for k in ("visits", "total_reward", "best_action", "sims_run"):
        assert torch.equal(out[k], out2[k]), k
    assert out2["rounds"] == out["rounds"]
    # launch accounting: a step is one kernel, the results one more
    search = b2.MCTSEvalSearch(batch, sims, seed=5)
    L = _lib.lib()
    c0 = L.b2s_launch_count()
    pending, k = search.step()
    assert L.b2s_launch_count() - c0 == 1 and k == n and bool(pending.all())
    v, p = evaluate_leaves(search.leaves, pending)
    c1 = L.b2s_launch_count()
    pending, k = search.step(v, p)
    assert L.b2s_launch_count() - c1 == 1
    c2 = L.b2s_launch_count()
    res = search.results()
    assert L.b2s_launch_count() - c2 == 1
    assert bool((res["sims_run"] == 1).all())                 # the root's evaluation finished simulation 1
    assert search.leaves.error_count()[0] == 0


def test_dirichlet_noise_helper():
    game = b2.load_game("go(board_size=5)")
    batch = game.new_batch(64)
    g = torch.Generator(device="cuda").manual_seed(3)
    z = b2.dirichlet_noise(batch, 0.03, generator=g)
    mask = batch.legal_actions_mask().bool()
    assert z.dtype == torch.float64 and z.shape == (64, game.num_distinct_actions())
    assert bool((z[~mask] == 0).all()) and bool((z >= 0).all())
    assert torch.allclose(z.sum(dim=1), torch.ones(64, dtype=torch.float64, device=z.device))
    g.manual_seed(3)
    assert torch.equal(z, b2.dirichlet_noise(batch, 0.03, generator=g))
    out = b2.mcts_search_evaluated(batch, evaluate_leaves, 32, seed=1, root_noise=z, dirichlet_epsilon=0.25,
                                   child_selection_policy=b2.ChildSelectionPolicy.PUCT)
    plain = b2.mcts_search_evaluated(batch, evaluate_leaves, 32, seed=1, child_selection_policy=b2.ChildSelectionPolicy.PUCT)
    assert not torch.equal(out["visits"], plain["visits"])


def test_evaluated_search_rejects_bad_arguments():
    game = b2.load_game("tic_tac_toe")
    batch = game.new_batch(16)
    with pytest.raises(b2.SpielError, match="same game"):
        b2.MCTSEvalSearch(batch, 10, leaves=b2.load_game("connect_four").new_batch(16))
    with pytest.raises(b2.SpielError, match="fewer lanes"):
        b2.MCTSEvalSearch(batch, 10, leaves=game.new_batch(8))
    with pytest.raises(b2.SpielError, match="max_wall_clock_time"):
        b2.MCTSEvalSearch(batch, 10, max_wall_clock_time=1.0)
    for gs in ("kuhn_poker", "leduc_poker"):
        poker = b2.load_game(gs).new_batch(8)
        with pytest.raises(b2.SpielError, match="no device MCTS"):
            b2.MCTSEvalSearch(poker, 10)
    search = b2.MCTSEvalSearch(batch, 10)
    search.step()
    with pytest.raises(b2.SpielError, match="values and priors"):
        search.step()
    with pytest.raises(b2.SpielError, match="float64"):
        search.step(torch.zeros((16, 2), device="cuda"), torch.zeros((16, 9), device="cuda"))
