"""Device AlphaBetaSearch (b2s_alpha_beta_search, open_spiel_b200.alpha_beta_search) against the restatement in
tests/alpha_beta_lib.py, which tests/test_alpha_beta_oracle_vs_reference.py pins to the reference's search.  Every search
here runs on roots whose oracle node count is small or under a budget: the kernels share the device."""
import math
import os
import random
import subprocess

import numpy as np
import pytest
import torch

import alpha_beta_lib as ab
import open_spiel_b200 as b2
from oracle_lib import OracleGame

pytestmark = pytest.mark.gpu


def make_batch(gs, roots, cap=None):
    """A batch whose lane i is the initial state after roots[i]."""
    g = b2.load_game(gs)
    batch = g.new_batch(cap or max(1, len(roots)))
    batch.reset()
    for t in range(max([len(h) for h in roots] + [0])):
        acts = torch.tensor([h[t] if t < len(h) else -1 for h in roots] + [-1] * (batch.n - len(roots)), dtype=torch.int32,
                            device=batch._dev)
        batch.apply_actions(acts)
    batch._reset_errors()
    return batch


def results(out, n=None):
    host = {k: v.cpu().numpy() for k, v in out.items()}
    n = len(host["value"]) if n is None else n
    return [dict(value=float(host["value"][i]), best_action=int(host["best_action"][i]), nodes=int(host["nodes"][i]),
                 status=int(host["status"][i])) for i in range(n)]


def check_against_oracle(gs, roots, got, depth=-1, maxp=-1, max_nodes=0):
    og = OracleGame(gs)
    for i, hist in enumerate(roots):
        want = ab.alpha_beta(ab.replay(og, hist), depth, maxp, max_nodes)
        assert ab.same(got[i], want), (gs, i, hist, depth, maxp, got[i], want)


@pytest.mark.parametrize("gs,plies,count", ab.VARIANTS, ids=[v[0] for v in ab.VARIANTS])
def test_device_equals_oracle(gs, plies, count):
    roots = ab.random_roots(OracleGame(gs), count, plies, seed=23)
    batch = make_batch(gs, roots)
    for depth, maxp in ((-1, -1), (-1, 0), (-1, 1), (2, -1), (3, 1)):
        out = b2.alpha_beta_search(batch, depth_limit=depth, maximizing_player=maxp)
        check_against_oracle(gs, roots, results(out), depth, maxp)


@pytest.mark.parametrize("n", [1, 33, 257, 1000, 4099])
def test_batch_sizes_tic_tac_toe(n):
    """One lane, a partial warp, a partial block, several blocks and a ragged multi-block batch; a larger batch capacity."""
    roots = ab.random_roots(OracleGame("tic_tac_toe"), n, (1, 9), seed=n)
    batch = make_batch("tic_tac_toe", roots, cap=n + 7)
    got = results(b2.alpha_beta_search(batch, n=n))
    check_against_oracle("tic_tac_toe", roots, got)


def test_ragged_connect_four_and_go():
    for gs, plies, n in (("connect_four", (30, 36), 777), ("go(board_size=3)", (6, 18), 300)):
        roots = ab.random_roots(OracleGame(gs), n, plies, seed=3)
        check_against_oracle(gs, roots, results(b2.alpha_beta_search(make_batch(gs, roots))))


def test_rejected_games():
    for gs in ("kuhn_poker", "leduc_poker", "go(board_size=13)", "go"):
        batch = b2.load_game(gs).new_batch(4)
        with pytest.raises(b2.SpielError, match="alpha_beta"):
            b2.alpha_beta_search(batch)
    batch = b2.load_game("tic_tac_toe").new_batch(4)
    with pytest.raises(b2.SpielError, match="maximizing_player"):
        b2.alpha_beta_search(batch, maximizing_player=2)


def test_budget_edge():
    """A root with max_nodes equal to its oracle count is solved with identical outputs; one less reports status 1.  Its
    neighbours keep their results."""
    gs = "connect_four"
    og = OracleGame(gs)
    roots = ab.random_roots(og, 64, (26, 32), seed=9)
    want = [ab.alpha_beta(ab.replay(og, h)) for h in roots]
    k = max(range(64), key=lambda i: want[i]["nodes"])
    budget = want[k]["nodes"]
    batch = make_batch(gs, roots)
    got = results(b2.alpha_beta_search(batch, max_nodes=budget))
    for i in range(64):
        assert ab.same(got[i], want[i] if want[i]["nodes"] <= budget else ab.alpha_beta(ab.replay(og, roots[i]), max_nodes=budget))
    assert ab.same(got[k], want[k])
    got = results(b2.alpha_beta_search(batch, max_nodes=budget - 1))
    assert got[k]["status"] == ab.BUDGET and got[k]["nodes"] == budget - 1 and math.isnan(got[k]["value"])
    assert got[k]["best_action"] == -1
    for i in range(64):
        if want[i]["nodes"] <= budget - 1:
            assert ab.same(got[i], want[i])
        else:
            assert got[i]["status"] == ab.BUDGET
    # terminal roots (maximizing_player -1) are the only counted lanes, once per call
    assert batch.error_count()[0] == 2 * sum(w["status"] == ab.TERMINAL_ROOT for w in want)


def test_scheduling_independence():
    gs, budget = "connect_four", 50000
    roots = ab.random_roots(OracleGame(gs), 600, (28, 36), seed=17)
    full = results(b2.alpha_beta_search(make_batch(gs, roots), max_nodes=budget))
    perm = list(range(600))
    random.Random(1).shuffle(perm)
    permuted = results(b2.alpha_beta_search(make_batch(gs, [roots[p] for p in perm]), max_nodes=budget))
    for j, p in enumerate(perm):
        assert ab.same(permuted[j], full[p])
    halves = results(b2.alpha_beta_search(make_batch(gs, roots[:300]), max_nodes=budget)) + \
        results(b2.alpha_beta_search(make_batch(gs, roots[300:]), max_nodes=budget))
    assert all(ab.same(a, b) for a, b in zip(halves, full))


def test_error_count():
    """Statuses 2 (depth 0 reached) and 3 (terminal root, maximizing_player -1) are counted on the roots batch, with the
    first such lane."""
    og = OracleGame("tic_tac_toe")
    roots = ab.random_roots(og, 200, (3, 9), seed=2)
    batch = make_batch("tic_tac_toe", roots)
    got = results(b2.alpha_beta_search(batch, depth_limit=3))
    bad = [i for i, r in enumerate(got) if r["status"] in (ab.DEPTH_ZERO, ab.TERMINAL_ROOT)]
    assert {got[i]["status"] for i in bad} == {ab.DEPTH_ZERO, ab.TERMINAL_ROOT}
    cnt, first = batch.error_count()
    assert cnt == len(bad) and first == bad[0]
    check_against_oracle("tic_tac_toe", roots, got, depth=3)


def _legal(batch, n):
    return batch.legal_actions_mask(n=n).bool()


def test_large_tic_tac_toe_invariants():
    """2^20 roots after 0-4 random plies: values in {-1, 0, 1}, legal best actions, the child of the best action has the root's
    value for the same maximizing player, and sampled lanes (block and warp edges, random) equal the oracle."""
    n = 1 << 20
    g = b2.load_game("tic_tac_toe")
    batch = g.new_batch(n)
    batch.reset()
    gen = torch.Generator(device="cuda").manual_seed(5)
    plies = torch.randint(0, 5, (n,), device="cuda", generator=gen)
    hist = torch.full((n, 4), -1, dtype=torch.int32, device="cuda")
    for t in range(4):
        mask = batch.legal_actions_mask().float()
        a = torch.multinomial(mask + 1e-30 * (mask.sum(1, keepdim=True) == 0), 1, generator=gen).squeeze(1).to(torch.int32)
        a = torch.where(plies > t, a, torch.full_like(a, -1))
        hist[:, t] = a
        batch.apply_actions(a)
    out = b2.alpha_beta_search(batch)
    status = out["status"]
    assert int((status != 0).sum()) == 0
    v = out["value"]
    assert bool(((v == -1) | (v == 0) | (v == 1)).all())
    best = out["best_action"].long()
    assert bool(_legal(batch, n).gather(1, best.unsqueeze(1)).all())
    # a MAX root's best child has the root's value, and so has a MIN root's: check it for either maximizing player
    child = g.new_batch(n)
    for p in (0, 1):
        r = b2.alpha_beta_search(batch, maximizing_player=p)
        child.copy_from(batch)
        child.apply_actions(r["best_action"])
        c = b2.alpha_beta_search(child, maximizing_player=p)
        assert bool((c["value"] == r["value"]).all()) and int((c["status"] != 0).sum()) == 0
    og = OracleGame("tic_tac_toe")
    hist_h = hist.cpu().numpy()
    sample = sorted({0, 31, 32, 127, 128, n - 1} | set(random.Random(0).sample(range(n), 200)))
    got = results(out)
    for i in sample:
        h = [int(a) for a in hist_h[i] if a >= 0]
        assert ab.same(got[i], ab.alpha_beta(ab.replay(og, h))), (i, h)


def test_large_connect_four_budget():
    """2^16 connect_four roots with 14 empty cells under a budget: solved lanes have values in {-1, 0, 1} and legal best actions;
    sampled lanes equal the oracle under the same budget."""
    n, budget = 1 << 16, 20000
    og = OracleGame("connect_four")
    rng = random.Random(4)
    roots = []
    while len(roots) < n:
        s, h = og.new_initial_state(), []
        while len(h) < 28 and not s.is_terminal():
            a = rng.choice(s.legal_actions())
            s.apply_action(a)
            h.append(a)
        if len(h) == 28 and not s.is_terminal():
            roots.append(h)
    batch = make_batch("connect_four", roots)
    out = b2.alpha_beta_search(batch, max_nodes=budget)
    st = out["status"]
    assert bool(((st == 0) | (st == 1)).all())
    solved = st == 0
    v = out["value"][solved]
    assert bool(((v == -1) | (v == 0) | (v == 1)).all())
    best = out["best_action"].long()
    legal = _legal(batch, n)
    assert bool(legal[solved].gather(1, best[solved].unsqueeze(1)).all())
    assert int(solved.sum()) > n // 2
    got = results(out)
    for i in sorted({0, 31, 32, 127, 128, n - 1} | set(rng.sample(range(n), 100))):
        assert ab.same(got[i], ab.alpha_beta(ab.replay(og, roots[i]), max_nodes=budget)), i


@pytest.mark.parametrize("gs,plies", [("tic_tac_toe", (2, 6)), ("connect_four", (30, 36))])
def test_mcts_solver_agrees(gs, plies):
    """Every root child MCTS-Solver reports as proven has that child's alpha-beta value for player 0."""
    og = OracleGame(gs)
    roots = [h for h in ab.random_roots(og, 64, plies, seed=8) if not ab.replay(og, h).is_terminal()]
    batch = make_batch(gs, roots)
    m = b2.mcts_search(batch, max_simulations=400, solve=True, seed=1)
    outcome = m["outcome_p0"].cpu().numpy()
    proven = 0
    for i, h in enumerate(roots):
        for a in np.nonzero(~np.isnan(outcome[i]))[0]:
            child = ab.replay(og, h + [int(a)])
            assert ab.alpha_beta(child, maximizing_player=0)["value"] == outcome[i][a], (i, h, a)
            proven += 1
    assert proven > 0


ADAPTER_TEST = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "open_spiel_b200", "adapter", "_build",
                            "alpha_beta_test")


@pytest.mark.skipif(not os.path.exists(ADAPTER_TEST), reason="alpha_beta_test not built (needs the reference headers)")
def test_cpp_drop_in_equals_stock_search():
    """b200::AlphaBetaSearch against the stock algorithms::AlphaBetaSearch (open_spiel_b200/adapter/alpha_beta_test.cc)."""
    out = subprocess.run([ADAPTER_TEST], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stdout[-2000:] + out.stderr[-2000:]
    assert "alpha_beta_test ok" in out.stdout
