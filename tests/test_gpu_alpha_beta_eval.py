"""Device AlphaBetaSearch with a caller-supplied value function (b2s_alpha_beta_eval_*, open_spiel_b200.AlphaBetaEvalSearch /
alpha_beta_search_evaluated) against the restatement alpha_beta_eval with the test value functions of
tests/alpha_beta_eval_lib.py, which tests/test_alpha_beta_eval_reference.py pins to the reference's minimax.py.  Values are
compared bit for bit; the leaves each root hands out are compared with the restatement's evaluated states, in order."""
import math
import random

import numpy as np
import pytest
import torch

import alpha_beta_eval_lib as abe
import alpha_beta_lib as ab
import open_spiel_b200 as b2
from oracle_lib import OracleGame
from test_gpu_alpha_beta import make_batch

pytestmark = pytest.mark.gpu

KEYS = ("value", "best_action", "nodes", "status", "evaluations")


def results(out, n=None):
    host = {k: out[k].cpu().numpy() for k in KEYS}
    n = len(host["value"]) if n is None else n
    return [dict(value=float(host["value"][i]), best_action=int(host["best_action"][i]), nodes=int(host["nodes"][i]),
                 status=int(host["status"][i]), evaluations=int(host["evaluations"][i])) for i in range(n)]


def search(gs, roots, depth, maxp, kind, max_nodes=0, cap=None):
    batch = make_batch(gs, roots, cap)
    out = b2.alpha_beta_search_evaluated(batch, abe.leaves_value_function(kind), depth, maxp, max_nodes, n=len(roots))
    return results(out), out


def check_against_restatement(gs, roots, got, depth, maxp, kind, max_nodes=0):
    og = OracleGame(gs)
    for i, hist in enumerate(roots):
        want = abe.restated(og, hist, depth, maxp, kind, max_nodes)
        assert abe.same_bits(got[i], want), (gs, i, hist, depth, maxp, kind, got[i], want)


@pytest.mark.parametrize("gs,plies,count", ab.VARIANTS, ids=[v[0] for v in ab.VARIANTS])
def test_device_equals_restatement(gs, plies, count):
    roots = ab.random_roots(OracleGame(gs), count, plies, seed=31)
    for depth in range(5):
        for maxp, kind in ((-1, "hash"), (0, "edge"), (1, "hash"), (-1, "edge")):
            got, out = search(gs, roots, depth, maxp, kind)
            check_against_restatement(gs, roots, got, depth, maxp, kind)
            assert out["rounds"] == max(g["evaluations"] for g in got)


@pytest.mark.parametrize("n", [1, 33, 257, 1000, 4099])
def test_batch_sizes(n):
    """One root, a partial warp, a partial block, several blocks and a ragged multi-block batch in a larger batch."""
    roots = ab.random_roots(OracleGame("tic_tac_toe"), n, (0, 6), seed=n)
    got, _ = search("tic_tac_toe", roots, 2, -1, "hash", cap=n + 7)
    check_against_restatement("tic_tac_toe", roots, got, 2, -1, "hash")


def leaf_sequences(gs, roots, depth, maxp, kind):
    """Drives the search by hand; returns (results, per root the list of (state bytes, legal mask row) of its leaves)."""
    batch = make_batch(gs, roots)
    s = b2.AlphaBetaEvalSearch(batch, depth, maxp)
    sb = batch.info.state_bytes
    seq = [[] for _ in roots]
    values = None
    while True:
        pending, cnt = s.step(values)
        if cnt == 0:
            break
        mask = s.leaves.legal_actions_mask().cpu().numpy()
        for i in torch.nonzero(pending).flatten().tolist():
            seq[i].append((s.leaves.state_blob(i)[:sb], mask[i]))
        values = abe.batch_values(s.leaves.observation_tensor(), kind)
    return results(s.results()), seq


def check_leaf_sequences(gs, roots, depth, maxp, kind):
    og = OracleGame(gs)
    got, seq = leaf_sequences(gs, roots, depth, maxp, kind)
    want_hist = []
    for i, hist in enumerate(roots):
        want = abe.restated(og, hist, depth, maxp, kind)
        assert abe.same_bits(got[i], want), (gs, i, hist, got[i], want)
        assert len(seq[i]) == len(want["histories"])
        want_hist += want["histories"]
    if not want_hist:
        return 0
    exp = make_batch(gs, want_hist)
    sb = exp.info.state_bytes
    emask = exp.legal_actions_mask().cpu().numpy()
    flat = [x for s in seq for x in s]
    for k, (blob, mask) in enumerate(flat):
        assert blob == exp.state_blob(k)[:sb], (gs, k, want_hist[k])
        assert np.array_equal(mask, emask[k]), (gs, k, want_hist[k])
    return len(flat)


@pytest.mark.parametrize("gs,plies,depth", [("tic_tac_toe", (0, 5), 3), ("connect_four", (6, 14), 3), ("othello", (20, 30), 2),
                                            ("breakthrough(rows=6,columns=6)", (6, 12), 2), ("hex(board_size=5)", (4, 10), 2)])
def test_leaves_are_the_evaluated_states(gs, plies, depth):
    """The k-th leaf each root hands out is the restatement's k-th evaluated state (lane blob and legal mask)."""
    roots = ab.random_roots(OracleGame(gs), 6, plies, seed=12)
    assert check_leaf_sequences(gs, roots, depth, -1, "hash") > 0


@pytest.mark.parametrize("size,plies,depth", [(2, (3, 8), 4), (3, (6, 14), 4), (4, (10, 20), 3), (5, (14, 30), 3), (6, (20, 40), 2),
                                              (7, (25, 45), 2), (8, (30, 60), 2), (9, (40, 70), 2)])
def test_go_leaves_carry_superko_history(size, plies, depth):
    """go 2..9 mid-game roots: every leaf lane equals the evaluated state replayed from the start, legal mask included, which
    needs the root's superko history plus the path's moves in the leaves batch."""
    gs = "go(board_size=%d)" % size
    roots = ab.random_roots(OracleGame(gs), 3, plies, seed=size)
    assert check_leaf_sequences(gs, roots, depth, -1, "hash") > 0


@pytest.mark.parametrize("depth", [1, 2])
def test_go_19x19(depth):
    """The wide go rule core, whose unlimited stack is too large, at small depths from late positions."""
    gs = "go"
    roots = ab.random_roots(OracleGame(gs), 2, (250, 300), seed=depth)
    got, _ = search(gs, roots, depth, -1, "hash")
    check_against_restatement(gs, roots, got, depth, -1, "hash")
    if depth == 1:
        assert check_leaf_sequences(gs, roots[:1], depth, 0, "edge") > 0


def test_budget_edge():
    """max_nodes equal to a root's count solves it unchanged; one less reports status 1 with the restatement's counts; the
    neighbours keep their results."""
    gs, depth = "connect_four", 4
    og = OracleGame(gs)
    roots = [h for h in ab.random_roots(og, 32, (8, 14), seed=9) if not ab.replay(og, h).is_terminal()]
    want = [abe.restated(og, h, depth, -1, "hash") for h in roots]
    k = max(range(len(roots)), key=lambda i: want[i]["nodes"])
    budget = want[k]["nodes"]
    got, _ = search(gs, roots, depth, -1, "hash", max_nodes=budget)
    check_against_restatement(gs, roots, got, depth, -1, "hash", max_nodes=budget)
    assert abe.same_bits(got[k], want[k])
    got, _ = search(gs, roots, depth, -1, "hash", max_nodes=budget - 1)
    check_against_restatement(gs, roots, got, depth, -1, "hash", max_nodes=budget - 1)
    assert got[k]["status"] == ab.BUDGET and got[k]["nodes"] == budget - 1 and math.isnan(got[k]["value"])
    assert got[k]["best_action"] == -1


def test_terminal_roots_and_error_count():
    """maximizing_player -1 on a terminal root is status 3, counted on the leaves batch; an explicit player scores it."""
    og = OracleGame("tic_tac_toe")
    roots = ab.random_roots(og, 200, (5, 9), seed=2)
    terminal = [i for i, h in enumerate(roots) if ab.replay(og, h).is_terminal()]
    assert terminal
    batch = make_batch("tic_tac_toe", roots)
    s = b2.AlphaBetaEvalSearch(batch, 2)
    values = None
    while True:
        pending, cnt = s.step(values)
        if cnt == 0:
            break
        values = abe.batch_values(s.leaves.observation_tensor(), "hash")
    got = results(s.results())
    cnt, first = s.leaves.error_count()
    assert cnt == len(terminal) and first == terminal[0]
    assert [i for i, g in enumerate(got) if g["status"] == ab.TERMINAL_ROOT] == terminal
    assert batch.error_count()[0] == 0
    check_against_restatement("tic_tac_toe", roots, got, 2, -1, "hash")
    got, _ = search("tic_tac_toe", roots, 2, 1, "hash")
    check_against_restatement("tic_tac_toe", roots, got, 2, 1, "hash")


def test_rejected_configurations():
    def make(gs, n, depth=2, leaves=None, maxp=-1):
        batch = b2.load_game(gs).new_batch(n)
        batch.reset()
        return b2.AlphaBetaEvalSearch(batch, depth, maxp, leaves=leaves)

    for gs in ("kuhn_poker", "leduc_poker"):
        with pytest.raises(b2.SpielError, match="alpha_beta_eval: AlphaBetaSearch needs a deterministic game"):
            make(gs, 4)
    with pytest.raises(b2.SpielError, match="same game, parameters and device"):
        make("connect_four", 4, leaves=b2.load_game("tic_tac_toe").new_batch(4))
    with pytest.raises(b2.SpielError, match="same game, parameters and device"):
        make("connect_four", 4, leaves=b2.load_game("connect_four(rows=5,columns=6)").new_batch(4))
    with pytest.raises(b2.SpielError, match="fewer lanes than n"):
        make("connect_four", 4, leaves=b2.load_game("connect_four").new_batch(3))
    with pytest.raises(b2.SpielError, match="B2S_ALPHA_BETA_THREAD_STACK_BYTES"):
        make("go", 2, depth=-1)
    with pytest.raises(b2.SpielError, match="maximizing_player"):
        make("tic_tac_toe", 2, maxp=2)
    make("go", 2, depth=2)                     # a small depth limit fits


def test_scheduling_independence():
    gs, depth = "connect_four", 4
    roots = ab.random_roots(OracleGame(gs), 600, (6, 14), seed=17)
    full, _ = search(gs, roots, depth, -1, "edge")
    perm = list(range(600))
    random.Random(1).shuffle(perm)
    permuted, _ = search(gs, [roots[p] for p in perm], depth, -1, "edge")
    for j, p in enumerate(perm):
        assert abe.same_bits(permuted[j], full[p])
    halves = search(gs, roots[:300], depth, -1, "edge")[0] + search(gs, roots[300:], depth, -1, "edge")[0]
    assert all(abe.same_bits(a, b) for a, b in zip(halves, full))


@pytest.mark.parametrize("gs,plies", [("tic_tac_toe", (2, 6)), ("connect_four", (30, 36))])
def test_depth_beyond_the_game_equals_exact_search(gs, plies):
    """Unlimited, or at least the remaining plies: the exact search's value, best action and nodes, no evaluation, and a first
    step with nothing pending."""
    roots = ab.random_roots(OracleGame(gs), 64, plies, seed=6)
    batch = make_batch(gs, roots)
    exact = b2.alpha_beta_search(batch, maximizing_player=0)
    for depth in (-1, 42):
        s = b2.AlphaBetaEvalSearch(batch, depth, 0)
        _, cnt = s.step()
        assert cnt == 0
        r = s.results()
        assert int(r["evaluations"].sum()) == 0
        for k in ("value", "best_action", "nodes", "status"):
            assert torch.equal(r[k], exact[k]), k


def test_exact_search_as_value_function():
    """alpha_beta_search on the leaves batch (exact values, maximizing player 0) as the value function gives the exact search's
    root value and best action at every depth limit."""
    gs = "tic_tac_toe"
    roots = [h for h in ab.random_roots(OracleGame(gs), 128, (2, 5), seed=7)]
    batch = make_batch(gs, roots)
    exact = b2.alpha_beta_search(batch, maximizing_player=0)
    leaves = b2.load_game(gs).new_batch(len(roots))
    leaves.reset()                              # every lane a valid state, pending or not

    def exact_values(lv, pending):
        v = b2.alpha_beta_search(lv, maximizing_player=0)["value"]
        return torch.stack([v, -v], dim=1)

    for depth in (1, 2, 3):
        out = b2.alpha_beta_search_evaluated(batch, exact_values, depth, 0, leaves=leaves)
        assert int(out["evaluations"].sum()) > 0
        assert torch.equal(out["value"], exact["value"]) and torch.equal(out["best_action"], exact["best_action"])


def test_large_connect_four():
    """65,536 connect_four roots after 8 plies at depth 4 with the hash function: every root solved, values among the hash
    values and the terminal returns, legal best actions, a round per evaluation of the busiest root; 2,000 sampled roots
    equal the restatement."""
    n, depth = 1 << 16, 4
    og = OracleGame("connect_four")
    rng = random.Random(4)
    roots = []
    while len(roots) < n:
        s, h = og.new_initial_state(), []
        while len(h) < 8 and not s.is_terminal():
            a = rng.choice(s.legal_actions())
            s.apply_action(a)
            h.append(a)
        if len(h) == 8 and not s.is_terminal():
            roots.append(h)
    batch = make_batch("connect_four", roots)
    out = b2.alpha_beta_search_evaluated(batch, abe.leaves_value_function("hash"), depth)
    assert int((out["status"] != 0).sum()) == 0
    allowed = torch.tensor(sorted({(k - 4) / 7.0 for k in range(9)} | {-1.0, 0.0, 1.0}), dtype=torch.float64, device="cuda")
    assert bool(torch.isin(out["value"], allowed).all())
    legal = batch.legal_actions_mask().bool()
    assert bool(legal.gather(1, out["best_action"].long().unsqueeze(1)).all())
    assert bool((out["evaluations"] <= out["nodes"]).all())
    assert out["rounds"] == int(out["evaluations"].max())
    got = results(out)
    for i in sorted({0, 31, 32, 127, 128, n - 1} | set(rng.sample(range(n), 2000 - 6))):
        want = abe.restated(og, roots[i], depth, -1, "hash")
        assert abe.same_bits(got[i], want), (i, got[i], want)
