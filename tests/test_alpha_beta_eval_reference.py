"""AlphaBetaSearch with a value function: the restatement (alpha_beta_eval in tests/alpha_beta_eval_lib.py) against the reference's
own search, the unmodified python/algorithms/minimax.py of the OpenSpiel checkout loaded by path and run over the unmodified
reference games (oracle/_ref, tests/ref_lib.py) with value_function = lambda s: f(s)[maxp] for the test value functions of
tests/alpha_beta_eval_lib.py.  Value (bit for bit), best action, node count, evaluation count and the sequence of evaluated
states must agree on every case of alpha_beta_eval_lib.reference_cases().  Where no checkout exists, the restatement is checked
against tests/golden/alpha_beta_eval_reference.json, written from the same comparison by
tests/golden/make_alpha_beta_eval_reference.py."""
import json
import math
import os

import pytest

import alpha_beta_eval_lib as abe
import alpha_beta_lib as ab
import ref_lib
from oracle_lib import OracleGame
from test_alpha_beta_oracle_vs_reference import _Game, _minimax, _State

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "alpha_beta_eval_reference.json")


def reference_alpha_beta_eval(minimax, case):
    """The reference's result in b2s_alpha_beta_eval_*'s terms, plus the histories of the states its value function saw."""
    gs, hist, depth, maxp, kind = case
    g = ref_lib.RefGame(gs)
    s = g.new_initial_state()
    for a in hist:
        s.apply_action(a)
    n = [0]
    root = _State(s, n)
    m = maxp if maxp >= 0 else (s.current_player() if not s.is_terminal() else 0)
    seen = []

    def value_function(state):
        seen.append(state._s.history())
        return abe.state_values(state._s, kind)[m]

    try:
        v, best = minimax.alpha_beta_search(_Game(g), root, value_function=value_function, maximum_depth=depth,
                                            maximizing_player_id=None if maxp < 0 else maxp)
    except IndexError:
        return dict(value=math.nan, best_action=-1, nodes=n[0], status=ab.TERMINAL_ROOT, evaluations=len(seen), histories=seen)
    # minimax.py returns best_action None for a terminal or depth-0 root and -1 when no child beat the initial value
    return dict(value=float(v), best_action=-1 if best is None else int(best), nodes=n[0], status=ab.SOLVED,
                evaluations=len(seen), histories=seen)


def oracle_alpha_beta_eval(case):
    gs, hist, depth, maxp, kind = case
    return abe.restated(OracleGame(gs), hist, depth, maxp, kind)


def golden_entry(r):
    return [abe.bits(r["value"]), r["best_action"], r["nodes"], r["status"], r["evaluations"], abe.digest(r["histories"])]


def test_oracle_equals_reference_minimax():
    minimax = _minimax()
    cases = abe.reference_cases()
    seen_values = set()
    for case in cases:
        want, got = reference_alpha_beta_eval(minimax, case), oracle_alpha_beta_eval(case)
        assert abe.same_bits(got, want), (case, got, want)
        assert got["histories"] == want["histories"], case
        seen_values.add(abe.bits(want["value"]))
    # the edge function's specials reach the root: +-inf, -0.0 and a depth-0 NaN
    for x in (math.inf, -math.inf, -0.0, math.nan):
        assert abe.bits(x) in seen_values or abe.bits(-x) in seen_values, x


def test_oracle_equals_golden_reference():
    golden = json.load(open(GOLDEN))
    cases = abe.reference_cases()
    assert len(golden) == len({abe.case_id(c) for c in cases})
    for case in cases:
        assert golden_entry(oracle_alpha_beta_eval(case)) == golden[abe.case_id(case)], case


def test_beyond_the_game_equals_exact_restatement():
    """A depth limit the game never reaches is the exact search (alpha_beta_lib.alpha_beta): the same results, no evaluation."""
    og = OracleGame("tic_tac_toe")
    for hist in ab.random_roots(og, 24, (0, 6), seed=1):
        for depth, maxp in ((-1, -1), (9, 0), (12, 1)):
            want = ab.alpha_beta(ab.replay(og, hist), depth, maxp)
            got = abe.alpha_beta_eval(ab.replay(og, hist), depth, maxp, 0, lambda s: 0.5)
            assert got.pop("evaluations") == 0 and got.pop("evaluated") == []
            assert ab.same(got, want), (hist, depth, maxp)


def test_depth_zero_root_and_special_values():
    """A depth-0 non-terminal root is its own single evaluation with best action -1; NaN children are never taken and all
    children at -inf leave best action -1."""
    og = OracleGame("tic_tac_toe")
    root = ab.replay(og, [4])
    r = abe.alpha_beta_eval(root, 0, -1, 0, lambda s: -0.0)
    assert abe.bits(r["value"]) == abe.bits(-0.0) and r["best_action"] == -1 and r["nodes"] == 0 and r["evaluations"] == 1
    r = abe.alpha_beta_eval(root, 1, -1, 0, lambda s: math.nan)
    assert r["value"] == -math.inf and r["best_action"] == -1 and r["evaluations"] == 8
    r = abe.alpha_beta_eval(root, 1, -1, 0, lambda s: -math.inf)
    assert r["value"] == -math.inf and r["best_action"] == -1
    r = abe.alpha_beta_eval(root, 1, -1, 0, lambda s: 0.0 if s.history()[-1] == 0 else -0.0)
    assert abe.bits(r["value"]) == abe.bits(0.0) and r["best_action"] == 0      # ties keep the first child


@pytest.mark.parametrize("gs", ["tic_tac_toe", "connect_four", "go(board_size=5)", "othello"])
def test_torch_value_functions_equal_numpy(gs):
    import numpy as np
    import torch
    og = OracleGame(gs)
    for hist in ab.random_roots(og, 12, (0, 12), seed=4):
        s = ab.replay(og, hist)
        if s.is_terminal():
            continue
        obs = s.observation_tensor(s.current_player())
        for kind in abe.KINDS:
            t = abe.batch_values(torch.from_numpy(np.asarray(obs))[None, :], kind)[0].tolist()
            assert [abe.bits(x) for x in t] == [abe.bits(x) for x in abe.state_values(s, kind)]
