"""The AlphaBetaSearch restatement (tests/alpha_beta_lib.py) against the reference's own search: the unmodified
python/algorithms/minimax.py of the OpenSpiel checkout, loaded by path, searching the unmodified reference games
(oracle/_ref, tests/ref_lib.py).  minimax.py searches with state.clone() + apply_action per child, as the C++ search does with
use_undo = false; the child states it generates are counted through apply_action.  Value, best action, node count and the
depth-0 error must agree on every case of alpha_beta_lib.reference_cases().  Where no checkout exists, the restatement is
checked against tests/golden/alpha_beta_reference.json, written from the same comparison by
tests/golden/make_alpha_beta_reference.py."""
import importlib.util
import json
import math
import os
import sys
import types

import pytest

import alpha_beta_lib as ab
import ref_lib
from __graft_entry__ import REFERENCE
from oracle_lib import OracleGame

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MINIMAX_PY = os.path.join(REFERENCE, "open_spiel", "python", "algorithms", "minimax.py")
GOLDEN = os.path.join(ROOT, "tests", "golden", "alpha_beta_reference.json")


class _GameType:
    """pyspiel.GameType's enums as minimax.py reads them; every served game is deterministic, perfect-information,
    sequential and zero-sum."""
    class ChanceMode:
        DETERMINISTIC = "deterministic"

    class Information:
        PERFECT_INFORMATION = "perfect"

    class Dynamics:
        SEQUENTIAL = "sequential"

    class Utility:
        ZERO_SUM = "zero_sum"

    chance_mode, information, dynamics, utility = "deterministic", "perfect", "sequential", "zero_sum"


class _State:
    def __init__(self, s, counter):
        self._s, self._n = s, counter

    def clone(self):
        return _State(self._s.clone(), self._n)

    def apply_action(self, a):
        self._n[0] += 1
        self._s.apply_action(a)

    def player_return(self, p):
        if p < 0:
            raise IndexError("player_return(%d)" % p)
        return self._s.returns()[p]

    def is_terminal(self):
        return self._s.is_terminal()

    def current_player(self):
        return self._s.current_player()

    def legal_actions(self):
        return self._s.legal_actions()


class _Game:
    def __init__(self, g):
        self._g = g

    def get_type(self):
        return _GameType

    def num_players(self):
        return self._g.num_players


def _minimax():
    if not ref_lib.available() or not os.path.exists(MINIMAX_PY):
        pytest.skip("needs the OpenSpiel checkout and the reference library built from it (oracle/_ref)")
    stub = types.ModuleType("pyspiel")
    stub.GameType = _GameType
    saved = sys.modules.get("pyspiel")
    sys.modules["pyspiel"] = stub
    try:
        spec = importlib.util.spec_from_file_location("reference_minimax", MINIMAX_PY)
        m = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(m)
    finally:
        if saved is None:
            del sys.modules["pyspiel"]
        else:
            sys.modules["pyspiel"] = saved
    return m


def reference_alpha_beta(minimax, case):
    """The reference's result in b2s_alpha_beta_search's terms."""
    gs, hist, depth, maxp = case
    g = ref_lib.RefGame(gs)
    s = g.new_initial_state()
    for a in hist:
        s.apply_action(a)
    n = [0]
    root = _State(s, n)
    try:
        v, best = minimax.alpha_beta_search(_Game(g), root, maximum_depth=depth, maximizing_player_id=None if maxp < 0 else maxp)
    except NotImplementedError:
        return dict(value=math.nan, best_action=-1, nodes=n[0], status=ab.DEPTH_ZERO)
    except IndexError:
        return dict(value=math.nan, best_action=-1, nodes=n[0], status=ab.TERMINAL_ROOT)
    return dict(value=float(v), best_action=-1 if best is None else int(best), nodes=n[0], status=ab.SOLVED)


def oracle_alpha_beta(case):
    gs, hist, depth, maxp = case
    return ab.alpha_beta(ab.replay(OracleGame(gs), hist), depth, maxp)


def test_oracle_equals_reference_minimax():
    minimax = _minimax()
    cases = ab.reference_cases()
    statuses = set()
    for case in cases:
        want, got = reference_alpha_beta(minimax, case), oracle_alpha_beta(case)
        assert ab.same(got, want), (case, got, want)
        statuses.add(want["status"])
    assert statuses == {ab.SOLVED, ab.DEPTH_ZERO, ab.TERMINAL_ROOT}
    assert len(cases) > 300


def test_minimax_test_cases():
    """minimax_test.cc: tic_tac_toe is a draw; after 4, 1 the mover wins; after 5, 4, 3, 8 the mover loses."""
    assert [oracle_alpha_beta(c)["value"] for c in ab.reference_cases()[:3]] == [0.0, 1.0, -1.0]


def test_oracle_equals_golden_reference():
    golden = json.load(open(GOLDEN))
    cases = ab.reference_cases()
    assert len(golden) == len({ab.case_id(c) for c in cases})
    for case in cases:
        v, best, nodes, status = golden[ab.case_id(case)]
        want = dict(value=math.nan if v is None else v, best_action=best, nodes=nodes, status=status)
        assert ab.same(oracle_alpha_beta(case), want), case
