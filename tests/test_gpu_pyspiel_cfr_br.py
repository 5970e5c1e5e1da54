"""pyspiel.CFRBRSolver (python/pybind11/policy.cc:264-280) of the pyspiel-compatible module on device tables: the known
answers of algorithms/cfr_br_test.cc, the reference's own Exploitability on the device policy, and a pickle round trip that
continues bit for bit."""
import glob
import os
import pickle
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BUILD = os.path.join(ROOT, "open_spiel_b200", "adapter", "_build")
if not glob.glob(os.path.join(BUILD, "pyspiel*.so")):
    pytest.skip("pyspiel module not built (needs the reference headers)", allow_module_level=True)
sys.path.insert(0, BUILD)
import pyspiel  # noqa: E402

pytestmark = pytest.mark.gpu


def expected_returns(state, policy):
    if state.is_terminal():
        return state.returns()
    if state.is_chance_node():
        outcomes = state.chance_outcomes()
    else:
        outcomes = sorted(policy.action_probabilities(state).items())
    total = [0.0, 0.0]
    for a, p in outcomes:
        v = expected_returns(state.child(a), policy)
        total = [t + p * x for t, x in zip(total, v)]
    return total


def test_cfr_br_solver_known_answers_and_pickle():
    game = pyspiel.load_game("kuhn_poker")
    solver = pyspiel.CFRBRSolver(game)
    e0 = pyspiel.exploitability(game, solver.average_policy())
    for _ in range(50):
        solver.evaluate_and_update_policy()
    e1 = pyspiel.exploitability(game, solver.average_policy())
    assert e0 > e1                                       # cfr_br_test.cc CFRBRTest_CFRBRSolverSerialization
    clone = pickle.loads(pickle.dumps(solver))
    assert isinstance(clone, pyspiel.CFRBRSolver)
    assert abs(pyspiel.exploitability(game, clone.average_policy()) - e1) <= 1e-12
    clone.iterate(250)
    solver.iterate(250)
    assert clone.average_policy().policy_table() == solver.average_policy().policy_table()
    assert clone.current_policy().policy_table() == solver.current_policy().policy_table()
    avg = solver.average_policy()                        # cfr_br_test.cc CFRBRTest_KuhnPoker, 300 iterations
    ret = expected_returns(game.new_initial_state(), avg)
    assert abs(ret[0] + 1 / 18) <= 1e-3 and abs(ret[1] - 1 / 18) <= 1e-3
    expl = pyspiel.exploitability(game, avg)
    assert expl <= 0.05 and abs(solver.nash_conv() / 2 - expl) < 1e-9
    assert e1 > expl
