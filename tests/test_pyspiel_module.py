"""The pyspiel-compatible module (open_spiel_b200/adapter/pyspiel_module.cc) on the CPU: scalar State methods run on the
host rule cores, so everything except MCTSBot / CFRSolver works without a GPU.  The core check is the reference's own
playthrough regression (python/tests/playthrough_test.py): every recorded playthrough of the seven games is regenerated
through the module by open_spiel_b200/playthrough.py and must come out byte-identical."""
import glob
import hashlib
import json
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

from __graft_entry__ import REFERENCE  # noqa: E402
from open_spiel_b200 import playthrough as pt  # noqa: E402

HASHES = json.load(open(os.path.join(ROOT, "tests", "golden", "playthrough_sha256.json")))
REF_DIR = os.path.join(REFERENCE, "open_spiel", "integration_tests", "playthroughs")


@pytest.mark.parametrize("name", sorted(HASHES))
def test_reference_playthrough_regenerates_byte_identically(name):
    rec = HASHES[name]
    text = pt.playthrough(pyspiel, rec["game"], rec["actions"], observation_params_string=rec["observation_params"])
    assert len(text.encode("utf-8")) == rec["bytes"]
    assert hashlib.sha256(text.encode("utf-8")).hexdigest() == rec["sha256"]
    ref = os.path.join(REF_DIR, name + ".txt")
    if os.path.exists(ref):                      # where the reference checkout exists: its own replay() comparison
        original = open(ref, encoding="utf-8").read()
        assert pt.replay(original, pyspiel) == original


def test_load_game_returns_the_dropins():
    for s in ["tic_tac_toe", "connect_four", "connect_four(rows=4,columns=5,x_in_row=3)", "breakthrough(rows=6,columns=6)",
              "hex(board_size=5,swap=True)", "go(board_size=9,komi=7.5)", "kuhn_poker", "leduc_poker(starting_player=1)"]:
        g = pyspiel.load_game(s)
        assert g.is_b200(), s
    # parameter sets outside the packed layouts are served by the stock games (the previous factory)
    assert pyspiel.load_game("kuhn_poker(players=3)").is_b200()          # kuhn 2..5 / leduc 2..4 players fit the packed layouts
    assert pyspiel.load_game("leduc_poker(players=3)").is_b200()
    for s in ["go(board_size=19)", "kuhn_poker(players=6)", "leduc_poker(players=5)", "hex(board_size=13)"]:
        assert not pyspiel.load_game(s).is_b200(), s
    g = pyspiel.load_game("go", {"board_size": 9, "komi": 6.5})
    assert g.is_b200() and g.get_parameters()["komi"] == 6.5 and g.num_distinct_actions() == 82
    assert str(g) == "go(board_size=9,komi=6.5)"
    assert g.observation_tensor_shape() == [4, 9, 9] and g.max_game_length() == 162


def test_state_surface():
    g = pyspiel.load_game("connect_four")
    s = g.new_initial_state()
    assert s.current_player() == 0 and s.legal_actions() == list(range(7)) and s.legal_actions_mask() == [1] * 7
    s.apply_action(3)
    c = s.child(3)
    assert s.history() == [3] and c.history() == [3, 3] and s.move_number() == 1
    assert s.action_to_string(1, 4) == "o4" and s.string_to_action("o4") == 4
    assert len(s.observation_tensor(0)) == 126 and sum(s.observation_tensor(0)) == 42
    assert s.clone().history() == [3] and not s.is_terminal() and s.returns() == [0.0, 0.0]
    c.undo_action(1, 3)
    assert str(c) == str(s)
    assert pickle.loads(pickle.dumps(c)).history() == [3]
    assert str(pickle.loads(pickle.dumps(g))) == "connect_four()"
    game2, state2 = pyspiel.deserialize_game_and_state(pyspiel.serialize_game_and_state(g, s))
    assert str(state2) == str(s) and game2.is_b200()
    assert len(s.packed_state()) == 16                      # the b2s lane: one 128-bit chunk
    with pytest.raises(pyspiel.SpielError):                  # SpielFatalError -> pyspiel.SpielError (pyspiel.cc:831-837)
        for _ in range(7):
            s.apply_action(3)


def test_poker_surface_and_policies():
    g = pyspiel.load_game("kuhn_poker")
    s = g.new_initial_state()
    assert s.is_chance_node() and s.chance_outcomes() == [(0, 1 / 3), (1, 1 / 3), (2, 1 / 3)]
    for a in [2, 0, 1, 1]:
        s.apply_action(a)
    assert s.is_terminal() and s.returns() == [2.0, -2.0]
    assert s.information_state_string(0) == "2bb" and s.observation_string(1) == "022"
    assert s.information_state_tensor(1) == [0, 1, 1, 0, 0, 0, 1, 0, 1, 0, 0]
    uniform = pyspiel.get_uniform_policy(g)
    assert abs(pyspiel.nash_conv(g, uniform) - 0.9166666666666666) < 1e-12       # the reference's value for kuhn
    assert abs(pyspiel.exploitability(g, uniform) - 0.4583333333333333) < 1e-12


def test_mcts_bot_with_a_foreign_evaluator_uses_the_stock_host_search():
    # the Evaluator plug point (mcts.h:83-92): anything that is not the rollout evaluator stays on the reference's bot
    g = pyspiel.load_game("tic_tac_toe")
    ev = pyspiel.RandomRolloutEvaluator(n_rollouts=2, seed=1)
    bot = pyspiel.MCTSBot(g, ev, 2.0, 50, 10, True, 3, False, dirichlet_alpha=0.3, dirichlet_epsilon=0.25)
    assert not bot.on_device()
    a = bot.step(g.new_initial_state())
    assert 0 <= a < 9
