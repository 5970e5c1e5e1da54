"""Pins the oracle restatement against the UNMODIFIED reference (oracle/_ref, built from the OpenSpiel checkout by
oracle/ref_build.mk with the abseil shim): random playouts, every observable compared after every move.
Skipped when oracle/_ref has not been built (it is built by __graft_entry__.build() when that checkout exists)."""
import numpy as np
import pytest

import ref_lib
from oracle_lib import OracleGame

pytestmark = pytest.mark.skipif(not ref_lib.available(), reason="oracle/_ref not built")

GAMES = [
    ("tic_tac_toe", 60), ("connect_four", 60), ("connect_four(rows=4,columns=5,x_in_row=3)", 30),
    ("connect_four(rows=7,columns=8,x_in_row=5)", 30), ("connect_four(egocentric_obs_tensor=True)", 20),
    ("breakthrough", 30), ("breakthrough(rows=6,columns=6)", 20), ("breakthrough(rows=5,columns=4)", 20),
    ("hex", 25), ("hex(board_size=5)", 40), ("hex(num_cols=4,num_rows=3)", 40), ("hex(board_size=4,swap=True)", 40),
    ("hex(board_size=5,plain_obs_tensor=True)", 20), ("hex(num_cols=5,num_rows=3,plain_obs_tensor=True)", 20),
    ("go(board_size=9)", 25), ("go(board_size=5)", 60), ("go(board_size=7,komi=4.5)", 30),
    ("go(board_size=9,max_game_length=60)", 20), ("go(board_size=4,komi=0.5)", 80), ("go(board_size=3,komi=0.5)", 80),
    ("kuhn_poker", 100), ("kuhn_poker(players=3)", 100),
    ("havannah", 12), ("havannah(board_size=4)", 150), ("havannah(board_size=4,swap=True)", 150), ("havannah(board_size=6)", 40),
    ("havannah(board_size=2)", 100), ("havannah(board_size=3,swap=True)", 100), ("havannah(board_size=1)", 2),
    ("y(board_size=9)", 60), ("y(board_size=11)", 30), ("y(board_size=4)", 100), ("y(board_size=1)", 2), ("y", 5),
    ("othello", 60), ("mnk", 6), ("mnk(m=3,n=3,k=3)", 100), ("mnk(m=7,n=5,k=4)", 30), ("mnk(m=15,n=15,k=3)", 10), ("mnk(m=4,n=15,k=5)", 20),
    ("mnk(m=5,n=5,k=7)", 20), ("mnk(m=1,n=1,k=1)", 3),
    ("leduc_poker", 150), ("leduc_poker(players=3)", 80), ("leduc_poker(starting_player=1)", 50),
]


def compare(o, r, game_string, check_strings=True):
    assert o.current_player() == r.current_player()
    assert o.is_terminal() == r.is_terminal()
    assert o.legal_actions() == r.legal_actions(), (game_string, o.to_string())
    ro, rr = o.returns(), r.returns()
    assert ro == rr and [np.signbit(x) for x in ro] == [np.signbit(x) for x in rr]
    if check_strings:
        assert o.to_string() == r.to_string()
    P = o.game.num_players
    for p in range(P):
        np.testing.assert_array_equal(o.observation_tensor(p), r.observation_tensor(p))
        if o.game.information_state_tensor_size:
            np.testing.assert_array_equal(o.information_state_tensor(p), r.information_state_tensor(p))
        if check_strings:
            assert o.information_state_string(p) == r.information_state_string(p)
            assert o.observation_string(p) == r.observation_string(p)
    if o.is_chance_node():
        assert o.chance_outcomes() == r.chance_outcomes()


@pytest.mark.parametrize("game_string,n_games", GAMES, ids=[g for g, _ in GAMES])
def test_oracle_equals_reference_on_random_playouts(game_string, n_games):
    og, rg = OracleGame(game_string), ref_lib.RefGame(game_string)
    for attr in ("num_distinct_actions", "num_players", "max_game_length", "observation_tensor_size",
                 "information_state_tensor_size", "max_chance_outcomes"):
        assert getattr(og, attr) == getattr(rg, attr), attr
    rng = np.random.RandomState(abs(hash(game_string)) % (2 ** 31))
    for _ in range(n_games):
        o, r = og.new_initial_state(), rg.new_initial_state()
        while True:
            compare(o, r, game_string)
            if o.is_terminal():
                break
            la = o.legal_actions()
            a = la[rng.randint(len(la))]
            o.apply_action(a)
            r.apply_action(a)
        assert o.history() == r.history()
