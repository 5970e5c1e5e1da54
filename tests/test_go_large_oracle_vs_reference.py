"""CPU: go on boards 10..19 — the oracle and the host build of the device's 384-bit rule core against the UNMODIFIED reference.
Everywhere: the reference's seeded games stored in tests/golden/go_large_reference.json (13x13, 19x19, handicap stones) are
replayed on both, every position's observables compared.  Where oracle/_ref is built: random games in lock-step with the
reference's State objects, and small MCTSBot searches on the reference's own random streams (the pattern of
test_mcts_oracle_vs_reference.py), including a max_memory_mb = 1 search that collects."""
import hashlib
import json
import os
import random

import numpy as np
import pytest

import ref_lib
from oracle_lib import OracleGame, oracle_mcts
from test_rule_cores_host import Emu
from go_wide_emul import use_wide_libraries


@pytest.fixture(autouse=True)
def _wide_host_build(monkeypatch):
    """Emu / Emv / run_emulated on the host build that also holds go 10..19 (tests/host_emul/go_wide.mk)."""
    use_wide_libraries(monkeypatch)


GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "go_large_reference.json")
_GAMES = json.load(open(GOLD, encoding="utf-8"))["games"]
needs_ref = pytest.mark.skipif(not ref_lib.available(), reason="oracle/_ref not built")


def _digest(player, terminal, returns, legal, obs):
    """A position as tests/golden/make_go_large_reference.py stores it."""
    return [int(player), int(terminal)] + [repr(float(x)) for x in returns] + [
        hashlib.sha256(json.dumps([int(a) for a in legal]).encode()).hexdigest()[:12],
        hashlib.sha256(b"".join(np.asarray(o, dtype=np.float32).tobytes() for o in obs)).hexdigest()[:12]]


@pytest.mark.parametrize("k", range(len(_GAMES)), ids=["%s-%d" % (g["game"], g["seed"]) for g in _GAMES])
def test_oracle_and_wide_core_replay_reference_games(k):
    g = _GAMES[k]
    st = OracleGame(g["game"]).new_initial_state()
    emu = Emu(g["game"], 1)
    for ply, want in enumerate(g["positions"]):
        assert _digest(st.current_player(), st.is_terminal(), st.returns(), st.legal_actions(),
                       [st.observation_tensor(p) for p in range(2)]) == want, ("oracle", ply)
        cur, term, rets = emu.status()
        assert _digest(cur[0], term[0], rets[0].tolist(), emu.legal()[0], [emu.tensor(p, 0)[0] for p in range(2)]) == want, ("core", ply)
        assert [bool(np.signbit(x)) for x in rets[0]] == [t.startswith("-") for t in want[2:4]]
        if ply < len(g["actions"]):
            st.apply_action(g["actions"][ply])
            emu.apply([g["actions"][ply]])
            assert emu.errors() == 0
    assert st.is_terminal()


REF_GAMES = [("go(board_size=10)", 8), ("go(board_size=13)", 6), ("go(board_size=16,komi=0.5)", 4), ("go(board_size=19)", 4),
             ("go(board_size=19,handicap=4)", 3), ("go(board_size=19,handicap=9,max_game_length=200)", 3), ("go(board_size=19,handicap=11)", 2)]


@needs_ref
@pytest.mark.parametrize("gs,games", REF_GAMES, ids=[g for g, _ in REF_GAMES])
def test_oracle_equals_reference_in_lockstep(gs, games):
    from test_ref_vs_oracle import compare
    rng = random.Random(len(gs))
    og, rg = OracleGame(gs), ref_lib.RefGame(gs)
    for _ in range(games):
        o, r = og.new_initial_state(), rg.new_initial_state()
        while True:
            compare(o, r, gs)
            if o.is_terminal():
                break
            a = rng.choice(r.legal_actions())
            o.apply_action(a)
            r.apply_action(a)


# game, prefix plies, simulations, n_rollouts, solve, seed, max_memory_mb
MCTS = [("go(board_size=19)", 10, 40, 1, True, 31, 1000), ("go(board_size=13)", 8, 80, 1, True, 32, 1000),
        ("go(board_size=19,handicap=3)", 4, 30, 2, False, 33, 1000), ("go(board_size=19)", 2, 450, 1, False, 34, 1)]


@needs_ref
@pytest.mark.parametrize("gs,prefix,sims,nroll,solve,seed,mb", MCTS, ids=["%s-%d-%dmb" % (c[0], c[2], c[6]) for c in MCTS])
def test_oracle_mcts_equals_reference_mctsbot_on_large_boards(gs, prefix, sims, nroll, solve, seed, mb):
    rng = random.Random(seed)
    rg, og = ref_lib.RefGame(gs), OracleGame(gs)
    rs, os_ = rg.new_initial_state(), og.new_initial_state()
    for _ in range(prefix):
        a = rng.choice(rs.legal_actions()[:-1])                  # not the pass
        rs.apply_action(a)
        os_.apply_action(a)
    ref = ref_lib.ref_mcts(rg, rs, 2.0, sims, nroll, solve, seed, max_memory_mb=mb)
    max_nodes = (mb << 20) // ref_lib.sizeof_search_node() + 1
    mine = oracle_mcts(os_, 2.0, sims, nroll, solve, seed, reference_rng=True, max_nodes=max_nodes)
    assert [c[:3] for c in mine["children"]] == [tuple(c) for c in ref["children"]]   # order, visits, exact total rewards
    assert mine["best_action"] == ref["best_action"] and mine["root_visits"] == ref["root_visits"]
    if mb == 1:
        assert mine["gc_runs"] >= 1
