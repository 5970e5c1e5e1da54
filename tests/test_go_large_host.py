"""CPU: go on boards 10..19 — the 384-bit rule core (GoWideRules, open_spiel_b200/csrc/rules_go.cuh) and the k_mcts /
k_mcts_eval_step kernel bodies on it, compiled for the host by tests/host_emul/go_wide.mk — against the oracle: every observable after
every move of random games (boards 10, 13, 16 and 19, komi, short games, handicap stones), full 19x19 games to the end with
captures and positional superko, the rollout kernel's Philox stream, both MCTS searches, and go_test.cc's known answers."""
import numpy as np
import pytest

import open_spiel_b200 as b2
from oracle_lib import OracleGame, oracle_mcts
from philox_ref import philox_uniform
from test_mcts_eval_host import check_against_oracle, run_emulated
from test_rule_cores_host import Emu, _lockstep
from go_wide_emul import use_wide_libraries


@pytest.fixture(autouse=True)
def _wide_host_build(monkeypatch):
    """Emu / Emv / run_emulated on the host build that also holds go 10..19 (tests/host_emul/go_wide.mk)."""
    use_wide_libraries(monkeypatch)


GAMES = [("go(board_size=10)", 24), ("go(board_size=11,komi=0.5)", 16), ("go(board_size=13)", 16), ("go(board_size=14,komi=6.0)", 12),
         ("go(board_size=16)", 12), ("go(board_size=17,komi=-2.5)", 8), ("go(board_size=19)", 12), ("go", 8),
         ("go(board_size=19,komi=0.0)", 8), ("go(board_size=13,max_game_length=40)", 32), ("go(board_size=19,max_game_length=7)", 16),
         ("go(board_size=19,max_game_length=1000)", 4), ("go(board_size=16,handicap=2)", 8), ("go(board_size=18,handicap=9)", 8)]
GAMES += [("go(board_size=19,handicap=%d)" % h, 6) for h in range(2, 11)] + [("go(board_size=19,handicap=1)", 6),
                                                                           ("go(board_size=19,handicap=17,komi=0.5)", 6)]


@pytest.mark.parametrize("gs,n", GAMES, ids=[g for g, _ in GAMES])
def test_wide_core_lockstep_vs_oracle(gs, n):
    """Current player, terminal flag, returns with the sign of zero, legal actions and both players' observation tensors after
    every move (the lock-step of test_rule_cores_host.py)."""
    _lockstep(gs, n, OracleGame)


def _superko_and_captures(gs, n, seed):
    """Random games on the host core with the rollout kernel's Philox stream; returns (plies, returns, lanes ended by superko)."""
    emu = Emu(gs, n)
    rets, plies = emu.rollout(seed)
    superko = [i for i in range(n) if plies[i] < emu.info.max_game_length and rets[i, 0] == 0.0]   # komi 7.5: no score draws
    return emu, rets, plies, superko


def test_full_19x19_games_with_superko_in_lockstep():
    """Full random 19x19 games played to the end by the host rule core on the Philox stream.  Every game that ends by
    positional superko, and a sample of the others, is replayed by the oracle on the same stream (candidate rejection
    sampling, test_rule_cores_host.py's playout test) — equal lengths and returns — and then move by move in lock-step with
    every observable compared.  Together with the lock-step tests above this checks the exact one-liberty test against the
    oracle's pseudo-liberty sums (kept in the reference's 16 / 32-bit types) over thousands of 19x19 positions per game."""
    gs, n, seed = "go(board_size=19)", 1200, 0x5EED19
    emu, rets, plies, superko = _superko_and_captures(gs, n, seed)
    assert len(superko) >= 1, "this seed has games that end by positional superko"
    og = OracleGame(gs)
    games, captures = {}, 0
    for i in sorted(set(superko) | set(range(0, n, 100))):
        st = og.new_initial_state()
        ply, acts, stones = 0, [], 0
        while not st.is_terminal():
            la, cand = st.legal_actions(), st.rollout_candidates()
            retry = 0
            while True:
                a = cand[philox_uniform(seed, i, ply + 4096 * retry, len(cand))]
                if a in la:
                    break
                retry += 1
            st.apply_action(a)
            acts.append(a)
            now = int(np.sum(st.observation_tensor(0)[:2 * 361]))
            captures += now < stones + (a != 361)
            stones = now
            ply += 1
        assert ply == plies[i] and st.returns() == rets[i].tolist(), (i, ply, plies[i])
        games[i] = acts
    assert captures > 100
    # replay the chosen games move by move on a fresh batch, one lane per game
    lanes = sorted(games)
    emu2 = Emu(gs, len(lanes))
    states = [og.new_initial_state() for _ in lanes]
    for ply in range(max(len(g) for g in games.values()) + 1):
        cur, term, r = emu2.status()
        legal = emu2.legal()
        obs = [emu2.tensor(p, 0) for p in range(2)]
        acts = np.full(len(lanes), -1, dtype=np.int32)
        for j, (lane, st) in enumerate(zip(lanes, states)):
            assert int(cur[j]) == st.current_player() and bool(term[j]) == st.is_terminal(), (lane, ply)
            assert legal[j] == st.legal_actions(), (lane, ply)
            assert r[j].tolist() == st.returns() and np.array_equal(np.signbit(r[j]), np.signbit(np.array(st.returns())))
            for p in range(2):
                np.testing.assert_array_equal(obs[p][j], st.observation_tensor(p))
            if ply < len(games[lane]):
                acts[j] = games[lane][ply]
                st.apply_action(int(acts[j]))
        emu2.apply(acts)
        assert emu2.errors() == 0
    assert emu2.status()[1].all()


@pytest.mark.parametrize("gs", ["go(board_size=13)", "go(board_size=19)", "go(board_size=19,handicap=5)"])
def test_wide_playout_step_matches_oracle_given_same_random_stream(gs):
    from test_rule_cores_host import test_playout_step_matches_oracle_given_same_random_stream as playout
    playout(gs)


@pytest.mark.parametrize("gs", ["go(board_size=%d,handicap=2)" % n for n in range(2, 16)] +
                         ["go(board_size=12,handicap=10)", "go(board_size=9,handicap=5)", "go(board_size=20)", "go(board_size=1)"])
def test_unsupported_configurations_are_rejected(gs):
    """Handicap stones sit on 19x19 coordinates up to row / column 16 (go.cc:72-93): boards 2..15 reject handicap >= 2 when the
    game is configured, as the hex swap rule is rejected where the reference's mirror is undefined.  Sizes beyond 2..19 too."""
    with pytest.raises(b2.SpielError):
        b2.load_game(gs)


def test_go_test_cc_known_answers_on_the_wide_core():
    # go_test.cc:54-67: 13x13 has 169 + 1 legal actions at the start
    emu = Emu("go(board_size=13)", 1)
    assert emu.info.num_distinct_actions == 170 and len(emu.legal()[0]) == 170
    # go_test.cc:43-52 HandicapTest: 19x19, komi 7.5, handicap 2 -> white to play, black stones on d4 and q16
    emu = Emu("go(board_size=19,komi=7.5,handicap=2)", 1)
    cur, term, _ = emu.status()
    assert int(cur[0]) == 1 and term[0] == 0
    black = emu.tensor(0, 0)[0][:361]
    assert black[3 * 19 + 3] == 1.0 and black[15 * 19 + 15] == 1.0 and black.sum() == 2
    assert emu.tensor(0, 0)[0][3 * 361:].all()                # plane 3: white to play
    # handicap > 9 places no stone but white still moves first (HandicapStones returns {}, ResetBoard go.cc:290-296)
    emu = Emu("go(board_size=19,handicap=12)", 1)
    assert int(emu.status()[0][0]) == 1 and emu.tensor(0, 0)[0][:722].sum() == 0


# game, trees, prefix plies, sims, n_rollouts, solve, PUCT[, node budget]
MCTS_CASES = [("go(board_size=13)", 4, 12, 40, 1, True, False), ("go(board_size=13)", 3, 6, 30, 3, False, True),
              ("go(board_size=19)", 3, 10, 25, 1, True, False), ("go(board_size=19)", 3, 4, 20, 2, False, True),
              ("go(board_size=19,handicap=4)", 2, 6, 20, 1, True, True),
              # max_memory_mb = 1: MCTSBot::max_nodes_ = (1 << 20) / 80 + 1 = 13108, i.e. about 36 expansions of 362 children
              ("go(board_size=19)", 2, 4, 480, 1, True, False, 13108), ("go(board_size=13)", 2, 4, 300, 1, False, True, 13108)]


@pytest.mark.parametrize("case", MCTS_CASES, ids=["%s-%d-%d%s%s" % (c[0], c[3], c[4], "-puct" if c[6] else "", "-gc" if len(c) > 7 else "")
                                                  for c in MCTS_CASES])
def test_mcts_kernel_body_on_wide_core_equals_oracle(case):
    """k_mcts (mcts.cuh) on the host, one tree at a time, vs the oracle's MCTS on the same Philox stream: 362-child expansions
    in the 9-bit child-count field, the 16-bit collector cursor, 16- and 24-byte nodes."""
    import math
    gs, n, prefix, sims, nroll, solve, puct = case[:7]
    budget = case[7] if len(case) > 7 else 0
    rng = np.random.RandomState(len(gs) + sims)
    og = OracleGame(gs)
    emu = Emu(gs, n)
    states = [og.new_initial_state() for _ in range(n)]
    for t in range(prefix):
        acts = np.full(n, -1, dtype=np.int32)
        for i, st in enumerate(states):
            la = st.legal_actions()
            acts[i] = la[rng.randint(len(la))]
            st.apply_action(int(acts[i]))
        emu.apply(acts)
    assert emu.errors() == 0
    visits, reward, outcome, best, ran = emu.mcts(sims, 2.0, nroll, solve, seed=0xC0FFEE, offset=17, puct=puct, budget=budget)
    assert emu.errors() == 0
    collections = 0
    for i, st in enumerate(states):
        o = oracle_mcts(st, 2.0, sims, nroll, solve, 0xC0FFEE, tree_index=i + 17, puct=puct, max_nodes=budget or 1)
        assert ran[i] == o["sims_run"] and emu.gc_runs[i] == o["gc_runs"], (gs, i)
        collections += o["gc_runs"]
        assert len(o["children"]) == len(st.legal_actions())
        for a, v, r, oc in o["children"]:
            assert visits[i, a] == v and reward[i, a] == r, (gs, i, a)
            assert (math.isnan(oc) and math.isnan(outcome[i, a])) or outcome[i, a] == oc, (gs, i, a)
        assert int(visits[i].sum()) == sum(v for _, v, _, _ in o["children"])
        assert best[i] == o["best_action"], (gs, i)
    if budget:
        assert collections >= n, "the budget must actually trigger garbage collections in this case"


# game, trees, prefix plies, sims, solve, PUCT, node budget, dirichlet alpha
EVAL_CASES = [("go(board_size=13)", 4, 8, 40, True, True, 0, 0.03), ("go(board_size=19)", 3, 6, 30, False, True, 0, 0.0),
              ("go(board_size=19,handicap=3)", 2, 4, 25, True, False, 0, 0.3), ("go(board_size=19)", 2, 2, 1000, True, True, 13108, 0.0)]


@pytest.mark.parametrize("gs,n,prefix,sims,solve,puct,budget,alpha", EVAL_CASES,
                         ids=["%s-%d%s%s%s" % (c[0], c[3], "-puct" if c[5] else "", "-gc" if c[6] else "", "-noise" if c[7] else "")
                              for c in EVAL_CASES])
def test_eval_kernel_body_on_wide_core_equals_oracle(gs, n, prefix, sims, solve, puct, budget, alpha):
    """k_mcts_eval_step on the host, round by round with tests/mcts_eval_lib.py's evaluator, vs oracle/algorithms/mcts_eval.cc."""
    out, rounds, states, noise = run_emulated(gs, n, prefix, sims, solve, puct, budget, alpha)
    collections = check_against_oracle(out, states, sims, solve, puct, budget, noise, alpha, tag=gs)
    assert rounds <= int((out["sims_run"] + out["prior_requests"]).max())
    if budget:
        assert collections >= n and int(out["prior_requests"].sum()) > 0
