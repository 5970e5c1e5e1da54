"""Pins tests/exact_policy_eval.py, the exact-arithmetic NashConv / best-response evaluator the device NashConv kernel is
checked against: exactly 0 on Kuhn's closed-form equilibria, the stored NashConv of the unmodified reference at the CFR
checkpoints, and (where oracle/_ref was built) the live reference on random and sparse average-policy tables."""
from fractions import Fraction

import numpy as np
import pytest

import exact_policy_eval as E
import golden_lib
import ref_lib
from oracle_lib import OracleCFR, OracleGame, infostate_tensors


def test_kuhn_closed_form_equilibria_are_exact():
    """The standard equilibrium family of 2-player Kuhn poker, alpha in [0, 1/3]: NashConv exactly 0, game value exactly
    -1/18 for player 0, and every best-response value equal to the on-policy value.  With the deal probabilities as the
    oracle's doubles every deal still has the same probability, so NashConv stays exactly 0."""
    gs = "kuhn_poker"
    t = E.tree(gs)
    layout = t.layout()
    for alpha in (Fraction(0), Fraction(1, 6), Fraction(1, 3)):
        policy = E.kuhn_equilibrium(gs, layout, alpha)
        assert all(isinstance(p, Fraction) for p in policy)
        for average in (False, True):
            r = E.evaluate(gs, layout, policy, average, rational_chance=True)
            assert r["nash_conv"] == 0, alpha
            assert r["values"] == [Fraction(-1, 18), Fraction(1, 18), Fraction(-1, 18), Fraction(1, 18)], alpha
            assert E.evaluate(gs, layout, policy, average)["nash_conv"] == 0, alpha
    # a policy away from the family is exploitable: player 1 always calling with the jack loses to a bluffing jack
    policy = E.kuhn_equilibrium(gs, layout, Fraction(1, 3))
    k = E.row_strings(gs, layout).index("0b")
    lo = layout["offsets"][k]
    policy[lo], policy[lo + 1] = Fraction(0), Fraction(1)
    assert E.evaluate(gs, layout, policy, False)["nash_conv"] > 0


def test_uniform_fallback_of_all_zero_rows():
    """CFRAveragePolicy: an all-zero cumulative row is the uniform policy, like a row of equal entries."""
    for gs in ("kuhn_poker", "leduc_poker"):
        layout = E.tree(gs).layout()
        zero = E.evaluate(gs, layout, np.zeros(len(layout["legal_actions"])), True)
        ones = E.evaluate(gs, layout, np.ones(len(layout["legal_actions"])), True)
        assert zero["values"] == ones["values"]
    assert float(zero["nash_conv"]) == golden_lib.reference_results()["cfr"]["checkpoints"]["leduc_poker"][0]["nash_conv"]


@pytest.mark.parametrize("gs", ["kuhn_poker", "leduc_poker"])
def test_matches_stored_reference_nash_conv_of_cfr(gs):
    """The oracle's CFR equals the reference bit for bit; the exact NashConv of its average policy must be within 1e-12 of
    the reference's double NashConv at every stored checkpoint."""
    gold = golden_lib.reference_results()["cfr"]["checkpoints"][gs]
    og = OracleGame(gs)
    cfr = OracleCFR(og)
    t = E.tree(gs)
    layout = t.layout()
    done = 0
    for g in gold:
        cfr.iterate(g["iterations"] - done)
        done = g["iterations"]
        table = cfr.table()
        cum = np.concatenate([table[s]["cum_policy"] for s in t.is_string])
        r = E.evaluate(gs, layout, cum, True)
        assert abs(r["nash_conv"] - Fraction(g["nash_conv"])) <= 1e-12, (gs, g["iterations"], float(r["nash_conv"]))
        assert abs(r["nash_conv"] / 2 - Fraction(g["exploitability"])) <= 1e-12


def test_tree_keys_match_oracle_information_state_tensors():
    for gs in ("kuhn_poker", "leduc_poker", "leduc_poker(starting_player=1)"):
        t = E.tree(gs)
        tensors = infostate_tensors(t.oracle_game)
        assert len(tensors) == len(t.is_key)
        assert all(tensors[s] == k for s, k in zip(t.is_string, t.is_key))


@pytest.mark.skipif(not ref_lib.available(), reason="the unmodified reference was not built (oracle/_ref)")
@pytest.mark.parametrize("gs", ["kuhn_poker", "leduc_poker", "leduc_poker(starting_player=1)"])
def test_matches_live_reference_on_random_tables(gs):
    """Cumulative-policy tables the reference never produces by training, loaded into the unmodified reference's
    CFRSolver through its own DeserializeCFRSolver: Dirichlet rows, sparse rows (exact zeros), all-zero rows, rows
    scaled by 1e-30 / 1e+30.  The reference's NashConv of the average policy must be within 1e-12 of the exact one."""
    from open_spiel_b200 import serialization as ser
    t = E.tree(gs)
    layout = t.layout()
    rg = ref_lib.RefGame(gs)
    n = len(layout["legal_actions"])
    cases = [E.dirichlet(layout, s) for s in (0, 1)] + [E.sparse(layout, s) for s in (2, 3)] + \
            [E.pure(layout, 4), E.tiny(layout, 5), E.cum_mixed(layout, 6)]
    for case, cum in enumerate(cases):
        table = dict(layout, regrets=np.zeros(n), cum_policy=np.asarray(cum, dtype=np.float64), cur_policy=E.uniform(layout))
        text = ser.serialize_cfr_solver(ref_lib.game_to_string(rg), "CFRSolver", 0, t.is_string, table)
        ref = ref_lib.cfr_deserialize(rg, text)
        exact = E.evaluate(gs, layout, table["cum_policy"], True)["nash_conv"]
        assert abs(Fraction(ref.nash_conv()) - exact) <= 1e-12, (gs, case, ref.nash_conv(), float(exact))
