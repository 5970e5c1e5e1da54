"""The oracle's CFRBRSolver and TabularBestResponse (oracle/algorithms/cfr_br.cc) against the unmodified reference
(oracle/_ref, live) or, without it, against the reference's pinned results (tests/golden/cfr_br_reference.json): tables
bit for bit after several iteration splits and after deserializing a non-uniform table, best responses in actions and
value bits, and the known answers of algorithms/cfr_br_test.cc."""
import pytest

import cfr_br_lib as L
import golden_lib
import oracle_lib
import ref_lib

needs_ref = pytest.mark.skipif(not L.ref_available(), reason="needs the reference build in oracle/_ref")


@needs_ref
@pytest.mark.parametrize("gs", sorted(L.SPLITS))
def test_oracle_tables_equal_reference_after_each_split(gs):
    o, r = L.OracleCFRBR(oracle_lib.OracleGame(gs)), L.RefCFRBR(ref_lib.RefGame(gs))
    for k in L.SPLITS[gs]:
        o.iterate(k)
        r.iterate(k)
        L.assert_tables_equal(o.table(), r.table())


@needs_ref
@pytest.mark.parametrize("gs", sorted(L.SPLITS))
@pytest.mark.parametrize("iteration", [0, 7])
def test_oracle_equals_reference_after_deserializing_nonuniform_table(gs, iteration):
    """A solver deserialized at iteration 0 answers the uniform policy on its first iteration (SetPolicy is skipped while
    iteration_ == 1), one deserialized at iteration 7 the imported current policy."""
    og, rg = oracle_lib.OracleGame(gs), ref_lib.RefGame(gs)
    table = L.nonuniform_table(L.legal_actions_by_key(og), seed=iteration + 1)
    o = L.OracleCFRBR(og)
    o.load(table, iteration)
    r = L.RefCFRBR(rg)
    r = L.RefCFRBR.deserialize(rg, _reserialize(r.serialize(), table, iteration))
    L.assert_tables_equal(o.table(), r.table())
    for k in (1, 2, 5):
        o.iterate(k)
        r.iterate(k)
        L.assert_tables_equal(o.table(), r.table())


def _reserialize(text, table, iteration):
    """A reference Serialize() text with the iteration and values table replaced (lossless hex doubles)."""
    from open_spiel_b200 import serialization as ser
    head = text.partition("[SolverSpecificState]\n")[0]
    body = "<~>".join("%s<~>%s" % (k, ";".join(",".join(str(x) if f == "legal" else ser.hex_double(x) for x in v[f])
                                                for f in ("legal", "regrets", "cum_policy", "cur_policy")))
                      for k, v in table.items())
    return head + "[SolverSpecificState]\n%d\n[SolverValuesTable]\n%s" % (iteration, body)


@pytest.mark.parametrize("gs", sorted(L.SPLITS))
def test_oracle_best_response_equals_reference(gs):
    """50 seeded random policies per game with exact zeros and ties: chosen actions and value bits, for both players."""
    og = oracle_lib.OracleGame(gs)
    legal = L.legal_actions_by_key(og)
    pins = L.golden()["best_response"]
    rg = ref_lib.RefGame(gs) if L.ref_available() else None
    for seed, player in L.br_cases():
        pol = L.random_policy(legal, seed)
        acts, value = L.oracle_tabular_br(og, player, pol)
        assert [L.br_digest(acts), value.hex()] == pins["%s/%d/%d" % (gs, seed, player)], (seed, player)
        if rg is not None:
            assert (acts, value.hex()) == (lambda a, v: (a, v.hex()))(*L.ref_tabular_br(rg, player, pol)), (seed, player)


@pytest.mark.parametrize("gs,iters", [("kuhn_poker", 300), ("leduc_poker", 100)])
def test_oracle_tables_equal_pinned_reference(gs, iters):
    pin = L.golden()["tables"]["%s@%d" % (gs, iters)]
    o = L.OracleCFRBR(oracle_lib.OracleGame(gs))
    o.iterate(iters)
    assert golden_lib.table_digest(o.table()) == pin["table_sha256"]
    assert abs(o.nash_conv() - pin["nash_conv"]) <= 1e-12


def test_known_answers_kuhn_300():
    """cfr_br_test.cc CFRBRTest_KuhnPoker: expected returns within 1e-3 of the Nash value -1/18, exploitability <= 0.05."""
    pin = L.golden()["tables"]["kuhn_poker@300"]
    o = L.OracleCFRBR(oracle_lib.OracleGame("kuhn_poker"))
    o.iterate(300)
    v = o.average_values()
    for ret in (pin["expected_returns"], v[2:]):
        assert abs(ret[0] - (-1 / 18)) <= 1e-3 and abs(ret[1] - 1 / 18) <= 1e-3
    assert o.exploitability() <= 0.05 and pin["exploitability"] <= 0.05
    if L.ref_available():
        r = L.RefCFRBR(ref_lib.RefGame("kuhn_poker"))
        r.iterate(300)
        ev = r.average_eval()
        assert abs(ev["expected_returns"][0] + 1 / 18) <= 1e-3 and ev["exploitability"] <= 0.05
        assert abs(ev["exploitability"] - o.exploitability()) <= 1e-12


def test_known_answers_serialization_round_trip():
    """cfr_br_test.cc CFRBRTest_CFRBRSolverSerialization: exploitability falls over 50 iterations, survives a
    serialize / deserialize, and falls over 50 more."""
    og = oracle_lib.OracleGame("kuhn_poker")
    o = L.OracleCFRBR(og)
    e0 = o.exploitability()
    o.iterate(50)
    e1 = o.exploitability()
    assert e0 > e1
    o2 = L.OracleCFRBR(og)
    o2.load(o.table(), o.iteration)
    assert abs(o2.exploitability() - e1) <= 1e-4
    o2.iterate(50)
    assert e1 > o2.exploitability()
    if L.ref_available():
        r = L.RefCFRBR(ref_lib.RefGame("kuhn_poker"))
        r0 = r.average_eval()["exploitability"]
        r.iterate(50)
        r1 = r.average_eval()["exploitability"]
        r2 = L.RefCFRBR.deserialize(r.game, r.serialize())
        assert r0 > r1 and abs(r2.average_eval()["exploitability"] - r1) <= 1e-4
        r2.iterate(50)
        assert r1 > r2.average_eval()["exploitability"]
        L.assert_tables_equal(o2.table(), r2.table())
