"""The oracle's Discounted CFR (oracle/algorithms/dcfr.cc) against the reference's own Python solver: the checkout's
python/algorithms/discounted_cfr.py, loaded by path with cfr.py, policy.py and get_all_states.py over the unmodified
reference games (oracle/_ref), or, without the checkout, against its pinned digests (tests/golden/dcfr_reference.json,
written by tests/golden/make_dcfr_reference.py).  Key set, regrets with the sign of zero, cumulative policy, current policy
and average policy bit for bit after each split, for every variant; a seeded table whose zero-reach pruning decides
stored bits; and the known answers of discounted_cfr_test.py."""
import pytest

import cfr_br_lib
import dcfr_lib as L
import oracle_lib
from exact_policy_eval import evaluate

needs_ref = pytest.mark.skipif(not L.ref_available(), reason="needs the OpenSpiel checkout and oracle/_ref")


def _check(o, r):
    ot = o.table()
    L.assert_tables_equal(ot, r.table())
    assert L.average_policy(ot) == r.average_policy()


@needs_ref
@pytest.mark.parametrize("variant", sorted(L.VARIANTS))
@pytest.mark.parametrize("gs", sorted(L.REF_SPLITS))
def test_oracle_equals_reference_after_each_split(gs, variant):
    o, r = L.OracleDCFR(oracle_lib.OracleGame(gs), *L.VARIANTS[variant]), L.RefDCFR(gs, variant)
    for k in L.REF_SPLITS[gs]:
        o.iterate(k)
        r.iterate(k)
        _check(o, r)


@needs_ref
@pytest.mark.parametrize("gs", sorted(L.REF_SPLITS))
def test_integral_floats_give_the_bits_of_ints(gs):
    """DCFRSolver(game, 1.5, 0.0, 2.0) and DCFRSolver(game, 1.0, 1.0, 1.0) in the reference compute t**k in floats, the
    defaults in Python ints: the tables agree bit for bit."""
    for ints, floats in (("dcfr", "dcfr_floats"), ("lcfr", "lcfr_floats")):
        a, b = L.RefDCFR(gs, ints), L.RefDCFR(gs, floats)
        a.iterate(L.REF_SPLITS[gs][-1])
        b.iterate(L.REF_SPLITS[gs][-1])
        L.assert_tables_equal(a.table(), b.table())


@needs_ref
@pytest.mark.parametrize("gs", sorted(L.ZERO_REACH_SPLITS))
def test_zero_reach_pruning_decides_bits_as_in_the_reference(gs):
    """A seeded table with a pure current policy and -0.0 regrets, loaded into both solvers (numpy float64 on the
    reference side) at iteration 3: the oracle equals the reference after each split.  Its stored bits differ from those
    of the oracle without pruning, and from those of the oracle that prunes the table updates but not the values, so
    both halves of the pruning are exercised."""
    og = oracle_lib.OracleGame(gs)
    table = L.zero_reach_table(cfr_br_lib.legal_actions_by_key(og), seed=L.ZERO_REACH_SEED)
    o, r = L.OracleDCFR(og, *L.VARIANTS["dcfr"]), L.RefDCFR(gs, "dcfr")
    contrasts = [L.OracleDCFR(og, *L.VARIANTS["dcfr"], prune=m) for m in (L.PRUNE_NONE, L.PRUNE_UPDATES)]
    for s in (o, r, *contrasts):
        s.load(table, 3)
    _check(o, r)
    differ = [0, 0]
    for k in L.ZERO_REACH_SPLITS[gs]:
        for s in (o, r, *contrasts):
            s.iterate(k)
        _check(o, r)
        t = o.table()
        for i, c in enumerate(contrasts):
            differ[i] = max(differ[i], min(L.negative_zeros(t), L.sign_differences(t, c.table())))
    assert min(differ) > 0, differ


@pytest.mark.parametrize("variant", sorted(L.VARIANTS))
@pytest.mark.parametrize("gs", sorted(L.REF_SPLITS))
def test_oracle_equals_pinned_reference(gs, variant):
    pins = L.golden()["splits"]["%s/%s" % (gs, variant)]
    o = L.OracleDCFR(oracle_lib.OracleGame(gs), *L.VARIANTS[variant])
    done = 0
    for k in L.REF_SPLITS[gs]:
        o.iterate(k)
        done += k
        assert L.digests(o.table()) == pins[str(done)], done


@pytest.mark.parametrize("gs", sorted(L.ZERO_REACH_SPLITS))
def test_zero_reach_oracle_equals_pinned_reference(gs):
    og = oracle_lib.OracleGame(gs)
    table = L.zero_reach_table(cfr_br_lib.legal_actions_by_key(og), seed=L.ZERO_REACH_SEED)
    pins = L.golden()["zero_reach"][gs]
    o = L.OracleDCFR(og, *L.VARIANTS["dcfr"])
    o.load(table, 3)
    done = 3
    for k in L.ZERO_REACH_SPLITS[gs]:
        o.iterate(k)
        done += k
        assert L.digests(o.table()) == pins[str(done)], done


def _nash_conv(gs, table):
    """Exact NashConv of the average policy of a {key: ...} table, through exact_policy_eval in the device layout."""
    import numpy as np
    og = oracle_lib.OracleGame(gs)
    tensors = oracle_lib.infostate_tensors(og)
    keys = list(table)
    offsets = np.cumsum([0] + [len(table[k]["legal"]) for k in keys]).astype(np.int32)
    dev = {"offsets": offsets, "legal_actions": np.array([a for k in keys for a in table[k]["legal"]], dtype=np.int32),
           "keys": np.stack([np.frombuffer(tensors[k], dtype=np.float32) for k in keys])}
    cum = np.array([x for k in keys for x in table[k]["cum_policy"]])
    return evaluate(gs, dev, cum, average=True)


def test_known_answers():
    """discounted_cfr_test.py: after 300 iterations on kuhn_poker the average policy's expected values are within 1e-3 of
    (-1/18, 1/18), for DCFRSolver and LCFRSolver; leduc_poker runs 10 iterations."""
    for variant in ("dcfr", "lcfr"):
        o = L.OracleDCFR(oracle_lib.OracleGame("kuhn_poker"), *L.VARIANTS[variant])
        o.iterate(300)
        v = _nash_conv("kuhn_poker", o.table())["values"]
        assert abs(float(v[2]) + 1 / 18) < 1e-3 and abs(float(v[3]) - 1 / 18) < 1e-3, variant
    o = L.OracleDCFR(oracle_lib.OracleGame("leduc_poker"), *L.VARIANTS["dcfr"])
    o.iterate(10)
    assert o.iteration == 10
