"""GPU: the device DCFRSolver / LCFRSolver (k_dcfr) against the oracle's restatement of discounted_cfr.py
(oracle/algorithms/dcfr.cc) and the reference's pinned digests (tests/golden/dcfr_reference.json): regrets with the sign
of zero, cumulative, current and average policy of every information state bit for bit after each split, for every
variant, to 10,000 iterations; the seeded zero-reach case; launch splits on two streams, resuming at an imported iteration,
NashConv, the known answers of discounted_cfr_test.py, and the errors a DCFR solver reports."""
import ctypes as C
import math

import numpy as np
import pytest

import cfr_br_lib
import dcfr_lib as L
import golden_lib
import open_spiel_b200 as b2
from exact_policy_eval import evaluate
from open_spiel_b200 import serialization as ser
from open_spiel_b200._lib import B2SError, check, lib
from oracle_lib import OracleGame, infostate_tensors

pytestmark = pytest.mark.gpu


def solver(gs, variant):
    game = b2.load_game(gs)
    if variant == "dcfr":
        return b2.DCFRSolver(game)
    if variant == "lcfr":
        return b2.LCFRSolver(game)
    return b2.DCFRSolver(game, *L.VARIANTS[variant])


def by_key(dev, og):
    return golden_lib.device_table_by_key(dev.table(), infostate_tensors(og))


def load_by_key(dev, table, iteration):
    t = dev.table()
    r, c, p = ser.table_arrays_from(table, ser.table_keys(dev.game._name, t), t)
    dev.load_table(r, c, p, iteration=iteration)


def check_equal(dev, og, cpu_table):
    table = by_key(dev, og)
    L.assert_tables_equal(table, cpu_table)
    avg = {k: [p for _, p in v] for k, v in dev.tabular_average_policy().items()}
    assert avg == L.average_policy(cpu_table)
    return table


@pytest.mark.parametrize("variant", sorted(L.VARIANTS))
@pytest.mark.parametrize("gs", sorted(L.DEV_SPLITS))
def test_device_equals_oracle_after_each_split(gs, variant):
    og = OracleGame(gs)
    dev, cpu = solver(gs, variant), L.OracleDCFR(og, *L.VARIANTS[variant])
    for k in L.DEV_SPLITS[gs]:
        dev.evaluate_and_update_policy(k)
        cpu.iterate(k)
        check_equal(dev, og, cpu.table())
    assert dev.info().iteration == sum(L.DEV_SPLITS[gs]) == 10000


@pytest.mark.parametrize("variant", sorted(L.VARIANTS))
@pytest.mark.parametrize("gs", sorted(L.REF_SPLITS))
def test_device_equals_pinned_reference(gs, variant):
    pins = L.golden()["splits"]["%s/%s" % (gs, variant)]
    og = OracleGame(gs)
    dev = solver(gs, variant)
    done = 0
    for k in L.REF_SPLITS[gs]:
        dev.evaluate_and_update_policy(k)
        done += k
        assert L.digests(by_key(dev, og)) == pins[str(done)], done


@pytest.mark.parametrize("gs", sorted(L.ZERO_REACH_SPLITS))
def test_zero_reach_seeded_table(gs):
    """-0.0 regrets below zero-probability edges of both players: the device prunes as the reference does (pinned
    digests, oracle after each split).  Its stored bits differ from the oracle's without pruning and from the oracle's
    that prunes the table updates but keeps the unpruned values, so both the skipped updates and the pruned values count."""
    og = OracleGame(gs)
    table = L.zero_reach_table(cfr_br_lib.legal_actions_by_key(og), seed=L.ZERO_REACH_SEED)
    pins = L.golden()["zero_reach"][gs]
    dev, cpu = b2.DCFRSolver(b2.load_game(gs)), L.OracleDCFR(og, *L.VARIANTS["dcfr"])
    contrasts = [L.OracleDCFR(og, *L.VARIANTS["dcfr"], prune=m) for m in (L.PRUNE_NONE, L.PRUNE_UPDATES)]
    load_by_key(dev, table, 3)
    for s in (cpu, *contrasts):
        s.load(table, 3)
    done, differ = 3, [0, 0]
    for k in L.ZERO_REACH_SPLITS[gs]:
        dev.evaluate_and_update_policy(k)
        for s in (cpu, *contrasts):
            s.iterate(k)
        done += k
        t = check_equal(dev, og, cpu.table())
        assert L.digests(t) == pins[str(done)], done
        for i, c in enumerate(contrasts):
            differ[i] = max(differ[i], min(L.negative_zeros(t), L.sign_differences(t, c.table())))
    assert min(differ) > 0, differ


@pytest.mark.parametrize("gs,n", [("kuhn_poker", 70000), ("leduc_poker", 9)])
@pytest.mark.parametrize("side_stream", [False, True])
def test_launch_splits_agree(gs, n, side_stream):
    """One call of n iterations = n calls of 1 = mixed splits; on kuhn_poker every split leaves the first 65,536-iteration
    factor window while earlier launches are still queued."""
    import torch
    runs = {"one": [n], "ones": [1] * n, "mixed": [2, 1, n - 6, 3]}
    stream = torch.cuda.Stream() if side_stream else torch.cuda.current_stream()
    tables = {}
    with torch.cuda.stream(stream):
        for name, split in runs.items():
            dev = b2.DCFRSolver(b2.load_game(gs))
            for k in split:
                dev.evaluate_and_update_policy(k)
            tables[name] = dev.table()
    for name in ("ones", "mixed"):
        for f in ("regrets", "cum_policy", "cur_policy"):
            assert tables[name][f].tobytes() == tables["one"][f].tobytes(), (name, f)


@pytest.mark.parametrize("variant", ["dcfr", "a2_b0.5_g3"])
def test_import_at_iteration_continues_with_its_factors(variant):
    """Export after k iterations, import into a fresh solver at iteration k, continue: the same bits as an uninterrupted
    run, so the resumed solver reads factor k + 1 on (its factor window starts at an iteration it never ran)."""
    gs = "leduc_poker"
    for k in (12, 1500):
        a, b = solver(gs, variant), solver(gs, variant)
        a.evaluate_and_update_policy(k)
        t = a.table()
        b.load_table(t["regrets"], t["cum_policy"], t["cur_policy"], iteration=k)
        a.evaluate_and_update_policy(7)
        b.evaluate_and_update_policy(7)
        ta, tb = a.table(), b.table()
        for f in ("regrets", "cum_policy", "cur_policy"):
            assert ta[f].tobytes() == tb[f].tobytes(), (k, f)
        c = solver(gs, variant)                  # a wrong counter gives other bits
        c.load_table(t["regrets"], t["cum_policy"], t["cur_policy"], iteration=k + 1)
        c.evaluate_and_update_policy(7)
        assert c.table()["regrets"].tobytes() != ta["regrets"].tobytes()


def test_long_calls_run_as_several_launches():
    """A call of more than 2**20 iterations runs as several launches, each with its own factor window: the same bits as
    calls split elsewhere."""
    a, b = b2.DCFRSolver(b2.load_game("kuhn_poker")), b2.DCFRSolver(b2.load_game("kuhn_poker"))
    a.evaluate_and_update_policy(2**20 + 3)
    for k in (70000, 2**20 - 70000, 3):
        b.evaluate_and_update_policy(k)
    assert a.info().iteration == b.info().iteration == 2**20 + 3
    ta, tb = a.table(), b.table()
    for f in ("regrets", "cum_policy", "cur_policy"):
        assert ta[f].tobytes() == tb[f].tobytes(), f


@pytest.mark.parametrize("gs", sorted(L.ZERO_REACH_SPLITS))
def test_counter_runs_to_int_max(gs):
    """A table imported 3 iterations below INT_MAX runs its last 3 iterations with the factors of t = 2**31 - 3 .. 2**31 - 1,
    as the oracle does, and the counter then refuses to go further."""
    og = OracleGame(gs)
    table = L.zero_reach_table(cfr_br_lib.legal_actions_by_key(og), seed=L.ZERO_REACH_SEED)
    dev, cpu = b2.DCFRSolver(b2.load_game(gs)), L.OracleDCFR(og, *L.VARIANTS["dcfr"])
    load_by_key(dev, table, 2**31 - 4)
    cpu.load(table, 2**31 - 4)
    for k in (1, 2):
        dev.evaluate_and_update_policy(k)
        cpu.iterate(k)
        check_equal(dev, og, cpu.table())
    assert dev.info().iteration == 2**31 - 1
    with pytest.raises(B2SError, match="iteration counter"):
        dev.evaluate_and_update_policy(1)


@pytest.mark.parametrize("gs,iters", [("kuhn_poker", 1000), ("leduc_poker", 100)])
def test_nash_conv_equals_exact_evaluation(gs, iters):
    dev = b2.DCFRSolver(b2.load_game(gs))
    dev.evaluate_and_update_policy(iters)
    t = dev.table()
    want = evaluate(gs, t, t["cum_policy"], average=True)
    assert abs(dev.nash_conv() - float(want["nash_conv"])) <= 1e-9
    assert all(abs(a - float(b)) <= 1e-9 for a, b in zip(dev.last_values, want["values"]))


def test_known_answers_kuhn_300():
    """discounted_cfr_test.py: after 300 iterations the average policy's expected values are within 1e-3 of
    (-1/18, 1/18), for DCFRSolver and LCFRSolver."""
    for dev in (b2.DCFRSolver(b2.load_game("kuhn_poker")), b2.LCFRSolver(b2.load_game("kuhn_poker"))):
        dev.evaluate_and_update_policy(300)
        dev.nash_conv()
        v = dev.last_values[2:]
        assert abs(v[0] + 1 / 18) < 1e-3 and abs(v[1] - 1 / 18) < 1e-3, type(dev).__name__
    leduc = b2.DCFRSolver(b2.load_game("leduc_poker"))
    leduc.evaluate_and_update_policy(10)
    assert leduc.info().iteration == 10


def test_errors_leave_tables_untouched():
    L_ = lib()
    game = b2.load_game("kuhn_poker")
    for bad in ((math.nan, 0.0, 2.0), (1.5, math.inf, 2.0), (1.5, 0.0, -math.inf)):
        h = C.c_void_p()
        with pytest.raises(B2SError, match="finite"):
            check(L_.b2s_dcfr_create(game._gid, C.byref(game._cparams), *bad, game.device, C.byref(h)))
        assert not h.value
    with pytest.raises(B2SError):
        b2.DCFRSolver(b2.load_game("kuhn_poker(players=3)"))
    dev = b2.DCFRSolver(game)
    dev.evaluate_and_update_policy(5)
    before = dev.table()
    with pytest.raises(B2SError, match="DCFR"):
        check(L_.b2s_cfr_traverse_shard(dev._h, 0, 6, 0, 1, None))
    with pytest.raises(B2SError, match="DCFR"):
        check(L_.b2s_cfr_apply_deltas(dev._h, None))
    with pytest.raises(B2SError, match="DCFR"):
        check(L_.b2s_cfr_iterate_sharded(dev._h, 2, None))
    with pytest.raises(B2SError):
        check(L_.b2s_mccfr_external_iterate(dev._h, 1, 1, 0, None))
    with pytest.raises(B2SError):
        check(L_.b2s_mccfr_outcome_iterate(dev._h, 1, 1, 0, 0.6, None))
    with pytest.raises(B2SError, match="DCFRSolver.serialize"):
        dev.serialize()
    with pytest.raises(B2SError, match="DCFRSolver.load_serialized"):
        dev.load_serialized(b2.CFRSolver(game).serialize())
    check(L_.b2s_cfr_set_iteration(dev._h, -1))
    with pytest.raises(B2SError, match="iteration counter"):
        dev.evaluate_and_update_policy(1)
    check(L_.b2s_cfr_set_iteration(dev._h, 2**31 - 3))
    with pytest.raises(B2SError, match="iteration counter"):
        dev.evaluate_and_update_policy(3)
    with pytest.raises(B2SError, match="iteration counter"):
        dev.evaluate_and_update_policy(2**31 - 1)
    check(L_.b2s_cfr_set_iteration(dev._h, 5))
    after = dev.table()
    for f in ("regrets", "cum_policy", "cur_policy"):
        assert before[f].tobytes() == after[f].tobytes(), f
    assert dev.info().iteration == 5
    ref = b2.DCFRSolver(game)
    ref.evaluate_and_update_policy(5)
    dev.evaluate_and_update_policy(3)
    ref.evaluate_and_update_policy(3)
    for f in ("regrets", "cum_policy", "cur_policy"):
        assert dev.table()[f].tobytes() == ref.table()[f].tobytes(), f
