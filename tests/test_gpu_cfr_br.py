"""GPU: the device CFRBRSolver (k_cfr_br) against the oracle's restatement of algorithms/cfr_br.cc and the unmodified
reference (live when oracle/_ref is present, else its digests in tests/golden/cfr_br_reference.json): regrets, cumulative
policy and current policy of every information state bit for bit, across launch splits, streams, checkpoints and the
reference's own serialized text; and the errors a CFR-BR solver reports."""
import ctypes as C

import numpy as np
import pytest

import cfr_br_lib as L
import golden_lib
import open_spiel_b200 as b2
import ref_lib
from open_spiel_b200 import serialization as ser
from open_spiel_b200._lib import B2SError, check, lib
from oracle_lib import OracleGame, infostate_tensors

pytestmark = pytest.mark.gpu

TREE = {"kuhn_poker": (4, 24, 30, 12), "leduc_poker": (157, 3780, 5520, 936)}   # api_test.py:77-104


def by_key(dev, og):
    return golden_lib.device_table_by_key(dev.table(), infostate_tensors(og))


def load_by_key(dev, table, iteration):
    t = dev.table()
    r, c, p = ser.table_arrays_from(table, ser.table_keys(dev.game._name, t), t)
    dev.load_table(r, c, p, iteration=iteration)


@pytest.mark.parametrize("gs", sorted(L.SPLITS))
def test_device_equals_oracle_after_each_split(gs):
    og = OracleGame(gs)
    dev, cpu = b2.CFRBRSolver(b2.load_game(gs)), L.OracleCFRBR(og)
    info = dev.info()
    assert (info.chance_nodes, info.decision_nodes, info.terminal_nodes, info.num_infosets) == TREE[gs]
    for k in L.SPLITS[gs]:
        dev.evaluate_and_update_policy(k)
        cpu.iterate(k)
        L.assert_tables_equal(by_key(dev, og), cpu.table())
    assert dev.info().iteration == sum(L.SPLITS[gs])


@pytest.mark.parametrize("gs,iters", L.PINNED)
def test_device_equals_pinned_and_live_reference(gs, iters):
    pin = L.golden()["tables"]["%s@%d" % (gs, iters)]
    og = OracleGame(gs)
    dev = b2.CFRBRSolver(b2.load_game(gs))
    dev.evaluate_and_update_policy(iters)
    table = by_key(dev, og)
    assert golden_lib.table_digest(table) == pin["table_sha256"]
    assert abs(dev.nash_conv() - pin["nash_conv"]) <= 1e-9
    if L.ref_available() and iters <= 100:
        ref = L.RefCFRBR(ref_lib.RefGame(gs))
        ref.iterate(iters)
        L.assert_tables_equal(table, ref.table())


def test_device_known_answers_kuhn_300():
    """cfr_br_test.cc CFRBRTest_KuhnPoker on the device tables: expected returns of the average policy within 1e-3 of
    (-1/18, 1/18), exploitability <= 0.05."""
    dev = b2.CFRBRSolver(b2.load_game("kuhn_poker"))
    dev.evaluate_and_update_policy(300)
    expl = dev.exploitability()
    on_policy = dev.last_values[2:]
    assert abs(on_policy[0] + 1 / 18) <= 1e-3 and abs(on_policy[1] - 1 / 18) <= 1e-3
    assert expl <= 0.05


@pytest.mark.parametrize("gs,n", [("kuhn_poker", 23), ("leduc_poker", 9)])
@pytest.mark.parametrize("side_stream", [False, True])
def test_launch_splits_agree(gs, n, side_stream):
    import torch
    game = b2.load_game(gs)
    runs = {"one": [n], "ones": [1] * n, "mixed": [2, 1, n - 6, 3]}
    stream = torch.cuda.Stream() if side_stream else torch.cuda.current_stream()
    tables = {}
    with torch.cuda.stream(stream):
        for name, split in runs.items():
            dev = b2.CFRBRSolver(game)
            for k in split:
                dev.evaluate_and_update_policy(k)
            tables[name] = dev.table()
    for name in ("ones", "mixed"):
        for f in ("regrets", "cum_policy", "cur_policy"):
            assert np.array_equal(tables[name][f], tables["one"][f]), (name, f)


def test_export_import_resumes_exactly():
    game = b2.load_game("leduc_poker")
    a, b = b2.CFRBRSolver(game), b2.CFRBRSolver(game)
    a.evaluate_and_update_policy(12)
    t = a.table()
    b.load_table(t["regrets"], t["cum_policy"], t["cur_policy"], iteration=12)
    a.evaluate_and_update_policy(7)
    b.evaluate_and_update_policy(7)
    ta, tb = a.table(), b.table()
    for f in ("regrets", "cum_policy", "cur_policy"):
        assert np.array_equal(ta[f], tb[f]), f


@pytest.mark.parametrize("gs", sorted(L.SPLITS))
def test_iteration_zero_import_answers_the_uniform_policy(gs):
    """A non-uniform table imported at iteration 0: iteration 1's best responses answer the uniform policy, as
    CFRBRSolver's; at iteration 7 they answer the imported current policy."""
    og = OracleGame(gs)
    table = L.nonuniform_table(L.legal_actions_by_key(og), seed=3)
    for iteration in (0, 7):
        dev, cpu = b2.CFRBRSolver(b2.load_game(gs)), L.OracleCFRBR(og)
        load_by_key(dev, table, iteration)
        cpu.load(table, iteration)
        for k in (1, 1, 4):
            dev.evaluate_and_update_policy(k)
            cpu.iterate(k)
            L.assert_tables_equal(by_key(dev, og), cpu.table())


def test_serialized_text_round_trips_with_the_reference():
    og = OracleGame("kuhn_poker")
    dev = b2.CFRBRSolver(b2.load_game("kuhn_poker"))
    dev.evaluate_and_update_policy(40)
    text = dev.serialize()
    assert "[SolverType]\nCFRBRSolver\n" in text
    resumed = b2.CFRBRSolver(b2.load_game("kuhn_poker"))
    resumed.load_serialized(text)
    assert resumed.info().iteration == 40
    cpu = L.OracleCFRBR(og)
    cpu.iterate(40)
    L.assert_tables_equal(by_key(resumed, og), cpu.table())
    with pytest.raises(B2SError):
        resumed.load_serialized(text.replace("[SolverType]\nCFRBRSolver", "[SolverType]\nCFRSolver"))
    if not L.ref_available():
        return
    rg = ref_lib.RefGame("kuhn_poker")
    ref = L.RefCFRBR.deserialize(rg, text)              # DeserializeCFRBRSolver loads the device's text ...
    ref.iterate(25)
    dev.evaluate_and_update_policy(25)                  # ... and continues bit for bit with the device
    L.assert_tables_equal(by_key(dev, og), ref.table())
    ref.iterate(5)
    back = b2.CFRBRSolver(b2.load_game("kuhn_poker"))   # the device resumes from the reference's Serialize()
    back.load_serialized(ref.serialize())
    ref.iterate(10)
    back.evaluate_and_update_policy(10)
    L.assert_tables_equal(by_key(back, og), ref.table())


def test_errors_leave_tables_untouched():
    L_ = lib()
    game = b2.load_game("kuhn_poker")
    for flags in (8 | 1, 8 | 2, 8 | 3, 8 | 4):
        h = C.c_void_p()
        with pytest.raises(B2SError, match="BEST_RESPONSE_OPPONENTS"):
            check(L_.b2s_cfr_create(game._gid, C.byref(game._cparams), flags, game.device, C.byref(h)))
        assert not h.value
    with pytest.raises(B2SError):
        b2.CFRBRSolver(b2.load_game("kuhn_poker(players=3)"))
    plain = b2.CFRSolver(game)
    plain.evaluate_and_update_policy(5)
    dev = b2.CFRBRSolver(game)
    dev.evaluate_and_update_policy(5)
    before = dev.table()
    with pytest.raises(B2SError, match="sharded"):
        check(L_.b2s_cfr_traverse_shard(dev._h, 0, 6, 0, 1, None))
    with pytest.raises(B2SError, match="sharded"):
        check(L_.b2s_cfr_apply_deltas(dev._h, None))
    with pytest.raises(B2SError, match="sharded"):
        check(L_.b2s_cfr_iterate_sharded(dev._h, 2, None))
    with pytest.raises(B2SError):
        check(L_.b2s_mccfr_external_iterate(dev._h, 1, 1, 0, None))
    with pytest.raises(B2SError):
        check(L_.b2s_mccfr_outcome_iterate(dev._h, 1, 1, 0, 0.6, None))
    after = dev.table()
    for f in ("regrets", "cum_policy", "cur_policy"):
        assert np.array_equal(before[f], after[f]), f
    assert dev.info().iteration == 5
    ref = b2.CFRSolver(game)
    ref.evaluate_and_update_policy(5)
    plain.evaluate_and_update_policy(0)
    for f in ("regrets", "cum_policy", "cur_policy"):
        assert np.array_equal(plain.table()[f], ref.table()[f]), f
