"""Device NashConv and best response (k_cfr_nashconv) against the exact-arithmetic evaluator of tests/exact_policy_eval.py,
on policies CFR never produces as well as on the solvers' own tables, for kuhn_poker, leduc_poker and
leduc_poker(starting_player=1).  Plus CFR / CFR+ / MCCFR training on leduc_poker(starting_player=1) bit for bit against
the oracle, and training that is interleaved with evaluations, which share the solver's scratch arrays.

Error bound.  Every device value is built by at most D levels of convex combinations (D <= 12 for leduc) of at most A + 1
products (A = 3 actions) of doubles, over utilities |u| <= U = 13.  Each level adds a relative error of at most
(A + 1) * 2^-53 (the sums are contracted into FMAs, which only removes roundings), so every value is within
D * (A + 1) * 2^-53 * U ~ 7e-14 of the exact one, and NashConv, which combines four values, within ~3e-13.  The tolerance
TOL = 1e-12 leaves more than 3x headroom.  The average policy adds one rounding per entry (cum / sum, with sum rounded),
which is inside the same per-level budget.  Best-response actions: the device's q(I, a) = sum_h cf_reach(h) * V(child)
is exact up to TOL * (1 + U * sum_h cf_reach(h)), so the chosen action's exact q must be within that of the maximum, must
be THE maximiser where that is unique by more than it, and must be index 0 (the reference's first-maximum rule) where
every history of I has cf reach exactly 0 in double."""
from fractions import Fraction

import numpy as np
import pytest

import exact_policy_eval as E
import open_spiel_b200 as b2
from oracle_lib import OracleCFR, OracleGame, OracleMCCFR, OracleOSMCCFR, infostate_tensors
from test_gpu_cfr import compare as compare_cfr
from test_gpu_mccfr import compare as compare_mccfr

pytestmark = pytest.mark.gpu

TOL = 1e-12
SP1 = "leduc_poker(starting_player=1)"
GAMES = ["kuhn_poker", "leduc_poker", SP1]
WORST = {}      # largest |device - exact| NashConv seen, per game


@pytest.fixture(scope="module", autouse=True)
def report_worst():
    yield
    for gs, w in sorted(WORST.items()):
        print("\nlargest |device - exact| NashConv, %s: %.3g" % (gs, w))


_SOLVERS = {}


def probe_solver(gs):
    """One CFRSolver per game whose tables the tests overwrite with load_table."""
    if gs not in _SOLVERS:
        _SOLVERS[gs] = b2.CFRSolver(b2.load_game(gs))
    return _SOLVERS[gs]


def check_against_exact(gs, s, average):
    """Device nash_conv / last_values / best_response of solver `s` vs the exact evaluation of its own table."""
    t = s.table()
    ex = E.evaluate(gs, t, t["cum_policy"] if average else t["cur_policy"], average)
    nc = s.nash_conv(average=average)
    vals = list(s.last_values)
    actions, br_vals = s.best_response(average=average)
    assert br_vals == vals
    err = abs(Fraction(nc) - ex["nash_conv"])
    WORST[gs] = max(WORST.get(gs, 0.0), float(err))
    assert err <= TOL, (gs, average, nc, float(ex["nash_conv"]))
    for i in range(4):
        assert abs(Fraction(vals[i]) - ex["values"][i]) <= TOL, (gs, average, i, vals[i], float(ex["values"][i]))
    U = E.tree(gs).max_abs_utility
    off, legal = t["offsets"], t["legal_actions"]
    for k, qs in ex["q"].items():
        chosen = legal[off[k]:off[k + 1]].tolist().index(actions[k])
        tol_q = TOL * (1 + U * ex["cf_reach_sum"][k])
        ranked = sorted(qs, reverse=True)
        assert qs[chosen] >= ranked[0] - tol_q, (gs, average, k, chosen, qs)
        if ranked[0] - ranked[1] > tol_q:
            assert chosen == ex["best"][k], (gs, average, k, chosen, qs)
        if ex["cf_reach_zero"][k]:
            assert chosen == 0, (gs, average, k, chosen)
    return ex


FAMILIES = {"uniform": lambda t: E.uniform(t),
            **{"dirichlet-%d" % s: (lambda t, s=s: E.dirichlet(t, s)) for s in (0, 1, 2)},
            **{"sparse-%d" % s: (lambda t, s=s: E.sparse(t, s)) for s in (10, 11, 12)},
            **{"pure-%d" % s: (lambda t, s=s: E.pure(t, s)) for s in (20, 21)},
            **{"tiny-%d" % s: (lambda t, s=s: E.tiny(t, s)) for s in (30, 31)}}


@pytest.mark.parametrize("family", sorted(FAMILIES))
@pytest.mark.parametrize("gs", GAMES)
def test_policy_tables_match_exact(gs, family):
    """Each policy as the current policy (average=False) and as a cumulative policy (average=True)."""
    s = probe_solver(gs)
    pol = FAMILIES[family](s.table())
    s.load_table(cur_policy=pol)
    ex = check_against_exact(gs, s, average=False)
    # the first-maximum rule at zero-reach information states is exercised (kuhn's few sparse rows rarely cut off every
    # history of an information state)
    if family.startswith("pure") or (family.startswith("sparse") and gs != "kuhn_poker"):
        assert any(ex["cf_reach_zero"].values())
    s.load_table(cum_policy=pol)
    check_against_exact(gs, s, average=True)


@pytest.mark.parametrize("seed", [40, 41, 42])
@pytest.mark.parametrize("gs", GAMES)
def test_cumulative_tables_match_exact(gs, seed):
    """All-zero rows (the uniform fallback), rows mixing zeros and nonzeros, rows scaled by 1e-30 and 1e+30."""
    s = probe_solver(gs)
    cum = E.cum_mixed(s.table(), seed)
    s.load_table(cum_policy=cum)
    check_against_exact(gs, s, average=True)
    # the fallback matters: the same table with the all-zero rows made uniform is the same policy, bit for bit
    t = s.table()
    nc = s.nash_conv(average=True)
    for k in range(len(t["players"])):
        lo, hi = t["offsets"][k], t["offsets"][k + 1]
        if not cum[lo:hi].any():
            cum[lo:hi] = 0.5
    s.load_table(cum_policy=cum)
    assert s.nash_conv(average=True) == nc


@pytest.mark.parametrize("alpha", [0.0, 1.0 / 6.0, 1.0 / 3.0])
def test_kuhn_equilibria_as_doubles(alpha):
    gs = "kuhn_poker"
    s = probe_solver(gs)
    pol = np.array(E.kuhn_equilibrium(gs, s.table(), alpha))
    for average in (False, True):
        if average:
            s.load_table(cum_policy=pol)
        else:
            s.load_table(cur_policy=pol)
        check_against_exact(gs, s, average)
        assert abs(s.nash_conv(average=average)) <= TOL
        assert abs(s.last_values[2] + 1.0 / 18.0) <= TOL


@pytest.mark.parametrize("gs", GAMES)
@pytest.mark.parametrize("plus", [False, True])
def test_cfr_tables_match_exact(gs, plus):
    s = b2.CFRSolver(b2.load_game(gs), linear_averaging=plus, regret_matching_plus=plus)
    done = 0
    for it in (1, 3, 12):
        s.evaluate_and_update_policy(it - done)
        done = it
        check_against_exact(gs, s, average=True)
        check_against_exact(gs, s, average=False)


MCCFR_CASES = [("es", 1, 40), ("es", 64, 4), ("es-full", 1, 40), ("es-full", 64, 4), ("os", 1, 200), ("os", 256, 4)]


def mccfr_solver(gs, kind, K, seed):
    game = b2.load_game(gs)
    if kind == "os":
        return b2.OutcomeSamplingMCCFRSolver(game, seed=seed, trajectories_per_update=K)
    return b2.ExternalSamplingMCCFRSolver(game, seed=seed, traversals_per_update=K, full_average=kind == "es-full")


@pytest.mark.parametrize("kind,K,iters", MCCFR_CASES)
@pytest.mark.parametrize("gs", GAMES)
def test_mccfr_tables_match_exact(gs, kind, K, iters):
    s = mccfr_solver(gs, kind, K, seed=9)
    s.run_iteration(iters)
    check_against_exact(gs, s, average=True)


def test_sampling_solvers_have_no_current_policy():
    """The reference's sampling solvers keep no current policy, and simple averaging never writes the current-policy
    table: every current-policy call must raise instead of evaluating the initial uniform table."""
    for kind in ("es", "es-full", "os"):
        s = mccfr_solver("kuhn_poker", kind, 1, seed=3)
        s.run_iteration(5)
        for call in (lambda: s.nash_conv(average=False), lambda: s.best_response(average=False),
                     lambda: s.exploitability(average=False), s.current_policy, s.tabular_current_policy):
            with pytest.raises(b2.SpielError, match="no current policy"):
                call()
        nc = s.nash_conv()
        assert nc == s.nash_conv(average=True) and 0.0 < nc < 2.0
        assert len(s.best_response()[0]) == 12 and len(s.average_policy()) == 12


# ---- leduc_poker(starting_player=1) training ------------------------------------------------------------------------
def test_starting_player_1_tree_matches_default_leduc():
    a, b = b2.CFRSolver(b2.load_game(SP1)).info(), b2.CFRSolver(b2.load_game("leduc_poker")).info()
    counts = lambda i: (i.chance_nodes, i.decision_nodes, i.terminal_nodes, i.num_infosets, i.num_entries, i.num_nodes)   # noqa: E731
    assert counts(a) == counts(b)
    assert counts(a)[:4] == (157, 3780, 5520, 936)


@pytest.mark.parametrize("plus", [False, True])
def test_starting_player_1_cfr_equals_oracle_bitwise(plus):
    og = OracleGame(SP1)
    dev = b2.CFRSolver(b2.load_game(SP1), linear_averaging=plus, regret_matching_plus=plus)
    cpu = OracleCFR(og, linear_averaging=plus, regret_matching_plus=plus)
    tensors = infostate_tensors(og)
    for k in (1, 1, 3, 6):
        dev.evaluate_and_update_policy(k)
        cpu.iterate(k)
        compare_cfr(dev.table(), cpu.table(), tensors)


@pytest.mark.parametrize("kind,K,steps", [("es", 1, [1, 10, 60]), ("es", 256, [1, 2, 5]), ("es-full", 1, [1, 10, 30]),
                                          ("os", 1, [1, 10, 200]), ("os", 256, [1, 2, 5])])
def test_starting_player_1_mccfr_equals_oracle_bitwise(kind, K, steps):
    og = OracleGame(SP1)
    seed = 0x5EED + K
    dev = mccfr_solver(SP1, kind, K, seed)
    if kind == "os":
        cpu = OracleOSMCCFR(og, seed=seed, rng_mode=1, trajectories_per_update=K, epsilon=0.6)
    else:
        cpu = OracleMCCFR(og, seed=seed, rng_mode=1, traversals_per_update=K, full_average=kind == "es-full")
    tensors = infostate_tensors(og)
    for n in steps:
        dev.run_iteration(n)
        cpu.iterate(n)
        compare_mccfr(dev.table(), cpu.table(), tensors)


# ---- evaluation interleaved with training ---------------------------------------------------------------------------
def evaluate_everything(s, current=True):
    s.nash_conv(average=True)
    s.best_response(average=True)
    if current:
        s.nash_conv(average=False)
        s.best_response(average=False)


def same_tables(a, b, fields=("regrets", "cum_policy", "cur_policy")):
    ta, tb = a.table(), b.table()
    for f in fields:
        assert np.array_equal(ta[f], tb[f]), f


@pytest.mark.parametrize("gs", ["leduc_poker", SP1])
def test_evaluation_between_cfr_plus_iterations_changes_nothing(gs):
    """nash_conv / best_response reuse the solver's reach, value and edge-probability arrays; training resumed after
    them must equal an uninterrupted run bit for bit (the evaluate-then-iterate loop of cfr_example.cc:37-46)."""
    game = b2.load_game(gs)
    a = b2.CFRSolver(game, linear_averaging=True, regret_matching_plus=True)
    b = b2.CFRSolver(game, linear_averaging=True, regret_matching_plus=True)
    for _ in range(8):
        a.evaluate_and_update_policy(1)
        evaluate_everything(a)
    b.evaluate_and_update_policy(8)
    same_tables(a, b)


@pytest.mark.parametrize("K", [1, 64])
def test_evaluation_between_full_average_mccfr_iterations_changes_nothing(K):
    """External sampling with full averaging shares the level passes (cfr_level_passes) with full-width CFR."""
    a, b = (mccfr_solver("leduc_poker", "es-full", K, seed=17) for _ in range(2))
    for _ in range(10):
        a.run_iteration(1)
        evaluate_everything(a, current=False)
    b.run_iteration(10)
    same_tables(a, b)


def test_evaluation_inside_the_sharded_traversal_path_changes_nothing():
    """The multi-GPU code path driven by hand with 3 shards, as in test_gpu_cfr.py, with evaluations between every
    traversal, all-reduce and apply step: the tables must equal the single-GPU kernel's bit for bit."""
    import torch
    from open_spiel_b200 import parallel
    from open_spiel_b200._lib import check, lib
    iters, shards = 12, 3
    for plus in (False, True):
        game = b2.load_game("leduc_poker")
        ref = b2.CFRSolver(game, linear_averaging=plus, regret_matching_plus=plus)
        ref.evaluate_and_update_policy(iters)
        multi = parallel.DistributedCFRSolver(game, linear_averaging=plus, regret_matching_plus=plus, in_library=False)
        s, L = multi.solver, lib()
        for it in range(1, iters + 1):
            for player in (0, 1):
                acc = torch.zeros_like(multi.delta)
                for shard in range(shards):
                    check(L.b2s_cfr_traverse_shard(s._h, player, it, shard, shards, None))
                    torch.cuda.synchronize()
                    acc += multi.delta
                    evaluate_everything(s)
                multi.delta.copy_(acc)
                evaluate_everything(s)
                check(L.b2s_cfr_apply_deltas(s._h, None))
            evaluate_everything(s)
        same_tables(s, ref)
