"""GPU: the loops bench.py times besides the connect_four step, run at the sizes, seeds and call sequences it runs them
(bench.py run_gpu, "the loops that drive the step kernels"), rank 0 and, where the bench offsets by rank, rank 1.

The results are compared with the oracle (tests/oracle_lib.py) bit for bit on sampled trees, lanes and episodes: block
and warp edges plus random indices from a fixed seed.  The oracle work runs in a process pool while the device works.
Runs the oracle would need minutes for (100k-iteration CFR, 52 MCCFR iterations of 16,384 traversals) are compared with
tests/golden/long_run_reference.json (tests/golden/make_long_cfr_reference.py).  Only sampled rows leave the device, and
every section frees its buffers before the next one starts.  tests/test_bench_loop_config.py checks that bench.py still
makes the calls restated here."""
import json
import os
import subprocess
import sys
import tempfile
import threading

import numpy as np
import pytest
import torch

import bench_loops_oracle as bo
import golden_lib
import open_spiel_b200 as b2
from oracle_lib import OracleGame, infostate_tensors
from open_spiel_b200 import parallel
from test_gpu_mccfr import compare as compare_mccfr
from test_gpu_mcts_many_trees import assert_matches_oracle

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
LONG = os.path.join(HERE, "golden", "long_run_reference.json")

# bench.py's literals
MCTS_TREES, MCTS_SIMS, MCTS_WARMUP_SIMS, MCTS_SEED = 65536, 128, 8, 1
DEEP_TREES, DEEP_SIMS, DEEP_NODES_PER_TREE = 8192, 10000, 240000
ROLLOUT_GAMES, ROLLOUT_SEED, ROLLOUT_WARMUP = 1 << 20, 9, 1024
CFR_WARMUP, CFR_ITERS = 10, 100000
MCCFR_K, MCCFR_SEED, MCCFR_WARMUP, MCCFR_ITERS = 16384, 11, 2, 50
EPISODES = 1 << 18


def free():
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def sample(n, count=30, seed=0, extra=()):
    """Block and warp edges of an n-lane launch plus `count` random indices from a fixed seed."""
    edges = {0, 1, 31, 32, 127, 128, 255, 256, 511, 512, n // 2, n - 1} | set(extra)
    rng = np.random.RandomState(seed)
    return sorted(i for i in edges | set(rng.choice(n, size=count, replace=False).tolist()) if 0 <= i < n)


def rows(out, idx, keys=("visits", "total_reward", "outcome_p0", "best_action", "sims_run")):
    """Rows `idx` of a search result, on the host."""
    i = torch.as_tensor(idx, dtype=torch.int64, device=out["sims_run"].device)
    host = {k: out[k].index_select(0, i).cpu().numpy() for k in keys}
    return [{k: host[k][j] for k in keys} for j in range(len(idx))]


def check_search(out, sims):
    """Every tree: all simulations ran unless the root was proven, and every simulation after the first (which expands
    the root) descended into exactly one child."""
    proven = ~torch.isnan(out["outcome_p0"]).all(dim=1)
    ran = out["sims_run"]
    assert bool(((ran == sims) | proven).all())
    assert bool((out["visits"].sum(dim=1) == ran - 1).all())


# ---- 1. MCTS, wide: loops["mcts_go9x9"] ------------------------------------------------------------------------------
@pytest.mark.parametrize("rank", [0, 1])
def test_mcts_wide_line(rank):
    trees, offset = MCTS_TREES, rank * MCTS_TREES
    idx = sample(trees, seed=10 + rank)
    with bo.pool() as p:
        oracle = p.map_async(bo.mcts_tree, [("go(board_size=9)", MCTS_SIMS, MCTS_SEED, t + offset) for t in idx], chunksize=1)
        go = b2.Game("go", {"board_size": 9}, device=0)
        roots = go.new_batch(trees)
        b2.mcts_search(roots, MCTS_WARMUP_SIMS, seed=MCTS_SEED, tree_index_offset=offset, max_nodes_total=0)
        out = b2.mcts_search(roots, MCTS_SIMS, uct_c=2.0, n_rollouts=1, solve=True, seed=MCTS_SEED, tree_index_offset=offset,
                             max_nodes_total=0)
        assert roots.error_count()[0] == 0
        check_search(out, MCTS_SIMS)
        dev = rows(out, idx)
        del roots, out
        free()
        for t, d, o in zip(idx, dev, oracle.get()):
            assert_matches_oracle(d, o, "rank %d tree %d" % (rank, t))


# ---- 2. MCTS, deep: loops["mcts_go9x9_deep"] -------------------------------------------------------------------------
DEEP_SAMPLE = [0, 1, 127, 128, 4095, 8191] + np.random.RandomState(20).choice(np.arange(2, 8190), 6, replace=False).tolist()


def concurrent(calls):
    """Runs each call in its own thread on its own CUDA stream (ctypes releases the GIL for a library call, and a search
    synchronises only its own stream), so one-tree searches proceed side by side; returns the results in order."""
    res = [None] * len(calls)
    errors = []

    def run(k):
        try:
            with torch.cuda.stream(torch.cuda.Stream()):
                res[k] = calls[k]()
                torch.cuda.current_stream().synchronize()
        except BaseException as e:                      # noqa: B902 - re-raised in the caller
            errors.append(e)

    threads = [threading.Thread(target=run, args=(k,)) for k in range(len(calls))]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    if errors:
        raise errors[0]
    return res


def test_mcts_deep_line():
    """8,192 trees of 10,000 simulations in arenas of 240,000 nodes per tree.  Sampled trees equal the oracle; re-run alone,
    each allocates exactly the nodes MCTSBot creates (nodes_ = 1, += children.size(): the arena bump-allocates one block
    per expansion and never frees without garbage collection), fits an arena of exactly that many nodes, and with a few
    nodes fewer it stops and is reported by the batch's error record while its neighbours are untouched."""
    go = b2.Game("go", {"board_size": 9}, device=0)
    nodes_total = DEEP_TREES * DEEP_NODES_PER_TREE
    triples = sorted({t + d for t in DEEP_SAMPLE for d in (-1, 0, 1) if 0 <= t + d < DEEP_TREES})
    with bo.pool() as p:
        oracle = p.map_async(bo.mcts_tree, [("go(board_size=9)", DEEP_SIMS, MCTS_SEED, t) for t in triples], chunksize=1)
        roots = go.new_batch(DEEP_TREES)
        b2.mcts_search(roots, MCTS_WARMUP_SIMS, seed=MCTS_SEED, tree_index_offset=0, max_nodes_total=nodes_total)
        out = b2.mcts_search(roots, DEEP_SIMS, uct_c=2.0, n_rollouts=1, solve=True, seed=MCTS_SEED, tree_index_offset=0,
                             max_nodes_total=nodes_total)
        assert roots.error_count()[0] == 0                 # no tree ran out of its 240,000 nodes
        assert bool((out["sims_run"] == DEEP_SIMS).all())
        check_search(out, DEEP_SIMS)
        used = b2.mcts_nodes_used(roots)
        dev = dict(zip(triples, rows(out, triples)))
        del roots, out
        free()
        o = dict(zip(triples, oracle.get()))
    for t in DEEP_SAMPLE:
        assert_matches_oracle(dev[t], o[t], "deep tree %d" % t)
    nodes = {t: o[t]["nodes"] for t in triples}
    assert max(nodes.values()) <= DEEP_NODES_PER_TREE
    # the tree to exhaust: a sampled tree that needs more than 3 nodes above both neighbours
    t_ex = max((t for t in DEEP_SAMPLE if 0 < t < DEEP_TREES - 1 and nodes[t] - 3 >= max(nodes[t - 1], nodes[t + 1])),
               key=lambda t: nodes[t])
    cap = nodes[t_ex] - 3

    def alone(t, cap_nodes):
        def call():
            b = go.new_batch(1)
            r = b2.mcts_search(b, DEEP_SIMS, uct_c=2.0, n_rollouts=1, solve=True, seed=MCTS_SEED, tree_index_offset=t,
                               max_nodes_total=cap_nodes)
            return rows(r, [0])[0], b.error_count(), b2.mcts_nodes_used(b)
        return call

    def exhausted():
        b = go.new_batch(3)
        r = b2.mcts_search(b, DEEP_SIMS, uct_c=2.0, n_rollouts=1, solve=True, seed=MCTS_SEED, tree_index_offset=t_ex - 1,
                           max_nodes_total=3 * cap)
        return rows(r, [0, 1, 2]), b.error_count(), b2.mcts_nodes_used(b)

    runs = concurrent([alone(t, DEEP_NODES_PER_TREE) for t in DEEP_SAMPLE] + [alone(t, nodes[t]) for t in DEEP_SAMPLE] +
                      [exhausted])
    free()
    device_nodes = {}
    for k, t in enumerate(DEEP_SAMPLE):
        for run, what in ((runs[k], "240000-node arena"), (runs[len(DEEP_SAMPLE) + k], "arena of exactly its nodes")):
            res, err, used_one = run
            assert err[0] == 0, (t, what)
            assert used_one == nodes[t], (t, what, used_one, nodes[t])
            assert_matches_oracle(res, o[t], "deep tree %d alone, %s" % (t, what))
        device_nodes[t] = runs[k][2]
    res, err, _ = runs[-1]
    assert err == (1, 1), (t_ex, cap, err)
    assert res[1]["sims_run"] < DEEP_SIMS
    for lane, t in ((0, t_ex - 1), (2, t_ex + 1)):
        for key in ("visits", "total_reward", "outcome_p0", "best_action", "sims_run"):
            assert np.asarray(res[lane][key]).tobytes() == np.asarray(dev[t][key]).tobytes(), (t, t_ex, key)
    top = max(device_nodes.values())
    print("deep line: %d nodes used over %d trees (mean %.0f); sampled trees %s; largest %d, %d below the %d-node arena" % (
        used, DEEP_TREES, used / DEEP_TREES, sorted(device_nodes.values()), top, DEEP_NODES_PER_TREE - top, DEEP_NODES_PER_TREE))


# ---- 3. breakthrough rollouts: loops["rollouts_breakthrough"] -----------------------------------------------------------
ROLLOUT_EDGES = (2, 3, 63, 64, 257, 510, 513, 767, 768, 1022, 1023, 1024, 1025)   # ILP = 2 lane pairs, the warm-up's end


@pytest.mark.parametrize("rank", [0, 1])
def test_rollout_line(rank):
    games, offset = ROLLOUT_GAMES, rank * ROLLOUT_GAMES
    idx = sample(games, seed=30 + rank, extra=ROLLOUT_EDGES)
    with bo.pool() as p:
        oracle = p.map_async(bo.rollout_lane, [("breakthrough", ROLLOUT_SEED, offset + i) for i in idx], chunksize=1)
        bt = b2.Game("breakthrough", device=0)
        bb = bt.new_batch(games)
        bb.rollout(seed=ROLLOUT_SEED, lane_offset=offset, n=ROLLOUT_WARMUP)
        bb.reset()
        rets, plies = bb.rollout(seed=ROLLOUT_SEED, lane_offset=offset)
        assert bb.error_count()[0] == 0
        _, term, rets_status = bb.status()
        assert bool(term.all()) and torch.equal(rets_status, rets)
        del bb, term, rets_status
        fresh = bt.new_batch(games)
        rets_f, plies_f = fresh.rollout(seed=ROLLOUT_SEED, lane_offset=offset)
        del fresh
        # reset() restored every lane.  The warm-up played these very games on lanes < 1024, so a lane it missed would keep
        # its returns and give itself away by its 0 plies.
        assert torch.equal(plies, plies_f) and torch.equal(rets, rets_f)
        del rets_f, plies_f
        assert bool((rets.sum(dim=1) == 0).all())
        assert int(plies.min()) >= 1 and int(plies.max()) <= bt.max_game_length()
        st = parallel.rollout_stats(rets, plies).tolist()
        r0, pl = rets[:, 0].cpu().numpy(), plies.cpu().numpy().astype(np.int64)
        assert st == [int((r0 > 0).sum()), int((r0 < 0).sum()), int((r0 == 0).sum()), int(pl.sum()), games]
        i = torch.as_tensor(idx, device=rets.device)
        dev_rets, dev_plies = rets.index_select(0, i).cpu().numpy(), plies.index_select(0, i).cpu().numpy()
        del rets, plies, r0, pl
        free()
        for k, (ply, ret) in enumerate(oracle.get()):
            assert dev_plies[k] == ply and dev_rets[k].tolist() == ret, (rank, idx[k])


# ---- 4. leduc CFR / CFR+, 100k iterations: loops["cfr_leduc"] ----------------------------------------------------------
@pytest.mark.parametrize("plus", [False, True], ids=["cfr", "cfr_plus"])
def test_cfr_long_run(plus):
    gold = json.load(open(LONG))["cfr_plus" if plus else "cfr"]["checkpoints"]
    assert [g["iterations"] for g in gold] == [1000, 10000, CFR_WARMUP + CFR_ITERS]
    leduc = b2.Game("leduc_poker", device=0)
    tensors = infostate_tensors(OracleGame("leduc_poker"))

    def check(solver, g):
        assert golden_lib.table_digest(golden_lib.device_table_by_key(solver.table(), tensors)) == g["table_sha256"], \
            (plus, g["iterations"])
        assert abs(solver.nash_conv() - g["nash_conv"]) <= 1e-9, (plus, g["iterations"], solver.nash_conv(), g["nash_conv"])
        assert abs(solver.exploitability() - g["exploitability"]) <= 1e-9

    solver = b2.CFRSolver(leduc, linear_averaging=plus, regret_matching_plus=plus)
    done = 0
    for g in gold[:2]:
        solver.evaluate_and_update_policy(g["iterations"] - done)
        done = g["iterations"]
        check(solver, g)
    solver = b2.CFRSolver(leduc, linear_averaging=plus, regret_matching_plus=plus)    # bench.py's two calls
    solver.evaluate_and_update_policy(CFR_WARMUP)
    solver.evaluate_and_update_policy(CFR_ITERS)
    check(solver, gold[2])
    del solver
    free()


# ---- 5. external-sampling MCCFR, 16,384 traversals per update: loops["mccfr_external_leduc"] --------------------------
def mccfr_digest(dev_table, tensors):
    t = golden_lib.device_table_by_key(dev_table, tensors)
    return golden_lib.table_digest({k: {f: v[f] for f in ("legal", "regrets", "cum_policy")} for k, v in t.items()})


def test_mccfr_bench_line_live_oracle():
    """The bench's rank-0 solver, its warm-up call and one more iteration, bit for bit against the oracle."""
    og = OracleGame("leduc_poker")
    with bo.pool() as p:
        oracle = p.map_async(bo.mccfr_tables, [("es", "leduc_poker", MCCFR_K, MCCFR_SEED, [MCCFR_WARMUP, 1])])
        tensors = infostate_tensors(og)
        mc = b2.ExternalSamplingMCCFRSolver(b2.Game("leduc_poker", device=0), seed=MCCFR_SEED, traversals_per_update=MCCFR_K)
        mc.run_iteration(MCCFR_WARMUP)
        t2 = mc.table()
        mc.run_iteration(1)
        t3 = mc.table()
        del mc
        free()
        o2, o3 = oracle.get()[0]
    compare_mccfr(t2, o2, tensors)
    compare_mccfr(t3, o3, tensors)


@pytest.mark.parametrize("rank", [0, 1])
def test_mccfr_bench_line_golden(rank):
    """The bench's full sequence (2 + 50 iterations) against the generator's oracle digests, seeds 11 (rank 0) and 12."""
    seed = MCCFR_SEED + rank
    gold = json.load(open(LONG))["mccfr_external"][str(seed)]
    assert gold["traversals_per_update"] == MCCFR_K and [g["iterations"] for g in gold["checkpoints"]] == \
        [MCCFR_WARMUP, MCCFR_WARMUP + MCCFR_ITERS]
    tensors = infostate_tensors(OracleGame("leduc_poker"))
    mc = b2.ExternalSamplingMCCFRSolver(b2.Game("leduc_poker", device=0), seed=seed, traversals_per_update=MCCFR_K)
    mc.run_iteration(MCCFR_WARMUP)
    assert mccfr_digest(mc.table(), tensors) == gold["checkpoints"][0]["table_sha256"]
    mc.run_iteration(MCCFR_ITERS)
    assert mccfr_digest(mc.table(), tensors) == gold["checkpoints"][1]["table_sha256"]
    assert abs(mc.nash_conv() - gold["checkpoints"][1]["nash_conv"]) <= 1e-9
    del mc
    free()


# K that leave some of the 64 reduction lanes a traversal short, or empty (K < 64)
RAGGED_K = [2, 37, 63, 65, 100, 777, 16383]
RAGGED = [(kind, K) for K in RAGGED_K for kind in ("es", "es_full", "os")]


def ragged_steps(K):
    return [1] if K > 4096 else [1, 2]


_RAGGED_SCRIPT = r"""
import json
import sys
import numpy as np
sys.path.insert(0, sys.argv[1])
import open_spiel_b200 as b2
cases, out = json.loads(sys.argv[2]), {}
for kind, K, seed, steps in cases:
    game = b2.load_game("leduc_poker")
    if kind == "os":
        s = b2.OutcomeSamplingMCCFRSolver(game, seed=seed, trajectories_per_update=K)
    else:
        s = b2.ExternalSamplingMCCFRSolver(game, seed=seed, traversals_per_update=K, full_average=kind == "es_full")
    for j, n in enumerate(steps):
        s.run_iteration(n)
        t = s.table()
        for f in ("regrets", "cum_policy"):
            out["%s_%d_%d_%s" % (kind, K, j, f)] = t[f]
np.savez(sys.argv[3], **out)
"""


def test_mccfr_ragged_k_both_update_paths():
    """K not a multiple of 64: external sampling (simple and full averaging) and outcome sampling bit for bit against the
    oracle, on the scatter update path and on the lanes path (B2S_MCCFR_MODE; the lanes path is the default for tables
    beyond 8 GiB).  Each mode runs in its own process, as the library reads the switch once."""
    cases = [(kind, K, 0xC0DE + K, ragged_steps(K)) for kind, K in RAGGED]
    og = OracleGame("leduc_poker")
    with bo.pool() as p:
        oracle = p.map_async(bo.mccfr_tables, [(kind, "leduc_poker", K, seed, steps) for kind, K, seed, steps in cases],
                             chunksize=1)
        tensors = infostate_tensors(og)
        layout = b2.ExternalSamplingMCCFRSolver(b2.load_game("leduc_poker")).table()
        root = os.path.dirname(HERE)
        dev = {}
        with tempfile.TemporaryDirectory() as tmp:
            for mode in ("scatter", "lanes"):
                path = os.path.join(tmp, mode + ".npz")
                env = dict(os.environ, B2S_MCCFR_MODE=mode)
                r = subprocess.run([sys.executable, "-c", _RAGGED_SCRIPT, root, json.dumps(cases), path], capture_output=True,
                                   text=True, env=env, timeout=900)
                assert r.returncode == 0, r.stderr[-2000:]
                with np.load(path) as z:
                    dev[mode] = {k: z[k] for k in z.files}
        tables = oracle.get()
    for mode in ("scatter", "lanes"):
        for (kind, K, _, steps), o in zip(cases, tables):
            for j in range(len(steps)):
                t = dict(layout, regrets=dev[mode]["%s_%d_%d_regrets" % (kind, K, j)],
                         cum_policy=dev[mode]["%s_%d_%d_cum_policy" % (kind, K, j)])
                try:
                    compare_mccfr(t, o[j], tensors)
                except AssertionError as e:
                    raise AssertionError("%s path, %s K=%d after step %d: %s" % (mode, kind, K, j, str(e)[:300])) from None


# ---- 6. connect_four trajectory recorder: loops["trajectories_connect_four"] ----------------------------------------
@pytest.mark.parametrize("rank", [0, 1])
def test_trajectory_line(rank):
    eps, offset = EPISODES, rank * EPISODES
    idx = sample(eps, seed=60 + rank, extra=(1023, 1024))
    c4 = b2.Game("connect_four", device=0)
    T, A = c4.max_game_length(), c4.num_distinct_actions()
    with bo.pool() as p:
        oracle = p.map_async(bo.trajectory, [("connect_four", 2, offset + i, T) for i in idx], chunksize=1)
        tb = c4.new_batch(eps)
        tb.record_trajectories(seed=1, lane_offset=offset)
        tb.reset()
        tr = tb.record_trajectories(seed=2, lane_offset=offset)
        assert tb.error_count()[0] == 0
        assert bool(tb.status()[1].all())                           # the batch is left terminal
        assert int(tr.valid.sum()) == int(tr.lengths.sum())
        assert int(tr.lengths.min()) >= 7                          # no lane was left at the warm-up's terminal state
        i = torch.as_tensor(idx, device=tr.lengths.device)
        dev = {k: getattr(tr, k).index_select(0, i).cpu().numpy()
               for k in ("observations", "legal_mask", "actions", "player_ids", "valid", "next_is_terminal", "rewards", "lengths")}
        keep = {k: getattr(tr, k).clone() for k in ("actions", "lengths", "rewards")}
        del tb, tr
        free()
        fresh = c4.new_batch(eps)
        tf = fresh.record_trajectories(seed=2, lane_offset=offset)
        for k, v in keep.items():                                    # reset() restored every lane
            assert torch.equal(getattr(tf, k), v), k
        del fresh, tf, keep
        free()
        bits = (dev["legal_mask"][..., None] >> np.arange(32, dtype=dev["legal_mask"].dtype)) & 1
        legal = bits.reshape(*dev["legal_mask"].shape[:2], -1)[..., :A].astype(np.int32)
        for k, o in enumerate(oracle.get()):
            what = (rank, idx[k])
            assert dev["lengths"][k] == o["length"], what
            for f in ("actions", "player_ids", "valid", "next_is_terminal", "observations"):
                assert np.array_equal(dev[f][k], o[f]), (what, f)
            assert np.array_equal(legal[k], o["legal_actions"]), what
            assert np.array_equal(dev["rewards"][k].astype(np.float64), o["rewards"]), what
