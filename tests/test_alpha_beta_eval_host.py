"""CPU: the KERNEL BODY of AlphaBetaSearch with a value function (k_alpha_beta_eval_step, open_spiel_b200/csrc/alpha_beta.cuh),
compiled for the host by tests/host_emul/ab_eval.mk (emul_ab_eval.cc), run round by round: after every step the test value
function is computed on the host from the leaves lanes (their observation tensor, read by the product's rule cores) and handed
back.  Every variant's roots must give the restatement's results (tests/alpha_beta_eval_lib.py's alpha_beta_eval, pinned to the
reference's minimax.py by test_alpha_beta_eval_reference.py), and the k-th leaf each root hands out must be the restatement's
k-th evaluated state, with the same observation and legal actions."""
import ctypes as C
import os

import numpy as np
import pytest

import alpha_beta_eval_lib as abe
import alpha_beta_lib as ab
import open_spiel_b200 as b2
from open_spiel_b200._lib import GameInfo
from oracle_lib import OracleGame

SO = os.path.join(os.path.dirname(os.path.abspath(__file__)), "host_emul", "libemul_ab_eval.so")
_LIB = None


def _lib():
    global _LIB
    if _LIB is None:
        if not os.path.exists(SO):
            pytest.skip("host emulation library not built (needs g++ and the CUDA headers)")
        L = C.CDLL(SO)
        L.eab_last_error.restype = C.c_char_p
        L.eab_create.restype = C.c_void_p
        L.eab_create.argtypes = [C.c_int, C.c_void_p, C.c_longlong]
        L.eab_destroy.argtypes = [C.c_void_p]
        L.eab_info.argtypes = [C.c_void_p, C.c_void_p]
        L.eab_apply.argtypes = [C.c_void_p, C.c_void_p, C.c_longlong]
        L.eab_error_count.restype = C.c_longlong
        L.eab_error_count.argtypes = [C.c_void_p]
        L.eab_search_create.argtypes = [C.c_void_p, C.c_longlong, C.c_int, C.c_int, C.c_longlong]
        L.eab_step.restype = C.c_longlong
        L.eab_step.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        L.eab_leaves.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        L.eab_results.argtypes = [C.c_void_p] + [C.c_void_p] * 5
        _LIB = L
    return _LIB


class Eab:
    """A host batch of n roots at the initial state (tests/host_emul/emul_ab_eval.cc)."""

    def __init__(self, game_string, n):
        self.L = _lib()
        g = b2.load_game(game_string)                       # parameter parsing only; no device is touched
        self.h = self.L.eab_create(g._gid, C.byref(g._cparams), n)
        assert self.h, self.L.eab_last_error()
        self.info = GameInfo()
        self.L.eab_info(self.h, C.byref(self.info))
        self.n = n

    def __del__(self):
        try:
            self.L.eab_destroy(self.h)
        except Exception:
            pass


def run_emulated(gs, roots, depth, maxp, kind, max_nodes=0):
    """Roots = the initial state after each history of `roots`; returns (results, rounds, leaves) where leaves[i] is the list
    of (observation, legal mask) root i handed out, in order."""
    n = len(roots)
    emu = Eab(gs, n)
    L = emu.L
    for t in range(max([len(h) for h in roots] + [0])):
        a = np.array([h[t] if t < len(h) else -1 for h in roots], dtype=np.int32)
        L.eab_apply(emu.h, a.ctypes.data, n)
    assert L.eab_error_count(emu.h) == 0
    assert L.eab_search_create(emu.h, n, depth, maxp, max_nodes) == 0
    A, F, W = emu.info.num_distinct_actions, emu.info.observation_tensor_size, emu.info.mask_words
    pending = np.zeros(n, dtype=np.uint8)
    obs = np.zeros((n, F), dtype=np.float32)
    words = np.zeros((n, W), dtype=np.uint32)
    values = None
    rounds = 0
    leaves = [[] for _ in range(n)]
    while True:
        cnt = L.eab_step(emu.h, values.ctypes.data if values is not None else None, pending.ctypes.data)
        assert cnt == int(pending.sum())
        if cnt == 0:
            break
        rounds += 1
        L.eab_leaves(emu.h, obs.ctypes.data, words.ctypes.data)
        mask = ((words[:, :, None] >> np.arange(32, dtype=np.uint32)) & 1).reshape(n, -1)[:, :A]
        values = np.zeros((n, 2), dtype=np.float64)
        for i in np.nonzero(pending)[0]:
            values[i] = abe.obs_values(obs[i], kind)
            leaves[i].append((obs[i].copy(), np.nonzero(mask[i])[0].tolist()))
    out = {"value": np.zeros(n, dtype=np.float64), "best_action": np.zeros(n, dtype=np.int32), "nodes": np.zeros(n, dtype=np.int64),
           "status": np.zeros(n, dtype=np.uint8), "evaluations": np.zeros(n, dtype=np.int64)}
    L.eab_results(emu.h, *[out[k].ctypes.data for k in ("value", "best_action", "nodes", "status", "evaluations")])
    got = [dict(value=float(out["value"][i]), best_action=int(out["best_action"][i]), nodes=int(out["nodes"][i]),
                status=int(out["status"][i]), evaluations=int(out["evaluations"][i])) for i in range(n)]
    errors = L.eab_error_count(emu.h)
    assert errors == sum(g["status"] == ab.TERMINAL_ROOT for g in got)
    return got, rounds, leaves


def check(gs, roots, depth, maxp, kind, max_nodes=0):
    og = OracleGame(gs)
    got, rounds, leaves = run_emulated(gs, roots, depth, maxp, kind, max_nodes)
    for i, hist in enumerate(roots):
        root = ab.replay(og, hist)
        m = maxp if maxp >= 0 else (root.current_player() if not root.is_terminal() else 0)
        want = abe.alpha_beta_eval(root, depth, maxp, max_nodes, lambda s: abe.state_values(s, kind)[m])
        assert abe.same_bits(got[i], want), (gs, hist, depth, maxp, kind, got[i], want)
        assert len(leaves[i]) == want["evaluations"]
        for (o, legal), s in zip(leaves[i], want["evaluated"]):
            assert np.array_equal(o, s.observation_tensor(s.current_player())), (gs, hist, s.history())
            assert legal == s.legal_actions(), (gs, hist, s.history())
    assert rounds == max([g["evaluations"] for g in got] + [0])      # one leaf per root and round
    return got


@pytest.mark.parametrize("gs,plies,count", ab.VARIANTS, ids=[v[0] for v in ab.VARIANTS])
def test_emulated_equals_restatement(gs, plies, count):
    roots = ab.random_roots(OracleGame(gs), min(count, 8), (plies[0] // 2, plies[1]), seed=29)
    evaluated = 0
    for depth in range(5):
        for maxp, kind in ((-1, "hash"), (0, "edge"), (1, "hash"), (-1, "edge")):
            got = check(gs, roots, depth, maxp, kind)
            evaluated += sum(g["evaluations"] for g in got)
    assert evaluated > 0


def test_emulated_go_13x13_depth_one():
    """go 13x13 (the wide rule core) from a mid-game position: every legal move is one evaluated leaf whose legal actions
    depend on the superko history the leaves lane carries."""
    gs = "go(board_size=13)"
    roots = ab.random_roots(OracleGame(gs), 2, 60, seed=3)
    for kind, maxp in (("hash", -1), ("edge", 1)):
        got = check(gs, roots, 1, maxp, kind)
        if kind == "hash":                     # finite values never cut at the root: every child is a leaf
            assert all(g["evaluations"] == g["nodes"] > 100 for g in got)


@pytest.mark.parametrize("gs,plies,depth", [("connect_four", (8, 12), 4), ("hex(board_size=4)", (2, 6), 3),
                                            ("go(board_size=3)", (2, 6), 4)])
def test_emulated_budget_edge(gs, plies, depth):
    """max_nodes equal to a root's count solves it with identical results; one less stops it with status 1 after as many
    evaluations as the restatement made before its budget ran out."""
    og = OracleGame(gs)
    roots = [h for h in ab.random_roots(og, 6, plies, seed=8) if not ab.replay(og, h).is_terminal()]
    for i, hist in enumerate(roots):
        m = ab.replay(og, hist).current_player()
        nodes = abe.alpha_beta_eval(ab.replay(og, hist), depth, -1, 0, lambda s: abe.state_values(s, "hash")[m])["nodes"]
        got = check(gs, [hist], depth, -1, "hash", max_nodes=nodes)
        assert got[0]["status"] == ab.SOLVED and got[0]["nodes"] == nodes
        got = check(gs, [hist], depth, -1, "hash", max_nodes=nodes - 1)
        assert got[0]["status"] == ab.BUDGET and got[0]["nodes"] == nodes - 1


def test_emulated_stack_limit():
    """The per-root frame stack: go 19x19 unlimited exceeds B2S_ALPHA_BETA_THREAD_STACK_BYTES, depth 2 fits."""
    emu = Eab("go", 1)
    assert emu.L.eab_search_create(emu.h, 1, -1, -1, 0) == 2
    assert emu.L.eab_search_create(emu.h, 1, 2, -1, 0) == 0
