"""CPU: the KERNEL BODY of the caller-evaluated search (k_mcts_eval_step / k_mcts_eval_report, open_spiel_b200/csrc/
mcts_eval.cuh), compiled for the host by tests/host_emul/eval.mk (emul_eval.cc), run round by round: after every step the test evaluator is computed
on the host from the leaves lanes (their observation and legal mask, read by the product's rule cores) and handed back.  The
root statistics must equal the oracle's MCTS with the same evaluator on the Philox stream (oracle/algorithms/mcts_eval.cc, pinned to
the unmodified reference by test_mcts_eval_oracle_vs_reference.py) for all nine games, UCT and PUCT, the root's Dirichlet noise
and the node budget's garbage collection."""
import ctypes as C
import math
import os

import numpy as np
import pytest

import open_spiel_b200 as b2
from open_spiel_b200._lib import GameInfo, MctsEvalConfig
from mcts_eval_lib import dirichlet_rows, hash_evaluator, oracle_mcts_eval, oracle_test_evaluator
from oracle_lib import OracleGame

SO = os.path.join(os.path.dirname(os.path.abspath(__file__)), "host_emul", "libemul_eval.so")
_LIB = None


def _lib():
    global _LIB
    if _LIB is None:
        if not os.path.exists(SO):
            pytest.skip("host emulation library not built (needs g++ and the CUDA headers)")
        L = C.CDLL(SO)
        L.emv_last_error.restype = C.c_char_p
        L.emv_create.restype = C.c_void_p
        L.emv_create.argtypes = [C.c_int, C.c_void_p, C.c_longlong]
        L.emv_destroy.argtypes = [C.c_void_p]
        L.emv_info.argtypes = [C.c_void_p, C.c_void_p]
        L.emv_apply.argtypes = [C.c_void_p, C.c_void_p, C.c_longlong]
        L.emv_error_count.restype = C.c_longlong
        L.emv_error_count.argtypes = [C.c_void_p]
        L.emv_mcts_eval_create.argtypes = [C.c_void_p, C.c_longlong, C.c_void_p]
        L.emv_mcts_eval_step.restype = C.c_longlong
        L.emv_mcts_eval_step.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        L.emv_mcts_eval_leaves.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        L.emv_mcts_eval_results.argtypes = [C.c_void_p] + [C.c_void_p] * 7
        _LIB = L
    return _LIB


class Emv:
    """A host batch of n roots at the initial state (tests/host_emul/emul_eval.cc)."""

    def __init__(self, game_string, n):
        self.L = _lib()
        g = b2.load_game(game_string)                       # parameter parsing only; no device is touched
        self.h = self.L.emv_create(g._gid, C.byref(g._cparams), n)
        assert self.h, self.L.emv_last_error()
        self.info = GameInfo()
        self.L.emv_info(self.h, C.byref(self.info))
        self.n = n

    def __del__(self):
        try:
            self.L.emv_destroy(self.h)
        except Exception:
            pass

    def apply(self, actions):
        a = np.ascontiguousarray(actions, dtype=np.int32)
        self.L.emv_apply(self.h, a.ctypes.data, self.n)

    def errors(self):
        return self.L.emv_error_count(self.h)


def run_emulated(gs, n, prefix, sims, solve, puct, budget=0, alpha=0.0, seed=0xBEEF, offset=5):
    """Roots = n random positions (the same actions on the emulated batch and on oracle states); returns (results, rounds,
    oracle states, noise)."""
    L = _lib()
    emu = Emv(gs, n)
    og = OracleGame(gs)
    states = [og.new_initial_state() for _ in range(n)]
    rng = np.random.RandomState(sum(map(ord, gs)) % 1000)
    ks = rng.randint(0, prefix + 1, size=n)
    for t in range(prefix):
        acts = np.full(n, -1, dtype=np.int32)
        for i, st in enumerate(states):
            if t < ks[i]:
                la = st.legal_actions()
                a = la[rng.randint(len(la))]
                nxt = st.clone()
                nxt.apply_action(a)
                if nxt.is_terminal():
                    continue
                states[i] = nxt
                acts[i] = a
        emu.apply(acts)
    assert emu.errors() == 0
    A, F, W = emu.info.num_distinct_actions, emu.info.observation_tensor_size, emu.info.mask_words
    noise = dirichlet_rows([st.legal_actions() for st in states], A, alpha, seed=7) if alpha > 0 else None
    cfg = MctsEvalConfig(sims, int(solve), int(puct), 0, 2.0, seed, offset, 0, budget, 0.25 if alpha > 0 else 0.0,
                         noise.ctypes.data if noise is not None else None)
    assert L.emv_mcts_eval_create(emu.h, n, C.byref(cfg)) == 0
    pending = np.zeros(n, dtype=np.uint8)
    obs = np.zeros((n, F), dtype=np.float32)
    words = np.zeros((n, W), dtype=np.uint32)
    values = priors = None
    rounds = 0
    while True:
        cnt = L.emv_mcts_eval_step(emu.h, values.ctypes.data if values is not None else None,
                                   priors.ctypes.data if priors is not None else None, pending.ctypes.data)
        assert cnt == int(pending.sum())
        if cnt == 0:
            break
        rounds += 1
        L.emv_mcts_eval_leaves(emu.h, obs.ctypes.data, words.ctypes.data)
        mask = ((words[:, :, None] >> np.arange(32, dtype=np.uint32)) & 1).reshape(n, -1)[:, :A]
        with np.errstate(all="ignore"):
            v, p = hash_evaluator(obs, mask)
        values, priors = np.ascontiguousarray(v.numpy()), np.ascontiguousarray(p.numpy())
    out = {k: np.zeros((n, A), dtype=d) for k, d in (("visits", np.int32), ("total_reward", np.float64), ("outcome_p0", np.float32))}
    for k in ("best_action", "sims_run", "gc_runs", "prior_requests"):
        out[k] = np.zeros(n, dtype=np.int32)
    L.emv_mcts_eval_results(emu.h, *[out[k].ctypes.data for k in ("visits", "total_reward", "outcome_p0", "best_action", "sims_run",
                                                                   "gc_runs", "prior_requests")])
    assert emu.errors() == 0
    return out, rounds, states, noise


def check_against_oracle(out, states, sims, solve, puct, budget, noise, alpha, seed=0xBEEF, offset=5, tag=""):
    collections = 0
    for i, st in enumerate(states):
        o = oracle_mcts_eval(st, 2.0, sims, solve, seed, tree_index=i + offset, puct=puct, max_nodes=budget or 1,
                             root_noise=noise[i] if noise is not None else None, dirichlet_epsilon=0.25 if alpha > 0 else 0.0)
        assert out["sims_run"][i] == o["sims_run"], (tag, i)
        assert out["gc_runs"][i] == o["gc_runs"], (tag, i)
        collections += o["gc_runs"]
        for a, v, r, oc in o["children"]:
            assert out["visits"][i, a] == v, (tag, i, a)
            assert out["total_reward"][i, a] == r, (tag, i, a, out["total_reward"][i, a], r)     # exact doubles
            assert (math.isnan(oc) and math.isnan(out["outcome_p0"][i, a])) or out["outcome_p0"][i, a] == oc, (tag, i, a)
        assert int(out["visits"][i].sum()) == sum(v for _, v, _, _ in o["children"]), (tag, i)
        assert out["best_action"][i] == o["best_action"], (tag, i)
    return collections


CASES = [
    # game, trees, prefix plies, sims, solve, PUCT, node budget, dirichlet alpha
    ("tic_tac_toe", 24, 3, 200, True, False, 0, 0.0),
    ("tic_tac_toe", 24, 2, 200, False, True, 0, 0.3),
    ("connect_four", 16, 8, 200, True, True, 0, 0.0),
    ("connect_four(rows=4,columns=5,x_in_row=3)", 16, 4, 300, True, False, 0, 1.0),
    ("breakthrough(rows=6,columns=6)", 8, 8, 100, True, True, 0, 0.0),
    ("hex(board_size=5)", 12, 6, 150, False, True, 0, 0.5),
    ("go(board_size=5)", 8, 8, 100, True, True, 0, 0.03),
    ("go(board_size=2)", 16, 6, 80, True, False, 0, 0.0),
    ("go(board_size=3)", 16, 10, 120, False, True, 0, 0.0),
    ("othello", 8, 30, 100, True, True, 0, 0.0),
    ("mnk(m=5,n=5,k=4)", 8, 6, 120, True, False, 0, 0.3),
    ("y(board_size=5)", 8, 4, 120, True, True, 0, 0.0),
    ("havannah(board_size=3)", 8, 4, 150, True, False, 0, 0.0),
    ("havannah(board_size=4,swap=True)", 8, 8, 100, False, True, 0, 0.3),
    # node budget: collections free children and cached priors; freed nodes ask again for their prior
    ("connect_four", 8, 4, 1500, False, True, 200, 0.0),
    ("tic_tac_toe", 8, 1, 1200, True, False, 100, 0.3),
    ("hex(board_size=4)", 6, 2, 1200, True, True, 250, 0.0),
    ("go(board_size=3)", 8, 4, 1000, True, False, 150, 0.0),
]


@pytest.mark.parametrize("gs,n,prefix,sims,solve,puct,budget,alpha", CASES,
                         ids=["%s-%d%s%s%s" % (c[0], c[3], "-puct" if c[5] else "", "-gc" if c[6] else "", "-noise" if c[7] else "")
                              for c in CASES])
def test_emulated_eval_kernel_equals_oracle(gs, n, prefix, sims, solve, puct, budget, alpha):
    out, rounds, states, noise = run_emulated(gs, n, prefix, sims, solve, puct, budget, alpha)
    collections = check_against_oracle(out, states, sims, solve, puct, budget, noise, alpha, tag=gs)
    # one request per tree and round: at most one Evaluate per simulation plus the prior-only re-expansions
    assert rounds <= int((out["sims_run"] + out["prior_requests"]).max())
    if budget:
        assert collections >= n and int(out["prior_requests"].sum()) > 0
    else:
        assert int(out["prior_requests"].sum()) == 0          # without collections every expansion finds its cached prior


@pytest.mark.parametrize("gs", ["tic_tac_toe", "connect_four", "go(board_size=5)", "othello", "havannah(board_size=4)", "mnk"])
def test_torch_test_evaluator_equals_oracle(gs):
    og = OracleGame(gs)
    rng = np.random.RandomState(3)
    st = og.new_initial_state()
    A = og.num_distinct_actions
    for _ in range(12):
        if st.is_terminal():
            break
        obs = st.observation_tensor(st.current_player())
        mask = np.zeros(A, dtype=np.int64)
        mask[st.legal_actions()] = 1
        v, p = hash_evaluator(obs[None, :], mask[None, :])
        ov, op = oracle_test_evaluator(st)
        assert v[0].tolist() == ov and p[0].tolist() == op
        la = st.legal_actions()
        st.apply_action(la[rng.randint(len(la))])
