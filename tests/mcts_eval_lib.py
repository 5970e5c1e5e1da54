"""The test evaluator of the caller-evaluated search (b2s_mcts_eval_*), in torch, plus shared helpers.  Test infrastructure.

The same evaluator is defined in oracle/algorithms/mcts_eval.cc (TestEvaluate / TestPrior) and as a reference Evaluator in
oracle/ref_glue/ref_mcts_eval.cc.  With x = ObservationTensor(CurrentPlayer()) and I its non-zero indices:
  h1 = sum_{i in I} (7i + 3) mod 11,  h2 = sum_{i in I} i mod 13
  Evaluate = {v, -v}, v = ((h1 mod 9) - 4) / 7.0
  Prior(a) = w_a / sum_b w_b over the legal actions, w_a = 1 + (h2 + 13a) mod 5
Integer sums and one correctly rounded float64 division each, so torch on the CPU or the GPU gives the oracle's doubles."""
import ctypes as C
import os

import numpy as np
import torch


def hash_evaluator(obs, mask):
    """obs [n, F] (the observation of the player to move), mask [n, A] legal 0/1 -> (values [n, 2], priors [n, A]) float64.
    Lanes without legal actions get NaN priors (the search never asks for them)."""
    obs, mask = torch.as_tensor(obs), torch.as_tensor(mask)
    nz = (obs != 0).to(torch.int64)
    idx = torch.arange(obs.shape[1], dtype=torch.int64, device=obs.device)
    h1 = (nz * ((7 * idx + 3) % 11)).sum(dim=1)
    h2 = (nz * (idx % 13)).sum(dim=1)
    v = ((h1 % 9) - 4).to(torch.float64) / 7.0
    values = torch.stack([v, -v], dim=1)
    a = torch.arange(mask.shape[1], dtype=torch.int64, device=obs.device)
    w = (1 + (h2[:, None] + 13 * a) % 5) * mask.to(torch.int64)
    priors = w.to(torch.float64) / w.sum(dim=1, keepdim=True).to(torch.float64)
    return values, priors


def evaluate_leaves(leaves, pending):
    """mcts_search_evaluated's `evaluate` for the test evaluator, from the leaves batch's own kernels."""
    return hash_evaluator(leaves.observation_tensor(), leaves.legal_actions_mask())


def dirichlet_rows(legal_lists, A, alpha, seed):
    """Per root a Dirichlet(alpha) vector over its legal actions, scattered by action id ([n, A] float64, numpy)."""
    rng = np.random.RandomState(seed)
    out = np.zeros((len(legal_lists), A), dtype=np.float64)
    for i, legal in enumerate(legal_lists):
        out[i, legal] = rng.dirichlet([alpha] * len(legal))
    return out


# ---- the oracle's MCTS with the test evaluator (oracle/algorithms/mcts_eval.cc, part of oracle/liboracle.so) ----------------
def oracle_mcts_eval(state, uct_c, max_simulations, solve=True, seed=0, tree_index=0, puct=False, reference_rng=False, max_nodes=1,
                     root_noise=None, dirichlet_alpha=0.0, dirichlet_epsilon=0.0):
    """One search from an oracle_lib.OracleState; dict(children=[(action, visits, total reward, outcome_p0)], best_action,
    root_visits, sims_run, gc_runs).  root_noise (Philox stream only): the root's Dirichlet noise by action id;
    dirichlet_alpha (reference streams only): drawn as the reference's dirichlet_noise."""
    import oracle_lib
    L = oracle_lib.lib()
    f = L.orc_mcts_eval_search
    f.restype = C.c_int
    f.argtypes = [C.c_void_p, C.c_void_p, C.c_double, C.c_int, C.c_int, C.c_uint64, C.c_uint64, C.c_int, C.c_int, C.c_int,
                  C.POINTER(C.c_double), C.c_double, C.c_double, C.POINTER(C.c_int64), C.POINTER(C.c_int), C.POINTER(C.c_double),
                  C.POINTER(C.c_double), C.c_int, C.POINTER(C.c_int64), C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_int)]
    cap = state.game.num_distinct_actions + 4
    acts, vis = (C.c_int64 * cap)(), (C.c_int * cap)()
    rew, outc = (C.c_double * cap)(), (C.c_double * cap)()
    best, rv, ran, gcs = C.c_int64(), C.c_int(), C.c_int(), C.c_int()
    noise = None
    if root_noise is not None:
        noise = (C.c_double * state.game.num_distinct_actions)(*[float(x) for x in root_noise])
    n = f(state.game._g, state._s, uct_c, max_simulations, int(solve), seed, tree_index, int(puct), int(reference_rng), int(max_nodes),
          noise, float(dirichlet_alpha), float(dirichlet_epsilon), acts, vis, rew, outc, cap, C.byref(best), C.byref(rv), C.byref(ran),
          C.byref(gcs))
    return {"children": [(acts[i], vis[i], rew[i], outc[i]) for i in range(n)], "best_action": best.value,
            "root_visits": rv.value, "sims_run": ran.value, "gc_runs": gcs.value}


def oracle_test_evaluator(state):
    """The oracle's test evaluator on one state: (values [num_players], priors [A] by action id)."""
    import oracle_lib
    L = oracle_lib.lib()
    L.orc_mcts_eval_test_evaluator.argtypes = [C.c_void_p, C.c_void_p, C.POINTER(C.c_double), C.POINTER(C.c_double)]
    v = (C.c_double * state.game.num_players)()
    p = (C.c_double * state.game.num_distinct_actions)()
    L.orc_mcts_eval_test_evaluator(state.game._g, state._s, v, p)
    return list(v), list(p)


# ---- the unmodified reference's MCTSBot with the test evaluator (oracle/_ref/libspiel_ref_mcts_eval.so, oracle/ref_eval.mk) ---
_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_EVAL_SO = os.path.join(_ROOT, "oracle", "_ref", "libspiel_ref_mcts_eval.so")
_REF_EVAL = None


def ref_eval_available():
    return os.path.exists(REF_EVAL_SO)


def _ref_eval_lib():
    global _REF_EVAL
    if _REF_EVAL is None:
        L = C.CDLL(REF_EVAL_SO)
        L.refe_last_error.restype = C.c_char_p
        L.refe_mcts_eval_search.argtypes = [C.c_char_p, C.POINTER(C.c_int64), C.c_int, C.c_double, C.c_int, C.c_int, C.c_int, C.c_int,
                                            C.c_double, C.c_double, C.c_int, C.POINTER(C.c_int64), C.POINTER(C.c_int),
                                            C.POINTER(C.c_double), C.c_int, C.POINTER(C.c_int64), C.POINTER(C.c_int)]
        _REF_EVAL = L
    return _REF_EVAL


def ref_sizeof_search_node():
    return _ref_eval_lib().refe_sizeof_search_node()


def ref_mcts_eval(game_string, history, num_distinct_actions, uct_c, max_simulations, solve=True, seed=0, puct=False,
                  dirichlet_alpha=0.0, dirichlet_epsilon=0.0, max_memory_mb=1000):
    """The unmodified reference's MCTSBot::MCTSearch with the test evaluator, from the position after `history`."""
    L = _ref_eval_lib()
    cap = num_distinct_actions + 4
    acts, vis, rew = (C.c_int64 * cap)(), (C.c_int * cap)(), (C.c_double * cap)()
    best, rv = C.c_int64(), C.c_int()
    hist = (C.c_int64 * max(1, len(history)))(*history)
    n = L.refe_mcts_eval_search(game_string.encode(), hist, len(history), uct_c, max_simulations, int(solve), seed, int(puct),
                                float(dirichlet_alpha), float(dirichlet_epsilon), int(max_memory_mb), acts, vis, rew, cap,
                                C.byref(best), C.byref(rv))
    assert n >= 0, L.refe_last_error()
    return {"children": [(acts[i], vis[i], rew[i]) for i in range(n)], "best_action": best.value, "root_visits": rv.value}
