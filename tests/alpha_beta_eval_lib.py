"""Restatement of AlphaBetaSearch with a value function (reference open_spiel/algorithms/minimax.cc:49-137, 221-258; device:
b2s_alpha_beta_eval_*), its test value functions and the cases the reference comparison and its golden fixture run.  Test
infrastructure.  The search without a value function is tests/alpha_beta_lib.py's; this module reuses its status codes, roots
and variants.

Both value functions read ObservationTensor(CurrentPlayer()) of the evaluated state; with I its non-zero indices and
h1 = sum_{i in I} (7i + 3) mod 11 (mcts_eval_lib.hash_evaluator's hash), k = h1 mod 9:
  hash  {v, -v}, v = (k - 4) / 7.0: nine values, so ties and cuts at equality are common;
  edge  the same except k = 0 -> {-inf, +inf}, k = 1 -> {NaN, NaN}, k = 4 -> {-0.0, +0.0}, k = 8 -> {+inf, -inf} (the NaN is
        Python's and torch's quiet NaN 0x7ff8000000000000 in both columns: no arithmetic touches it).
Integer sums and one correctly rounded float64 division, so numpy on one state and torch on a batch give the same doubles."""
import hashlib
import math
import struct

import numpy as np

import alpha_beta_lib as ab

KINDS = ("hash", "edge")


def _h1(nz_idx):
    return int(((7 * nz_idx + 3) % 11).sum())


EDGE = {0: (-math.inf, math.inf), 1: (math.nan, math.nan), 4: (-0.0, 0.0), 8: (math.inf, -math.inf)}


def obs_values(obs, kind):
    """[num_players] values of one state from its observation tensor (numpy / list)."""
    k = _h1(np.nonzero(np.asarray(obs))[0].astype(np.int64)) % 9
    v = (k - 4) / 7.0
    if kind == "edge" and k in EDGE:
        return list(EDGE[k])
    return [v, -v]


def state_values(state, kind):
    """[num_players] values of an oracle or reference state."""
    return obs_values(state.observation_tensor(state.current_player()), kind)


def batch_values(obs, kind):
    """obs [n, F] torch (the observation of the player to move) -> values [n, 2] float64 on obs's device."""
    import torch
    nz = (obs != 0).to(torch.int64)
    idx = torch.arange(obs.shape[1], dtype=torch.int64, device=obs.device)
    k = (nz * ((7 * idx + 3) % 11)).sum(dim=1) % 9
    v = (k - 4).to(torch.float64) / 7.0
    out = torch.stack([v, -v], dim=1)
    if kind == "edge":
        for kk, pair in EDGE.items():
            out = torch.where((k == kk)[:, None], torch.tensor(pair, dtype=torch.float64, device=obs.device), out)
    return out


def leaves_value_function(kind):
    """alpha_beta_search_evaluated's value_function from the leaves batch's own observation kernel."""
    return lambda leaves, pending: batch_values(leaves.observation_tensor(), kind)


def bits(x):
    """The float64's 8 bytes as hex: the bitwise identity of a value, NaN sign and -0.0 included."""
    return struct.pack("<d", float(x)).hex()


def digest(histories):
    """One hash of a sequence of evaluated states, each given as its action history."""
    return hashlib.sha256(";".join(",".join(map(str, h)) for h in histories).encode()).hexdigest()[:16]


def alpha_beta_eval(root, depth_limit, maximizing_player, max_nodes, value_function):
    """dict(value, best_action, nodes, status, evaluations, evaluated) exactly as lane i of b2s_alpha_beta_eval_* reports them
    (evaluated: the states value_function was called with, in order).  value_function(state) is the maximizing player's value
    of a non-terminal state at depth 0 (minimax.cc:67-69); terminal states are scored first (:60-62).  Statuses and the per-root
    budget are alpha_beta_lib.alpha_beta's; status 2 cannot occur."""
    nodes = [0]
    evaluated = []

    def search(state, depth, alpha, beta, maxp, at_root):          # minimax.cc:49-137
        if state.is_terminal():
            return state.returns()[maxp], -1
        if depth == 0:
            evaluated.append(state)
            return value_function(state), -1
        is_max = state.current_player() == maxp
        value, best = (-math.inf, -1) if is_max else (math.inf, -1)
        for a in state.legal_actions():
            if max_nodes and nodes[0] == max_nodes:
                raise ab._Stop(ab.BUDGET)
            nodes[0] += 1
            child = state.clone()
            child.apply_action(a)
            v, _ = search(child, depth - 1, alpha, beta, maxp, False)
            if (v > value) if is_max else (v < value):
                value, best = v, (a if at_root else best)
            if is_max:
                alpha = max(alpha, value)
            else:
                beta = min(beta, value)
            if alpha >= beta:
                break
        return value, best

    def result(**kw):
        kw.update(evaluations=len(evaluated), evaluated=evaluated)
        return kw

    if maximizing_player < 0:
        if root.is_terminal():
            return result(value=math.nan, best_action=-1, nodes=0, status=ab.TERMINAL_ROOT)
        maximizing_player = root.current_player()
    try:
        v, best = search(root, depth_limit, -math.inf, math.inf, maximizing_player, True)
    except ab._Stop as e:
        return result(value=math.nan, best_action=-1, nodes=nodes[0], status=e.status)
    return result(value=float(v), best_action=best, nodes=nodes[0], status=ab.SOLVED)


def restated(game, hist, depth, maxp, kind, max_nodes=0):
    """alpha_beta_eval with the test value function from the root after `hist` of an OracleGame."""
    root = ab.replay(game, hist)
    m = maxp if maxp >= 0 else (root.current_player() if not root.is_terminal() else 0)
    r = alpha_beta_eval(root, depth, maxp, max_nodes, lambda s: state_values(s, kind)[m])
    r["histories"] = [s.history() for s in r.pop("evaluated")]
    return r


def same_bits(a, b):
    """Equal results with the value compared bit for bit."""
    return bits(a["value"]) == bits(b["value"]) and all(a[k] == b[k] for k in ("best_action", "nodes", "status", "evaluations"))


C4_OPENINGS = [[], [3], [3, 3], [0, 6, 1], [3, 2, 4, 3], [6, 5, 4, 3, 2], [3, 3, 3, 3, 2, 4], [1, 2, 3, 4, 5, 6, 0], [3, 4, 2, 5, 3, 4, 2, 5]]


def reference_cases():
    """(game string, root history, depth_limit, maximizing_player, kind) of the reference comparison and its golden fixture:
    seeded roots of every variant (terminal roots included), depth limits 0 to 4, each maximizing player, both value
    functions; and connect_four openings of 0 to 8 plies at depth 6."""
    from oracle_lib import OracleGame
    cases = []
    for gs, plies, _ in ab.VARIANTS:
        for hist in ab.random_roots(OracleGame(gs), 3, plies, seed=11):
            for depth in range(5):
                for maxp in (-1, 0, 1):
                    for kind in KINDS:
                        cases.append((gs, hist, depth, maxp, kind))
    for hist in C4_OPENINGS:
        for kind in KINDS:
            cases.append(("connect_four", hist, 6, -1, kind))
    return cases


def case_id(case):
    gs, hist, depth, maxp, kind = case
    return "%s|%s|%d|%d|%s" % (gs, ",".join(map(str, hist)), depth, maxp, kind)
