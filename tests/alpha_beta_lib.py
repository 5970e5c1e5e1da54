"""Restatement of algorithms::AlphaBetaSearch (reference open_spiel/algorithms/minimax.cc:49-137, 221-258) over any State with
clone / apply_action / legal_actions / returns / is_terminal / current_player (the CPU oracle's or the reference's), with the
device's additions: the count of generated child states, the per-root budget and the status codes of b2s_alpha_beta_search
(include/b2s.h).  Test infrastructure."""
import math
import random

SOLVED, BUDGET, DEPTH_ZERO, TERMINAL_ROOT = 0, 1, 2, 3


class _Stop(Exception):
    def __init__(self, status):
        self.status = status


def alpha_beta(root, depth_limit=-1, maximizing_player=-1, max_nodes=0):
    """dict(value, best_action, nodes, status) exactly as lane i of b2s_alpha_beta_search reports them."""
    nodes = [0]

    def search(state, depth, alpha, beta, maxp, at_root):          # minimax.cc:49-137
        if state.is_terminal():
            return state.returns()[maxp], -1
        if depth == 0:
            raise _Stop(DEPTH_ZERO)                                # SpielFatalError: no value function
        is_max = state.current_player() == maxp
        value, best = (-math.inf, -1) if is_max else (math.inf, -1)
        for a in state.legal_actions():
            if max_nodes and nodes[0] == max_nodes:
                raise _Stop(BUDGET)
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

    if maximizing_player < 0:
        if root.is_terminal():
            return dict(value=math.nan, best_action=-1, nodes=0, status=TERMINAL_ROOT)
        maximizing_player = root.current_player()
    try:
        v, best = search(root, depth_limit, -math.inf, math.inf, maximizing_player, True)
    except _Stop as e:
        return dict(value=math.nan, best_action=-1, nodes=nodes[0], status=e.status)
    return dict(value=float(v), best_action=best, nodes=nodes[0], status=SOLVED)


def random_roots(game, count, plies, seed):
    """`count` action histories of seeded uniform play from the initial state, each `plies` long or cut at a terminal state.
    plies may be an int or a (lo, hi) range."""
    rng = random.Random(seed)
    out = []
    for _ in range(count):
        k = plies if isinstance(plies, int) else rng.randint(plies[0], plies[1])
        s, hist = game.new_initial_state(), []
        while len(hist) < k and not s.is_terminal():
            a = rng.choice(s.legal_actions())
            s.apply_action(a)
            hist.append(a)
        out.append(hist)
    return out


def replay(game, hist):
    s = game.new_initial_state()
    for a in hist:
        s.apply_action(a)
    return s


def same(a, b):
    """Equal results, NaN values included."""
    va, vb = a["value"], b["value"]
    return ((math.isnan(va) and math.isnan(vb)) or va == vb) and all(a[k] == b[k] for k in ("best_action", "nodes", "status"))


# Every served variant on a size whose unlimited searches stay small: (game string, root plies, roots).  go 5x5 and othello are
# late positions; connect_four 6x7 leaves about a dozen empty cells.
VARIANTS = [
    ("tic_tac_toe", (0, 9), 24),
    ("connect_four", (28, 34), 16),
    ("connect_four(rows=4,columns=4,x_in_row=3)", (4, 16), 16),
    ("breakthrough(rows=4,columns=4)", (6, 14), 12),
    ("hex(board_size=3)", (0, 9), 16),
    ("hex(board_size=4)", (6, 16), 12),
    ("othello", (48, 60), 8),
    ("mnk(m=4,n=4,k=3)", (4, 16), 16),
    ("y(board_size=4)", (3, 10), 12),
    ("havannah(board_size=3)", (10, 19), 12),
    ("go(board_size=2)", (0, 6), 12),
    ("go(board_size=3)", (4, 18), 10),
    ("go(board_size=5)", (36, 46), 6),
]


def reference_cases():
    """(game string, root history, depth_limit, maximizing_player) of the reference comparison and its golden fixture: seeded
    roots of every variant (terminal roots included), unlimited and small depth limits, each maximizing player, and the three
    tic_tac_toe cases of the reference's minimax_test.cc."""
    from oracle_lib import OracleGame
    cases = [("tic_tac_toe", [], -1, -1), ("tic_tac_toe", [4, 1], -1, -1), ("tic_tac_toe", [5, 4, 3, 8], -1, -1)]
    for gs, plies, count in VARIANTS:
        for k, hist in enumerate(random_roots(OracleGame(gs), count, plies, seed=5)):
            for depth, maxp in ((-1, -1), (-1, 0), (-1, 1), (2, -1), (3, 1)):
                if (k + depth + maxp) % 2 == 0 or depth < 0:
                    cases.append((gs, hist, depth, maxp))
    return cases


def case_id(case):
    gs, hist, depth, maxp = case
    return "%s|%s|%d|%d" % (gs, ",".join(map(str, hist)), depth, maxp)
