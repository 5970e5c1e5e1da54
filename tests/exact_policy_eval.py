"""Exact-arithmetic NashConv / best response of a tabular policy in a two-player game: a plain restatement of
algorithms::NashConv (tabular_exploitability.cc) and TabularBestResponse (best_response.cc) in fractions.Fraction over
the oracle's game tree.  Test infrastructure, CPU only.

The policy comes as a device-table-shaped table (CFRSolver.table(): offsets, legal_actions, keys) with either a current
policy, used as it is, or a cumulative policy, normalised with the rule of CFRAveragePolicy (cfr.cc:104-125): uniform
where the row sums to exactly 0.  Information states are keyed by their information-state tensor bytes, as the device
table keys its rows.  Chance probabilities, terminal utilities and policy entries are the exact values of the doubles the
oracle and the table hold, so the result is the device's computation without rounding.

The only rounding-aware output is `cf_reach_zero`: whether every history of a responder's information state has
counterfactual reach exactly 0 as a double product, accumulated in the device's order (parents before children, one
multiplication per edge).  There every q(I, a) is 0 on the device and TabularBestResponse's first-maximum rule picks
action index 0."""
import functools
from fractions import Fraction

import numpy as np

from oracle_lib import OracleGame


class ExactTree:
    """The game tree of `game_string`, walked on the oracle like oracle_lib.infostate_tensors.  Node 0 is the root;
    nodes are numbered in DFS order, children in legal-action order."""

    def __init__(self, game_string):
        self.game_string = game_string
        self.kind, self.player, self.depth, self.children, self.infoset = [], [], [], [], []
        self.chance_p, self.chance_p_double, self.chance_p_rational, self.ret = {}, {}, {}, {}
        self.is_key, self.is_string, self.is_player, self.is_legal, self.hists = [], [], [], [], []
        key_to_is = {}

        def walk(st, depth):
            n = len(self.kind)
            self.kind.append(0)
            self.player.append(-1)
            self.depth.append(depth)
            self.children.append([])
            self.infoset.append(-1)
            if st.is_terminal():
                self.ret[n] = tuple(Fraction(r) for r in st.returns())
                return n
            if st.is_chance_node():
                self.kind[n] = 1
                outcomes = st.chance_outcomes()
                self.chance_p[n] = [Fraction(p) for _, p in outcomes]
                self.chance_p_double[n] = [p for _, p in outcomes]
                self.chance_p_rational[n] = [Fraction(p).limit_denominator(1 << 20) for _, p in outcomes]
                assert [float(p) for p in self.chance_p_rational[n]] == self.chance_p_double[n]
                actions = [a for a, _ in outcomes]
            else:
                p = st.current_player()
                self.kind[n], self.player[n] = 2, p
                key = st.information_state_tensor(p).tobytes()
                actions = st.legal_actions()
                I = key_to_is.get(key)
                if I is None:
                    I = key_to_is[key] = len(self.is_key)
                    self.is_key.append(key)
                    self.is_string.append(st.information_state_string(p))
                    self.is_player.append(p)
                    self.is_legal.append(actions)
                    self.hists.append([])
                assert self.is_legal[I] == actions and self.is_player[I] == p
                self.infoset[n] = I
                self.hists[I].append(n)
            for a in actions:
                c = st.clone()
                c.apply_action(a)
                self.children[n].append(walk(c, depth + 1))
            return n

        self.oracle_game = OracleGame(game_string)
        walk(self.oracle_game.new_initial_state(), 0)
        self.num_nodes = len(self.kind)
        self.num_levels = max(self.depth) + 1
        self.by_depth = [[] for _ in range(self.num_levels)]
        for n in range(self.num_nodes):
            self.by_depth[self.depth[n]].append(n)
        self.is_depth = [self.depth[h[0]] for h in self.hists]
        assert all(self.depth[h] == self.is_depth[I] for I, hs in enumerate(self.hists) for h in hs)
        self.max_abs_utility = max(abs(v) for r in self.ret.values() for v in r)

    def layout(self):
        """A table shaped like CFRSolver.table() (offsets, legal_actions, players, keys), rows in this tree's order."""
        offsets = np.zeros(len(self.is_key) + 1, dtype=np.int32)
        for I, legal in enumerate(self.is_legal):
            offsets[I + 1] = offsets[I] + len(legal)
        return {"offsets": offsets, "legal_actions": np.array([a for legal in self.is_legal for a in legal], dtype=np.int32),
                "players": np.array(self.is_player, dtype=np.int32),
                "keys": np.stack([np.frombuffer(k, dtype=np.float32) for k in self.is_key])}


@functools.lru_cache(maxsize=None)
def tree(game_string):
    return ExactTree(game_string)


def row_strings(game_string, table):
    """The information-state string of every row of `table`."""
    t = tree(game_string)
    strings = {key: s for key, s in zip(t.is_key, t.is_string)}
    return [strings[table["keys"][k].tobytes()] for k in range(len(table["offsets"]) - 1)]


# ---- policy tables in the layout of a table: num_entries entries, one row per information state ----------------------
def _rows(table):
    off = table["offsets"]
    return [(int(off[k]), int(off[k + 1])) for k in range(len(off) - 1)]


def uniform(table):
    out = np.empty(len(table["legal_actions"]))
    for lo, hi in _rows(table):
        out[lo:hi] = 1.0 / (hi - lo)
    return out


def dirichlet(table, seed):
    rng = np.random.default_rng(seed)
    out = np.empty(len(table["legal_actions"]))
    for lo, hi in _rows(table):
        out[lo:hi] = rng.dirichlet(np.ones(hi - lo))
    return out


def sparse(table, seed):
    """About a third of the actions exactly 0 (never a whole row), so whole subtrees have zero reach for the opponent
    and for the responder."""
    rng = np.random.default_rng(seed)
    out = np.empty(len(table["legal_actions"]))
    for lo, hi in _rows(table):
        keep = rng.random(hi - lo) >= 1 / 3
        keep[rng.integers(hi - lo)] = True
        w = rng.dirichlet(np.ones(hi - lo)) * keep
        out[lo:hi] = w / w.sum()
    return out


def pure(table, seed):
    rng = np.random.default_rng(seed)
    out = np.zeros(len(table["legal_actions"]))
    for lo, hi in _rows(table):
        out[lo + rng.integers(hi - lo)] = 1.0
    return out


def tiny(table, seed):
    """One action of most rows at probability 1e-300, so that a path through two of them has a reach product that
    underflows to 0 (or a subnormal) in double."""
    rng = np.random.default_rng(seed)
    out = dirichlet(table, seed + 1000)
    for lo, hi in _rows(table):
        if rng.random() < 0.7:
            out[lo + rng.integers(hi - lo)] = 1e-300
    return out


def cum_mixed(table, seed):
    """A cumulative-policy table: rows all zero (the uniform fallback), rows mixing zeros and nonzeros, rows scaled by
    1e-30 and by 1e+30, and plain rows.  Sums large enough to overflow to inf are left out: the reference divides by
    inf too, so such a table is not a meaningful input."""
    rng = np.random.default_rng(seed)
    out = np.empty(len(table["legal_actions"]))
    for lo, hi in _rows(table):
        w = rng.random(hi - lo) * 10
        kind = rng.integers(5)
        if kind == 0:
            w[:] = 0.0
        elif kind == 1:
            w[rng.random(hi - lo) < 0.5] = 0.0
        elif kind == 2:
            w *= 1e-30
        elif kind == 3:
            w *= 1e+30
        out[lo:hi] = w
    return out


def kuhn_equilibrium(game_string, table, alpha):
    """The standard equilibrium family of 2-player Kuhn poker (action 0 = pass, 1 = bet; cards 0 = J, 1 = Q, 2 = K).
    Player 0 bets J with alpha, checks Q, bets K with 3 alpha, and after check-bet calls with Q with alpha + 1/3 (never
    with J, always with K).  Player 1 after a check bets J with 1/3, checks Q, bets K; after a bet calls with Q with 1/3,
    never with J, always with K.  `alpha` may be a Fraction (the policy is then exact) or a float.  List in the layout
    of `table`."""
    third = Fraction(1, 3) if isinstance(alpha, Fraction) else 1.0 / 3.0
    bet = {"0": alpha, "1": 0, "2": 3 * alpha, "0pb": 0, "1pb": alpha + third, "2pb": 1,
           "0p": third, "1p": 0, "2p": 1, "0b": 0, "1b": third, "2b": 1}
    out = [None] * len(table["legal_actions"])
    for (lo, hi), s in zip(_rows(table), row_strings(game_string, table)):
        assert table["legal_actions"][lo:hi].tolist() == [0, 1]
        b = bet[s]
        out[lo], out[lo + 1] = 1 - b, b
    if isinstance(alpha, Fraction):
        return [Fraction(v) for v in out]
    return [float(v) for v in out]


def _row_policy(values, average):
    """(exact, double) probabilities of one table row: the row itself, or CFRAveragePolicy's normalisation of it (the
    double version in the device's order: sequential sum, then one division per entry).  A row sum that overflows to inf
    is not handled here; the reference computes NaN probabilities from it just as the device does.  Entries may be
    doubles or exact Fractions."""
    exact, vals = [Fraction(v) for v in values], [float(v) for v in values]
    if not average:
        return exact, vals
    na = len(vals)
    s = sum(exact)
    sd = 0.0
    for v in vals:
        sd += v
    exact = [Fraction(1, na)] * na if s == 0 else [v / s for v in exact]
    dbl = [1.0 / na] * na if sd == 0.0 else [v / sd for v in vals]
    return exact, dbl


def evaluate(game_string, table, policy, average, rational_chance=False):
    """Exact NashConv of the policy given by `policy` (num_entries doubles in the layout of `table`): the current policy
    when `average` is false, else the average policy normalised from `policy` as a cumulative-policy table.
    rational_chance: take chance probabilities as the simple fractions (1/3, 1/6, ...) the oracle's doubles are the
    roundings of, instead of the doubles themselves, for closed-form game values.

    Returns dict(values=[BR_0, BR_1, v_0, v_1], nash_conv, and per row k of `table` that is a decision point:
    q[k] = [sum_h cf_reach(h) * V_b(child(h, a)) for each action], cf_reach_sum[k], cf_reach_zero[k] and best[k], the
    first exact maximiser of q[k]), all exact Fractions except the boolean cf_reach_zero and the index best."""
    t = tree(game_string)
    by_key = {table["keys"][k].tobytes(): k for k in range(len(table["offsets"]) - 1)}
    assert len(by_key) == len(t.is_key), (len(by_key), len(t.is_key))
    rows = [by_key[key] for key in t.is_key]
    pol, pol_d = [], []
    for I, k in enumerate(rows):
        lo, hi = int(table["offsets"][k]), int(table["offsets"][k + 1])
        assert table["legal_actions"][lo:hi].tolist() == t.is_legal[I]
        e, d = _row_policy(policy[lo:hi], average)
        pol.append(e)
        pol_d.append(d)
    chance_p = t.chance_p_rational if rational_chance else t.chance_p

    def edge(n):
        """(exact, double) probabilities of the edges below chance or decision node n."""
        if t.kind[n] == 1:
            return chance_p[n], t.chance_p_double[n]
        return pol[t.infoset[n]], pol_d[t.infoset[n]]

    # on-policy values
    val = [None] * t.num_nodes
    for level in reversed(t.by_depth):
        for n in level:
            if t.kind[n] == 0:
                val[n] = t.ret[n]
            else:
                v0 = v1 = Fraction(0)
                for p, c in zip(edge(n)[0], t.children[n]):
                    if p:
                        v0 += p * val[c][0]
                        v1 += p * val[c][1]
                val[n] = (v0, v1)
    values = [None, None, val[0][0], val[0][1]]
    q, cf_sum, cf_zero, best = {}, {}, {}, {}
    for b in (0, 1):
        # counterfactual reach for responder b: every probability but b's own
        reach, reach_d = [None] * t.num_nodes, [None] * t.num_nodes
        reach[0], reach_d[0] = Fraction(1), 1.0
        for level in t.by_depth:
            for n in level:
                if t.kind[n] == 0:
                    continue
                if t.kind[n] == 2 and t.player[n] == b:
                    for c in t.children[n]:
                        reach[c], reach_d[c] = reach[n], reach_d[n]
                else:
                    pe, pd = edge(n)
                    for p, p_d, c in zip(pe, pd, t.children[n]):
                        reach[c], reach_d[c] = reach[n] * p, reach_d[n] * p_d
        br = [None] * t.num_nodes
        for depth in range(t.num_levels - 1, -1, -1):
            choice = {}
            for I in range(len(t.is_key)):
                if t.is_player[I] != b or t.is_depth[I] != depth:
                    continue
                qs = [sum((reach[h] * br[t.children[h][a]] for h in t.hists[I]), Fraction(0))
                      for a in range(len(t.is_legal[I]))]
                arg = max(range(len(qs)), key=lambda a: (qs[a], -a))       # first maximum
                choice[I] = arg
                k = rows[I]
                q[k], best[k] = qs, arg
                cf_sum[k] = sum((reach[h] for h in t.hists[I]), Fraction(0))
                cf_zero[k] = all(reach_d[h] == 0.0 for h in t.hists[I])
            for n in t.by_depth[depth]:
                if t.kind[n] == 0:
                    br[n] = t.ret[n][b]
                elif t.kind[n] == 2 and t.player[n] == b:
                    br[n] = br[t.children[n][choice[t.infoset[n]]]]
                else:
                    br[n] = sum((p * br[c] for p, c in zip(edge(n)[0], t.children[n]) if p), Fraction(0))
        values[b] = br[0]
    return {"values": values, "nash_conv": (values[0] - values[2]) + (values[1] - values[3]),
            "q": q, "cf_reach_sum": cf_sum, "cf_reach_zero": cf_zero, "best": best, "rows": rows}
