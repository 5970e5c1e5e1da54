"""Test infrastructure for Discounted CFR: ctypes bindings of the oracle's restatement (oracle/algorithms/dcfr.cc), the
reference's own Python solver (python/algorithms/discounted_cfr.py of the OpenSpiel checkout, with cfr.py, policy.py and
get_all_states.py, loaded by path over the unmodified reference games of oracle/_ref through a small pyspiel stand-in), the
variants, iteration splits and seeded tables the tests share, and table helpers."""
import collections
import ctypes as C
import hashlib
import importlib.util
import json
import os
import sys
import types

import numpy as np

import golden_lib
import oracle_lib
import ref_lib

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "dcfr_reference.json")

# name -> (alpha, beta, gamma) as the reference receives them: DCFRSolver() and LCFRSolver() as constructed, one all-float
# set, and integral-valued floats that must give the bits of the same ints.
VARIANTS = {
    "dcfr": (3 / 2, 0, 2),
    "lcfr": (1, 1, 1),
    "a2_b0.5_g3": (2.0, 0.5, 3.0),
    "dcfr_floats": (1.5, 0.0, 2.0),
    "lcfr_floats": (1.0, 1.0, 1.0),
}
# Iteration splits the reference and the oracle are compared on (the Python reference takes about 0.3 s per leduc
# iteration), and the longer ones the device and the oracle are compared on.
REF_SPLITS = {"kuhn_poker": [1, 1, 3, 5, 40, 250, 700], "leduc_poker": [1, 1, 3, 5]}
DEV_SPLITS = {"kuhn_poker": [1, 1, 3, 5, 40, 250, 700, 9000], "leduc_poker": [1, 1, 3, 5, 40, 250, 700, 9000]}
ZERO_REACH_SPLITS = {"kuhn_poker": [1, 2, 7, 40], "leduc_poker": [1, 2, 3]}
ZERO_REACH_SEED = 25
PRUNE_NONE, PRUNE, PRUNE_UPDATES = 0, 1, 2

_dp, _vp, _cp = C.POINTER(C.c_double), C.c_void_p, C.c_char_p


def _oracle():
    L = oracle_lib.lib()
    if not getattr(L, "_dcfr_bound", False):
        L.orc_dcfr_new.restype = _vp
        L.orc_dcfr_new.argtypes = [_vp, C.c_double, C.c_double, C.c_double, C.c_int]
        L.orc_dcfr_free.argtypes = [_vp]
        L.orc_dcfr_iterate.argtypes = [_vp, C.c_int]
        L.orc_dcfr_iteration.argtypes = [_vp]
        L.orc_dcfr_set_iteration.argtypes = [_vp, C.c_int]
        L.orc_dcfr_num_infosets.argtypes = [_vp]
        L.orc_dcfr_get.argtypes = [_vp, C.c_int, _cp, C.c_int, C.POINTER(C.c_int64), _dp, _dp, _dp, C.c_int,
                                   C.POINTER(C.c_int)]
        L.orc_dcfr_set.argtypes = [_vp, _cp, _dp, _dp, _dp, C.c_int]
        L._dcfr_bound = True
    return L


class OracleDCFR:
    """oracle/algorithms/dcfr.cc: restatement of _DCFRSolver.  prune: PRUNE (the reference's), or, as contrasts,
    PRUNE_UPDATES (table updates only, unpruned values) or PRUNE_NONE."""

    def __init__(self, game, alpha, beta, gamma, prune=None):
        prune = PRUNE if prune is None else prune
        self.game = game
        self._c = _oracle().orc_dcfr_new(game._g, float(alpha), float(beta), float(gamma), int(prune))
        assert self._c

    def __del__(self):
        try:
            _oracle().orc_dcfr_free(self._c)
        except Exception:
            pass

    def iterate(self, iters=1):
        _oracle().orc_dcfr_iterate(self._c, iters)

    @property
    def iteration(self):
        return _oracle().orc_dcfr_iteration(self._c)

    def table(self):
        L = _oracle()
        out = {}
        key = C.create_string_buffer(4096)
        legal = (C.c_int64 * 16)()
        r, cu, cp = (C.c_double * 16)(), (C.c_double * 16)(), (C.c_double * 16)()
        pl = C.c_int()
        for k in range(L.orc_dcfr_num_infosets(self._c)):
            n = L.orc_dcfr_get(self._c, k, key, 4096, legal, r, cu, cp, 16, C.byref(pl))
            out[key.value.decode()] = {"legal": list(legal[:n]), "regrets": list(r[:n]), "cum_policy": list(cu[:n]),
                                       "cur_policy": list(cp[:n])}
        return out

    def load(self, table, iteration):
        L = _oracle()
        for key, v in table.items():
            arrs = [(C.c_double * len(v[f]))(*v[f]) for f in ("regrets", "cum_policy", "cur_policy")]
            assert L.orc_dcfr_set(self._c, key.encode(), *arrs, len(v["regrets"])) == 0, key
        L.orc_dcfr_set_iteration(self._c, iteration)


# ---- the reference's Python solver ----------------------------------------------------------------------------------

def _reference_dir():
    from __graft_entry__ import REFERENCE
    return os.path.join(REFERENCE, "open_spiel", "python")


def ref_available():
    return ref_lib.available() and os.path.exists(os.path.join(_reference_dir(), "algorithms", "discounted_cfr.py"))


class _GameType:
    """The pyspiel.GameType fields cfr.py, policy.py and get_all_states.py read for kuhn_poker and leduc_poker."""
    class Dynamics:
        SEQUENTIAL, MEAN_FIELD = "sequential", "mean_field"

    dynamics = "sequential"
    provides_information_state_string = provides_information_state_tensor = True
    provides_observation_string = provides_observation_tensor = True


class _State:
    """pyspiel.State over a reference state (ref_lib.RefState), with the methods the Python solver calls."""

    def __init__(self, s):
        self._s = s

    def clone(self):
        return _State(self._s.clone())

    def child(self, a):
        c = self._s.clone()
        c.apply_action(a)
        return _State(c)

    def is_terminal(self):
        return self._s.is_terminal()

    def is_chance_node(self):
        return self._s.is_chance_node()

    def is_simultaneous_node(self):
        return False

    def current_player(self):
        return self._s.current_player()

    def legal_actions(self, player=None):
        return self._s.legal_actions()

    def legal_actions_mask(self, player):
        mask = [0] * self._s.game.num_distinct_actions
        for a in self._s.legal_actions():
            mask[a] = 1
        return mask

    def chance_outcomes(self):
        return self._s.chance_outcomes()

    def returns(self):
        return self._s.returns()

    def history_str(self):
        return " ".join(str(a) for a in self._s.history())

    def information_state_string(self, player=None):
        return self._s.information_state_string(self._s.current_player() if player is None else player)

    def information_state_tensor(self, player=None):
        return self._s.information_state_tensor(self._s.current_player() if player is None else player)


class _Game:
    def __init__(self, g):
        self._g = g

    def get_type(self):
        return _GameType

    def num_players(self):
        return self._g.num_players

    def num_distinct_actions(self):
        return self._g.num_distinct_actions

    def new_initial_state(self):
        return _State(self._g.new_initial_state())

    def new_initial_states(self):
        return [self.new_initial_state()]


_REF_MODULE = None


def reference_module():
    """discounted_cfr.py with its imports (cfr.py, policy.py, get_all_states.py) loaded by path from the checkout, under a
    pyspiel stand-in; sys.modules is restored afterwards."""
    global _REF_MODULE
    if _REF_MODULE is not None:
        return _REF_MODULE
    py = _reference_dir()
    pyspiel = types.ModuleType("pyspiel")
    pyspiel.GameType = _GameType
    pyspiel.PlayerId = types.SimpleNamespace(MEAN_FIELD=-5)
    pyspiel.Game, pyspiel.State, pyspiel.TabularPolicy = _Game, _State, object     # annotations only
    names = ["pyspiel", "open_spiel", "open_spiel.python", "open_spiel.python.games", "open_spiel.python.algorithms",
             "open_spiel.python.algorithms.get_all_states", "open_spiel.python.policy", "open_spiel.python.algorithms.cfr"]
    saved = {n: sys.modules.get(n) for n in names}
    try:
        sys.modules["pyspiel"] = pyspiel
        for pkg in ("open_spiel", "open_spiel.python", "open_spiel.python.games", "open_spiel.python.algorithms"):
            sys.modules[pkg] = types.ModuleType(pkg)
        sys.modules["open_spiel"].python = sys.modules["open_spiel.python"]
        sys.modules["open_spiel.python"].algorithms = sys.modules["open_spiel.python.algorithms"]
        sys.modules["open_spiel.python"].games = sys.modules["open_spiel.python.games"]

        def load(name, path, parent, attr):
            spec = importlib.util.spec_from_file_location(name, path)
            m = importlib.util.module_from_spec(spec)
            sys.modules[name] = m
            spec.loader.exec_module(m)
            setattr(sys.modules[parent], attr, m)
            return m
        load("open_spiel.python.algorithms.get_all_states", os.path.join(py, "algorithms", "get_all_states.py"),
             "open_spiel.python.algorithms", "get_all_states")
        load("open_spiel.python.policy", os.path.join(py, "policy.py"), "open_spiel.python", "policy")
        load("open_spiel.python.algorithms.cfr", os.path.join(py, "algorithms", "cfr.py"), "open_spiel.python.algorithms", "cfr")
        spec = importlib.util.spec_from_file_location("reference_discounted_cfr", os.path.join(py, "algorithms", "discounted_cfr.py"))
        m = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(m)
    finally:
        for n, mod in saved.items():
            if mod is None:
                sys.modules.pop(n, None)
            else:
                sys.modules[n] = mod
    _REF_MODULE = m
    return m


class RefDCFR:
    """The reference's DCFRSolver / LCFRSolver over the unmodified reference game."""

    def __init__(self, game_string, variant):
        m = reference_module()
        game = _Game(ref_lib.RefGame(game_string))
        if variant == "dcfr":
            self.solver = m.DCFRSolver(game)
        elif variant == "lcfr":
            self.solver = m.LCFRSolver(game)
        else:
            self.solver = m.DCFRSolver(game, *VARIANTS[variant])

    def iterate(self, iters=1):
        for _ in range(iters):
            self.solver.evaluate_and_update_policy()

    def table(self):
        s = self.solver
        cur = s._current_policy.action_probability_array
        out = {}
        for key, node in s._info_state_nodes.items():
            legal = list(node.legal_actions)
            out[key] = {"legal": legal,
                        "regrets": [float(node.cumulative_regret.get(a, 0.0)) for a in legal],
                        "cum_policy": [float(node.cumulative_policy.get(a, 0.0)) for a in legal],
                        "cur_policy": [float(cur[node.index_in_tabular_policy][a]) for a in legal]}
        return out

    def average_policy(self):
        """{key: [probabilities in legal-action order]} of the reference's average_policy()."""
        avg = self.solver.average_policy().action_probability_array
        return {key: [float(avg[node.index_in_tabular_policy][a]) for a in node.legal_actions]
                for key, node in self.solver._info_state_nodes.items()}

    def load(self, table, iteration):
        """Seed the tables as numpy float64 values (what the solver's own += and *= store) and the iteration counter."""
        s = self.solver
        for key, v in table.items():
            node = s._info_state_nodes[key]
            node.cumulative_regret = collections.defaultdict(float, {a: np.float64(x) for a, x in zip(v["legal"], v["regrets"])})
            node.cumulative_policy = collections.defaultdict(float, {a: np.float64(x) for a, x in zip(v["legal"], v["cum_policy"])})
            for a, x in zip(v["legal"], v["cur_policy"]):
                s._current_policy.action_probability_array[node.index_in_tabular_policy][a] = x
        s._iteration = iteration


# ---- tables ---------------------------------------------------------------------------------------------------------

def average_policy(table):
    """cfr.py _update_average_policy (:100-123) on a {key: {legal, cum_policy}} table: sequential sum, 1 / n where it is 0."""
    out = {}
    for key, v in table.items():
        s = 0
        for x in v["cum_policy"]:
            s = s + x
        n = len(v["legal"])
        out[key] = [1 / n] * n if s == 0 else [x / s for x in v["cum_policy"]]
    return out


def assert_tables_equal(a, b):
    """Equal key sets, legal actions and bit-identical regrets (sign of zero included), cumulative and current policy."""
    assert sorted(a) == sorted(b)
    for key in a:
        assert a[key]["legal"] == b[key]["legal"], key
        for f in ("regrets", "cum_policy", "cur_policy"):
            x, y = np.array(a[key][f], dtype=np.float64), np.array(b[key][f], dtype=np.float64)
            assert x.tobytes() == y.tobytes(), (key, f, a[key][f], b[key][f])


def average_digest(avg):
    h = hashlib.sha256()
    for key in sorted(avg):
        h.update(key.encode() + b"\0" + np.asarray(avg[key], dtype=np.float64).tobytes())
    return h.hexdigest()


def digests(table):
    return {"table_sha256": golden_lib.table_digest(table), "average_sha256": average_digest(average_policy(table))}


def negative_zeros(table):
    return sum(int(np.signbit(x) and x == 0) for v in table.values() for x in v["regrets"])


def sign_differences(a, b):
    """Entries whose regret bits differ between two tables with the same keys."""
    return sum(int(np.float64(x).tobytes() != np.float64(y).tobytes())
               for key in a for x, y in zip(a[key]["regrets"], b[key]["regrets"]))


def zero_reach_table(legal_by_key, seed):
    """A seeded table whose current policy is pure, so that many histories lie below two zero-probability edges, one of
    each player: each information state has one positive regret (50..100) at a random action and -0.0 elsewhere, a random
    positive cumulative policy, and the current policy regret matching gives.  Information states no player reaches keep
    their -0.0 regrets under the reference's pruning; the unpruned rule would add +0.0 to some of them."""
    rng = np.random.default_rng(seed)
    out = {}
    for key, legal in legal_by_key.items():
        n = len(legal)
        k = int(rng.integers(n))
        regrets = [-0.0] * n
        regrets[k] = float(50 + 50 * rng.random())
        cur = [0.0] * n
        cur[k] = 1.0
        out[key] = {"legal": [int(a) for a in legal], "regrets": regrets,
                    "cum_policy": [float(x) for x in rng.random(n) * 3], "cur_policy": cur}
    return out


def golden():
    with open(GOLDEN) as f:
        return json.load(f)
