"""Test infrastructure for CFR-BR: ctypes bindings of the oracle's CFRBRSolver / TabularBestResponse restatement
(oracle/algorithms/cfr_br.cc) and of the unmodified reference's (oracle/_ref/libspiel_ref_cfr_br.so, built by
oracle/ref_cfr_br.mk from oracle/ref_glue/ref_cfr_br.cc), the iteration splits and
best-response cases the tests share, and table helpers."""
import ctypes as C
import hashlib
import json
import os

import numpy as np

import oracle_lib
import ref_lib

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "cfr_br_reference.json")
REF_SO = os.path.join(ref_lib.ROOT, "oracle", "_ref", "libspiel_ref_cfr_br.so")
_REF = None

# Iteration splits the oracle and the device are compared on, after every step.
SPLITS = {"kuhn_poker": [1, 1, 3, 5, 40, 250], "leduc_poker": [1, 1, 3, 10]}
# Iteration counts pinned by tests/golden/cfr_br_reference.json.
PINNED = [("kuhn_poker", 300), ("leduc_poker", 100), ("leduc_poker", 1000)]
BR_SEEDS = 50

_i64p, _dp, _vp, _cp = C.POINTER(C.c_int64), C.POINTER(C.c_double), C.c_void_p, C.c_char_p


def _oracle():
    L = oracle_lib.lib()
    if not getattr(L, "_cfrbr_bound", False):
        L.orc_cfrbr_new.restype = _vp
        L.orc_cfrbr_new.argtypes = [_vp]
        L.orc_cfrbr_free.argtypes = [_vp]
        L.orc_cfrbr_iterate.argtypes = [_vp, C.c_int]
        L.orc_cfrbr_iteration.argtypes = [_vp]
        L.orc_cfrbr_num_infosets.argtypes = [_vp]
        L.orc_cfrbr_get.argtypes = [_vp, C.c_int, _cp, C.c_int, _i64p, _dp, _dp, _dp, C.c_int, C.POINTER(C.c_int)]
        L.orc_cfrbr_set.argtypes = [_vp, _cp, _dp, _dp, _dp, C.c_int]
        L.orc_cfrbr_set_iteration.argtypes = [_vp, C.c_int]
        L.orc_cfrbr_average_values.argtypes = [_vp, _dp]
        L.orc_tabular_br.argtypes = [_vp, C.c_int, _cp, C.POINTER(C.c_int), _dp, C.c_int, _i64p, _dp]
        L._cfrbr_bound = True
    return L


def ref_available():
    """The reference's CFRBRSolver glue is built (and with it libspiel_ref_c.so, which it links against)."""
    return ref_lib.available() and os.path.exists(REF_SO)


def _ref():
    global _REF
    if _REF is None:
        ref_lib.lib()                  # the reference's games, the error handler, and the one copy of the library
        L = C.CDLL(REF_SO)
        L.ref_cfrbr_last_error.restype = _cp
        L.ref_cfrbr_new.restype = _vp
        L.ref_cfrbr_new.argtypes = [_vp]
        L.ref_cfrbr_free.argtypes = [_vp]
        L.ref_cfrbr_iterate.argtypes = [_vp, C.c_int]
        L.ref_cfrbr_get.argtypes = [_vp, _cp, _i64p, _dp, _dp, _dp, C.c_int]
        L.ref_cfrbr_keys.argtypes = [_vp, _cp, C.c_int]
        L.ref_cfrbr_serialize.argtypes = [_vp, _cp, C.c_int]
        L.ref_cfrbr_deserialize.restype = _vp
        L.ref_cfrbr_deserialize.argtypes = [_cp]
        L.ref_cfrbr_average_eval.argtypes = [_vp, _vp, _dp]
        L.ref_tabular_br.argtypes = [_vp, C.c_int, _cp, C.POINTER(C.c_int), _i64p, _dp, C.c_int, _i64p, _dp]
        _REF = L
    return _REF


def _ref_error():
    return _ref().ref_cfrbr_last_error()


class OracleCFRBR:
    """oracle/algorithms/cfr_br.cc: restatement of algorithms::CFRBRSolver."""

    def __init__(self, game):
        self.game = game
        self._c = _oracle().orc_cfrbr_new(game._g)

    def __del__(self):
        try:
            _oracle().orc_cfrbr_free(self._c)
        except Exception:
            pass

    def iterate(self, iters=1):
        _oracle().orc_cfrbr_iterate(self._c, iters)

    @property
    def iteration(self):
        return _oracle().orc_cfrbr_iteration(self._c)

    def table(self):
        L = _oracle()
        out = {}
        key = C.create_string_buffer(4096)
        legal = (C.c_int64 * 16)()
        r, cu, cp = (C.c_double * 16)(), (C.c_double * 16)(), (C.c_double * 16)()
        pl = C.c_int()
        for k in range(L.orc_cfrbr_num_infosets(self._c)):
            n = L.orc_cfrbr_get(self._c, k, key, 4096, legal, r, cu, cp, 16, C.byref(pl))
            out[key.value.decode()] = {"legal": list(legal[:n]), "regrets": list(r[:n]), "cum_policy": list(cu[:n]),
                                       "cur_policy": list(cp[:n])}
        return out

    def load(self, table, iteration):
        """Tables and counter of a deserialized solver: {key: dict(regrets, cum_policy, cur_policy)}."""
        L = _oracle()
        for key, v in table.items():
            arrs = [(C.c_double * len(v[f]))(*v[f]) for f in ("regrets", "cum_policy", "cur_policy")]
            assert L.orc_cfrbr_set(self._c, key.encode(), *arrs, len(v["regrets"])) == 0, key
        L.orc_cfrbr_set_iteration(self._c, iteration)

    def average_values(self):
        """[BR value p0, BR value p1, on-policy value p0, on-policy value p1] of the average policy."""
        out = (C.c_double * 4)()
        _oracle().orc_cfrbr_average_values(self._c, out)
        return list(out)

    def nash_conv(self):
        v = self.average_values()
        return (v[0] - v[2]) + (v[1] - v[3])

    def exploitability(self):
        return self.nash_conv() / 2


class RefCFRBR:
    """The unmodified reference's algorithms::CFRBRSolver."""

    def __init__(self, game, _ptr=None):
        self.game = game
        self._c = _ptr if _ptr is not None else _ref().ref_cfrbr_new(game._g)
        assert self._c, _ref_error()

    def __del__(self):
        try:
            _ref().ref_cfrbr_free(self._c)
        except Exception:
            pass

    def iterate(self, iters=1):
        assert _ref().ref_cfrbr_iterate(self._c, iters) == 0, _ref_error()

    def table(self):
        L = _ref()
        buf = C.create_string_buffer(1 << 20)
        L.ref_cfrbr_keys(self._c, buf, 1 << 20)
        out = {}
        legal = (C.c_int64 * 16)()
        r, cu, cp = (C.c_double * 16)(), (C.c_double * 16)(), (C.c_double * 16)()
        for key in buf.value.decode().split("\n"):
            n = L.ref_cfrbr_get(self._c, key.encode(), legal, r, cu, cp, 16)
            if n >= 0:
                out[key] = {"legal": list(legal[:n]), "regrets": list(r[:n]), "cum_policy": list(cu[:n]),
                            "cur_policy": list(cp[:n])}
        return out

    def serialize(self):
        buf = C.create_string_buffer(1 << 22)
        n = _ref().ref_cfrbr_serialize(self._c, buf, 1 << 22)
        assert 0 <= n < 1 << 22, _ref_error()
        return buf.value.decode()

    @classmethod
    def deserialize(cls, game, text):
        """DeserializeCFRBRSolver(text)."""
        return cls(game, _ref().ref_cfrbr_deserialize(text.encode()))

    def average_eval(self):
        """{nash_conv, exploitability, expected_returns} of the average policy (tabular_exploitability.cc,
        expected_returns.cc)."""
        out = (C.c_double * 4)()
        assert _ref().ref_cfrbr_average_eval(self.game._g, self._c, out) == 0, _ref_error()
        return {"nash_conv": out[0], "exploitability": out[1], "expected_returns": [out[2], out[3]]}


def _policy_args(policy):
    keys = list(policy)
    counts = (C.c_int * len(keys))(*[len(policy[k]) for k in keys])
    legal = [a for k in keys for a, _ in policy[k]]
    probs = [p for k in keys for _, p in policy[k]]
    return keys, "\n".join(keys).encode(), counts, legal, probs


def oracle_tabular_br(game, player, policy):
    """The oracle's TabularBestResponse on {key: [(action, prob)]}: ({key: action} of the player's states, root value)."""
    keys, kb, counts, _, probs = _policy_args(policy)
    acts, val = (C.c_int64 * len(keys))(), C.c_double()
    _oracle().orc_tabular_br(game._g, player, kb, counts, (C.c_double * len(probs))(*probs), len(keys), acts, C.byref(val))
    return {k: a for k, a in zip(keys, acts) if a >= 0}, val.value


def ref_tabular_br(game, player, policy):
    """The unmodified reference's TabularBestResponse(game, player, TabularPolicy(policy)): as oracle_tabular_br."""
    keys, kb, counts, legal, probs = _policy_args(policy)
    acts, val = (C.c_int64 * len(keys))(), C.c_double()
    rc = _ref().ref_tabular_br(game._g, player, kb, counts, (C.c_int64 * len(legal))(*legal),
                               (C.c_double * len(probs))(*probs), len(keys), acts, C.byref(val))
    assert rc == 0, _ref_error()
    return {k: a for k, a in zip(keys, acts) if a >= 0}, val.value


def legal_actions_by_key(game):
    """{information state string: legal actions} of every decision node of the oracle's game tree, in first-visit order."""
    out = {}

    def walk(st):
        if st.is_terminal():
            return
        if not st.is_chance_node():
            out.setdefault(st.information_state_string(st.current_player()), st.legal_actions())
        for a in st.legal_actions():
            c = st.clone()
            c.apply_action(a)
            walk(c)
    walk(game.new_initial_state())
    return out


def random_policy(legal_by_key, seed):
    """A seeded random tabular policy with exact zeros and exact ties: each state draws one of uniform, a pure action,
    two tied actions, a random distribution with zeros, or a random distribution."""
    rng = np.random.default_rng(seed)
    pol = {}
    for key, legal in legal_by_key.items():
        n = len(legal)
        kind = int(rng.integers(5))
        if kind == 0:
            p = [1.0 / n] * n
        elif kind == 1:
            p = [0.0] * n
            p[int(rng.integers(n))] = 1.0
        elif kind == 2 and n >= 2:
            p = [0.0] * n
            for a in rng.choice(n, 2, replace=False):
                p[int(a)] = 0.5
        else:
            w = rng.random(n)
            if kind == 3:
                w[int(rng.integers(n))] = 0.0
            w = w / w.sum()
            p = [float(x) for x in w]
        pol[key] = list(zip([int(a) for a in legal], p))
    return pol


def nonuniform_table(legal_by_key, seed):
    """A seeded non-uniform CFR table (regrets of both signs, positive cumulative policy, a normalised current policy) for
    deserialized-solver cases."""
    rng = np.random.default_rng(seed)
    out = {}
    for key, legal in legal_by_key.items():
        n = len(legal)
        cur = rng.random(n)
        out[key] = {"legal": [int(a) for a in legal], "regrets": [float(x) for x in rng.normal(size=n)],
                    "cum_policy": [float(x) for x in rng.random(n) * 3], "cur_policy": [float(x) for x in cur / cur.sum()]}
    return out


def assert_tables_equal(a, b):
    """Equal key sets, legal actions and bit-identical regrets, cumulative policy and current policy."""
    assert sorted(a) == sorted(b)
    for key in a:
        assert a[key]["legal"] == b[key]["legal"], key
        for f in ("regrets", "cum_policy", "cur_policy"):
            assert np.array_equal(np.array(a[key][f]), np.array(b[key][f])), (key, f, a[key][f], b[key][f])


def br_digest(actions):
    """SHA-256 of a best response's {information state: action}, keys sorted."""
    return hashlib.sha256(json.dumps(sorted(actions.items())).encode()).hexdigest()


def br_cases():
    """(seed, player) of every best-response case, the same on each game."""
    return [(seed, player) for seed in range(BR_SEEDS) for player in (0, 1)]


def golden():
    with open(GOLDEN) as f:
        return json.load(f)
