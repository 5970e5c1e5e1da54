"""CPU rehearsal of the device AlphaBetaSearch: the kernel body k_alpha_beta (open_spiel_b200/csrc/alpha_beta.cuh), compiled for
the host by tests/host_emul/emul_ab.cc over the product's rule cores, against the restatement in tests/alpha_beta_lib.py.
Value, best action, generated-node count and status must be equal on every served variant: unlimited searches, depth limits
that end in the depth-0 error, every maximizing player, and budgets at the oracle's count and one below it."""
import ctypes as C
import math
import os
import subprocess

import pytest

import alpha_beta_lib as ab
import open_spiel_b200 as b2
from oracle_lib import OracleGame

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMUL = os.path.join(ROOT, "tests", "host_emul")
SO = os.path.join(EMUL, "libemul_ab.so")


def _lib():
    if not os.path.isdir("/usr/local/cuda/include"):
        pytest.skip("CUDA headers not available for the host build of the rule cores")
    if not os.path.exists(SO):
        subprocess.check_call(["make", "-s", "-C", EMUL, "-f", "ab.mk"])
    L = C.CDLL(SO)
    L.emu_ab_last_error.restype = C.c_char_p
    L.emu_ab_search.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_longlong, C.POINTER(C.c_double),
                                C.POINTER(C.c_int), C.POINTER(C.c_longlong), C.POINTER(C.c_int)]
    return L


def host_search(game, hist, depth_limit=-1, maximizing_player=-1, max_nodes=0):
    L = _lib()
    acts = (C.c_int * max(1, len(hist)))(*hist)
    v, best, nodes, status = C.c_double(), C.c_int(), C.c_longlong(), C.c_int()
    rc = L.emu_ab_search(game._gid, C.addressof(game._cparams), acts, len(hist), depth_limit, maximizing_player, max_nodes,
                         C.byref(v), C.byref(best), C.byref(nodes), C.byref(status))
    assert rc == 0, L.emu_ab_last_error()
    return dict(value=v.value, best_action=best.value, nodes=nodes.value, status=status.value)


@pytest.mark.parametrize("gs,plies,count", ab.VARIANTS, ids=[v[0] for v in ab.VARIANTS])
def test_host_kernel_body_equals_oracle(gs, plies, count):
    og, dg = OracleGame(gs), b2.load_game(gs)
    roots = ab.random_roots(og, count, plies, seed=11)
    checked = 0
    for k, hist in enumerate(roots):
        settings = [(-1, -1), (-1, 0), (-1, 1), (2, -1), (1, 1)]
        for depth, maxp in settings:
            want = ab.alpha_beta(ab.replay(og, hist), depth, maxp)
            got = host_search(dg, hist, depth, maxp)
            assert ab.same(got, want), (gs, hist, depth, maxp, got, want)
            checked += 1
        want = ab.alpha_beta(ab.replay(og, hist))
        if want["status"] == ab.SOLVED and want["nodes"] > 0:      # budget edge: the oracle's count solves, one less stops
            assert ab.same(host_search(dg, hist, max_nodes=want["nodes"]), want)
            cut = host_search(dg, hist, max_nodes=want["nodes"] - 1) if want["nodes"] > 1 else None
            if cut is not None:
                assert cut["status"] == ab.BUDGET and cut["nodes"] == want["nodes"] - 1 and math.isnan(cut["value"])
                assert ab.same(cut, ab.alpha_beta(ab.replay(og, hist), max_nodes=want["nodes"] - 1))
    assert checked == 5 * count


def test_host_minimax_test_cases():
    """The three tic_tac_toe cases of the reference's minimax_test.cc."""
    g = b2.load_game("tic_tac_toe")
    assert host_search(g, [])["value"] == 0.0
    assert host_search(g, [4, 1])["value"] == 1.0
    assert host_search(g, [5, 4, 3, 8])["value"] == -1.0
    r = host_search(g, [])
    assert (r["best_action"], r["nodes"], r["status"]) == (0, 18296, 0)
