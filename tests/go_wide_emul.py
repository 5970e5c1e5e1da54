"""Test infrastructure: the host builds of the rule cores and MCTS kernel bodies that also hold go 10..19
(tests/host_emul/go_wide.mk: libemul_go_wide.so, libemul_eval_go_wide.so).  They export the same C functions as
libemul.so / libemul_eval.so; use_wide_libraries(monkeypatch) points the helpers of test_rule_cores_host.py (Emu,
_lockstep, the playout test) and test_mcts_eval_host.py (Emv, run_emulated) at them for the duration of one test."""
import ctypes as C
import os
import subprocess

import pytest

import test_mcts_eval_host
import test_rule_cores_host

HERE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "host_emul")
_LIBS = {}


def _load(name):
    if name not in _LIBS:
        so = os.path.join(HERE, name)
        if not os.path.exists(so):
            subprocess.run(["make", "-s", "-C", HERE, "-f", "go_wide.mk"], capture_output=True)
        if not os.path.exists(so):
            pytest.skip("host emulation library not built (needs g++ and the CUDA headers)")
        _LIBS[name] = C.CDLL(so)
    return _LIBS[name]


def emu_lib():
    """libemul_go_wide.so with test_rule_cores_host._lib's signatures."""
    L = _load("libemul_go_wide.so")
    L.emu_create.restype = C.c_void_p
    L.emu_create.argtypes = [C.c_int, C.c_void_p, C.c_longlong]
    L.emu_last_error.restype = C.c_char_p
    for name, args in (("emu_destroy", [C.c_void_p]), ("emu_info", [C.c_void_p, C.c_void_p]),
                       ("emu_reset", [C.c_void_p, C.c_longlong]), ("emu_apply", [C.c_void_p, C.c_void_p, C.c_longlong]),
                       ("emu_legal_mask", [C.c_void_p, C.c_void_p, C.c_longlong]),
                       ("emu_status", [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_longlong]),
                       ("emu_observation", [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_longlong])):
        getattr(L, name).argtypes = args
    L.emu_error_count.restype = C.c_longlong
    L.emu_error_count.argtypes = [C.c_void_p]
    L.emu_rollout.argtypes = [C.c_void_p, C.c_ulonglong, C.c_longlong, C.c_void_p, C.c_void_p, C.c_longlong]
    L.emu_mcts.argtypes = [C.c_void_p, C.c_longlong, C.c_void_p] + [C.c_void_p] * 5
    return L


def emv_lib():
    """libemul_eval_go_wide.so with test_mcts_eval_host._lib's signatures."""
    L = _load("libemul_eval_go_wide.so")
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
    return L


def use_wide_libraries(monkeypatch):
    monkeypatch.setattr(test_rule_cores_host, "_lib", emu_lib)
    monkeypatch.setattr(test_mcts_eval_host, "_lib", emv_lib)
