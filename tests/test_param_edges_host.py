"""CPU: every accepted variant of tests/param_edges.py through the host build of the rule cores (tests/host_emul), in
lock-step with the oracle (test_rule_cores_host.py's check: status, returns with the sign of zero, legal actions and every
player's tensors after every move), plus the rollout kernel's Philox stream.  The host build runs the same source as the
device with g++ semantics, so a shift past the word size in a rule core shows up here without a GPU; and every shape past
a limit must be refused by the host build as by the device."""
import ctypes as C

import pytest

import open_spiel_b200 as b2
import test_rule_cores_host
from oracle_lib import OracleGame
from param_edges import ACCEPTED, REJECTED, host_lanes, raw_params
from philox_ref import philox_uniform
from test_rule_cores_host import Emu, _lockstep
from go_wide_emul import use_wide_libraries


def _wide(gs, monkeypatch):
    if gs.startswith("go"):            # go 10..19 is only in the wide host build; it also holds go 2..9
        use_wide_libraries(monkeypatch)


@pytest.mark.parametrize("gs,lanes", ACCEPTED, ids=[g for g, _ in ACCEPTED])
def test_rule_core_lockstep_at_layout_edges(gs, lanes, monkeypatch):
    _wide(gs, monkeypatch)
    _lockstep(gs, host_lanes(gs, lanes), OracleGame)


@pytest.mark.parametrize("gs,lanes", ACCEPTED, ids=[g for g, _ in ACCEPTED])
def test_playout_at_layout_edges(gs, lanes, monkeypatch):
    """common.cuh playout_step on the host against the oracle replaying the same Philox words, on the device test's lanes
    and stream (test_gpu_param_edges.py::test_rollout_at_layout_edges).  The host build's playout loop stops after
    max_game_length + 4 plies, which a 5-player kuhn_poker game (5 deals and up to 9 moves) can pass; b2s_rollout leaves room
    for the chance plies, and the device test checks those lanes."""
    _wide(gs, monkeypatch)
    n = lanes
    emu = Emu(gs, n)
    rets, plies = emu.rollout(0xED6E, 5000)
    og = OracleGame(gs)
    for i in range(n):
        st = og.new_initial_state()
        ply = 0
        while not st.is_terminal():
            la, cand = st.legal_actions(), st.rollout_candidates()
            retry = 0
            while True:
                a = cand[philox_uniform(0xED6E, 5000 + i, ply + 4096 * retry, len(cand))]
                if a in la:
                    break
                retry += 1
            st.apply_action(a)
            ply += 1
        if ply > emu.info.max_game_length + 4:
            assert plies[i] == emu.info.max_game_length + 4, (gs, i)
            continue
        assert ply == plies[i] and st.returns() == rets[i].tolist(), (gs, i)
    assert emu.errors() == 0


@pytest.mark.parametrize("gs", REJECTED)
def test_shapes_past_a_limit_are_refused(gs, monkeypatch):
    """load_game refuses the shape, and so does the host build's make_cfg when handed the parameters directly."""
    _wide(gs, monkeypatch)
    with pytest.raises(b2.SpielError):
        b2.load_game(gs)
    gid, cp = raw_params(gs)
    L = test_rule_cores_host._lib()
    assert not L.emu_create(gid, C.byref(cp), 4)
    assert L.emu_last_error()
