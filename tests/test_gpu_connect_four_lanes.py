"""GPU: how a connect_four batch addresses its lanes, checked where a lane format that groups lanes (e.g. in 32-lane tiles)
would break first: lane get / set at lanes 0, 31, 32, 33 and cap-1 of a batch whose capacity is not a multiple of 32, copies
between unaligned lane ranges, the chunked host-buffer step (it steps sub-range views of the batch) and two boards on either
side of 54 key bits (6x7: 49, 7x7: 56) through every batched observable, all against the oracle."""
import os
import struct
import subprocess
import sys

import numpy as np
import pytest
import torch

import open_spiel_b200 as b2
from oracle_lib import OracleGame, oracle_record_trajectory
from parity import lockstep

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BOARDS = ["connect_four", "connect_four(rows=7,columns=7)"]     # 49 and 56 key bits


def random_play(game_string, n, plies, seed):
    """n oracle states after up to `plies` random moves each (lane i stops after i % (plies + 1) of them), and a device batch
    of capacity n driven through the same moves."""
    game, og = b2.load_game(game_string), OracleGame(game_string)
    batch = game.new_batch(n)
    rng = np.random.RandomState(seed)
    states = [og.new_initial_state() for _ in range(n)]
    for ply in range(plies):
        acts = np.full(n, -1, dtype=np.int32)
        for i, st in enumerate(states):
            if ply < i % (plies + 1) and not st.is_terminal():
                la = st.legal_actions()
                acts[i] = la[rng.randint(len(la))]
                st.apply_action(int(acts[i]))
        batch.apply_actions(torch.from_numpy(acts).to(batch._dev))
    assert batch.error_count()[0] == 0
    return game, batch, states


def expected_blob(st, rows, cols):
    """The lane blob {x, o} (rules_connect_four.cuh: bit col*(rows+1)+row, cached outcome ^ 2 in bits 62-63 of x) of an
    oracle state, from its observation tensor (plane 0: player 0's stones, plane 1: player 1's)."""
    obs = np.asarray(st.observation_tensor(0)).reshape(3, rows, cols)
    x = o = 0
    for r in range(rows):
        for c in range(cols):
            bit = 1 << (c * (rows + 1) + r)
            x |= bit if obs[0, r, c] else 0
            o |= bit if obs[1, r, c] else 0
    rets = st.returns()
    oc = 2 if not st.is_terminal() else 0 if rets[0] > 0 else 1 if rets[1] > 0 else 3
    return struct.pack("<QQ", x | (oc ^ 2) << 62, o)


@pytest.mark.parametrize("gs,rows,cols", [("connect_four", 6, 7), ("connect_four(rows=7,columns=7)", 7, 7)])
def test_state_get_set_at_tile_edges(gs, rows, cols):
    n = 77
    game, batch, states = random_play(gs, n, 30, seed=11)
    edges = [0, 31, 32, 33, n - 1]
    for i in edges:
        assert batch.state_blob(i) == expected_blob(states[i], rows, cols), (gs, i)
    # set: lanes of a fresh batch take the blobs of other lanes; only those lanes change
    fresh = game.new_batch(n)
    start = fresh.state_blob(0)
    src = {lane: (lane * 7 + 3) % n for lane in edges}
    for lane, s in src.items():
        fresh.set_state_blob(lane, batch.state_blob(s))
    cur, term, rets = fresh.status()
    obs = fresh.observation_tensor(0).cpu().numpy()
    legal = fresh.legal_actions_mask().cpu().numpy()
    for lane in range(n):
        st = states[src[lane]] if lane in src else OracleGame(gs).new_initial_state()
        assert fresh.state_blob(lane) == (batch.state_blob(src[lane]) if lane in src else start), (gs, lane)
        assert int(cur[lane]) == st.current_player() and bool(term[lane]) == st.is_terminal(), (gs, lane)
        assert rets[lane].tolist() == st.returns(), (gs, lane)
        np.testing.assert_array_equal(obs[lane], st.observation_tensor(0))
        assert np.nonzero(legal[lane])[0].tolist() == st.legal_actions(), (gs, lane)


@pytest.mark.parametrize("gs", BOARDS)
def test_copy_between_unaligned_ranges(gs):
    game, src, states = random_play(gs, 100, 25, seed=5)
    dst = game.new_batch(90)
    blank = dst.state_blob(0)
    dst.copy_from(src, src_begin=5, dst_begin=37, count=41)
    assert dst.error_count()[0] == 0
    for lane in range(90):
        want = src.state_blob(lane - 32) if 37 <= lane < 78 else blank
        assert dst.state_blob(lane) == want, (gs, lane)
    cur, term, _ = dst.status()
    for lane in range(37, 78):
        assert int(cur[lane]) == states[lane - 32].current_player(), (gs, lane)


CHUNKED_STEP = r"""
import sys, numpy as np, torch
sys.path.insert(0, sys.argv[1])
import open_spiel_b200 as b2
game = b2.load_game(sys.argv[2])
n = int(sys.argv[3])
host, dev = game.new_batch(n), game.new_batch(n)
A, W, P = game.num_distinct_actions(), host.info.mask_words, game.num_players()
g = torch.Generator(device="cuda").manual_seed(1)
mask = dev.legal_actions_mask_words()
a_h = torch.empty(n, dtype=torch.int32).pin_memory()
m_h = torch.empty((n, W), dtype=torch.int32).pin_memory()
t_h = torch.empty(n, dtype=torch.uint8).pin_memory()
r_h = torch.empty((n, P), dtype=torch.float32).pin_memory()
for step in range(12):
    bits = (mask[:, :1] >> torch.arange(A, device="cuda", dtype=torch.int32)) & 1
    score = torch.rand((n, A), generator=g, device="cuda") * bits
    acts = torch.where(bits.any(1), score.argmax(1).to(torch.int32), torch.full((n,), -1, dtype=torch.int32, device="cuda"))
    acts[step::97] = -1                               # some lanes sit a step out
    a_h.copy_(acts.cpu())
    host.step_host(a_h, m_h, t_h, r_h)
    mask, term, rets = dev.step(acts)
    torch.cuda.synchronize()
    assert torch.equal(m_h, mask.cpu()) and torch.equal(t_h, term.cpu()) and torch.equal(r_h, rets.cpu()), step
assert host.error_count()[0] == 0 and dev.error_count()[0] == 0
for lane in (0, 31, 32, 1023, 1024, n // 3, n // 2 + 1, n - 1):
    assert host.state_blob(lane) == dev.state_blob(lane), lane
print("ok")
"""


@pytest.mark.parametrize("gs", BOARDS)
def test_chunked_host_step_equals_device_step(gs, tmp_path):
    # B2S_HOST_CHUNKS is read once per process: a child process steps in 3 chunks, each on a sub-range view of the batch
    script = tmp_path / "chunked.py"
    script.write_text(CHUNKED_STEP)
    env = dict(os.environ, B2S_HOST_CHUNKS="3")
    r = subprocess.run([sys.executable, str(script), ROOT, gs, str((1 << 18) + 4133)], capture_output=True, text=True,
                       env=env, timeout=600)
    assert r.returncode == 0 and r.stdout.strip().endswith("ok"), r.stdout + r.stderr


@pytest.mark.parametrize("gs", BOARDS)
def test_both_key_layouts_against_the_oracle(gs):
    assert lockstep(gs, n_lanes=77, seed=21, check_obs_every=1) > 0
    game, og = b2.load_game(gs), OracleGame(gs)
    n = 77
    batch = game.new_batch(n)
    tr = batch.record_trajectories(0x5EED, lane_offset=3)
    assert batch.error_count()[0] == 0
    actions, lengths, obs = tr.actions.cpu().numpy(), tr.lengths.cpu().numpy(), tr.observations.cpu().numpy()
    legal, rewards = tr.legal_actions().cpu().numpy(), tr.rewards.cpu().numpy()
    T = game.max_game_length()
    init = og.new_initial_state()
    for i in range(n):
        o = oracle_record_trajectory(init, 0x5EED, 3 + i, T)
        assert lengths[i] == o["length"] and np.array_equal(actions[i], o["actions"]), (gs, i)
        assert np.array_equal(legal[i], o["legal_actions"]) and np.array_equal(obs[i], o["observations"]), (gs, i)
        assert np.array_equal(rewards[i].astype(np.float64), o["rewards"]), (gs, i)
