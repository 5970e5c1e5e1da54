"""GPU: go on boards 10..19 (the 384-bit rule core, with handicap stones) on the device, bit for bit against the oracle — the
batched state functions through whole games, lane blobs, b2s_rollout, the trajectory recorder, both MCTS searches (16- and
24-byte nodes, garbage collection; PUCT, caller noise and a node budget for the evaluated one) — and, where oracle/_ref is
built, against the unmodified reference in lock-step."""
import numpy as np
import pytest
import torch

import open_spiel_b200 as b2
import ref_lib
from oracle_lib import OracleGame
from parity import lockstep
from philox_ref import philox_uniform

pytestmark = pytest.mark.gpu

LOCKSTEP = [("go(board_size=13)", 24), ("go(board_size=19)", 12), ("go(board_size=16,komi=0.5)", 12),
            ("go(board_size=19,handicap=4)", 12), ("go(board_size=19,handicap=9,max_game_length=120)", 16), ("go", 8)]


@pytest.mark.parametrize("gs,lanes", LOCKSTEP, ids=[g for g, _ in LOCKSTEP])
def test_device_state_functions_equal_oracle(gs, lanes):
    """apply / step / status / legal mask and list / observation tensors, played to the end of every game."""
    assert lockstep(gs, n_lanes=lanes, seed=19, check_obs_every=2) > lanes * 100


@pytest.mark.parametrize("gs,lanes", [("go(board_size=13)", 12), ("go(board_size=19)", 6), ("go(board_size=19,handicap=3)", 6)])
def test_device_equals_unmodified_reference(gs, lanes):
    if not ref_lib.available():
        pytest.skip("oracle/_ref not built")
    assert lockstep(gs, n_lanes=lanes, seed=23, check_obs_every=4, checker=ref_lib.RefGame) > lanes * 50


def test_lane_blobs_round_trip_mid_game():
    """b2s_state_get / b2s_state_set: 112 state bytes plus the superko history move a 19x19 lane to another batch, which then
    plays on exactly like the original (including repetition detection against the copied history)."""
    gs, n = "go(board_size=19,handicap=2)", 64
    game = b2.load_game(gs)
    a, b = game.new_batch(n), game.new_batch(n)
    assert a.info.state_bytes == 112
    rng = np.random.RandomState(2)
    for _ in range(150):
        m = a.legal_actions_mask_words().cpu().numpy()
        bits = ((m[:, :, None] >> np.arange(32, dtype=np.uint32)) & 1).reshape(n, -1)[:, :game.num_distinct_actions()]
        acts = np.array([rng.choice(np.flatnonzero(r)) if r.any() else -1 for r in bits], dtype=np.int32)
        a.apply_actions(torch.from_numpy(acts).cuda())
    for i in range(n):
        blob = a.state_blob(i)
        b.set_state_blob(i, blob)
        assert b.state_blob(i) == blob
    for x, y in zip(a.status(), b.status()):
        assert torch.equal(x, y)
    assert torch.equal(a.legal_actions_mask_words(), b.legal_actions_mask_words())
    assert torch.equal(a.observation_tensor(0), b.observation_tensor(0))
    ra, pa = a.rollout(seed=77)
    rb, pb = b.rollout(seed=77)
    assert torch.equal(ra, rb) and torch.equal(pa, pb)


@pytest.mark.parametrize("gs,n", [("go(board_size=13)", 1 << 14), ("go(board_size=19)", 1 << 13), ("go(board_size=19,handicap=6)", 4096)])
def test_device_rollout_equals_oracle(gs, n):
    """b2s_rollout on the Philox stream: every lane's length and returns; a sample of lanes replayed by the oracle on the same
    stream (candidate rejection sampling), the rest checked for the properties every game has."""
    game = b2.load_game(gs)
    batch = game.new_batch(n)
    rets, plies = batch.rollout(seed=0x60, lane_offset=100)
    rets, plies = rets.cpu().numpy(), plies.cpu().numpy()
    assert bool(batch.status()[1].all()) and int(plies.min()) >= 2 and int(plies.max()) <= game.max_game_length()
    assert (rets.sum(axis=1) == 0).all()
    og = OracleGame(gs)
    for i in list(range(0, n, n // 6)) + [n - 1]:
        st = og.new_initial_state()
        ply = 0
        while not st.is_terminal():
            la, cand = st.legal_actions(), st.rollout_candidates()
            retry = 0
            while True:
                a = cand[philox_uniform(0x60, 100 + i, ply + 4096 * retry, len(cand))]
                if a in la:
                    break
                retry += 1
            st.apply_action(a)
            ply += 1
        assert ply == plies[i] and st.returns() == rets[i].tolist(), (gs, i)


@pytest.mark.parametrize("gs,n", [("go(board_size=13)", 12), ("go(board_size=19)", 6), ("go(board_size=19,handicap=2)", 4)])
def test_device_recorder_equals_oracle_recorder(gs, n):
    from test_gpu_trajectories import test_device_recorder_equals_oracle_recorder as recorder
    recorder(gs, n, 0)


# game, trees, prefix plies, sims, n_rollouts, solve, PUCT, node budget (max_memory_mb = 1 -> 13108 nodes)
MCTS = [("go(board_size=13)", 24, 12, 60, 1, True, False, 0), ("go(board_size=19)", 16, 10, 40, 1, True, False, 0),
        ("go(board_size=19)", 8, 6, 30, 3, False, False, 0), ("go(board_size=19,handicap=5)", 8, 4, 40, 1, True, True, 0),
        ("go(board_size=13)", 8, 6, 30, 2, True, True, 0),
        ("go(board_size=19)", 4, 4, 480, 1, True, False, 13108), ("go(board_size=13)", 4, 4, 400, 1, False, True, 13108)]


@pytest.mark.parametrize("gs,n,prefix,sims,nroll,solve,puct,budget", MCTS,
                         ids=["%s-%d-%d%s%s" % (c[0], c[3], c[4], "-puct" if c[6] else "", "-gc" if c[7] else "") for c in MCTS])
def test_device_mcts_equals_oracle(gs, n, prefix, sims, nroll, solve, puct, budget):
    from test_gpu_mcts import _check_against_oracle
    collections = _check_against_oracle(gs, n, prefix, sims, nroll, solve, puct, budget)
    if budget:
        assert collections >= n


EVAL = [("go(board_size=13)", 16, 8, 60, True, True, 0, 0.0), ("go(board_size=19)", 8, 6, 40, False, True, 0, 0.03),
        ("go(board_size=19,handicap=4)", 8, 4, 40, True, False, 0, 0.3), ("go(board_size=19)", 4, 2, 1000, True, True, 13108, 0.0)]


@pytest.mark.parametrize("gs,n,prefix,sims,solve,puct,budget,alpha", EVAL,
                         ids=["%s-%d%s%s%s" % (c[0], c[3], "-puct" if c[5] else "", "-gc" if c[6] else "", "-noise" if c[7] else "")
                              for c in EVAL])
def test_device_evaluated_mcts_equals_oracle(gs, n, prefix, sims, solve, puct, budget, alpha):
    from test_gpu_mcts_eval import test_device_evaluated_mcts_equals_oracle as evaluated
    evaluated(gs, n, prefix, sims, solve, puct, budget, alpha)
