"""GPU: every accepted variant of tests/param_edges.py (each rule core's parameter range, sampled where the packed layouts change
code path) through the device kernels against the oracle, and every shape past a limit refused.  Per variant: lock-step random
games on a ragged batch (status, legal mask and list, apply and the fused step, observation and information-state tensors),
b2s_rollout against an oracle replay of the same Philox stream, mid-game state blobs round-tripped and cloned by copy_from and
b2s_gather_states, and b2s_observation into a buffer that starts one float past an aligned address.  Per deterministic game, a
small MCTS and a budgeted AlphaBetaSearch on its layout edges and at the longest game the search's path stack holds."""
import ctypes as C

import numpy as np
import pytest
import torch

import alpha_beta_lib as ab
import open_spiel_b200 as b2
from open_spiel_b200 import _lib
from oracle_lib import OracleGame
from param_edges import ACCEPTED, INFO_STATE, MCTS_REJECTED, REJECTED, SEARCH, SEARCH_REJECTED, BoardTextOracle, raw_params
from parity import lockstep, mask_words_to_lists
from philox_ref import philox_uniform
from test_gpu_alpha_beta import check_against_oracle, make_batch, results
from test_gpu_mcts import _check_against_oracle, make_roots

pytestmark = pytest.mark.gpu

IDS = [g for g, _ in ACCEPTED]


@pytest.mark.parametrize("gs,lanes", ACCEPTED, ids=IDS)
def test_lockstep_at_layout_edges(gs, lanes):
    assert lockstep(gs, n_lanes=lanes, seed=77, check_info_state=gs in INFO_STATE, checker=BoardTextOracle) >= lanes


@pytest.mark.parametrize("gs,lanes", ACCEPTED, ids=IDS)
def test_rollout_at_layout_edges(gs, lanes):
    """b2s_rollout from the initial state; sampled lanes replayed by the oracle on the same Philox words."""
    b = b2.load_game(gs).new_batch(lanes)
    rets, plies = (t.cpu().numpy() for t in b.rollout(seed=0xED6E, lane_offset=5000))
    og = OracleGame(gs)
    for i in range(0, lanes, max(1, lanes // 16)):
        st, ply = og.new_initial_state(), 0
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
        assert ply == plies[i] and st.returns() == rets[i].tolist(), (gs, i)
    _, term, rets2 = b.status()
    assert term.all() and np.array_equal(rets2.cpu().numpy(), rets)


def _assert_lanes(batch, states, lanes, what):
    """Lanes `lanes` of batch show the oracle states: status, legal mask, every player's tensors."""
    g = batch.game
    width = max(g.num_distinct_actions(), g.max_chance_outcomes())
    n = max(lanes) + 1
    cur, term, rets = (t.cpu().numpy() for t in batch.status(n=n))
    legal = mask_words_to_lists(batch.legal_actions_mask_words(n=n), width)
    P = g.num_players()
    obs = [batch.observation_tensor(p, n=n).cpu().numpy() for p in range(P)]
    ist = [batch.information_state_tensor(p, n=n).cpu().numpy() for p in range(P)] if g.information_state_tensor_size() else None
    for lane, st in zip(lanes, states):
        assert (int(cur[lane]), bool(term[lane])) == (st.current_player(), st.is_terminal()), (what, lane)
        assert legal[lane] == st.legal_actions() and rets[lane].tolist() == st.returns(), (what, lane)
        for p in range(P):
            np.testing.assert_array_equal(obs[p][lane], st.observation_tensor(p), err_msg="%s lane %d" % (what, lane))
            if ist is not None:
                np.testing.assert_array_equal(ist[p][lane], st.information_state_tensor(p), err_msg="%s lane %d" % (what, lane))


@pytest.mark.parametrize("gs,lanes", ACCEPTED, ids=IDS)
def test_state_blobs_and_clones_at_layout_edges(gs, lanes):
    """Mid-game lanes (tall connect_four columns included) through b2s_state_get / b2s_state_set, b2s_copy_states and
    b2s_gather_states: every copy shows the oracle's state, and a blob read back is the blob written."""
    game, src, states = make_roots(gs, lanes, b2.load_game(gs).max_game_length(), seed=lanes)
    rng = np.random.RandomState(len(gs))
    blobs = [src.state_blob(i) for i in range(lanes)]
    dst = game.new_batch(lanes)
    for i in rng.permutation(lanes):
        dst.set_state_blob(int(i), blobs[i])
    assert [dst.state_blob(i) for i in range(lanes)] == blobs
    _assert_lanes(dst, states, range(lanes), "state_set")
    cp = game.new_batch(lanes + 40)
    cp.copy_from(dst, src_begin=3, dst_begin=29, count=lanes - 3)
    _assert_lanes(cp, states[3:], range(29, 26 + lanes), "copy_states")
    _assert_lanes(cp, [OracleGame(gs).new_initial_state()] * 29, range(29), "copy_states (untouched)")
    idx = rng.randint(0, lanes, size=lanes + 11)
    ga = game.new_batch(lanes + 11)
    idx_d = torch.from_numpy(idx.astype(np.int64)).cuda()
    _lib.check(_lib.lib().b2s_gather_states(ga._h, dst._h, C.c_void_p(idx_d.data_ptr()), len(idx), ga._stream()))
    _assert_lanes(ga, [states[i] for i in idx], range(len(idx)), "gather_states")
    for b in (dst, cp, ga):
        assert b.error_count()[0] == 0


@pytest.mark.parametrize("gs,lanes", ACCEPTED, ids=IDS)
def test_tensors_into_a_buffer_one_float_off(gs, lanes):
    """b2s_observation / b2s_information_state into a float buffer that starts 4 bytes past an aligned address: k_obs's
    scalar peel runs for every tensor size.  Same values as into an aligned buffer, and nothing written outside."""
    game, batch, _ = make_roots(gs, lanes, game_len_half(gs), seed=5)
    which = [(batch.observation_tensor, game.observation_tensor_size())]
    if game.information_state_tensor_size():
        which.append((batch.information_state_tensor, game.information_state_tensor_size()))
    for fn, F in which:
        for p in range(game.num_players()):
            want = fn(p)
            buf = torch.full((lanes * F + 2,), -7.0, dtype=torch.float32, device=batch._dev)
            out = buf[1:1 + lanes * F].view(lanes, F)
            fn(p, out=out)
            assert torch.equal(out, want), (gs, p)
            assert buf[0].item() == -7.0 and buf[-1].item() == -7.0


def game_len_half(gs):
    return max(1, b2.load_game(gs).max_game_length() // 2)


@pytest.mark.parametrize("gs,n,prefix,sims", SEARCH, ids=[c[0] for c in SEARCH])
def test_mcts_at_layout_edges(gs, n, prefix, sims):
    _check_against_oracle(gs, n, prefix, sims, 1, True, puct=False)


@pytest.mark.parametrize("gs,n,prefix,sims", SEARCH, ids=[c[0] for c in SEARCH])
def test_alpha_beta_at_layout_edges(gs, n, prefix, sims):
    """A budgeted search (most roots run out of nodes), and an unlimited one of depth 2."""
    roots = ab.random_roots(OracleGame(gs), n, (0, prefix), seed=n)
    batch = make_batch(gs, roots)
    check_against_oracle(gs, roots, results(b2.alpha_beta_search(batch, max_nodes=150)), max_nodes=150)
    check_against_oracle(gs, roots, results(b2.alpha_beta_search(batch, depth_limit=2, max_nodes=400)), depth=2, max_nodes=400)


@pytest.mark.parametrize("gs", MCTS_REJECTED)
def test_searches_refuse_games_past_their_path_stack(gs):
    batch = b2.load_game(gs).new_batch(4)
    with pytest.raises(b2.SpielError, match="mcts"):
        b2.mcts_search(batch, 10)
    if gs in SEARCH_REJECTED:
        with pytest.raises(b2.SpielError, match="alpha_beta"):
            b2.alpha_beta_search(batch, max_nodes=10)


@pytest.mark.parametrize("gs", REJECTED)
def test_shapes_past_a_limit_are_refused(gs):
    with pytest.raises(b2.SpielError):
        b2.load_game(gs)
    gid, cp = raw_params(gs)
    h = C.c_void_p()
    assert _lib.lib().b2s_batch_create(gid, C.byref(cp), 8, 0, C.byref(h)) != 0
    assert not h.value
