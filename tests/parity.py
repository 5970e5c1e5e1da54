"""Lock-step parity harness: CUDA batch (through the C ABI) vs the CPU oracle on the same seeded inputs.

Mirrors the reference's RandomSimTest (tests/basic_tests.cc:321-581): play random games to the end and check
every observable after every move — here with the oracle supplying the expected values.
"""
import hashlib

import numpy as np
import torch

import open_spiel_b200 as b2
from oracle_lib import OracleGame


def mask_words_to_lists(words, width):
    """[n, W] int32 words -> list of ascending action lists."""
    w = words.cpu().numpy().astype(np.uint32)
    n = w.shape[0]
    bits = ((w[:, :, None] >> np.arange(32, dtype=np.uint32)) & 1).reshape(n, -1)[:, :width]
    return [np.nonzero(row)[0].tolist() for row in bits]


def absorb(h, cur, term, legal, rets, obs=None, ist=None):
    """Feeds what one lane shows at one ply into the sha256 object h: player to move, terminal flag, legal actions,
    returns (float64, sign of zero included) and, when checked at that ply, the observation / information-state tensor of
    every player (float32)."""
    h.update(np.array([int(cur), int(bool(term)), len(legal)] + list(legal), dtype=np.int64).tobytes())
    h.update(np.asarray(rets, dtype=np.float64).tobytes())
    for t in (obs or []) + (ist or []):
        h.update(np.asarray(t, dtype=np.float32).tobytes())


def games_digest(hashes):
    """The digest stored per game in tests/golden/reference_results.json: sha256 over the lanes' sha256 digests in order."""
    return hashlib.sha256("".join(h.hexdigest() for h in hashes).encode()).hexdigest()


def checker_digests(game_string, n_lanes, seed, checker, check_obs_every=3, check_info_state=False):
    """The games lockstep() plays, on the scalar checker alone (no device): same random actions, same observables fed
    to absorb() in the same order; returns games_digest().  Used to record the reference's digest."""
    rng = np.random.RandomState(seed)
    game = checker(game_string)
    states = [game.new_initial_state() for _ in range(n_lanes)]
    hashes = [hashlib.sha256() for _ in range(n_lanes)]
    P, ply = game.num_players, 0
    while True:
        check_obs = check_obs_every and ply % check_obs_every == 0
        alive = 0
        for i, st in enumerate(states):
            ola = st.legal_actions()
            absorb(hashes[i], st.current_player(), st.is_terminal(), ola, st.returns(),
                   [st.observation_tensor(p) for p in range(P)] if check_obs else None,
                   [st.information_state_tensor(p) for p in range(P)] if check_obs and check_info_state else None)
            if not st.is_terminal():
                st.apply_action(ola[rng.randint(len(ola))])
                alive += 1
        if alive == 0:
            return games_digest(hashes)
        ply += 1


def lockstep(game_string, n_lanes=512, seed=0, check_obs_every=3, max_plies=None, check_info_state=False,
             checker=OracleGame, hashes=None):
    """Play n_lanes random games in lock-step on device and on the checker (the oracle restatement, or — passing
    ref_lib.RefGame — the unmodified reference build); assert equality of everything after every move.  hashes: a list
    of n_lanes sha256 objects that absorb() what each device lane showed (compare with checker_digests())."""
    rng = np.random.RandomState(seed)
    game = b2.load_game(game_string)
    ogame = checker(game_string)
    assert game.num_distinct_actions() == ogame.num_distinct_actions
    assert game.max_game_length() == ogame.max_game_length
    assert game.num_players() == ogame.num_players
    assert game.observation_tensor_size() == ogame.observation_tensor_size
    batch = game.new_batch(n_lanes)
    ostates = [ogame.new_initial_state() for _ in range(n_lanes)]
    width = max(game.num_distinct_actions(), game.max_chance_outcomes())
    P = game.num_players()
    dev = batch._dev
    ply = 0
    total_steps = 0
    limit = max_plies or (game.max_game_length() + 8)
    while True:
        cur, term, rets = batch.status()
        cur, term, rets = cur.cpu().numpy(), term.cpu().numpy(), rets.cpu().numpy()
        legal = mask_words_to_lists(batch.legal_actions_mask_words(), width)
        acts_l, counts = batch.legal_actions_list()
        acts_l, counts = acts_l.cpu().numpy(), counts.cpu().numpy()
        obs = None
        if check_obs_every and ply % check_obs_every == 0:
            obs = [batch.observation_tensor(p).cpu().numpy() for p in range(P)]
            ist = [batch.information_state_tensor(p).cpu().numpy() for p in range(P)] if check_info_state else None
        actions = np.full(n_lanes, -1, dtype=np.int32)
        alive = 0
        for i, st in enumerate(ostates):
            if hashes is not None:
                absorb(hashes[i], cur[i], term[i], legal[i], rets[i], [o[i] for o in obs] if obs is not None else None,
                       [t[i] for t in ist] if obs is not None and check_info_state else None)
            assert int(cur[i]) == st.current_player(), (game_string, "current_player", i, ply)
            assert bool(term[i]) == st.is_terminal(), (game_string, "is_terminal", i, ply)
            ola = st.legal_actions()
            assert legal[i] == ola, (game_string, "legal", i, ply, legal[i], ola, st.to_string())
            assert counts[i] == len(ola) and acts_l[i, :len(ola)].tolist() == ola
            orets = st.returns()
            assert rets[i].tolist() == orets, (game_string, "returns", i, ply, rets[i], orets)
            assert np.array_equal(np.signbit(rets[i]), np.signbit(np.array(orets))), (game_string, "sign of zero")
            if obs is not None:
                for p in range(P):
                    np.testing.assert_array_equal(obs[p][i], st.observation_tensor(p),
                                                  err_msg="%s obs lane %d ply %d player %d\n%s" % (game_string, i, ply, p, st.to_string()))
                    if check_info_state:
                        np.testing.assert_array_equal(ist[p][i], st.information_state_tensor(p))
            if not st.is_terminal():
                a = ola[rng.randint(len(ola))]
                actions[i] = a
                st.apply_action(a)
                alive += 1
        if alive == 0:
            break
        total_steps += alive
        # alternate between the plain and the fused entry point
        a_d = torch.from_numpy(actions).to(dev)
        if ply % 2 == 0:
            batch.apply_actions(a_d)
        else:
            m, t, r = batch.step(a_d)
            # fused outputs must equal the separate calls made at the top of the next iteration
            cur2, term2, rets2 = batch.status()
            assert torch.equal(t, term2) and torch.equal(r, rets2)
            assert torch.equal(m, batch.legal_actions_mask_words())
        cnt, first = batch.error_count()
        assert cnt == 0, (game_string, "unexpected rejected lanes", cnt, first)
        ply += 1
        assert ply <= limit, "game did not end"
    return total_steps
