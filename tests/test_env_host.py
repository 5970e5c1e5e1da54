"""CPU rehearsal of the device RL environment: the per-lane body of k_env_step (open_spiel_b200/csrc/env_step.cuh), compiled
for the host by tests/host_emul/emul_env.cc over the product's rule cores, stepped lock-step with the restatement of
rl_environment.Environment / SyncVectorEnv (tests/env_lib.py).  Every output of every call must be equal: observations of
every player, legal mask, rewards, done, step type, current player and the illegal-action count."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import env_lib
import open_spiel_b200 as b2

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMUL = os.path.join(ROOT, "tests", "host_emul")
SO = os.path.join(EMUL, "libemul_env.so")

GAMES = ["tic_tac_toe", "connect_four", "connect_four(rows=4,columns=5,x_in_row=3)", "breakthrough(rows=6,columns=6)",
         "hex(board_size=5)", "hex(board_size=5,swap=True)", "go(board_size=5)", "go(board_size=13)", "go(board_size=19,handicap=4)",
         "kuhn_poker", "kuhn_poker(players=3)", "leduc_poker", "leduc_poker(players=3)", "othello", "mnk(m=5,n=5,k=4)",
         "y(board_size=7)", "havannah(board_size=4,swap=True)"]


def _lib():
    if not os.path.isdir("/usr/local/cuda/include"):
        pytest.skip("CUDA headers not available for the host build of the rule cores")
    if not os.path.exists(SO):
        subprocess.check_call(["make", "-s", "-C", EMUL, "-f", "env.mk"])
    L = C.CDLL(SO)
    L.emu_env_create.restype = C.c_void_p
    L.emu_env_create.argtypes = [C.c_int, C.c_void_p, C.c_longlong, C.c_ulonglong, C.c_longlong, C.c_int]
    L.emu_env_destroy.argtypes = [C.c_void_p]
    L.emu_env_call.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_longlong] + [C.c_void_p] * 6
    L.emu_env_error_count.restype = C.c_longlong
    L.emu_env_error_count.argtypes = [C.c_void_p]
    L.emu_env_last_error.restype = C.c_char_p
    return L


class HostEnv:
    """The emulated b2s_env_* over n lanes; call(actions or None, reset_if_done) returns env_lib's dict layout."""

    def __init__(self, gs, n, seed, lane_offset, observation):
        self.L, self.game, self.n = _lib(), b2.load_game(gs), n
        self.h = self.L.emu_env_create(self.game._gid, C.addressof(self.game._cparams), n, seed, lane_offset, observation)
        assert self.h, self.L.emu_env_last_error()
        info = self.game._info
        which = observation if observation >= 0 else (1 if info.information_state_tensor_size > 0 else 0)
        self.F = info.information_state_tensor_size if which else info.observation_tensor_size
        self.P, self.A, self.W = info.num_players, info.num_distinct_actions, info.mask_words

    def __del__(self):
        if getattr(self, "h", None):
            self.L.emu_env_destroy(self.h)

    def call(self, actions=None, reset_if_done=False):
        n, P = self.n, self.P
        obs = np.zeros((P, n, self.F), np.float32)
        words = np.zeros((n, self.W), np.uint32)
        rew, done = np.zeros((n, P), np.float32), np.zeros(n, np.uint8)
        st, cur = np.zeros(n, np.uint8), np.zeros(n, np.int8)
        a = None if actions is None else np.ascontiguousarray(actions, dtype=np.int32)
        self.L.emu_env_call(self.h, None if a is None else a.ctypes.data, int(reset_if_done), n,
                            *[x.ctypes.data for x in (obs, words, rew, done, st, cur)])
        bits = ((words[:, :, None] >> np.arange(32, dtype=np.uint32)) & 1).reshape(n, -1)[:, :self.A].astype(bool)
        return {"obs": obs.transpose(1, 0, 2), "mask": bits, "cur": cur, "rewards": rew, "done": done, "step_type": st}

    def errors(self):
        return self.L.emu_env_error_count(self.h)


def assert_same(got, want, where):
    for k in ("obs", "mask", "cur", "rewards", "done", "step_type"):
        assert np.array_equal(got[k], want[k]), (where, k, np.argwhere(np.asarray(got[k] != want[k]))[:4].tolist())


def sample_actions(rng, mask, p_skip=0.0, p_illegal=0.0, A=None):
    """A uniformly random legal action per lane (0 where none: a LAST lane ignores it), some -1, some illegal."""
    acts = np.zeros(len(mask), np.int32)
    for i, m in enumerate(mask):
        legal = np.flatnonzero(m)
        if len(legal):
            acts[i] = rng.choice(legal)
            u = rng.rand()
            if u < p_skip:
                acts[i] = -1
            elif u < p_skip + p_illegal:
                illegal = np.flatnonzero(~m[:A])
                if len(illegal):
                    acts[i] = rng.choice(illegal)
    return acts


@pytest.mark.parametrize("gs", GAMES)
@pytest.mark.parametrize("reset_if_done", [False, True])
def test_emulated_env_step_equals_restatement(gs, reset_if_done):
    n, steps, seed, off = 12, 40, 0x5EED, 77
    game = b2.load_game(gs)
    obs_kinds = [-1, 0] + ([1] if game.information_state_tensor_size() > 0 else [])
    for observation in obs_kinds:
        dev = HostEnv(gs, n, seed, off, observation)
        ref = env_lib.VectorEnv(gs, n, seed, off, {-1: None, 0: "OBSERVATION", 1: "INFORMATION_STATE"}[observation])
        rng = np.random.RandomState(len(gs) + observation)
        got, want = dev.call(), ref.reset()
        assert_same(got, want, (gs, observation, "reset"))
        for t in range(steps):
            acts = sample_actions(rng, want["mask"], p_skip=0.1, p_illegal=0.05, A=dev.A)
            got, want = dev.call(acts, reset_if_done), ref.step(acts, reset_if_done)
            assert_same(got, want, (gs, observation, t))
            assert dev.errors() == ref.errors
        want = ref.reset()                                    # Environment.reset mid-episode
        assert_same(dev.call(), want, (gs, observation, "reset again"))
        for t in range(5):
            acts = sample_actions(rng, want["mask"])
            got, want = dev.call(acts, reset_if_done), ref.step(acts, reset_if_done)
            assert_same(got, want, (gs, observation, "after reset", t))
