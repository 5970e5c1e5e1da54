"""Restatement of the reference's RL environment (python/rl_environment.py Environment.reset / step / get_time_step and
python/vector_env.py SyncVectorEnv.step) over the CPU oracle's OracleGame / OracleState, with chance outcomes drawn from
the Philox stream b2s_env_step uses (include/b2s.h), plus the batch API's extensions: action -1 leaves a lane untouched
and an illegal action is counted and leaves the lane as it was.  The device env (b2s_env_*) must equal it lane by lane;
tests/test_env_reference.py pins it to the reference's own Environment code.  Test infrastructure."""
import numpy as np

from oracle_lib import OracleGame
from philox_ref import philox_uniform

FIRST, MID, LAST = 0, 1, 2


def block(c):
    """Random block of the call with counter c (include/b2s.h): chance node j after the action takes block(c) + 1 + j,
    after a reset block(c) + 32 + j."""
    return (64 * (c + 1)) & 0xFFFFFFFF


class PhiloxChanceSampler:
    """A chance_event_sampler for rl_environment.Environment (its ChanceEventSampler interface, rl_environment.py:
    135-150): the j-th chance node since `start(b)` takes the philox_uniform(seed, lane, b + j, #outcomes)-th outcome in
    ascending action order, as draw_legal takes the k-th set bit of the chance node's legal mask."""

    def __init__(self, seed, lane):
        self.seed, self.lane, self.b, self.j = seed, lane, 0, 0

    def start(self, b):
        self.b, self.j = b, 0

    def __call__(self, state):
        outcomes = sorted(a for a, _ in state.chance_outcomes())
        k = philox_uniform(self.seed, self.lane, (self.b + self.j) & 0xFFFFFFFF, len(outcomes))
        self.j += 1
        return outcomes[k]


class Env:
    """rl_environment.Environment (turn-based games) over an OracleGame."""

    def __init__(self, game, sampler, use_observation):
        self.game, self.sampler, self.use_observation = game, sampler, use_observation
        self.state, self.should_reset = None, True          # rl_environment.py:222-223
        self.P = game.num_players

    def _sample_external_events(self):                     # rl_environment.py:431-442
        while self.state.is_chance_node():
            self.state.apply_action(self.sampler(self.state))

    def _observation(self):
        st = self.state
        tensors = [st.observation_tensor(p) if self.use_observation else st.information_state_tensor(p) for p in range(self.P)]
        cur = st.current_player()
        legal = np.zeros(self.game.num_distinct_actions, dtype=bool)
        if cur >= 0:                                         # legal_actions(p) is empty but for the player to move
            legal[st.legal_actions()] = True
        return np.stack(tensors), legal, cur

    def get_time_step(self):                               # rl_environment.py:261-310
        step_type = LAST if self.state.is_terminal() else MID
        self.should_reset = step_type == LAST
        rewards = np.array(self.state.returns() if self.state.is_terminal() else [0.0] * self.P, dtype=np.float32)
        return self._observation() + (rewards, step_type)

    def reset(self, b):                                    # rl_environment.py:399-420 (rewards None -> 0)
        self.should_reset = False
        self.state = self.game.new_initial_state()
        self.sampler.start(b + 32)
        self._sample_external_events()
        return self._observation() + (np.zeros(self.P, dtype=np.float32), FIRST)

    def step(self, action, b):
        """Environment.step (rl_environment.py:337-383) plus the batch API's -1 and illegal-action conventions.  Returns
        (time step, illegal)."""
        if self.should_reset:
            return self.reset(b), False
        if action == -1:
            return self.get_time_step(), False
        if action not in self.state.legal_actions():
            return self.get_time_step(), True
        self.state.apply_action(int(action))
        self.sampler.start(b + 1)
        self._sample_external_events()
        return self.get_time_step(), False


class VectorEnv:
    """SyncVectorEnv (vector_env.py:18-80) of `n` Envs; lane i samples chance with lane index lane_offset + i.  Each
    reset() / step() returns dict(obs [n, P, F], mask [n, A] bool, cur [n], rewards [n, P], done [n], step_type [n]) and
    counts illegal actions in .errors."""

    def __init__(self, game_string, n, seed=0, lane_offset=0, observation_type=None, lanes=None):
        """lanes: the lane indices to keep (default range(n)), for checking a sample of a large batch."""
        self.game = OracleGame(game_string)
        has_info = self.game.information_state_tensor_size > 0
        use_observation = observation_type == "OBSERVATION" or (observation_type is None and not has_info)
        lanes = range(n) if lanes is None else lanes
        self.envs = [Env(self.game, PhiloxChanceSampler(seed, lane_offset + int(i)), use_observation) for i in lanes]
        self.c, self.errors = 0, 0

    def _stack(self, steps, done):
        obs, mask, cur, rewards, step_type = zip(*steps)
        return {"obs": np.stack(obs), "mask": np.stack(mask), "cur": np.array(cur, dtype=np.int8),
                "rewards": np.stack(rewards), "done": np.array(done, dtype=np.uint8), "step_type": np.array(step_type, dtype=np.uint8)}

    def reset(self):
        b = block(self.c)
        self.c += 1
        steps = [e.reset(b) for e in self.envs]
        return self._stack(steps, [0] * len(steps))

    def step(self, actions, reset_if_done=False):
        b = block(self.c)
        self.c += 1
        steps = []
        for e, a in zip(self.envs, actions):
            ts, illegal = e.step(int(a), b)
            self.errors += int(illegal)
            steps.append(ts)
        done = [int(ts[4] == LAST) for ts in steps]          # vector_env.py:56: step.last()
        rewards = [ts[3] for ts in steps]
        if reset_if_done:                                    # vector_env.py:62-63: SyncVectorEnv.reset(envs_to_reset=done)
            steps = [e.reset(b) if d else ts for e, d, ts in zip(self.envs, done, steps)]
        out = self._stack(steps, done)
        out["rewards"] = np.stack(rewards)
        return out


# ---- the runs tests/test_env_reference.py compares with the reference's Environment and pins in
# ---- tests/golden/env_reference.json (tests/golden/make_env_reference.py) ------------------------------------------
REFERENCE_GAMES = ["kuhn_poker", "kuhn_poker(players=3)", "leduc_poker", "leduc_poker(players=3)", "tic_tac_toe", "connect_four",
                   "hex(board_size=5)", "go(board_size=5)"]
REFERENCE_N, REFERENCE_STEPS, REFERENCE_SEED = 64, 200, 0xC0FFEE


def reference_cases():
    """(game, observation_type, reset_if_done): both observation types where the game has an information state tensor."""
    out = []
    for gs in REFERENCE_GAMES:
        kinds = ["INFORMATION_STATE", "OBSERVATION"] if gs.startswith(("kuhn", "leduc")) else ["OBSERVATION"]
        out += [(gs, kind, rid) for kind in kinds for rid in (False, True)]
    return out


def case_id(case):
    return "%s-%s-%s" % (case[0], case[1].lower(), "reset_if_done" if case[2] else "no_reset")


def run_calls(reset, step, n, steps, seed, reset_if_done):
    """reset() then `steps` step(actions, reset_if_done) calls, the actions uniformly random legal ones of the previous
    time step (0 for a lane at LAST, which ignores it) from numpy's RandomState(seed); yields every call's dict."""
    rng = np.random.RandomState(seed & 0xFFFFFFFF)
    ts = reset()
    yield ts
    for _ in range(steps):
        acts = np.array([rng.choice(np.flatnonzero(m)) if m.any() else 0 for m in ts["mask"]], dtype=np.int32)
        ts = step(acts, reset_if_done)
        yield ts


def digest(calls):
    import hashlib
    h = hashlib.sha256()
    for ts in calls:
        for k in ("obs", "mask", "cur", "rewards", "done", "step_type"):
            h.update(np.ascontiguousarray(ts[k]).tobytes())
    return h.hexdigest()
