"""The restatement tests/env_lib.py (which the device RL environment must equal lane by lane) against the reference's own
python/rl_environment.py Environment and python/vector_env.py SyncVectorEnv, loaded by path from the OpenSpiel checkout
and run over the pyspiel-compatible module (open_spiel_b200/adapter) with a Philox chance_event_sampler: every TimeStep
field of every call, 64 envs x 200 steps, with and without reset_if_done.  The digests of those runs are pinned in
tests/golden/env_reference.json, which keeps env_lib checked where no checkout exists."""
import glob
import importlib.util
import json
import os
import sys

import numpy as np
import pytest

import env_lib
from __graft_entry__ import REFERENCE

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BUILD = os.path.join(ROOT, "open_spiel_b200", "adapter", "_build")
REF_PY = os.path.join(REFERENCE, "open_spiel", "python")
GOLDEN = json.load(open(os.path.join(ROOT, "tests", "golden", "env_reference.json")))
CASES = env_lib.reference_cases()


def _reference_modules():
    if not glob.glob(os.path.join(BUILD, "pyspiel*.so")) or not os.path.exists(os.path.join(REF_PY, "rl_environment.py")):
        pytest.skip("needs the OpenSpiel checkout and the pyspiel module built against it")
    if BUILD not in sys.path:
        sys.path.insert(0, BUILD)
    mods = []
    for name in ("rl_environment", "vector_env"):
        spec = importlib.util.spec_from_file_location("reference_" + name, os.path.join(REF_PY, name + ".py"))
        m = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(m)
        mods.append(m)
    return mods


class _StepOutput:
    def __init__(self, action):
        self.action = action


def reference_calls(gs, kind, reset_if_done):
    """The reference's SyncVectorEnv of Environments over the same random actions as env_lib.run_calls; each call's
    time steps in env_lib's dict layout (rewards None -> 0)."""
    rl, ve_mod = _reference_modules()
    import pyspiel
    n, seed = env_lib.REFERENCE_N, env_lib.REFERENCE_SEED

    class PhiloxEnvironment(rl.Environment):
        """Environment with the device's chance keying: reset() draws from block b + 32 + j, step() from b + 1 + j."""
        block = 0

        def reset(self):
            self._chance_event_sampler.start(self.block + 32)
            return super().reset()

        def step(self, actions):
            self._chance_event_sampler.start(self.block + 1)
            return super().step(actions)

    game = pyspiel.load_game(gs)
    envs = [PhiloxEnvironment(game, chance_event_sampler=env_lib.PhiloxChanceSampler(seed, i),
                              observation_type=getattr(rl.ObservationType, kind)) for i in range(n)]
    vec = ve_mod.SyncVectorEnv(envs)
    A, P = game.num_distinct_actions(), game.num_players()
    counter = [0]

    def begin_call():
        for e in envs:
            e.block = env_lib.block(counter[0])
        counter[0] += 1

    def convert(time_steps, rewards=None, done=None):
        mask = np.zeros((n, A), dtype=bool)
        for i, ts in enumerate(time_steps):
            cur = ts.observations["current_player"]
            if cur >= 0:
                mask[i, ts.observations["legal_actions"][cur]] = True
        rw = rewards if rewards is not None else [ts.rewards for ts in time_steps]
        return {"obs": np.array([ts.observations["info_state"] for ts in time_steps], dtype=np.float32), "mask": mask,
                "cur": np.array([ts.observations["current_player"] for ts in time_steps], dtype=np.int8),
                "rewards": np.array([r if r is not None else [0.0] * P for r in rw], dtype=np.float32),
                "done": np.array(done if done is not None else [0] * n, dtype=np.uint8),
                "step_type": np.array([ts.step_type.value for ts in time_steps], dtype=np.uint8)}

    def reset():
        begin_call()
        return convert(vec.reset())

    def step(actions, rid):
        begin_call()
        time_steps, reward, done, _ = vec.step([_StepOutput(int(a)) for a in actions], reset_if_done=rid)
        return convert(time_steps, reward, done)

    return env_lib.run_calls(reset, step, n, env_lib.REFERENCE_STEPS, seed, reset_if_done)


@pytest.mark.parametrize("case", CASES, ids=[env_lib.case_id(c) for c in CASES])
def test_restatement_equals_reference_environment(case):
    gs, kind, rid = case
    mine = env_lib.VectorEnv(gs, env_lib.REFERENCE_N, env_lib.REFERENCE_SEED, 0, kind)
    calls = list(env_lib.run_calls(mine.reset, mine.step, env_lib.REFERENCE_N, env_lib.REFERENCE_STEPS, env_lib.REFERENCE_SEED, rid))
    for t, (got, want) in enumerate(zip(calls, reference_calls(gs, kind, rid))):
        for k in ("obs", "mask", "cur", "rewards", "done", "step_type"):
            assert np.array_equal(got[k], want[k]), (case, t, k)
    assert sum(int(c["done"].sum()) for c in calls) >= 2 * env_lib.REFERENCE_N      # every lane finishes episodes
    assert env_lib.digest(calls) == GOLDEN[env_lib.case_id(case)]


@pytest.mark.parametrize("case", CASES, ids=[env_lib.case_id(c) for c in CASES])
def test_restatement_matches_pinned_digests(case):
    gs, kind, rid = case
    mine = env_lib.VectorEnv(gs, env_lib.REFERENCE_N, env_lib.REFERENCE_SEED, 0, kind)
    calls = env_lib.run_calls(mine.reset, mine.step, env_lib.REFERENCE_N, env_lib.REFERENCE_STEPS, env_lib.REFERENCE_SEED, rid)
    assert env_lib.digest(calls) == GOLDEN[env_lib.case_id(case)]
