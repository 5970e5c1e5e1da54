"""GPU parity of the device RL environment (VectorEnv over b2s_env_reset / b2s_env_step) with the restatement of
rl_environment.Environment / SyncVectorEnv (tests/env_lib.py): every output of every call, lane by lane, on ragged
multi-block batches, both reset_if_done settings and every observation setting; -1 and illegal actions; sharded lanes;
CUDA-graph replay; and the full 2^20-lane size on a sample of lanes.  env_lib itself is pinned to the reference's own
Environment code by tests/test_env_reference.py."""
import numpy as np
import pytest
import torch

import env_lib
import open_spiel_b200 as b2
from test_gpu_trajectories import CASES

pytestmark = pytest.mark.gpu

GAMES = list(dict.fromkeys(c[0] for c in CASES)) + ["go(board_size=19,handicap=4)", "hex(board_size=5,swap=True)",
                                                   "connect_four(egocentric_obs_tensor=True)"]
LARGE = ("breakthrough", "hex", "go(board_size=9)", "go(board_size=19", "othello", "havannah")


def device_ts(ts, reward, done, idx=None):
    """The time step as env_lib's dict of numpy arrays, of lanes idx (a device index tensor) or all."""
    pick = (lambda x: x) if idx is None else (lambda x: x[idx])
    return {"obs": pick(ts.info_state).cpu().numpy(), "mask": pick(ts.legal_actions_mask).cpu().numpy(),
            "cur": pick(ts.current_player).cpu().numpy(), "rewards": pick(reward).cpu().numpy(),
            "done": pick(done).cpu().numpy().astype(np.uint8), "step_type": pick(ts.step_type).cpu().numpy()}


def assert_same(got, want, where, lanes=None):
    for k in ("obs", "mask", "cur", "rewards", "done", "step_type"):
        g = got[k] if lanes is None else got[k][lanes]
        assert np.array_equal(g, want[k]), (where, k, np.argwhere(np.asarray(g != want[k]))[:4].tolist())


def draw_actions(mask, gen, p_skip=0.0, p_illegal=0.0):
    """On the device: a uniformly random legal action per lane (0 where there is none), then -1 on a p_skip share of the
    lanes and the lowest illegal action on a p_illegal share."""
    m = mask.to(torch.int32)
    cnt = m.sum(1)
    u = torch.rand(mask.shape[0], device=mask.device, generator=gen)
    k = (u * cnt).to(torch.int32).clamp_(max=(cnt - 1).clamp(min=0))
    a = (m.cumsum(1) <= k.unsqueeze(1)).sum(1).to(torch.int32)
    a = torch.where(cnt > 0, a, torch.zeros_like(a))
    v = torch.rand(mask.shape[0], device=mask.device, generator=gen)
    a = torch.where((v < p_skip) & (cnt > 0), torch.full_like(a, -1), a)
    illegal = (~mask).to(torch.int32).argmax(1).to(torch.int32)
    has_illegal = (~mask).any(1) & (cnt > 0)
    return torch.where((v >= p_skip) & (v < p_skip + p_illegal) & has_illegal, illegal, a).contiguous()


@pytest.mark.parametrize("reset_if_done", [False, True])
@pytest.mark.parametrize("gs", GAMES)
def test_device_env_equals_restatement(gs, reset_if_done):
    game = b2.load_game(gs)
    n = 261 if gs.startswith(LARGE) else 1061            # ragged: several blocks at every game's lanes per thread
    steps = 12 if gs.startswith("go(board_size=19") else 30
    kinds = [None, "OBSERVATION"] + (["INFORMATION_STATE"] if game.information_state_tensor_size() > 0 else [])
    gen = torch.Generator(device="cuda").manual_seed(len(gs))
    for kind in kinds:
        env = b2.VectorEnv(game, n, seed=0xE17, observation_type=kind, lane_offset=5)
        ref = env_lib.VectorEnv(gs, n, 0xE17, 5, kind)
        ts = env.reset()
        assert_same(device_ts(ts, env.time_step.rewards, torch.zeros(n)), ref.reset(), (gs, kind, "reset"))
        for t in range(steps):
            acts = draw_actions(ts.legal_actions_mask, gen, p_skip=0.1, p_illegal=0.05)
            ts, reward, done = env.step(acts, reset_if_done=reset_if_done)
            assert_same(device_ts(ts, reward, done), ref.step(acts.cpu().numpy(), reset_if_done), (gs, kind, t))
            assert env.batch.error_count()[0] == ref.errors, (gs, kind, t)
            want_disc = np.where(ts.step_type.cpu().numpy() == 2, 0.0, 1.0)[:, None]
            assert np.array_equal(ts.discounts.cpu().numpy(), np.broadcast_to(want_disc, ts.discounts.shape).astype(np.float32))
        errors = env.batch.error_count()[0]
        assert_same(device_ts(env.reset(), env.time_step.rewards, torch.zeros(n)), ref.reset(), (gs, kind, "reset again"))
        assert env.batch.error_count()[0] == errors          # b2s_env_reset leaves the error counter alone


def test_step_before_reset_resets_and_info_state_is_a_view():
    env = b2.VectorEnv("leduc_poker", 64, seed=1)
    ref = env_lib.VectorEnv("leduc_poker", 64, 1)
    ts, reward, done = env.step(torch.zeros(64, dtype=torch.int32, device="cuda"))
    assert_same(device_ts(ts, reward, done), ref.reset(), "first step")
    assert bool((ts.step_type == b2.StepType.FIRST).all()) and not bool(done.any())
    assert ts.info_state.shape == (64, 2, 30) and ts.info_state.data_ptr() == env._obs.data_ptr()
    with pytest.raises(b2.SpielError):
        b2.VectorEnv("tic_tac_toe", 8, observation_type=b2.ObservationType.INFORMATION_STATE)


@pytest.mark.parametrize("gs", ["leduc_poker(players=3)", "connect_four"])
def test_two_half_batches_equal_one_full_batch(gs):
    n = 2 * 700
    full = b2.VectorEnv(gs, n, seed=9)
    halves = [b2.VectorEnv(gs, n // 2, seed=9, lane_offset=k * (n // 2)) for k in range(2)]
    gen = torch.Generator(device="cuda").manual_seed(3)
    ts = full.reset()
    for k, h in enumerate(halves):
        assert_same(device_ts(ts, ts.rewards, torch.zeros(n, device="cuda")), device_ts(h.reset(), h.time_step.rewards, torch.zeros(n // 2, device="cuda")),
                    (gs, "reset", k), lanes=slice(k * (n // 2), (k + 1) * (n // 2)))
    for t in range(25):
        acts = draw_actions(ts.legal_actions_mask, gen)
        ts, reward, done = full.step(acts, reset_if_done=True)
        outs = [h.step(acts[k * (n // 2):(k + 1) * (n // 2)].contiguous(), reset_if_done=True) for k, h in enumerate(halves)]
        got = device_ts(ts, reward, done)
        for k, o in enumerate(outs):
            part = device_ts(*o)
            assert_same(got, part, (gs, t, k), lanes=slice(k * (n // 2), (k + 1) * (n // 2)))


def test_cuda_graph_replay_equals_eager_steps():
    gs, n = "leduc_poker", 1500
    graph_env, twin = b2.VectorEnv(gs, n, seed=4), b2.VectorEnv(gs, n, seed=4)

    def policy(mask):                                    # deterministic, on the device: the lowest legal action
        return mask.to(torch.int32).argmax(1).to(torch.int32)

    ts = graph_env.reset()
    twin_ts = twin.reset()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(side):
        with torch.cuda.graph(g, stream=side):
            for _ in range(8):
                ts, reward, done = graph_env.step(policy(ts.legal_actions_mask), reset_if_done=True)
    torch.cuda.current_stream().wait_stream(side)
    seen = []
    for replay in range(3):
        g.replay()
        for _ in range(8):
            twin_ts, twin_r, twin_d = twin.step(policy(twin_ts.legal_actions_mask), reset_if_done=True)
        torch.cuda.synchronize()
        assert_same(device_ts(ts, reward, done), device_ts(twin_ts, twin_r, twin_d), ("replay", replay))
        seen.append(ts.info_state.cpu().numpy().copy())
    assert not np.array_equal(seen[0], seen[1]) and not np.array_equal(seen[1], seen[2])   # fresh chance draws per replay


@pytest.mark.parametrize("gs,kind", [("connect_four", None), ("leduc_poker", None)])
def test_full_size_sampled_lanes(gs, kind):
    n, steps = 1 << 20, 12
    lanes = np.sort(np.random.RandomState(0).choice(n, 2000, replace=False))
    env = b2.VectorEnv(gs, n, seed=21, observation_type=kind)
    ref = env_lib.VectorEnv(gs, n, 21, 0, kind, lanes=lanes)
    gen = torch.Generator(device="cuda").manual_seed(5)
    idx = torch.from_numpy(lanes).cuda()
    ts = env.reset()
    assert_same(device_ts(ts, env.time_step.rewards, torch.zeros(n, device="cuda"), idx), ref.reset(), (gs, "reset"))
    for t in range(steps):
        acts = draw_actions(ts.legal_actions_mask, gen, p_skip=0.05)
        ts, reward, done = env.step(acts, reset_if_done=True)
        assert_same(device_ts(ts, reward, done, idx), ref.step(acts[idx].cpu().numpy(), True), (gs, t))
    assert env.batch.error_count()[0] == 0
