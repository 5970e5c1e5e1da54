"""Parity of the BENCHED workload itself (SURVEY §8d config 2: "first 1M lanes replayed through the oracle"): the exact
1,048,576-lane U{0..20}-ply connect_four batch bench.py times (same builder, same seed) replayed lane by lane on the
UNMODIFIED reference — live where its build (oracle/_ref) exists, and everywhere through the digests of the reference's
outputs stored in tests/golden/reference_results.json — and every output of the benched step (legal mask before,
terminal, current player, returns, next legal mask and the full observation tensor after) must match on every lane.
Both host entry points (float and compact) are checked on the same batch."""
import os
import sys

import numpy as np
import pytest
import torch

import golden_lib
import ref_lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
pytestmark = pytest.mark.gpu


def test_benched_connect_four_batch_equals_reference_on_every_lane():
    import bench
    import open_spiel_b200 as b2
    gold = golden_lib.reference_results()["bench_workload"]
    n = bench.N_STATES
    assert gold["n"] == n and gold["seed"] == 0x5EED
    dev = torch.device("cuda", 0)
    game = b2.Game("connect_four", device=0)
    _, snap, actions, hist = bench.build_workload(torch, game, n, dev, seed=0x5EED, with_history=True)
    assert hist.shape == (n, bench.MAX_PREFIX)
    hist_np, actions_np = hist.cpu().numpy(), actions.cpu().numpy()
    assert golden_lib.array_digest(hist_np) == gold["inputs"]["hist"], "the benched inputs differ from the recorded ones"
    assert golden_lib.array_digest(actions_np) == gold["inputs"]["actions"], "the benched inputs differ from the recorded ones"
    # the device step on the benched batch
    work = game.new_batch(n)
    work.copy_from(snap)
    mask_before = work.legal_actions_mask_words().cpu().numpy().astype(np.uint32)
    mask = torch.empty((n, 1), dtype=torch.int32, device=dev)
    term = torch.empty((n,), dtype=torch.uint8, device=dev)
    rets = torch.empty((n, 2), dtype=torch.float32, device=dev)
    work.step(actions, mask, term, rets)
    work.check_errors()
    cur, term2, rets2 = work.status()
    obs = work.observation_tensor(player=0)                       # [n, 126] float32
    assert torch.equal(term, term2) and torch.equal(rets, rets2)
    F = obs.shape[1]
    pad = torch.zeros((n, (-F) % 32), dtype=obs.dtype, device=dev)
    bits = (torch.cat([obs, pad], dim=1) != 0).reshape(n, -1, 32).to(torch.int64)
    words = (bits << torch.arange(32, device=dev, dtype=torch.int64)).sum(dim=2).cpu().numpy().astype(np.uint32)
    out = {"mask_before": mask_before, "terminal": term.cpu().numpy().astype(np.uint8),
           "cur_player": cur.cpu().numpy().astype(np.int8), "returns": rets.cpu().numpy().astype(np.float32),
           "mask_after": mask.cpu().numpy().astype(np.uint32), "obs_bits": words}
    assert sorted(out) == sorted(gold["outputs"])
    if ref_lib.available():
        live = ref_lib.replay_batch("connect_four", hist_np, actions_np, mask_words=1)
        assert live["failed_lanes"] == 0
        for k, v in out.items():
            assert np.array_equal(v, live[k]), k
    for k, v in out.items():
        assert golden_lib.array_digest(v) == gold["outputs"][k], k
    ref = out                                                     # equal to the reference's outputs, lane for lane
    assert int(ref["terminal"].sum()) == gold["terminal_lanes"]
    assert int(ref["terminal"].sum()) > 0 and int((ref["terminal"] == 0).sum()) > n // 2      # the step does end some games
    # the two host entry points on the same batch
    work.copy_from(snap)
    act_h = actions.cpu().pin_memory()
    mask_h = torch.empty((n, 1), dtype=torch.int32).pin_memory()
    term_h = torch.empty((n,), dtype=torch.uint8).pin_memory()
    rets_h = torch.empty((n, 2), dtype=torch.float32).pin_memory()
    torch.cuda.synchronize()
    work.step_host(act_h, mask_h, term_h, rets_h)
    assert np.array_equal(term_h.numpy(), ref["terminal"]) and np.array_equal(rets_h.numpy(), ref["returns"])
    assert np.array_equal(mask_h.numpy().astype(np.uint32), ref["mask_after"])
    work.copy_from(snap)
    torch.cuda.synchronize()
    status_h = torch.empty((n,), dtype=torch.uint8).pin_memory()
    work.step_host_compact(actions.to(torch.uint8).cpu().pin_memory(), status_h)
    st = status_h.numpy()
    t = ref["terminal"].astype(bool)
    assert np.array_equal(st >> 7, ref["terminal"])
    assert np.array_equal(st[~t] & 0x7F, ref["mask_after"][~t, 0].astype(np.uint8))
    outcome = np.where(ref["returns"][:, 0] > 0, 1, np.where(ref["returns"][:, 0] < 0, 2, 0)).astype(np.uint8)
    assert np.array_equal(st[t] & 3, outcome[t])
    work.check_errors()


@pytest.mark.parametrize("n", [1, 3, 5, 33])
@pytest.mark.parametrize("gs", ["tic_tac_toe", "kuhn_poker", "leduc_poker", "connect_four", "hex(board_size=3)"])
def test_observation_rows_need_no_16_byte_alignment(gs, n):
    """ADVICE r01 (high): k_obs emits float4 stores; row t of the trajectory recorder starts at t*n*F floats, which is
    16-byte aligned only when n*F % 4 == 0.  Odd batch sizes must work and agree with the aligned call."""
    import open_spiel_b200 as b2
    game = b2.load_game(gs)
    batch = game.new_batch(n)
    tr = batch.record_trajectories(seed=5)
    assert batch.error_count()[0] == 0
    obs = tr.time_major["observations"]                      # [T, n, F]
    batch2 = game.new_batch(n)
    tr2 = batch2.record_trajectories(seed=5, include_full_observations=False)
    assert torch.equal(tr.time_major["actions"], tr2.time_major["actions"])
    # the first row is the tensor of the start state (after the initial chance moves): recompute it with an aligned buffer
    b3 = game.new_batch(n)
    F = obs.shape[2]
    base = torch.zeros((n * F + 8,), dtype=torch.float32, device=obs.device)
    for shift in (0, 1, 2, 3):                                # every 4-byte phase of the output pointer
        out = base[shift:shift + n * F].view(n, F)
        which = b3.information_state_tensor if b3.info.information_state_tensor_size > 0 else b3.observation_tensor
        if b3.info.max_chance_outcomes == 0:
            which(player=-1, out=out)
            assert torch.equal(out, obs[0]), (gs, n, shift)
    torch.cuda.synchronize()
