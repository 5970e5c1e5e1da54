"""Throughput of go on 13x13 and 19x19 boards on the device (the 384-bit rule core).  Per board, one JSON line with:
  apply_per_s      batched ApplyAction (b2s_apply) steps per second: lanes x steps over the CUDA-event time of the apply
                   launches only, 32 steps of random legal moves after 64 opening plies
  playouts_per_s   random playouts to the end of the game from the initial position (b2s_rollout)
  mcts_sims_per_s  mcts_search, UCT, n_rollouts 1, solver on, from 4-ply roots that differ between trees
  eval_step_ms     mcts_search_evaluated (PUCT) with the hash test evaluator of tests/mcts_eval_lib.py: mean time of one
                   b2s_mcts_eval_step launch, and the whole search's simulations per second
The batch sizes fit the history column of 8 (max_game_length + 1) bytes per lane (5.8 KB on 19x19).  The card's name and
power limit are printed with every line (nvidia-smi query, read only).
Usage: python scripts/bench_go_large.py [--repeat 3] [--only 19]"""
import argparse
import json
import subprocess
import sys
import time

import torch

sys.path.insert(0, ".")
sys.path.insert(0, "tests")
import open_spiel_b200 as b2  # noqa: E402
from mcts_eval_lib import hash_evaluator  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, limit = [x.strip() for x in out.split(",")]
        return name, limit
    except Exception:
        return torch.cuda.get_device_name(), "unknown"


def random_legal(batch, gen):
    """One uniformly random legal action per lane (-1 for finished lanes), drawn on the device."""
    acts, counts = batch.legal_actions_list()
    u = torch.rand(counts.shape, device=counts.device, generator=gen)
    k = (u * counts.clamp_min(1)).long().clamp_max(acts.shape[1] - 1)
    a = acts.gather(1, k[:, None]).squeeze(1).int()
    return torch.where(counts > 0, a, torch.full_like(a, -1))


def timed(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    r = fn()
    e1.record()
    torch.cuda.synchronize()
    return r, e0.elapsed_time(e1) * 1e-3


def roots(game, n):
    batch = game.new_batch(n)
    lane = torch.arange(n, device="cuda", dtype=torch.int64)
    for ply in range(4):                        # legal action (7 lane + 13 ply) mod (count - 1): never the pass
        acts, counts = batch.legal_actions_list()
        k = (7 * lane + 13 * ply) % (counts.long() - 1).clamp_min(1)
        batch.apply_actions(acts.gather(1, k[:, None]).squeeze(1).int())
    batch.check_errors()
    return batch


def run(size, lanes, trees, sims, eval_sims):
    gs = "go(board_size=%d)" % size
    game = b2.load_game(gs)
    gen = torch.Generator(device="cuda")
    gen.manual_seed(1)
    res = {"game": gs}
    # ApplyAction
    batch = game.new_batch(lanes)
    for _ in range(64):
        batch.apply_actions(random_legal(batch, gen))
    t = 0.0
    for _ in range(32):
        a = random_legal(batch, gen)
        torch.cuda.synchronize()
        _, dt = timed(lambda: batch.apply_actions(a))
        t += dt
    batch.check_errors()
    res["apply_lanes"] = lanes
    res["apply_per_s"] = lanes * 32 / t
    del batch
    # random playouts
    batch = game.new_batch(lanes)
    (rets, plies), dt = timed(lambda: batch.rollout(seed=3))
    res["playouts_per_s"] = lanes / dt
    res["playout_mean_plies"] = float(plies.float().mean())
    del batch, rets, plies
    # mcts_search (UCT, one rollout)
    batch = roots(game, trees)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = b2.mcts_search(batch, sims, uct_c=2.0, n_rollouts=1, solve=True, seed=5)
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    res["mcts_trees"], res["mcts_sims"] = trees, sims
    res["mcts_sims_per_s"] = int(out["sims_run"].sum()) / wall
    del batch, out
    # mcts_search_evaluated (PUCT, hash evaluator)
    batch = roots(game, trees)
    leaves = game.new_batch(trees)
    search = b2.MCTSEvalSearch(batch, eval_sims, uct_c=2.0, solve=False, seed=7, child_selection_policy=b2.ChildSelectionPolicy.PUCT,
                               leaves=leaves)
    values = priors = None
    steps = []
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    with torch.no_grad():
        while True:
            (pending, n_pending), dt = timed(lambda: search.step(values, priors))
            steps.append(dt)
            if n_pending == 0:
                break
            values, priors = hash_evaluator(leaves.observation_tensor(), leaves.legal_actions_mask())
    wall = time.perf_counter() - t0
    out = search.results()
    res["eval_trees"], res["eval_sims"], res["eval_rounds"] = trees, eval_sims, len(steps) - 1
    res["eval_step_ms"] = 1e3 * sum(steps) / len(steps)
    res["eval_sims_per_s"] = int(out["sims_run"].sum()) / wall
    res["eval_failed_trees"] = leaves.error_count()[0]
    name, limit = card()
    res["device"], res["power_limit"] = name, limit
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeat", type=int, default=3)
    ap.add_argument("--only", default="")
    args = ap.parse_args()
    # (size, ApplyAction / playout lanes, MCTS trees, MCTS sims, evaluated-search sims)
    configs = [c for c in ((13, 1 << 20, 4096, 32, 64), (19, 1 << 19, 2048, 32, 64)) if args.only in str(c[0])]
    run(13, 4096, 128, 4, 4)                    # warm-up: library load, torch kernels, allocator
    for r in range(args.repeat):
        for c in configs:
            res = run(*c)
            res["repeat"] = r
            print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
