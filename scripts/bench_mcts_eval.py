"""Throughput of the caller-evaluated device MCTS (mcts_search_evaluated, b2s_mcts_eval_*) and where its time goes.
For connect_four and go 9x9, 4,096 and 65,536 trees, 64 and 800 simulations, and two evaluators:
  hash  the deterministic test evaluator of the parity tests (tests/mcts_eval_lib.py), a few elementwise torch ops
  mlp   a small torch MLP on the observation tensor (obs -> 256 -> 256 -> value + policy logits, float32), masked softmax prior
Per configuration: simulations per second (sum of sims_run over the wall time of the whole search), rounds, and the device
time of the search steps (b2s_mcts_eval_step) and of the evaluator (leaves' observation + legal mask + evaluate), each summed
from CUDA events around every call.  The configurations are run --repeat times, one pass over all of them per repeat, so the
repeats of one configuration alternate with the others.  One JSON line per run.
Usage: python scripts/bench_mcts_eval.py [--repeat 3] [--only connect_four] [--trees 4096,65536] [--sims 64,800]"""
import argparse
import json
import sys
import time

import torch

sys.path.insert(0, ".")
sys.path.insert(0, "tests")
import open_spiel_b200 as b2  # noqa: E402
from mcts_eval_lib import hash_evaluator  # noqa: E402


class Mlp(torch.nn.Module):
    def __init__(self, F, A, H=256):
        super().__init__()
        self.body = torch.nn.Sequential(torch.nn.Linear(F, H), torch.nn.ReLU(), torch.nn.Linear(H, H), torch.nn.ReLU())
        self.value = torch.nn.Linear(H, 1)
        self.policy = torch.nn.Linear(H, A)

    def forward(self, obs, mask):
        h = self.body(obs)
        v = torch.tanh(self.value(h)).squeeze(1).double()
        logits = self.policy(h).masked_fill(mask == 0, float("-inf"))
        return torch.stack([v, -v], dim=1), torch.softmax(logits, dim=1).double()


def node_budget(game, trees, sims):
    """A per-tree node budget (MCTSBot::max_nodes_) where the unbudgeted arena would not fit in 60 % of free memory: 32-byte
    nodes, at most one expansion block and one cached prior block of <= A nodes per simulation."""
    A = game.num_distinct_actions()
    free, _ = torch.cuda.mem_get_info()
    per_tree = int(free * 0.5 / 32 / trees)
    if 2 * sims * A + 2 <= per_tree:
        return 0
    return max(1000, (per_tree - 16 * A - 128) // 4)


def run(gs, trees, sims, ev, model_cache):
    game = b2.load_game(gs)
    batch = game.new_batch(trees)
    # four opening plies that differ between lanes: legal action k = (7 lane + 13 ply) mod (count - 1) of the ascending list,
    # never the highest id (go's pass: two passes would end the game); lanes without a choice stay put (-1)
    lane = torch.arange(trees, device="cuda", dtype=torch.int64)
    for ply in range(4):
        acts, counts = batch.legal_actions_list()
        k = (7 * lane + 13 * ply) % (counts.long() - 1).clamp_min(1)
        a = acts.gather(1, k[:, None]).squeeze(1).int()
        batch.apply_actions(torch.where(counts > 1, a, torch.full_like(a, -1)))
    batch.check_errors()
    if ev == "mlp":
        key = gs
        if key not in model_cache:
            torch.manual_seed(0)
            model_cache[key] = Mlp(game.observation_tensor_size(), game.num_distinct_actions()).cuda().eval()
        model = model_cache[key]
    budget = node_budget(game, trees, sims)
    leaves = game.new_batch(trees)
    search = b2.MCTSEvalSearch(batch, sims, uct_c=2.0, solve=False, seed=7, child_selection_policy=b2.ChildSelectionPolicy.PUCT,
                               max_nodes_per_tree=budget, leaves=leaves)
    step_ev, eval_ev = [], []
    values = priors = None
    rounds = 0
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    with torch.no_grad():
        while True:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            pending, n_pending = search.step(values, priors)
            e1.record()
            step_ev.append((e0, e1))
            if n_pending == 0:
                break
            rounds += 1
            e2, e3 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e2.record()
            obs, mask = leaves.observation_tensor(), leaves.legal_actions_mask()
            values, priors = hash_evaluator(obs, mask) if ev == "hash" else model(obs, mask)
            e3.record()
            eval_ev.append((e2, e3))
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    out = search.results()
    sims_run = int(out["sims_run"].sum())
    return {"game": gs, "trees": trees, "sims": sims, "evaluator": ev, "node_budget": budget, "rounds": rounds,
            "wall_s": round(wall, 4), "sims_per_s": sims_run / wall,
            "step_ms": round(sum(a.elapsed_time(b) for a, b in step_ev), 2),
            "eval_ms": round(sum(a.elapsed_time(b) for a, b in eval_ev), 2),
            "prior_requests": int(out["prior_requests"].sum()), "failed_trees": leaves.error_count()[0],
            "device": torch.cuda.get_device_name()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeat", type=int, default=3)
    ap.add_argument("--only", default="")
    ap.add_argument("--trees", default="4096,65536")
    ap.add_argument("--sims", default="64,800")
    ap.add_argument("--evaluators", default="hash,mlp")
    args = ap.parse_args()
    games = [g for g in ("connect_four", "go(board_size=9)") if args.only in g]
    configs = [(gs, int(t), int(s), ev) for gs in games for t in args.trees.split(",") for s in args.sims.split(",")
               for ev in args.evaluators.split(",")]
    cache = {}
    run("connect_four", 256, 16, "mlp", cache)          # warm-up: library load, torch kernels, allocator
    for r in range(args.repeat):
        for c in configs:
            res = run(*c, cache)
            res["repeat"] = r
            print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
