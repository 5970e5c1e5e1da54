"""Device AlphaBetaSearch with a caller-supplied value function (open_spiel_b200.AlphaBetaEvalSearch): rounds, CUDA-event totals
of the search steps and of the evaluator kept apart, evaluated leaves/s and generated states/s, and the pending-lane count per
round (its tail decides the round count).  Two evaluators over the leaves' observation tensor: the test "hash" value function
(tests/alpha_beta_eval_lib.py) and a 2-layer, 256-wide torch MLP (float32, seeded weights).  The card's name and power limit
are read in the same run.  CPU baseline in the same run: the reference's stock AlphaBetaSearch with the hash value function
(open_spiel_b200/adapter/_build/alpha_beta_bench, built where the OpenSpiel checkout is) on the first --cpu-roots searched roots of
each workload, on one thread and on every hardware thread; its states/s use the device's node counts of those roots, which are the
reference's.  Prints one JSON line per workload and evaluator.

  python scripts/bench_alpha_beta_eval.py [--reps 2] [--roots 65536] [--cpu-roots 1000] [--only go]"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CPU_BENCH = os.path.join(ROOT, "open_spiel_b200", "adapter", "_build", "alpha_beta_bench")
sys.path.insert(0, ROOT)
import open_spiel_b200 as b2  # noqa: E402
from bench_alpha_beta import random_batch  # noqa: E402


def hash_values(obs):
    """tests/alpha_beta_eval_lib.py's "hash" function: {v, -v}, v = ((sum_{obs_i != 0} (7i + 3) mod 11) mod 9 - 4) / 7."""
    idx = torch.arange(obs.shape[1], dtype=torch.int64, device=obs.device)
    k = ((obs != 0).to(torch.int64) * ((7 * idx + 3) % 11)).sum(dim=1) % 9
    v = (k - 4).to(torch.float64) / 7.0
    return torch.stack([v, -v], dim=1)


def mlp(F, seed):
    torch.manual_seed(seed)
    net = torch.nn.Sequential(torch.nn.Linear(F, 256), torch.nn.ReLU(), torch.nn.Linear(256, 256), torch.nn.ReLU(),
                              torch.nn.Linear(256, 2), torch.nn.Tanh()).cuda()
    return lambda obs: net(obs).to(torch.float64)


def search(batch, depth, evaluator, n):
    """One search, rounds timed with CUDA events: (results, rounds, step seconds, evaluator seconds, pending per round)."""
    s = b2.AlphaBetaEvalSearch(batch, depth, n=n)
    obs = torch.empty((n, batch.info.observation_tensor_size), dtype=torch.float32, device="cuda")
    ev = []
    pending_counts = []
    values = None
    with torch.no_grad():
        while True:
            a, b, c = (torch.cuda.Event(enable_timing=True) for _ in range(3))
            a.record()
            _, cnt = s.step(values)             # synchronises to read the pending count
            b.record()
            if cnt == 0:
                ev.append((a, b, None))
                break
            pending_counts.append(cnt)
            values = evaluator(s.leaves.observation_tensor(out=obs)).contiguous()
            c.record()
            ev.append((a, b, c))
        out = s.results()
    torch.cuda.synchronize()
    step_s = sum(a.elapsed_time(b) for a, b, _ in ev) / 1e3
    eval_s = sum(b.elapsed_time(c) for _, b, c in ev if c is not None) / 1e3
    return out, len(pending_counts), step_s, eval_s, pending_counts


def cpu_baseline(gs, hist, lanes, nodes, depth):
    if not os.path.exists(CPU_BENCH) or len(lanes) == 0:
        return None
    text = gs + "\n" + "".join(",".join(str(a) for a in hist[i] if a >= 0) + "\n" for i in lanes)
    r = json.loads(subprocess.run([CPU_BENCH, "0", str(depth)], input=text, capture_output=True, text=True, check=True).stdout)
    states = float(nodes.sum())
    return {"roots": r["roots"], "threads": r["threads"], "one_core_seconds": r["one_core_seconds"],
            "one_core_states_per_s": states / r["one_core_seconds"], "all_cores_seconds": r["all_cores_seconds"],
            "all_cores_states_per_s": states / r["all_cores_seconds"]}


def pending_profile(counts, n):
    """The pending-lane count at tenths of the rounds, and the rounds spent after fewer than 1% / 0.1% of the roots remain."""
    c = np.asarray(counts)
    if len(c) == 0:
        return {}
    return {"at_round_fraction": {"%.1f" % f: int(c[min(len(c) - 1, int(f * len(c)))]) for f in np.linspace(0, 1, 11)},
            "rounds_below_1pct": int((c < 0.01 * n).sum()), "rounds_below_0.1pct": int((c < 0.001 * n).sum()),
            "first_round_pending": int(c[0])}


def run(name, gs, n, plies, depth, seed, reps, cpu_roots, evaluators):
    g, batch, hist = random_batch(gs, n, plies, seed)
    cpu = None
    for ename, evaluator in evaluators(batch.info.observation_tensor_size):
        search(batch, depth, evaluator, n)       # warm-up
        runs = [search(batch, depth, evaluator, n) for _ in range(reps)]
        out, rounds, _, _, counts = runs[0]
        nodes = out["nodes"].cpu().numpy()
        evals = out["evaluations"].cpu().numpy()
        searched = out["status"].cpu().numpy() == 0       # lanes whose random play ended are terminal roots (status 3)
        live = int(searched.sum())
        if ename == "hash" and cpu is None:
            lanes = np.flatnonzero(searched)[:cpu_roots]
            cpu = cpu_baseline(gs, hist, lanes, nodes[lanes], depth)
        steps = [r[2] for r in runs]
        evs = [r[3] for r in runs]
        totals = [r[2] + r[3] for r in runs]
        print(json.dumps({
            "workload": name, "game": gs, "roots": n, "non_terminal_roots": live, "depth_limit": depth, "evaluator": ename,
            "rounds": rounds, "step_seconds": [round(x, 4) for x in steps], "evaluator_seconds": [round(x, 4) for x in evs],
            "leaves": int(evals.sum()), "nodes": int(nodes.sum()),
            "leaves_per_s": [float(evals.sum()) / t for t in totals], "nodes_per_s": [float(nodes.sum()) / t for t in totals],
            "evaluations_per_root_median_max": [float(np.median(evals)), int(evals.max())],
            "pending": pending_profile(counts, n), "cpu_reference_hash": cpu if ename == "hash" else None}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--roots", type=int, default=1 << 16)
    ap.add_argument("--go19-roots", type=int, default=1 << 13)
    ap.add_argument("--cpu-roots", type=int, default=1000)
    ap.add_argument("--only", default="")
    args = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()[0]
    print(json.dumps({"card": card}), flush=True)

    def evaluators(F):
        return [("hash", hash_values), ("mlp_2x256", mlp(F, 0))]

    n = args.roots
    work = [("connect_four 6x7, 8 plies, depth 4", "connect_four", n, 8, 4, 1),
            ("connect_four 6x7, 8 plies, depth 6", "connect_four", n, 8, 6, 1),
            ("othello 8x8, 20 plies, depth 3", "othello", n, 20, 3, 2),
            ("go 9x9, 40 plies, depth 2", "go(board_size=9)", n, 40, 2, 3),
            ("go 19x19, 150 plies, depth 2", "go", args.go19_roots, 150, 2, 4)]
    for name, gs, roots, plies, depth, seed in work:
        if args.only and args.only not in name:
            continue
        run(name, gs, roots, plies, depth, seed, args.reps, args.cpu_roots, evaluators)


if __name__ == "__main__":
    main()
