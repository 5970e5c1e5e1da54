"""Device AlphaBetaSearch throughput (open_spiel_b200.alpha_beta_search): roots/s, generated states/s, the per-root node-count
distribution and the tail cost (kernel time over the time of the slowest root searched alone).  Each call is timed with CUDA
events after one warm-up call; the card's name and power limit are read in the same run.  CPU baseline in the same run: the
reference's stock AlphaBetaSearch (open_spiel_b200/adapter/_build/alpha_beta_bench, built where the OpenSpiel checkout is) on
the first --cpu-roots searched roots of each workload, on one thread and on every hardware thread; its states/s use the device's
node counts of those roots, which are the reference's.  Prints one JSON line per workload.

  python scripts/bench_alpha_beta.py [--reps 3] [--cpu-roots 2000]"""
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


def random_batch(gs, n, plies, seed):
    """n lanes after uniform random plies (an int, or a per-lane count drawn from range(lo, hi + 1)); a lane whose game ends
    earlier stays terminal."""
    g = b2.load_game(gs)
    batch = g.new_batch(n)
    gen = torch.Generator(device="cuda").manual_seed(seed)
    lo, hi = (plies, plies) if isinstance(plies, int) else plies
    batch.reset()
    k = torch.randint(lo, hi + 1, (n,), device="cuda", generator=gen)
    hist = torch.full((n, hi), -1, dtype=torch.int32, device="cuda")
    for t in range(hi):
        mask = batch.legal_actions_mask().float()
        none = mask.sum(1) == 0
        a = torch.multinomial(mask + none.unsqueeze(1).float(), 1, generator=gen).squeeze(1).to(torch.int32)
        a = torch.where((k > t) & ~none, a, torch.full_like(a, -1))
        hist[:, t] = a
        batch.apply_actions(a)
    batch._reset_errors()
    return g, batch, hist.cpu().numpy()


def timed(fn):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    out = fn()
    e.record()
    torch.cuda.synchronize()
    return out, s.elapsed_time(e) / 1e3


def cpu_baseline(gs, hist, lanes, nodes):
    """The stock search on the roots `lanes` (histories `hist`): seconds on one and on all hardware threads, as roots/s and
    states/s; None without the binary."""
    if not os.path.exists(CPU_BENCH):
        return None
    text = gs + "\n" + "".join(",".join(str(a) for a in hist[i] if a >= 0) + "\n" for i in lanes)
    undo = "1" if gs.split("(")[0] in ("tic_tac_toe", "breakthrough", "go", "mnk") else "0"   # the games with UndoAction
    r = json.loads(subprocess.run([CPU_BENCH, undo], input=text, capture_output=True, text=True, check=True).stdout)
    states = float(nodes.sum())
    return {"roots": r["roots"], "use_undo": r["use_undo"], "threads": r["threads"], "one_core_seconds": r["one_core_seconds"],
            "one_core_roots_per_s": r["roots"] / r["one_core_seconds"], "one_core_states_per_s": states / r["one_core_seconds"],
            "all_cores_seconds": r["all_cores_seconds"], "all_cores_roots_per_s": r["roots"] / r["all_cores_seconds"],
            "all_cores_states_per_s": states / r["all_cores_seconds"]}


def run(name, gs, n, plies, seed, max_nodes, reps, cpu_roots):
    g, batch, hist = random_batch(gs, n, plies, seed)
    b2.alpha_beta_search(batch, max_nodes=max_nodes)             # warm-up: module load, stack allocation
    torch.cuda.synchronize()
    times = []
    for _ in range(reps):
        out, t = timed(lambda: b2.alpha_beta_search(batch, max_nodes=max_nodes))
        times.append(t)
    status = out["status"].cpu().numpy()
    searched = status != 3                                        # lanes whose random play ended are terminal roots
    all_nodes = out["nodes"].cpu().numpy()
    nodes = all_nodes[searched]
    # CPU sample: the first cpu_roots solved roots (a budget-stopped root has no finite reference time)
    sample = np.flatnonzero(status == 0)[:cpu_roots]
    cpu = cpu_baseline(gs, hist, sample, all_nodes[sample])
    slowest = int(np.flatnonzero(searched)[np.argmax(nodes)])
    one = g.new_batch(1)
    one.copy_from(batch, src_begin=slowest, count=1)
    b2.alpha_beta_search(one, max_nodes=max_nodes)
    _, t1 = timed(lambda: b2.alpha_beta_search(one, max_nodes=max_nodes))
    t = min(times)
    print(json.dumps({
        "workload": name, "game": gs, "lanes": n, "searched_roots": int(searched.sum()), "max_nodes": max_nodes,
        "seconds": [round(x, 5) for x in times], "searched_roots_per_s": int(searched.sum()) / t, "states_per_s": float(nodes.sum()) / t, "solved": int((status == 0).sum()),
        "budget_stopped": int((status == 1).sum()), "nodes_median": float(np.median(nodes)),
        "nodes_p99": float(np.percentile(nodes, 99)), "nodes_max": int(nodes.max()), "slowest_root_seconds": t1,
        "kernel_over_slowest_root": t / t1, "cpu_reference": cpu}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--cpu-roots", type=int, default=2000)
    args = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()[0]
    print(json.dumps({"card": card}), flush=True)
    run("tic_tac_toe, 0-4 random plies", "tic_tac_toe", 1 << 20, (0, 4), 1, 0, args.reps, args.cpu_roots)
    run("connect_four 6x7, 14 empty cells", "connect_four", 1 << 16, 28, 2, 0, args.reps, args.cpu_roots)
    run("connect_four 6x7, 18 empty cells, budget 2e6", "connect_four", 1 << 14, 24, 3, 2_000_000, args.reps, args.cpu_roots)
    run("othello 8x8, 10 empty squares", "othello", 1 << 14, 50, 4, 0, args.reps, args.cpu_roots)


if __name__ == "__main__":
    main()
