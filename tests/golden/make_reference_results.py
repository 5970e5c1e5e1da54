#!/usr/bin/env python3
"""Generates tests/golden/reference_results.json from the UNMODIFIED reference (oracle/_ref, built by oracle/ref_build.mk):
what the GPU tests compare the device against, so that they need no reference build at test time (tests/golden_lib.py).
  lockstep        test_gpu_vs_reference: digest of the random games lockstep() plays, per game (tests/parity.py)
  cfr             test_gpu_cfr: digest of the CFRSolver table after N iterations; NashConv / exploitability at checkpoints
  mcts            test_gpu_mcts: mean share of root visits and mean root value over 256 seeded MCTSBot searches
  bench_workload  test_gpu_bench_workload: digests of the inputs and of every output of the benched connect_four step;
                  the inputs are drawn on the GPU, so this section is written only where a CUDA device exists
Existing sections of the output file are kept unless recomputed.
Usage: python tests/golden/make_reference_results.py [--out PATH] [--sections lockstep,cfr,mcts,bench_workload]"""
import argparse
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
TESTS = os.path.dirname(HERE)
sys.path.insert(0, TESTS)
sys.path.insert(0, os.path.dirname(TESTS))
import golden_lib  # noqa: E402
import ref_lib  # noqa: E402
from parity import checker_digests  # noqa: E402
from test_gpu_vs_reference import GAMES  # noqa: E402

LOCKSTEP_SEED = 99
CFR_TABLES = [("kuhn_poker", 300), ("leduc_poker", 25)]
CFR_CHECKPOINTS = [("kuhn_poker", [1, 10, 100, 300]), ("leduc_poker", [1, 5, 20])]
MCTS = {"game": "connect_four", "prefix": [3, 3, 2], "sims": 400, "uct_c": 2.0, "n_ref": 256}


def lockstep():
    return {"seed": LOCKSTEP_SEED,
            "digests": {gs: checker_digests(gs, lanes, LOCKSTEP_SEED, ref_lib.RefGame,
                                            check_info_state=gs in ("kuhn_poker", "leduc_poker")) for gs, lanes in GAMES}}


def cfr():
    tables = {}
    for gs, iters in CFR_TABLES:
        ref = ref_lib.RefCFR(ref_lib.RefGame(gs))
        ref.iterate(iters)
        tables[gs] = {"iterations": iters, "table_sha256": golden_lib.table_digest(ref.table()),
                      "exploitability": ref.exploitability()}
    checkpoints = {}
    for gs, its in CFR_CHECKPOINTS:
        ref, done, rows = ref_lib.RefCFR(ref_lib.RefGame(gs)), 0, []
        for it in its:
            ref.iterate(it - done)
            done = it
            rows.append({"iterations": it, "nash_conv": ref.nash_conv(), "exploitability": ref.exploitability()})
        checkpoints[gs] = rows
    return {"tables": tables, "checkpoints": checkpoints}


def mcts():
    rg = ref_lib.RefGame(MCTS["game"])
    st = rg.new_initial_state()
    for a in MCTS["prefix"]:
        st.apply_action(a)
    n_ref = MCTS["n_ref"]
    share, value = np.zeros(rg.num_distinct_actions), 0.0
    for seed in range(n_ref):
        r = ref_lib.ref_mcts(rg, st, MCTS["uct_c"], MCTS["sims"], 1, False, seed + 1)
        tot = sum(vv for _, vv, _ in r["children"])
        for a, vv, _ in r["children"]:
            share[a] += vv / tot / n_ref
        value += sum(rw for _, _, rw in r["children"]) / tot / n_ref
    return dict(MCTS, share=share.tolist(), value=value)


def bench_workload():
    import torch

    import bench
    import open_spiel_b200 as b2
    n = bench.N_STATES
    game = b2.Game("connect_four", device=0)
    _, _, actions, hist = bench.build_workload(torch, game, n, torch.device("cuda", 0), seed=0x5EED, with_history=True)
    hist, actions = hist.cpu().numpy(), actions.cpu().numpy()
    ref = ref_lib.replay_batch("connect_four", hist, actions, mask_words=1)
    assert ref.pop("failed_lanes") == 0
    return {"n": n, "seed": 0x5EED, "inputs": {"hist": golden_lib.array_digest(hist), "actions": golden_lib.array_digest(actions)},
            "outputs": {k: golden_lib.array_digest(v) for k, v in ref.items()},
            "terminal_lanes": int(ref["terminal"].sum())}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=golden_lib.PATH)
    ap.add_argument("--sections", default="lockstep,cfr,mcts,bench_workload")
    args = ap.parse_args()
    assert ref_lib.available(), "build oracle/_ref first (make -C oracle -f ref_build.mk REF=<open_spiel checkout>)"
    out = json.load(open(args.out)) if os.path.exists(args.out) else {}
    for name in args.sections.split(","):
        if name == "bench_workload":
            import torch
            if not torch.cuda.is_available():
                print("no CUDA device: bench_workload kept as it was")
                continue
        out[name] = globals()[name]()
    with open(args.out, "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
        f.write("\n")
    print("wrote", args.out, os.path.getsize(args.out), "bytes")


if __name__ == "__main__":
    main()
