#!/usr/bin/env python3
"""Generates tests/golden/long_run_reference.json: the leduc_poker solver runs bench.py times, at their full length, for
tests/test_gpu_bench_loops.py.

- CFR and CFR+ (linear averaging + regret matching plus): sha256 of regrets, cumulative policy and current policy
  (golden_lib.table_digest) after 1,000, 10,000 and 100,010 iterations (the bench's 10 warm-up + 100,000 timed), and
  NashConv / exploitability of the average policy there.
- External-sampling MCCFR with 16,384 traversals per update, seeds 11 and 12 (ranks 0 and 1 of the bench): sha256 of
  regrets and cumulative policy of every information state (the ones no traversal has reached yet at their initial
  value, as the device tables hold them) after 2 and after 2 + 50 iterations, and NashConv of the average policy at the
  end.

Plain CFR runs on the unmodified reference (ref_lib.RefCFR, its own NashConv) where oracle/_ref is built.  Everywhere
else the tables come from the oracle (tests/oracle_lib.py; test_cfr_oracle.py / test_mccfr_oracle.py pin it to the
reference bit for bit) and NashConv from the exact-arithmetic evaluator (tests/exact_policy_eval.py), rounded once to a
double.  Each entry records which one produced it.  The four runs go to separate processes; a 100k-iteration oracle
run takes about 40 minutes.
Usage: python tests/golden/make_long_cfr_reference.py"""
import json
import multiprocessing
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import exact_policy_eval  # noqa: E402
import golden_lib  # noqa: E402
import ref_lib  # noqa: E402
from oracle_lib import OracleCFR, OracleGame, OracleMCCFR  # noqa: E402

GAME = "leduc_poker"
CFR_CHECKPOINTS = [1000, 10000, 100010]
MCCFR_K = 16384
MCCFR_SEEDS = [11, 12]
MCCFR_ITERATIONS = [2, 52]
MCCFR_INIT = 0.000001          # external_sampling_mccfr.h: initial regret and average-policy entries


def exact_nash_conv(table):
    """NashConv of the average policy of an oracle-shaped table {information state string: {legal, cum_policy}}."""
    t = exact_policy_eval.tree(GAME)
    layout = t.layout()
    cum = np.concatenate([np.asarray(table[s]["cum_policy"], dtype=np.float64) for s in t.is_string])
    assert [table[s]["legal"] for s in t.is_string] == t.is_legal
    return float(exact_policy_eval.evaluate(GAME, layout, cum, average=True)["nash_conv"])


def cfr_run(plus):
    if not plus and ref_lib.available():
        solver, source = ref_lib.RefCFR(ref_lib.RefGame(GAME)), "reference"
    else:
        solver, source = OracleCFR(OracleGame(GAME), linear_averaging=plus, regret_matching_plus=plus), "oracle"
    rows, done = [], 0
    for it in CFR_CHECKPOINTS:
        solver.iterate(it - done)
        done = it
        table = solver.table()
        if source == "reference":
            nc, expl = solver.nash_conv(), solver.exploitability()
        else:
            nc = exact_nash_conv(table)
            expl = nc / 2
        rows.append({"iterations": it, "table_sha256": golden_lib.table_digest(table), "nash_conv": nc,
                     "exploitability": expl})
    return {"source": source, "checkpoints": rows}


def mccfr_full_table(table):
    """Every information state of the game, the ones the sampled traversals have not reached yet at the initial value
    the device tables hold (test_gpu_mccfr.INIT), regrets and cumulative policy only."""
    t = exact_policy_eval.tree(GAME)
    out = {}
    for s, legal in zip(t.is_string, t.is_legal):
        v = table.get(s)
        out[s] = {"legal": legal, "regrets": v["regrets"] if v else [MCCFR_INIT] * len(legal),
                  "cum_policy": v["cum_policy"] if v else [MCCFR_INIT] * len(legal)}
    return out


def mccfr_run(seed):
    solver = OracleMCCFR(OracleGame(GAME), seed=seed, rng_mode=1, traversals_per_update=MCCFR_K)
    rows, done = [], 0
    for it in MCCFR_ITERATIONS:
        solver.iterate(it - done)
        done = it
        table = mccfr_full_table(solver.table())
        rows.append({"iterations": it, "table_sha256": golden_lib.table_digest(table)})
    rows[-1]["nash_conv"] = exact_nash_conv(table)
    return {"source": "oracle", "traversals_per_update": MCCFR_K, "seed": seed, "checkpoints": rows}


def job(spec):
    kind, arg = spec
    return cfr_run(arg) if kind == "cfr" else mccfr_run(arg)


def main():
    specs = [("cfr", False), ("cfr", True)] + [("mccfr", s) for s in MCCFR_SEEDS]
    with multiprocessing.Pool(len(specs)) as pool:
        res = pool.map(job, specs)
    out = {"game": GAME, "cfr": res[0], "cfr_plus": res[1], "mccfr_external": {str(s): r for s, r in zip(MCCFR_SEEDS, res[2:])}}
    with open(os.path.join(HERE, "long_run_reference.json"), "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
        f.write("\n")
    print("wrote long_run_reference.json (cfr: %s)" % res[0]["source"])


if __name__ == "__main__":
    main()
