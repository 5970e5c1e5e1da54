#!/usr/bin/env python3
"""Generates tests/golden/mcts_eval_reference.json from the UNMODIFIED reference (oracle/_ref): MCTSBot::MCTSearch driven by
the test evaluator (oracle/ref_glue/ref_mcts_eval.cc TestEvaluator) for the cases of tests/test_mcts_eval_oracle_vs_reference.py
(UCT / PUCT, solver on and off, Dirichlet noise, max_memory_mb = 1 collections).  Per search: the root's history, the root's
children (action, visits, total reward as a hex float) in child order, BestChild and the root's visit count.  The stored
searches pin the oracle's evaluator mode where no reference build exists (tests/test_mcts_eval_golden.py).
Usage: python tests/golden/make_mcts_eval_reference.py"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from mcts_eval_lib import ref_eval_available, ref_mcts_eval, ref_sizeof_search_node  # noqa: E402
from oracle_lib import OracleGame  # noqa: E402
from test_mcts_eval_oracle_vs_reference import CASES, GC_CASES, _roots  # noqa: E402

assert ref_eval_available(), "build oracle/_ref first (make -C oracle -f ref_build.mk, then -f ref_eval.mk)"


def search(gs, hist, sims, solve, puct, alpha, seed, max_memory_mb):
    eps = 0.25 if alpha > 0 else 0.0
    r = ref_mcts_eval(gs, hist, OracleGame(gs).num_distinct_actions, 2.0, sims, solve, seed, puct=puct, dirichlet_alpha=alpha,
                      dirichlet_epsilon=eps, max_memory_mb=max_memory_mb)
    return {"game": gs, "history": hist, "sims": sims, "solve": solve, "puct": puct, "dirichlet_alpha": alpha,
            "dirichlet_epsilon": eps, "seed": seed, "max_memory_mb": max_memory_mb,
            "max_nodes": ((max_memory_mb << 20) // ref_sizeof_search_node() + 1) if max_memory_mb else 1,
            "children": [[a, n, float(w).hex()] for a, n, w in r["children"]], "best_action": r["best_action"],
            "root_visits": r["root_visits"]}


out = []
for gs, prefix, sims, solve, puct, alpha, seed in CASES:
    out.append(search(gs, _roots(gs, prefix, seed)[1], sims, solve, puct, alpha, seed, 1000))
for gs, sims, puct, seed in GC_CASES:
    out.append(search(gs, [], sims, False, puct, 0.0, seed, 1))
with open(os.path.join(HERE, "mcts_eval_reference.json"), "w") as f:
    json.dump({"mcts_eval": out}, f, indent=0)
    f.write("\n")
print("wrote %d searches" % len(out))
