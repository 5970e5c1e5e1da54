#!/usr/bin/env python3
"""Generates tests/golden/reference_vectors.json from the UNMODIFIED reference (oracle/_ref, built by oracle/ref_build.mk
where the reference checkout exists).  The vectors pin the oracle's algorithm restatements without needing the
reference at test time (tests/test_reference_vectors.py):
  mcts          MCTSBot::MCTSearch root children (action, visits, total reward as hex float) for seeded searches
  mccfr         ExternalSamplingMCCFRSolver tables after N iterations (hex floats)
  cfr           CFRSolver tables after N iterations (hex floats)
  trajectories  RecordBatchedTrajectory episodes (uniform policies): actions, players, legal masks, rewards, observations
Usage: python tests/golden/make_reference_vectors.py"""
import json
import os
import random
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import ref_lib  # noqa: E402

assert ref_lib.available(), "build oracle/_ref first (make -C oracle -f ref_build.mk)"
out = {"mcts": [], "mccfr": [], "cfr": [], "trajectories": []}

MCTS = [("tic_tac_toe", 0, 300, 1, True, 1), ("tic_tac_toe", 3, 200, 3, True, 7), ("connect_four", 0, 400, 1, True, 42),
        ("connect_four", 8, 300, 2, False, 5), ("breakthrough(rows=6,columns=6)", 4, 150, 1, True, 11),
        ("hex(board_size=5)", 3, 200, 1, True, 2), ("go(board_size=5)", 6, 120, 1, True, 9), ("go(board_size=9)", 10, 50, 1, True, 13)]
for gs, prefix, sims, nroll, solve, seed in MCTS:
    rng = random.Random(seed)
    g = ref_lib.RefGame(gs)
    s = g.new_initial_state()
    hist = []
    for _ in range(prefix):
        a = rng.choice(s.legal_actions())
        nxt = s.clone()
        nxt.apply_action(a)
        if nxt.is_terminal():
            break
        s.apply_action(a)
        hist.append(a)
    r = ref_lib.ref_mcts(g, s, 2.0, sims, nroll, solve, seed)
    out["mcts"].append({"game": gs, "history": hist, "sims": sims, "n_rollouts": nroll, "solve": solve, "seed": seed,
                        "children": [[a, v, float(w).hex()] for a, v, w in r["children"]], "best_action": r["best_action"],
                        "root_visits": r["root_visits"]})


def hex_table(t, fields):
    return {k: {"legal": v["legal"], **{f: [float(x).hex() for x in v[f]] for f in fields}} for k, v in sorted(t.items())}


for gs, seed, iters in [("kuhn_poker", 0, 200), ("kuhn_poker", 12345, 1000), ("leduc_poker", 3, 60)]:
    s = ref_lib.RefMCCFR(ref_lib.RefGame(gs), seed)
    s.iterate(iters)
    out["mccfr"].append({"game": gs, "seed": seed, "iterations": iters, "table": hex_table(s.table(), ("regrets", "cum_policy"))})

for gs, iters in [("kuhn_poker", 50)]:          # leduc tables (936 information states) are covered live by test_cfr_oracle.py
    s = ref_lib.RefCFR(ref_lib.RefGame(gs))
    s.iterate(iters)
    out["cfr"].append({"game": gs, "iterations": iters, "table": hex_table(s.table(), ("regrets", "cum_policy", "cur_policy"))})

for gs, T, B, seed in [("kuhn_poker", 5, 40, 99), ("leduc_poker", 10, 20, 7)]:
    t = ref_lib.ref_record_batched_trajectory(ref_lib.RefGame(gs), B, seed, T)
    out["trajectories"].append({"game": gs, "T": T, "seed": seed,
                                "episodes": [{k: t[k][b].tolist() for k in ("observations", "legal_actions", "actions", "player_ids",
                                                                            "valid", "next_is_terminal", "rewards")} for b in range(B)]})

path = os.path.join(HERE, "reference_vectors.json")
json.dump(out, open(path, "w"), separators=(",", ":"))
print("wrote", path, os.path.getsize(path), "bytes")
