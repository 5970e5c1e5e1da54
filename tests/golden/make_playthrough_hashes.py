#!/usr/bin/env python3
"""Writes tests/golden/playthrough_sha256.json: the SHA-256 (and game string, action count) of every reference
playthrough file of the seven b2s games, open_spiel/integration_tests/playthroughs/*.txt.  The files themselves are the
reference's and are not copied; tests/test_pyspiel_module.py regenerates each text through the drop-in pyspiel module
and compares hashes, so the byte-exact playthrough check also runs where the reference checkout does not exist."""
import hashlib
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from __graft_entry__ import REFERENCE  # noqa: E402
from open_spiel_b200.playthrough import recorded_params  # noqa: E402

SRC = os.path.join(REFERENCE, "open_spiel", "integration_tests", "playthroughs")
NAMES = ["tic_tac_toe", "connect_four", "connect_four_start_at", "breakthrough", "hex(board_size=5)", "go", "kuhn_poker_2p",
         "kuhn_poker_3p", "leduc_poker_1540482260", "leduc_poker_3977671846", "leduc_poker_773740114", "leduc_poker_3p",
         "leduc_poker_3p_single_tensor", "mnk", "othello", "y(board_size=9)", "havannah(board_size=4)", "havannah(board_size=4,swap=True)"]
out = {}
for n in NAMES:
    text = open(os.path.join(SRC, n + ".txt"), encoding="utf-8").read()
    game, actions, obs_params = recorded_params(text)
    out[n] = {"game": game, "actions": actions, "observation_params": obs_params,
              "sha256": hashlib.sha256(text.encode("utf-8")).hexdigest(), "bytes": len(text.encode("utf-8"))}
json.dump(out, open(os.path.join(ROOT, "tests", "golden", "playthrough_sha256.json"), "w"), indent=1, sort_keys=True)
print("wrote", len(out), "entries")
