#!/usr/bin/env python3
"""Generates tests/golden/go_large_reference.json from the UNMODIFIED reference (oracle/_ref): seeded random games on
go(board_size=13), go(board_size=19) and go(board_size=19,handicap=h), played to the end.  Per game the actions, and per
position (the initial one included) the current player, terminal flag, returns as text (sign of zero kept), and sha256 prefixes
of the legal action list and of both players' observation tensors (float32 bytes).  The traces pin the oracle's go on large
boards where no reference build exists (tests/test_go_large_oracle_vs_reference.py).
Usage: python tests/golden/make_go_large_reference.py"""
import hashlib
import json
import os
import random
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import ref_lib  # noqa: E402

assert ref_lib.available(), "build oracle/_ref first (make -C oracle -f ref_build.mk)"

# game, number of games, seed
GAMES = [("go(board_size=13)", 4, 1301), ("go(board_size=19)", 2, 1901), ("go(board_size=19,handicap=2)", 1, 1902),
         ("go(board_size=19,handicap=5)", 1, 1905), ("go(board_size=19,handicap=9,komi=0.5)", 1, 1909),
         ("go(board_size=19,handicap=10)", 1, 1910)]


def position(st):
    """The observables of one position as stored in the fixture: [current player, terminal, returns[0], returns[1] (text),
    first 12 hex digits of the sha256 of the legal action list (JSON) and of both observation tensors (float32 bytes)]."""
    legal = st.legal_actions()
    obs = b"".join(np.asarray(st.observation_tensor(p), dtype=np.float32).tobytes() for p in range(2))
    return [st.current_player(), int(st.is_terminal())] + [repr(float(x)) for x in st.returns()] + [
        hashlib.sha256(json.dumps(legal).encode()).hexdigest()[:12], hashlib.sha256(obs).hexdigest()[:12]]


def record(gs, seed):
    rng = random.Random(seed)
    st = ref_lib.RefGame(gs).new_initial_state()
    actions, positions = [], [position(st)]
    while not st.is_terminal():
        a = rng.choice(st.legal_actions())
        st.apply_action(a)
        actions.append(a)
        positions.append(position(st))
    return {"game": gs, "seed": seed, "actions": actions, "positions": positions}


def main():
    out = [record(gs, seed + k) for gs, n, seed in GAMES for k in range(n)]
    with open(os.path.join(HERE, "go_large_reference.json"), "w") as f:
        json.dump({"games": out}, f, separators=(",", ":"))
        f.write("\n")
    print("wrote %d games, %d positions" % (len(out), sum(len(g["positions"]) for g in out)))


if __name__ == "__main__":
    main()
