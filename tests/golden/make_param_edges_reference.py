#!/usr/bin/env python3
"""Generates tests/golden/param_edges_reference.json from the UNMODIFIED reference (oracle/_ref): for every accepted variant of
tests/param_edges.py, parity.checker_digests of seeded random games played to the end on the reference's State objects (player
to move, terminal flag, legal actions, returns with the sign of zero, and every third ply each player's observation tensor and,
for the poker games, information-state tensor).  tests/test_param_edges_reference.py requires the oracle to give the same
digests, which pins the oracle to the reference on these shapes where no reference build exists.
Usage: python tests/golden/make_param_edges_reference.py"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
import ref_lib  # noqa: E402
from param_edges import ACCEPTED, INFO_STATE, reference_lanes  # noqa: E402
from parity import checker_digests  # noqa: E402

assert ref_lib.available(), "build oracle/_ref first (make -C oracle -f ref_build.mk)"

SEED = 2027


def main():
    out = {}
    for gs, lanes in ACCEPTED:
        out[gs] = checker_digests(gs, reference_lanes(gs, lanes), SEED, ref_lib.RefGame, check_info_state=gs in INFO_STATE)
    with open(os.path.join(HERE, "param_edges_reference.json"), "w") as f:
        json.dump({"seed": SEED, "digests": out}, f, indent=1, sort_keys=True)
        f.write("\n")
    print("wrote %d digests" % len(out))


if __name__ == "__main__":
    main()
