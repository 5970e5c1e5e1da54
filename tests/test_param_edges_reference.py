"""CPU: the oracle against the UNMODIFIED reference on every accepted variant of tests/param_edges.py.  The reference's digests
of seeded random games (parity.checker_digests: player to move, terminal flag, legal actions, returns with the sign of zero,
observation and information-state tensors) are stored in golden/param_edges_reference.json by
golden/make_param_edges_reference.py; the oracle must reproduce each one.  Where oracle/_ref is built, the stored digests are
also checked against the reference itself."""
import json
import os

import pytest

import ref_lib
from oracle_lib import OracleGame
from param_edges import ACCEPTED, INFO_STATE, reference_lanes
from parity import checker_digests

GOLD = json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "param_edges_reference.json"),
                      encoding="utf-8"))


def test_every_accepted_variant_has_a_reference_digest():
    assert sorted(GOLD["digests"]) == sorted(gs for gs, _ in ACCEPTED)


@pytest.mark.parametrize("gs,lanes", ACCEPTED, ids=[g for g, _ in ACCEPTED])
def test_oracle_reproduces_reference_digest(gs, lanes):
    got = checker_digests(gs, reference_lanes(gs, lanes), GOLD["seed"], OracleGame, check_info_state=gs in INFO_STATE)
    assert got == GOLD["digests"][gs]


@pytest.mark.skipif(not ref_lib.available(), reason="oracle/_ref not built")
@pytest.mark.parametrize("gs,lanes", ACCEPTED[::7], ids=[g for g, _ in ACCEPTED[::7]])
def test_stored_digest_is_the_reference_s(gs, lanes):
    got = checker_digests(gs, reference_lanes(gs, lanes), GOLD["seed"], ref_lib.RefGame, check_info_state=gs in INFO_STATE)
    assert got == GOLD["digests"][gs]
