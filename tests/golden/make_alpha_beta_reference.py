"""Regenerates tests/golden/alpha_beta_reference.json: the reference's AlphaBetaSearch results (value, best action, generated
child states, status) on every case of alpha_beta_lib.reference_cases(), from the comparison in
tests/test_alpha_beta_oracle_vs_reference.py, so the restatement stays pinned where no reference checkout exists.  Needs the
OpenSpiel checkout and oracle/_ref:

  python tests/golden/make_alpha_beta_reference.py"""
import json
import math
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
import alpha_beta_lib as ab  # noqa: E402
import test_alpha_beta_oracle_vs_reference as t  # noqa: E402


def main():
    minimax = t._minimax()
    out = {}
    for case in ab.reference_cases():
        r = t.reference_alpha_beta(minimax, case)
        out[ab.case_id(case)] = [None if math.isnan(r["value"]) else r["value"], r["best_action"], r["nodes"], r["status"]]
    with open(os.path.join(HERE, "alpha_beta_reference.json"), "w") as f:
        json.dump(out, f, indent=0, sort_keys=True)
        f.write("\n")


if __name__ == "__main__":
    main()
