"""Regenerates tests/golden/alpha_beta_eval_reference.json: the reference's AlphaBetaSearch with the test value functions
(value bits, best action, generated child states, status, evaluation count and a digest of the evaluated states' histories) on
every case of alpha_beta_eval_lib.reference_cases(), from the comparison in tests/test_alpha_beta_eval_reference.py, so the
restatement stays pinned where no reference checkout exists.  Needs the OpenSpiel checkout and oracle/_ref:

  python tests/golden/make_alpha_beta_eval_reference.py"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
import alpha_beta_eval_lib as abe  # noqa: E402
import test_alpha_beta_eval_reference as t  # noqa: E402


def main():
    minimax = t._minimax()
    out = {}
    for case in abe.reference_cases():
        out[abe.case_id(case)] = t.golden_entry(t.reference_alpha_beta_eval(minimax, case))
    with open(os.path.join(HERE, "alpha_beta_eval_reference.json"), "w") as f:
        json.dump(out, f, indent=0, sort_keys=True)
        f.write("\n")


if __name__ == "__main__":
    main()
