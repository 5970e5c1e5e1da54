"""Regenerates tests/golden/cfr_br_reference.json from the unmodified reference (oracle/_ref): table digests of
CFRBRSolver after kuhn_poker 300 and leduc_poker 100 and 1,000 iterations, with NashConv, exploitability and expected
returns of their average policies, and TabularBestResponse's actions (digest) and value on the seeded random policies of
cfr_br_lib.random_policy.  tests/test_cfr_br_oracle.py and tests/test_gpu_cfr_br.py compare against it where no reference
checkout exists.  Run after those tests pass against the checkout:

  python tests/golden/make_cfr_br_reference.py"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import cfr_br_lib  # noqa: E402
import golden_lib  # noqa: E402
import oracle_lib  # noqa: E402
import ref_lib  # noqa: E402


def main():
    out = {"tables": {}, "best_response": {}}
    for gs, iters in cfr_br_lib.PINNED:
        ref = cfr_br_lib.RefCFRBR(ref_lib.RefGame(gs))
        ref.iterate(iters)
        out["tables"]["%s@%d" % (gs, iters)] = {"table_sha256": golden_lib.table_digest(ref.table()), **ref.average_eval()}
    for gs in cfr_br_lib.SPLITS:
        game = ref_lib.RefGame(gs)
        legal = cfr_br_lib.legal_actions_by_key(oracle_lib.OracleGame(gs))
        for seed, player in cfr_br_lib.br_cases():
            actions, value = cfr_br_lib.ref_tabular_br(game, player, cfr_br_lib.random_policy(legal, seed))
            out["best_response"]["%s/%d/%d" % (gs, seed, player)] = [cfr_br_lib.br_digest(actions), value.hex()]
    with open(cfr_br_lib.GOLDEN, "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
        f.write("\n")


if __name__ == "__main__":
    main()
