"""Regenerates tests/golden/dcfr_reference.json from the reference's own Python Discounted CFR (the checkout's
python/algorithms/discounted_cfr.py over the unmodified reference games, as tests/dcfr_lib.py loads it): digests of the
tables and of the average policy after each split of dcfr_lib.REF_SPLITS for every variant, and after each split of the
seeded zero-reach case, with the Python and numpy versions that computed them.  tests/test_dcfr_oracle.py and
tests/test_gpu_dcfr.py compare against it where no checkout exists.  Run after those tests pass against the checkout:

  python tests/golden/make_dcfr_reference.py"""
import json
import os
import platform
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
import cfr_br_lib  # noqa: E402
import dcfr_lib  # noqa: E402
import oracle_lib  # noqa: E402


def _digests(ref):
    t = ref.table()
    avg = ref.average_policy()
    assert avg == dcfr_lib.average_policy(t)
    return {"table_sha256": dcfr_lib.digests(t)["table_sha256"], "average_sha256": dcfr_lib.average_digest(avg)}


def main():
    assert dcfr_lib.ref_available(), "needs the OpenSpiel checkout and oracle/_ref"
    out = {"python": platform.python_version(), "numpy": np.__version__, "splits": {}, "zero_reach": {}}
    for gs, splits in dcfr_lib.REF_SPLITS.items():
        for variant in dcfr_lib.VARIANTS:
            ref = dcfr_lib.RefDCFR(gs, variant)
            pins, done = {}, 0
            for k in splits:
                ref.iterate(k)
                done += k
                pins[str(done)] = _digests(ref)
            out["splits"]["%s/%s" % (gs, variant)] = pins
    for gs, splits in dcfr_lib.ZERO_REACH_SPLITS.items():
        table = dcfr_lib.zero_reach_table(cfr_br_lib.legal_actions_by_key(oracle_lib.OracleGame(gs)), seed=dcfr_lib.ZERO_REACH_SEED)
        ref = dcfr_lib.RefDCFR(gs, "dcfr")
        ref.load(table, 3)
        pins, done = {}, 3
        for k in splits:
            ref.iterate(k)
            done += k
            pins[str(done)] = _digests(ref)
        out["zero_reach"][gs] = pins
    with open(dcfr_lib.GOLDEN, "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
        f.write("\n")


if __name__ == "__main__":
    main()
