"""What the unmodified reference computed for the GPU tests that compare against it, stored in
tests/golden/reference_results.json (written by tests/golden/make_reference_results.py), so that the comparisons hold
where the reference build (oracle/_ref) does not exist.  Large outputs are stored as sha256 digests."""
import hashlib
import json
import os

import numpy as np

PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_results.json")


def reference_results():
    with open(PATH) as f:
        return json.load(f)


def array_digest(a):
    """sha256 of an array's dtype, shape and C-ordered bytes."""
    a = np.ascontiguousarray(a)
    h = hashlib.sha256()
    h.update(("%s%s" % (a.dtype.str, a.shape)).encode())
    h.update(a.tobytes())
    return h.hexdigest()


def table_digest(table):
    """sha256 of a tabular solver's {information state string: {"legal": [...], field: [...]}} dict, in key order,
    values as float64."""
    h = hashlib.sha256()
    for key in sorted(table):
        v = table[key]
        h.update(key.encode() + b"\0")
        h.update(np.asarray(v["legal"], dtype=np.int64).tobytes())
        for f in ("regrets", "cum_policy", "cur_policy"):
            if f in v:
                h.update(np.asarray(v[f], dtype=np.float64).tobytes())
    return h.hexdigest()


def device_table_by_key(dev_table, tensors):
    """A device CFRSolver.table() as the dict table_digest() takes; tensors maps information state strings to the
    information-state tensor bytes that key the device table (oracle_lib.infostate_tensors)."""
    key_of = {t: k for k, t in tensors.items()}
    out = {}
    for i in range(len(dev_table["players"])):
        lo, hi = dev_table["offsets"][i], dev_table["offsets"][i + 1]
        out[key_of[dev_table["keys"][i].tobytes()]] = {
            "legal": dev_table["legal_actions"][lo:hi].tolist(),
            **{f: dev_table[f][lo:hi].tolist() for f in ("regrets", "cum_policy", "cur_policy")}}
    return out
