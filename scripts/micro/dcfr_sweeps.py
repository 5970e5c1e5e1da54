"""What k_dcfr's split sweeps cost: DCFR iterations/s of this tree's k_dcfr (the reach sweep runs to the bottom before the
value sweep, so values can be pruned as the reference prunes them) against a variant built from the same source with
cfr_level_passes' fused sweeps (pruning at the table update only, which is not bit-exact with the reference).  The
variant is built in a temporary directory: a copy of open_spiel_b200/ (its object files included, so only cfr_full.cu
recompiles) with k_dcfr's two sweeps replaced by one cfr_level_passes call.  The two libraries run alternately, each in its
own process, through scripts/bench_dcfr.py's device_rates.  Prints one JSON line per run, the card and its power limit
first; writes nothing into the tree.  Run after build():  python scripts/micro/dcfr_sweeps.py"""
import json
import os
import shutil
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
SCRIPTS = os.path.join(ROOT, "scripts")
SPLIT_BEGIN = "      for (int n = 1 + tid; n < N; n += nt) d.edge_prob[n] = CurrentPolicyEdge{}(d, n, 0);\n"
SPLIT_END = "      for (int I = tid; I < d.n_infosets; I += nt) {\n        const int off = d.is_off[I], na"
RATES = ("import json, sys; sys.path.insert(0, %r); import bench_dcfr as b; "
         "print(json.dumps({g: {k: v for k, v in b.device_rates(g).items() if k in ('dcfr', 'cfr')} "
         "for g in ('kuhn_poker', 'leduc_poker')}))" % SCRIPTS)


def build_fused(tmp):
    shutil.copytree(os.path.join(ROOT, "open_spiel_b200"), os.path.join(tmp, "open_spiel_b200"),
                    ignore=shutil.ignore_patterns("__pycache__", "_build"))
    shutil.copytree(os.path.join(ROOT, "include"), os.path.join(tmp, "include"))
    src = os.path.join(tmp, "open_spiel_b200", "csrc", "cfr_full.cu")
    text = open(src).read()
    k = text.index("k_dcfr(CfrDev d")
    a = text.index(SPLIT_BEGIN, k)
    b = text.index(SPLIT_END, a)
    open(src, "w").write(text[:a] + "      cfr_level_passes(d, tid, nt);\n" + text[b:])
    subprocess.check_call(["make", "-s", "-C", os.path.join(tmp, "open_spiel_b200", "csrc")])


def rates(root):
    out = subprocess.run([sys.executable, "-c", RATES], cwd=root, capture_output=True, text=True, check=True)
    return json.loads(out.stdout.strip().splitlines()[-1])


if __name__ == "__main__":
    import torch
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    print(json.dumps({"card": torch.cuda.get_device_name(0), "nvidia_smi": q[0] if q else None}), flush=True)
    tmp = tempfile.mkdtemp()
    try:
        build_fused(tmp)
        for run in (1, 2):
            for name, root in (("split", ROOT), ("fused", tmp)):
                print(json.dumps({"run": run, "k_dcfr": name, "iterations_per_s": rates(root)}), flush=True)
    finally:
        shutil.rmtree(tmp)
