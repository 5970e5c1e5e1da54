"""Device Discounted CFR (k_dcfr: DCFRSolver and LCFRSolver) iterations/s on kuhn_poker and leduc_poker beside k_cfr
(CFRSolver and CFRPlusSolver) in the same run, CUDA events around b2s_cfr_iterate(10,000) windows after a warm-up; NashConv
of the four solvers' average policies after 10^2, 10^3 and 10^4 iterations; the number of -0.0 regrets a 10^4-iteration
DCFR run ends with; and, as the CPU baseline, the host rate of the oracle's restatement of discounted_cfr.py
(oracle/algorithms/dcfr.cc; the reference's Python solver itself is about 400 times slower still on leduc_poker).  Prints one JSON line
per result, the card and its power limit first.  Usage: python scripts/bench_dcfr.py"""
import json
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, ".")
sys.path.insert(0, "tests")
import open_spiel_b200 as b2  # noqa: E402

ITERS = 10000      # b2s_cfr_iterate(N) per timed window
WINDOWS = 3
SOLVERS = {
    "dcfr": lambda g: b2.DCFRSolver(g),
    "lcfr": lambda g: b2.LCFRSolver(g),
    "cfr": lambda g: b2.CFRSolver(g),
    "cfr_plus": lambda g: b2.CFRSolver(g, linear_averaging=True, regret_matching_plus=True),
}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return {"card": torch.cuda.get_device_name(0), "nvidia_smi": q[0] if q else None}


def device_rates(gs):
    """Iterations/s of one b2s_cfr_iterate(ITERS) launch per solver and window, the solvers alternating within a window."""
    solvers = {name: make(b2.load_game(gs)) for name, make in SOLVERS.items()}
    for s in solvers.values():
        s.evaluate_and_update_policy(100)
    torch.cuda.synchronize()
    rates = {name: [] for name in solvers}
    for _ in range(WINDOWS):
        for name, s in solvers.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            s.evaluate_and_update_policy(ITERS)
            e1.record()
            e1.synchronize()
            rates[name].append(ITERS / (e0.elapsed_time(e1) * 1e-3))
    return rates


def restatement_seconds_per_iteration(gs, iters):
    import dcfr_lib
    import oracle_lib
    o = dcfr_lib.OracleDCFR(oracle_lib.OracleGame(gs), *dcfr_lib.VARIANTS["dcfr"])
    o.iterate(1)
    t0 = time.perf_counter()
    o.iterate(iters)
    return (time.perf_counter() - t0) / iters


def nash_conv_curve(gs):
    out = {}
    for name, make in SOLVERS.items():
        s, done = make(b2.load_game(gs)), 0
        for n in (100, 1000, 10000):
            s.evaluate_and_update_policy(n - done)
            done = n
            out.setdefault(name, {})[str(n)] = s.nash_conv()
        if name == "dcfr":
            r = s.table()["regrets"]
            out["dcfr_negative_zero_regrets_at_10000"] = int(np.sum((r == 0) & np.signbit(r)))
    return out


if __name__ == "__main__":
    print(json.dumps(card()), flush=True)
    for gs, host_iters in (("kuhn_poker", 20000), ("leduc_poker", 500)):
        rates = device_rates(gs)
        med = {k: sorted(v)[1] for k, v in rates.items()}
        print(json.dumps({"game": gs, "iterations_per_window": ITERS, "iterations_per_s": rates,
                          "dcfr_cost_over_cfr": med["cfr"] / med["dcfr"],
                          "restatement_dcfr_seconds_per_iteration": restatement_seconds_per_iteration(gs, host_iters)}),
              flush=True)
        print(json.dumps({"game": gs, "nash_conv": nash_conv_curve(gs)}), flush=True)
