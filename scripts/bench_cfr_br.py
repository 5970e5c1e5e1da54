"""Device CFR-BR (k_cfr_br) iterations/s on kuhn_poker and leduc_poker beside k_cfr in the same run, the unmodified
reference CFRBRSolver's seconds per iteration on the host CPU (when oracle/_ref exists), and NashConv of the CFR and CFR-BR
average policies after 10^2, 10^3 and 10^4 iterations.  Prints one JSON line per result, the card and its power limit
first.  Usage: python scripts/bench_cfr_br.py"""
import json
import subprocess
import sys
import time

import torch

sys.path.insert(0, ".")
sys.path.insert(0, "tests")
import open_spiel_b200 as b2  # noqa: E402

ITERS = 10000      # b2s_cfr_iterate(N) per timed window
WINDOWS = 3


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return {"card": torch.cuda.get_device_name(0), "nvidia_smi": q[0] if q else None}


def device_rate(solver_cls, gs):
    """Iterations/s of one b2s_cfr_iterate(ITERS) launch, CUDA events around it, after a warm-up; one per window."""
    s = solver_cls(b2.load_game(gs))
    s.evaluate_and_update_policy(100)
    torch.cuda.synchronize()
    rates = []
    for _ in range(WINDOWS):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        s.evaluate_and_update_policy(ITERS)
        e1.record()
        e1.synchronize()
        rates.append(ITERS / (e0.elapsed_time(e1) * 1e-3))
    return rates


def reference_seconds_per_iteration(gs, iters):
    import cfr_br_lib
    import ref_lib
    if not cfr_br_lib.ref_available():
        return None
    r = cfr_br_lib.RefCFRBR(ref_lib.RefGame(gs))
    r.iterate(1)
    t0 = time.perf_counter()
    r.iterate(iters)
    return (time.perf_counter() - t0) / iters


def nash_conv_curve(gs):
    out = {}
    for name, cls in (("cfr", b2.CFRSolver), ("cfr_br", b2.CFRBRSolver)):
        s, done = cls(b2.load_game(gs)), 0
        for n in (100, 1000, 10000):
            s.evaluate_and_update_policy(n - done)
            done = n
            out.setdefault(name, {})[str(n)] = s.nash_conv()
    return out


if __name__ == "__main__":
    print(json.dumps(card()), flush=True)
    for gs, ref_iters in (("kuhn_poker", 200), ("leduc_poker", 3)):
        br, cfr = device_rate(b2.CFRBRSolver, gs), device_rate(b2.CFRSolver, gs)
        print(json.dumps({"game": gs, "iterations_per_window": ITERS, "cfr_br_iterations_per_s": br,
                          "cfr_iterations_per_s": cfr, "cfr_br_cost_over_cfr": sorted(cfr)[1] / sorted(br)[1],
                          "reference_cfr_br_seconds_per_iteration": reference_seconds_per_iteration(gs, ref_iters)}),
              flush=True)
        print(json.dumps({"game": gs, "nash_conv": nash_conv_curve(gs)}), flush=True)
