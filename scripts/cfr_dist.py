#!/usr/bin/env python3
"""Multi-GPU CFR exchange, measured (run under torchrun, one rank per GPU):
  * exactness: in-library NCCL-sharded Leduc CFR and CFR+ vs the single-GPU solver at 1k / 10k / 100k iterations (max
    |delta| of cumulative regrets, cumulative policy, current policy; expected 0 — bit-identical).  CFR+'s linear averaging
    weights every average-policy increment by the iteration number, which the sharded loop keeps in a device counter
  * throughput: iterations/s of the sharded loop (16 iterations per CUDA-graph launch, no host code between the steps)
    vs the single-GPU persistent kernel
  * latency floor: device time of one ncclAllReduce of the contribution buffer (2C doubles), two of which every
    iteration needs whatever the kernels cost
  python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 --master-port 29531 scripts/cfr_dist.py [out.json]"""
import json
import os
import sys
import time

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import open_spiel_b200 as b2  # noqa: E402
from open_spiel_b200 import parallel  # noqa: E402

rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
torch.cuda.set_device(local)
dev = torch.device("cuda", local)
dist.init_process_group("nccl", device_id=dev)
game = b2.Game("leduc_poker", device=local)
VARIANTS = {"cfr": (False, False), "cfr_plus": (True, True)}      # (linear averaging, regret matching+)
solvers = {v: (parallel.DistributedCFRSolver(game, la, rm, in_library=True), b2.CFRSolver(game, la, rm))
           for v, (la, rm) in VARIANTS.items()}
sharded = solvers["cfr"][0]
res = {"world": world, "game": "leduc_poker", "contribution_doubles": int(sharded.delta.numel()),
       "checkpoints": {v: [] for v in VARIANTS}}
done = 0
for target in (1000, 10000, 100000):
    for v, (sh, single) in solvers.items():
        torch.cuda.synchronize(); dist.barrier()
        t0 = time.perf_counter()
        sh.evaluate_and_update_policy(target - done)
        torch.cuda.synchronize()
        t_sh = time.perf_counter() - t0
        t0 = time.perf_counter()
        single.evaluate_and_update_policy(target - done)
        torch.cuda.synchronize()
        t_1 = time.perf_counter() - t0
        ts, t1 = sh.table(), single.table()
        err = {f: float(np.abs(ts[f] - t1[f]).max()) for f in ("regrets", "cum_policy", "cur_policy")}
        res["checkpoints"][v].append({"iterations": target, "max_abs_diff": err,
                                      "bit_identical": all(np.array_equal(ts[f], t1[f]) for f in err),
                                      "iteration_counters": [sh.iteration, single.info().iteration],
                                      "sharded_iters_per_s": (target - done) / t_sh, "single_gpu_iters_per_s": (target - done) / t_1})
    done = target
for v, (sh, single) in solvers.items():
    res["exploitability_sharded_" + v] = sh.solver.exploitability()
    res["exploitability_single_" + v] = single.exploitability()
secs = sharded.allreduce_seconds(400)
res["allreduce_us"] = secs / 400 * 1e6
best = res["checkpoints"]["cfr"][-1]
res["iteration_us_single_gpu"] = 1e6 / best["single_gpu_iters_per_s"]
res["iteration_us_sharded"] = 1e6 / best["sharded_iters_per_s"]
res["floor_note"] = ("one iteration needs 2 all-reduces = %.1f us of exchange latency on top of two traversals whose level passes are "
                     "as long as the single-GPU kernel's (%.1f us per iteration): sharding a 9457-node tree cannot shorten them"
                     % (2 * res["allreduce_us"], res["iteration_us_single_gpu"]))
if rank == 0:
    print(json.dumps(res))
    if len(sys.argv) > 1:
        json.dump(res, open(sys.argv[1], "w"), indent=1)
dist.barrier()
dist.destroy_process_group()
