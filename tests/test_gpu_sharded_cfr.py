"""GPU: the sharded CFR loop at world size 1 — b2s_cfr_iterate_sharded (16 iterations per CUDA-graph launch, the rest one
by one, the iteration number kept in a device counter), the in-library communicator's lifecycle, DistributedCFRSolver on
both of its paths, resumed solvers, mixed sharded and single-GPU calls on one handle, and every CFRSolver call on a side
stream.  The reference is always CFRSolver with the same flags on the default stream, which test_gpu_cfr.py pins to the
oracle and to the unmodified reference: tables must be equal bit for bit, and so must the iteration counters.

Anything that creates an NCCL communicator or a torch process group runs in a child process, so the rest of the suite
never sees an initialised process group (DistributedCFRSolver's defaults and parallel.world() depend on it).  A child
prints one line per comparison, "@ <label> | ok" or "@ <label> | FAIL <what differs>", and this process asserts on them."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import open_spiel_b200 as b2

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FLAGS = {"vanilla": (False, False), "linear": (True, False), "rm_plus": (False, True), "cfr_plus": (True, True)}
FIELDS = ("regrets", "cum_policy", "cur_policy")
# calls of b2s_cfr_iterate_sharded: shorter than one graph, exactly one, one plus a remainder, several graph launches
SCHEDULES = ([1], [15], [16], [17], [16, 16], [1, 16, 3, 33], [100])

_CHILD = r"""
import ctypes as C, gc, json, math, sys
sys.path.insert(0, sys.argv[1])
import numpy as np
import torch
import torch.distributed as dist
import open_spiel_b200 as b2
from open_spiel_b200 import parallel
from open_spiel_b200._lib import check, lib

FLAGS = {"vanilla": (False, False), "linear": (True, False), "rm_plus": (False, True), "cfr_plus": (True, True)}
FIELDS = ("regrets", "cum_policy", "cur_policy")
GRAPH = 16        # kGraphIters: sharded iterations per CUDA-graph launch
DEV = torch.device("cuda", 0)


def line(label, problems):
    print("@ %s | %s" % (label, "ok" if not problems else "FAIL " + "; ".join(problems)), flush=True)


def snap(solver):
    t = solver.table()
    return {f: t[f] for f in FIELDS}, solver.info().iteration


def compare(label, got, want):
    (tg, ig), (tw, iw) = got, want
    problems = [f for f in FIELDS if not np.array_equal(tg[f], tw[f])]
    if ig != iw:
        problems.append("iteration %d, expected %d" % (ig, iw))
    line(label, problems)


def sharded_call(sh, n, label, captured):
    # b2s_launch_count counts k_cfr_traverse / k_cfr_apply when they are enqueued or captured into the graph, not when the
    # graph is replayed: 4 per iteration run without the graph, 4 * GRAPH once per capture.
    before = lib().b2s_launch_count()
    sh.evaluate_and_update_policy(n)
    counted = lib().b2s_launch_count() - before
    expect = 4 * (n % GRAPH) + (4 * GRAPH if n >= GRAPH and not captured else 0)
    line(label + " launches", [] if counted == expect else ["counted %d, expected %d" % (counted, expect)])
    return captured or n >= GRAPH


def nccl_group():
    # a world-1 NCCL process group without a TCP store; device_id creates its communicator now.  The library calls a
    # communicator it adopts with blocking NCCL calls, so the group's communicator is made blocking.
    opts = dist.ProcessGroupNCCL.Options()
    opts.config.blocking = 1
    dist.init_process_group("nccl", store=dist.HashStore(), rank=0, world_size=1, device_id=DEV, pg_options=opts)
    assert parallel.world() == (0, 1)


def case_schedules(gs, schedules):
    game = b2.load_game(gs)
    for name, (la, rm) in FLAGS.items():
        for sched in schedules:
            ref = b2.CFRSolver(game, la, rm)
            sh = parallel.DistributedCFRSolver(game, la, rm, in_library=True)
            done, captured = 0, False
            for n in sched:
                done += n
                label = "%s %s %s after %d" % (gs, name, sched, done)
                captured = sharded_call(sh, n, label, captured)
                ref.evaluate_and_update_policy(n)
                compare(label, snap(sh.solver), snap(ref))
            del sh, ref


def case_resume():
    for gs in ("kuhn_poker", "leduc_poker"):
        game = b2.load_game(gs)
        for name in ("linear", "cfr_plus"):
            la, rm = FLAGS[name]
            for k in (7, 40):
                src = b2.CFRSolver(game, la, rm)
                src.evaluate_and_update_policy(k)
                t = src.table()
                del src
                for in_library in (True, False):
                    ref = b2.CFRSolver(game, la, rm)
                    sh = parallel.DistributedCFRSolver(game, la, rm, in_library=in_library)
                    for s in (ref, sh.solver):
                        s.load_table(t["regrets"], t["cum_policy"], t["cur_policy"], iteration=k)
                    done = k
                    for n in (5, 16, 2):
                        done += n
                        label = "%s %s in_library=%s resumed at %d, after %d" % (gs, name, in_library, k, done)
                        sh.evaluate_and_update_policy(n)
                        ref.evaluate_and_update_policy(n)
                        compare(label, snap(sh.solver), snap(ref))
                        line(label + " DistributedCFRSolver.iteration",
                             [] if sh.iteration == done else ["%d, expected %d" % (sh.iteration, done)])
                    del sh, ref


def evaluations(solver):
    out = []
    for average in (True, False):
        nc = solver.nash_conv(average=average)
        actions, values = solver.best_response(average=average)
        out.append((nc, actions.tolist(), values))
    return out


def case_mixed():
    for gs in ("kuhn_poker", "leduc_poker"):
        game = b2.load_game(gs)
        for name in ("linear", "cfr_plus"):
            la, rm = FLAGS[name]
            ref = b2.CFRSolver(game, la, rm)
            sh = parallel.DistributedCFRSolver(game, la, rm, in_library=True)
            done = 0
            for how, n in (("sharded", 5), ("single", 3), ("sharded", 17), ("single", 1), ("sharded", 16),
                           ("single", 20), ("sharded", 3), ("sharded", 1)):
                done += n
                label = "%s %s %s %d, after %d" % (gs, name, how, n, done)
                if how == "sharded":
                    sh.evaluate_and_update_policy(n)
                else:
                    sh.solver.evaluate_and_update_policy(n)
                ref.evaluate_and_update_policy(n)
                before = snap(sh.solver)
                compare(label, before, snap(ref))
                got, want = evaluations(sh.solver), evaluations(ref)
                line(label + " nash_conv / best_response", [] if got == want else ["%r, expected %r" % (got, want)])
                compare(label + " tables after the evaluations", snap(sh.solver), before)
            del sh, ref


def case_side_stream():
    # Long calls (2,000 Leduc iterations) right before table() / nash_conv() / best_response(): a read that is not ordered
    # after them on the caller's stream sees tables half-way through.
    game = b2.load_game("leduc_poker")
    la, rm = FLAGS["cfr_plus"]
    src = b2.CFRSolver(game, la, rm)
    src.evaluate_and_update_policy(7)
    t = src.table()
    del src
    load = lambda s: s.load_table(t["regrets"], t["cum_policy"], t["cur_policy"], iteration=7)   # noqa: E731
    schedule = (16, 3, 2000)

    def run(solver, iterate):
        iterate(2000)          # still running when load_table is queued behind it
        load(solver)
        for n in schedule:
            iterate(n)
        first = snap(solver)
        iterate(2000)
        nc = [solver.nash_conv()]
        iterate(2000)
        actions, values = solver.best_response()
        return first, nc + [actions.tolist(), values], snap(solver)

    ref = b2.CFRSolver(game, la, rm)
    want = run(ref, ref.evaluate_and_update_policy)
    del ref
    s = torch.cuda.Stream()
    assert s.cuda_stream != 0
    for kind in ("CFRSolver", "DistributedCFRSolver"):
        with torch.cuda.stream(s):
            if kind == "CFRSolver":
                x = b2.CFRSolver(game, la, rm)
                got = run(x, x.evaluate_and_update_policy)
            else:
                x = parallel.DistributedCFRSolver(game, la, rm, in_library=True)
                got = run(x.solver, x.evaluate_and_update_policy)
        compare("%s on a side stream: table() after %s" % (kind, schedule), got[0], want[0])
        line("%s on a side stream: nash_conv(), best_response()" % kind,
             [] if got[1] == want[1] else ["%r, expected %r" % (got[1], want[1])])
        compare("%s on a side stream: final tables" % kind, got[2], want[2])
        s.synchronize()
        del x


def case_comm():
    game = b2.load_game("leduc_poker")
    la, rm = FLAGS["cfr_plus"]
    ref = b2.CFRSolver(game, la, rm)
    sh = parallel.DistributedCFRSolver(game, la, rm, in_library=True)
    state = {"done": 0, "captured": False}

    def step(what, n):
        state["done"] += n
        label = "%s, %d iterations (after %d)" % (what, n, state["done"])
        state["captured"] = sharded_call(sh, n, label, state["captured"])
        ref.evaluate_and_update_policy(n)
        compare(label, snap(sh.solver), snap(ref))

    step("own communicator", 20)
    # a second b2s_cfr_comm_init replaces the communicator and drops the graph captured with the old one: the next
    # call of 16 or more iterations captures again (visible in the launch count)
    ident = (C.c_char * 128)()
    check(lib().b2s_nccl_unique_id(ident))
    check(lib().b2s_cfr_comm_init(sh.solver._h, ident, 0, 1))
    state["captured"] = False
    step("re-initialised communicator", 17)
    step("re-initialised communicator", 16)
    secs = sh.allreduce_seconds(50)
    line("allreduce probe %r s" % secs, [] if math.isfinite(secs) and secs > 0 else ["not a positive time"])
    step("after the probe", 5)
    step("after the probe", 32)        # the probe's own graph leaves the cached one alone
    nccl_group()
    comm = dist.group.WORLD._get_backend(DEV)._comm_ptr()
    line("process group communicator", [] if comm else ["null"])
    check(lib().b2s_cfr_comm_adopt(sh.solver._h, C.c_void_p(comm), 0, 1))
    state["captured"] = False
    step("adopted communicator", 17)
    step("adopted communicator", 33)
    step("adopted communicator", 2)
    del sh, ref
    gc.collect()
    # the solver is gone; the communicator it adopted still belongs to the process group
    x = torch.arange(1, 9, dtype=torch.float64, device=DEV)
    dist.all_reduce(x)
    torch.cuda.synchronize()
    line("all_reduce after the adopting solver was destroyed",
         [] if torch.equal(x.cpu(), torch.arange(1, 9, dtype=torch.float64)) else ["%r" % x.tolist()])
    dist.destroy_process_group()


def case_mccfr():
    nccl_group()
    for gs, K in (("kuhn_poker", 1), ("kuhn_poker", 64), ("leduc_poker", 1), ("leduc_poker", 64), ("leduc_poker", 1000),
                  ("leduc_poker", 4096)):
        game = b2.load_game(gs)
        single = b2.ExternalSamplingMCCFRSolver(game, seed=29 + K, traversals_per_update=K)
        sh = parallel.DistributedExternalSamplingMCCFRSolver(game, seed=29 + K, traversals_per_update=K)
        single.run_iteration(3)
        sh.run_iteration(3)
        label = "%s K=%d after 3" % (gs, K)
        compare(label, snap(sh.solver), snap(single))
        a, b = sh.nash_conv(), single.nash_conv()
        line(label + " nash_conv", [] if a == b else ["%r, expected %r" % (a, b)])
        del sh, single
    dist.destroy_process_group()


case, args = sys.argv[2], json.loads(sys.argv[3])
globals()["case_" + case](*args)
gc.collect()
torch.cuda.synchronize()
print("@@ done", flush=True)
"""


def run_child(case, *args, timeout=600):
    """Runs one case of _CHILD in a fresh interpreter; returns its "@" lines as (label, verdict) pairs."""
    env = dict(os.environ, NCCL_SOCKET_IFNAME="lo")       # the NCCL bootstrap stays on loopback
    r = subprocess.run([sys.executable, "-c", _CHILD, ROOT, case, json.dumps(args)], capture_output=True, text=True,
                       env=env, timeout=timeout)
    assert r.returncode == 0, (r.stdout[-2000:], r.stderr[-4000:])
    out = r.stdout.splitlines()
    assert out and out[-1] == "@@ done", r.stdout[-2000:]
    lines = [ln[2:].split(" | ", 1) for ln in out if ln.startswith("@ ")]
    failed = [ln for ln in lines if ln[1] != "ok"]
    assert not failed, "\n".join("%s: %s" % tuple(ln) for ln in failed)
    return lines


@pytest.mark.parametrize("gs", ["kuhn_poker", "leduc_poker"])
def test_graph_and_remainder_schedules(gs):
    """DistributedCFRSolver(in_library=True) on a fresh solver per schedule, every flag combination: tables and iteration
    counter after every call, and the launch count of every call."""
    lines = run_child("schedules", gs, SCHEDULES)
    assert len(lines) == 2 * len(FLAGS) * sum(len(s) for s in SCHEDULES)


def test_resumed_solver_continues_from_its_iteration():
    """Tables and iteration k loaded through .solver.load_table, then 5, 16 and 2 more iterations, on both paths of
    DistributedCFRSolver, with linear averaging (where the iteration number weights the average policy)."""
    lines = run_child("resume")
    assert len(lines) == 2 * 2 * 2 * 2 * 3 * 2


def test_sharded_and_single_gpu_calls_on_one_handle():
    """Sharded and single-GPU iterations alternate on one solver, with NashConv and best responses of the average and the
    current policy in between: the evaluations change no table and equal the reference's."""
    lines = run_child("mixed")
    assert len(lines) == 2 * 2 * 8 * 3


def test_every_call_is_ordered_on_a_side_stream():
    """CFRSolver and the sharded solver driven entirely inside `with torch.cuda.stream(s)` (a non-blocking stream): a
    load_table queued behind running iterations, then table(), nash_conv() and best_response() right after long calls,
    with no synchronisation of the caller's."""
    lines = run_child("side_stream")
    assert len(lines) == 2 * 3


def test_communicator_lifecycle():
    """Re-initialising the communicator, the all-reduce probe and adopting a process group's communicator leave the tables
    bit-identical; destroying the adopting solver leaves that communicator usable."""
    lines = run_child("comm")
    assert len(lines) == 2 * 8 + 3


def test_sharded_mccfr_in_an_nccl_process_group():
    """DistributedExternalSamplingMCCFRSolver in a world-1 NCCL process group equals ExternalSamplingMCCFRSolver: tables,
    iteration counter and NashConv."""
    lines = run_child("mccfr")
    assert len(lines) == 6 * 2


def emulated_shards(game, la, rm, iters, shards):
    """The caller-driven sharded path with `shards` ranks evaluated one after the other on one GPU and their contribution
    buffers summed by hand — what the all-reduce does, every slot being one rank's value plus zeros."""
    import torch
    from open_spiel_b200 import parallel
    from open_spiel_b200._lib import check, lib
    multi = parallel.DistributedCFRSolver(game, la, rm, in_library=False)
    L, h = lib(), multi.solver._h
    for it in range(1, iters + 1):
        for player in (0, 1):
            acc = torch.zeros_like(multi.delta)
            for shard in range(shards):
                check(L.b2s_cfr_traverse_shard(h, player, it, shard, shards, None))
                torch.cuda.synchronize()
                acc += multi.delta
            multi.delta.copy_(acc)
            check(L.b2s_cfr_apply_deltas(h, None))
    return multi.table()


@pytest.mark.parametrize("gs,flag", [("kuhn_poker", "vanilla"), ("kuhn_poker", "linear"), ("kuhn_poker", "rm_plus"),
                                     ("kuhn_poker", "cfr_plus"), ("leduc_poker", "linear"), ("leduc_poker", "rm_plus")])
def test_emulated_multi_rank_path_every_flag(gs, flag):
    """test_gpu_cfr.py's emulated 3- and 8-rank exchange (Leduc, vanilla and CFR+ there) for the other flag combinations
    and for Kuhn, plus DistributedCFRSolver(in_library=False) at world 1."""
    from open_spiel_b200 import parallel
    la, rm = FLAGS[flag]
    game = b2.load_game(gs)
    iters = 40
    ref = b2.CFRSolver(game, la, rm)
    ref.evaluate_and_update_policy(iters)
    want = ref.table()
    one = parallel.DistributedCFRSolver(game, la, rm, in_library=False)
    one.evaluate_and_update_policy(iters)
    assert one.solver.info().iteration == iters
    tables = {1: one.table()}
    for shards in (3, 8):
        tables[shards] = emulated_shards(game, la, rm, iters, shards)
    for shards, t in tables.items():
        for f in FIELDS:
            assert np.array_equal(t[f], want[f]), (gs, flag, shards, f)
    assert np.abs(want["regrets"]).max() > 0.1
