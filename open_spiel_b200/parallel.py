"""Multi-GPU plumbing: one process per GPU (torchrun), torch.distributed for the collectives.

The hot path shards by independent lanes / search roots, so stepping, rollouts and MCTS need no data-path
collective — each rank owns a contiguous slice of the global lane range and a disjoint slice of the random
stream space (lane_offset / tree_index_offset).  Only two things are ever exchanged:
  * a handful of int64 statistics per batch (wins / draws / plies, visit totals): `allreduce_stats`;
  * CFR's regret / average-policy deltas, once per player traversal: `DistributedCFRSolver`.
Works with backend "nccl" (CUDA tensors) and "gloo" (CPU tensors; used by the CPU tests of this logic).
"""
import ctypes as C

import torch

from ._lib import check, lib


def world():
    import torch.distributed as dist
    if dist.is_available() and dist.is_initialized():
        return dist.get_rank(), dist.get_world_size()
    return 0, 1


def shard_range(total, rank=None, world_size=None):
    """Contiguous, balanced slice [lo, hi) of `total` global lanes owned by `rank` (sizes differ by at most 1)."""
    if rank is None or world_size is None:
        rank, world_size = world()
    base, rem = divmod(int(total), int(world_size))
    lo = rank * base + min(rank, rem)
    return lo, lo + base + (1 if rank < rem else 0)


def allreduce_stats(t):
    """Sum a small statistics tensor over all ranks in place (no-op for a single process)."""
    import torch.distributed as dist
    if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
        dist.all_reduce(t, op=dist.ReduceOp.SUM)
    return t


def rollout_stats(returns, plies):
    """[p0 wins, p1 wins, draws, total plies, games] of a batch of finished playouts, summed over ranks."""
    r0 = returns[:, 0]
    s = torch.stack([(r0 > 0).sum(), (r0 < 0).sum(), (r0 == 0).sum(), plies.sum(), torch.tensor(plies.numel(), device=plies.device)])
    return allreduce_stats(s.to(torch.int64))


def lane_range(rank=None, world_size=None, lanes=64):
    """The reduction lanes [lo, hi) a rank owns in the lane-sharded MCCFR (world size must divide `lanes`)."""
    if rank is None or world_size is None:
        rank, world_size = world()
    if lanes % world_size:
        raise ValueError("world size must divide %d" % lanes)
    per = lanes // world_size
    return rank * per, (rank + 1) * per


def gather_lanes(partials, lo, hi):
    """All-gather along dim 0 in place: every rank contributes rows [lo, hi) of `partials` ([lanes, E]) and ends up with
    all rows.  NCCL: one all_gather_into_tensor; gloo (CPU tests): list all_gather."""
    import torch.distributed as dist
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size() == 1:
        return partials
    mine = partials[lo:hi].clone()
    if partials.is_cuda:
        dist.all_gather_into_tensor(partials, mine)
    else:
        pieces = [torch.empty_like(mine) for _ in range(dist.get_world_size())]
        dist.all_gather(pieces, mine)
        partials.copy_(torch.cat(pieces, dim=0))
    return partials


class _DevArray:
    """__cuda_array_interface__ view of library-owned device memory, so torch / NCCL can operate on it in place."""

    def __init__(self, ptr, n, typestr="<f8"):
        self.__cuda_array_interface__ = {"shape": (int(n),), "typestr": typestr, "data": (int(ptr), False), "version": 2}


class DistributedCFRSolver:
    """CFRSolver whose per-history regret / average-policy contributions are computed by rank (slot mod world), summed by
    an all-reduce and applied by every rank in the reference's order — tables stay replicated and BIT-IDENTICAL to the
    single-GPU solver (include/b2s.h).  in_library=True (default on CUDA with world > 1): the library owns an NCCL
    communicator and enqueues traverse -> ncclAllReduce -> apply itself, 16 iterations per CUDA-graph launch
    (b2s_cfr_iterate_sharded); in_library=False: this class performs the all-reduce with torch.distributed between the
    two library calls (works with gloo-backed tests via a CPU bounce of the buffer)."""

    def __init__(self, game, linear_averaging=False, regret_matching_plus=False, in_library=None):
        from .spiel import CFRSolver
        import torch.distributed as dist
        self.solver = CFRSolver(game, linear_averaging, regret_matching_plus)
        self.rank, self.world = world()
        ptr, cnt = C.c_void_p(), C.c_int64()
        check(lib().b2s_cfr_delta_buffer(self.solver._h, C.byref(ptr)))
        check(lib().b2s_cfr_delta_count(self.solver._h, C.byref(cnt)))
        self.delta = torch.as_tensor(_DevArray(ptr.value, cnt.value), device=torch.device("cuda", game.device))
        if in_library is None:
            in_library = self.world > 1 and dist.is_initialized() and dist.get_backend() == "nccl"
        self.in_library = bool(in_library)
        if self.in_library:
            ident = (C.c_char * 128)()
            if self.rank == 0:
                check(lib().b2s_nccl_unique_id(ident))
            box = [bytes(ident)]
            if self.world > 1:
                dist.broadcast_object_list(box, src=0)
            check(lib().b2s_cfr_comm_init(self.solver._h, box[0], self.rank, self.world))

    @property
    def iteration(self):
        """The wrapped solver's iteration counter (it moves with single-GPU calls and load_table too)."""
        return self.solver.info().iteration

    def evaluate_and_update_policy(self, iterations=1):
        L, h = lib(), self.solver._h
        st = C.c_void_p(torch.cuda.current_stream(self.delta.device).cuda_stream)
        if self.in_library:
            check(L.b2s_cfr_iterate_sharded(h, int(iterations), st))
            return
        for _ in range(int(iterations)):
            iteration = self.iteration + 1
            for player in (0, 1):
                check(L.b2s_cfr_traverse_shard(h, player, iteration, self.rank, self.world, st))
                allreduce_stats(self.delta)
                check(L.b2s_cfr_apply_deltas(h, st))
            check(L.b2s_cfr_set_iteration(h, iteration))

    def allreduce_seconds(self, count=200):
        """Device seconds of `count` back-to-back all-reduces of the contribution buffer (latency floor of the exchange)."""
        secs = C.c_double()
        check(lib().b2s_cfr_allreduce_probe(self.solver._h, int(count), C.byref(secs)))
        return secs.value

    def table(self):
        return self.solver.table()


class DistributedExternalSamplingMCCFRSolver:
    """ExternalSamplingMCCFRSolver whose traversals are split over the ranks, BIT-IDENTICAL to the single-GPU solver:
    the 64 lanes of the fixed-order delta reduction are dealt out to the ranks (world size must divide 64), every rank
    runs the traversals of its lanes and reduces them to per-lane partial sums, the lanes are all-gathered (NCCL), and
    every rank finishes the same reduction tree on the same numbers — tables stay replicated and identical."""

    LANES = 64

    def __init__(self, game, seed=0, traversals_per_update=1):
        from .spiel import ExternalSamplingMCCFRSolver
        self.solver = ExternalSamplingMCCFRSolver(game, seed, traversals_per_update)
        self.rank, self.world = world()
        self.lo, self.hi = lane_range(self.rank, self.world, self.LANES)
        dev = torch.device("cuda", game.device)
        self.partials = torch.zeros((self.LANES, self.solver._info.num_entries), dtype=torch.float64, device=dev)

    def run_iteration(self, iterations=1):
        L, h, s = lib(), self.solver._h, self.solver
        st = C.c_void_p(torch.cuda.current_stream(self.partials.device).cuda_stream)
        for _ in range(int(iterations)):
            for player in (0, 1):
                check(L.b2s_mccfr_traverse_lanes(h, player, s.traversals_per_update, s.seed, self.lo, self.hi,
                                                 self.partials.data_ptr(), st))
                gather_lanes(self.partials, self.lo, self.hi)
                check(L.b2s_mccfr_apply_partials(h, player, self.partials.data_ptr(), st))

    def table(self):
        return self.solver.table()

    def nash_conv(self):
        return self.solver.nash_conv()
