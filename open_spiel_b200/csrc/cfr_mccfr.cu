// External-sampling and outcome-sampling MCCFR on the CFR solver's flattened tree and tables (cfr.cuh, cfr_tree.cu).
#include <string.h>

#include <algorithm>

#include "cfr.cuh"

namespace b2s {

// ---- external-sampling MCCFR (external_sampling_mccfr.cc) ----------------------------------------------------
// One thread = one UpdateRegrets traversal (:124-186) of traverser p over the flattened tree, as an explicit-stack
// DFS: chance and opponent nodes are sampled and followed (no frame), the traverser's decision nodes keep a frame
// (policy, child values) until all actions are explored.  Tables are read-only here; each traversal writes its deltas
// to its own delta log (in phase p an entry of player p receives a regret delta, an entry of the other player an
// average-policy delta, so one log serves both), which the reduction kernels below add in a fixed order.
// z(node) = U53(Philox4x32-10(seed; path hash, phase, k)) — the stream oracle/algorithms/mccfr.cc (rng_mode 1) restates.
constexpr int kMcMaxActions = 8;
constexpr int kMcMaxDepth = 32;

__device__ __forceinline__ double mc_uniform(u64 seed, u64 h, u32 phase, u32 k) {
  u32 r[4];
  philox4(seed, h, phase, k, r);
  u64 bits = (((u64)r[1] << 32) | r[0]) >> 11;
  return __dmul_rn((double)bits, 1.0 / 9007199254740992.0);
}
__device__ __forceinline__ u64 mc_child_hash(u64 h, int idx) { return h * 0x9E3779B97F4A7C15ull + (u64)(idx + 1); }

// SampleAction(ChanceOutcomes(), z), spiel.cc:372-409: the outcome whose cumulative-probability interval holds z.  When
// none does, the error counter is raised and the last outcome taken.
__device__ __forceinline__ int mc_chance_outcome(const double* prob, int n, double z, int* err) {
  double sum = 0.0;
  for (int c = 0; c < n; ++c) {
    if (sum <= z && z < __dadd_rn(sum, prob[c])) return c;
    sum = __dadd_rn(sum, prob[c]);
  }
  atomicAdd(err, 1);
  return n - 1;
}

// Sharding: the rank that owns reduction lanes [lane_begin, lane_begin + L) runs the traversals k with k mod 64 in
// that range; thread t is traversal k = lane_begin + t mod L + 64 (t div L) and owns log t.  One GPU: L = 64, k = t.
//
// A delta log is log[t][0 .. counts[t]) of {table entry, value} records.  A traversal touches an entry at most once (perfect
// recall: the information states on the paths of one traversal differ in the traverser's own actions), so a log holds the
// non-zero cells of a [E] delta row — a few dozen records instead of E cells.
struct McLog {
  int4* rec;      // [threads][cap]: {entry, 0, value bits lo, value bits hi}
  int* counts;    // [threads]
  int cap;        // records per traversal: an exact upper bound from the tree (mccfr_log_capacity)
};
__device__ __forceinline__ void mc_log_append(const McLog& lg, int t, int& cnt, int entry, double v, int* err) {
  if (v == 0.0) return;                                  // a dense row cannot tell a zero delta from an untouched cell either
  if (cnt >= lg.cap) { atomicAdd(err, 1); return; }
  const long long bits = __double_as_longlong(v);
  lg.rec[(size_t)t * lg.cap + cnt++] = make_int4(entry, 0, (int)(u32)bits, (int)(u32)((u64)bits >> 32));
}

__global__ void __launch_bounds__(128) k_mccfr_es(CfrDev d, int p, u32 phase, u64 seed, int K, int lane_begin, int L, int n_threads,
                                                   McLog lg, int* __restrict__ err, int simple_average) {
  int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n_threads) return;
  int k = lane_begin + t % L + 64 * (t / L);
  if (k >= K) { lg.counts[t] = 0; return; }
  int cnt = 0;
  struct Frame { int node, a, n, off; double v; u64 h; double cv[kMcMaxActions], sig[kMcMaxActions]; };
  Frame st[kMcMaxDepth];
  int sp = 0, node = 0;
  u64 h = 0;
  for (;;) {
    // ---- descend until a value is produced ----
    double r;
    for (;;) {
      const int4 rec = __ldg(d.mc_node + node);          // one 16-byte load per node instead of five dependent ones
      const int kind = rec.z & 0xff, actor = (rec.z >> 8) & 0xff, n = rec.z >> 16, fc = rec.x;
      if (kind == 0) { r = d.ret[2 * node + p]; break; }
      if (kind == 1) {
        double z = mc_uniform(seed, h, phase, (u32)k);
        int chosen = n == 1 ? 0 : mc_chance_outcome(d.chance_prob + fc, n, z, err);
        h = mc_child_hash(h, chosen);
        node = fc + chosen;
        continue;
      }
      const int off = rec.y;
      double sig[kMcMaxActions];
      regret_matching(d.regrets + off, sig, n);         // ApplyRegretMatching on a copy
      if (actor != p) {                                  // opponent: SampleActionIndex(0, z), cfr.cc:617-628
        double z = mc_uniform(seed, h, phase, (u32)k);
        int aidx = -1;
        double sum = 0.0;
        for (int a = 0; a < n; ++a) {
          if (z >= sum && z < __dadd_rn(sum, sig[a])) { aidx = a; break; }
          sum = __dadd_rn(sum, sig[a]);
        }
        if (aidx < 0) { atomicAdd(err, 1); aidx = n - 1; }
        if (simple_average && actor == ((p + 1) & 1))    // simple averaging at the next player's nodes (:176-183)
          for (int a = 0; a < n; ++a) mc_log_append(lg, t, cnt, off + a, sig[a], err);
        h = mc_child_hash(h, aidx);
        node = fc + aidx;
        continue;
      }
      Frame& f = st[sp++];                               // traverser: walk every action (:156-163)
      f.node = node; f.a = 0; f.n = n; f.off = off; f.v = 0.0; f.h = h;
      for (int a = 0; a < n; ++a) f.sig[a] = sig[a];
      h = mc_child_hash(f.h, 0);
      node = fc;
    }
    // ---- hand the value to the waiting frames ----
    bool done = false;
    for (;;) {
      if (sp == 0) { done = true; break; }
      Frame& f = st[sp - 1];
      f.cv[f.a] = r;
      f.v = __dadd_rn(f.v, __dmul_rn(f.sig[f.a], r));
      ++f.a;
      if (f.a < f.n) { node = d.first_child[f.node] + f.a; h = mc_child_hash(f.h, f.a); break; }
      for (int a = 0; a < f.n; ++a)                      // regret += child value - node value (:168-172)
        mc_log_append(lg, t, cnt, f.off + a, __dsub_rn(f.cv[a], f.v), err);
      r = f.v;
      --sp;
    }
    if (done) break;
  }
  lg.counts[t] = cnt;
}

// tables += the sum of the K traversal rows, in a FIXED order so the result is reproducible (and restated by the
// oracle): 64 partial sums, partial[q] = delta[q] + delta[q+64] + delta[q+128] + ... (sequential, from 0.0), combined
// by the tree partial[q] += partial[q+s], s = 32, 16, 8, 4, 2, 1; table += partial[0].  With K = 1 this is
// table += delta[0].  A block owns 16 consecutive table entries (x) and the 64 partial lanes (y): every row is read
// in 128-byte coalesced segments, 8 independent loads in flight per thread.  Touched cells are re-zeroed for the
// next phase.
constexpr int kMcLanes = 64, kMcTile = 16;
// The tree over the 64 lane partial sums part[.][ex] of table entry e, then the entry += partial[0]: an entry of player p receives
// a regret delta, an entry of the other player an average-policy delta (mode 0), every entry -> regrets (1) / cumulative policy (2).
__device__ __forceinline__ void mc_add_lanes(const CfrDev& d, int p, int mode, double (&part)[kMcLanes][kMcTile + 1], int q, int ex, int e) {
  __syncthreads();
  for (int s = kMcLanes / 2; s >= 1; s >>= 1) {
    if (q < s) part[q][ex] = __dadd_rn(part[q][ex], part[q + s][ex]);
    __syncthreads();
  }
  if (q == 0 && e < d.n_entries) {
    double* dst = mode == 0 ? (d.entry_player[e] == p ? d.regrets + e : d.cum_policy + e) : (mode == 1 ? d.regrets + e : d.cum_policy + e);
    *dst = __dadd_rn(*dst, part[0][ex]);
  }
}
// `stride` = doubles per row (E for external sampling, 2E for outcome sampling: two passes over the two halves of its rows).
__global__ void __launch_bounds__(kMcLanes * kMcTile) k_mccfr_apply(CfrDev d, int p, int K, double* __restrict__ rows, int stride, int mode) {
  __shared__ double part[kMcLanes][kMcTile + 1];
  const int E = d.n_entries;
  const int ex = threadIdx.x, q = threadIdx.y;
  const int e = blockIdx.x * kMcTile + ex;
  double acc = 0.0;
  if (e < E) {
    constexpr int U = 8;
    int k = q;
    for (; k + kMcLanes * (U - 1) < K; k += kMcLanes * U) {
      double v[U];
#pragma unroll
      for (int u = 0; u < U; ++u) v[u] = rows[(size_t)(k + kMcLanes * u) * stride + e];
#pragma unroll
      for (int u = 0; u < U; ++u)
        if (v[u] != 0.0) { acc = __dadd_rn(acc, v[u]); rows[(size_t)(k + kMcLanes * u) * stride + e] = 0.0; }
    }
    for (; k < K; k += kMcLanes) {
      double* cell = rows + (size_t)k * stride + e;
      double v = *cell;
      if (v != 0.0) { acc = __dadd_rn(acc, v); *cell = 0.0; }
    }
  }
  part[q][ex] = acc;
  mc_add_lanes(d, p, mode, part, q, ex, e);
}

// Sharded form of k_mccfr_apply, step 1: the partial sums of lanes [lane_begin, lane_begin + L) from this rank's rows
// (row t holds traversal k = lane_begin + t mod L + 64 (t div L)) into partials[64][E].
__global__ void __launch_bounds__(1024) k_mccfr_partial(CfrDev d, int K, int lane_begin, int L, double* __restrict__ rows, double* __restrict__ partials) {
  const int E = d.n_entries;
  const int e = blockIdx.x * kMcTile + threadIdx.x, ql = threadIdx.y;
  if (e >= E || ql >= L) return;
  double acc = 0.0;
  for (int j = 0; lane_begin + ql + 64 * j < K; ++j) {
    double* cell = rows + (size_t)(ql + L * j) * E + e;
    double v = *cell;
    if (v != 0.0) { acc = __dadd_rn(acc, v); *cell = 0.0; }
  }
  partials[(size_t)(lane_begin + ql) * E + e] = acc;
}
// The same partial sums straight from the delta logs.  The order is the row kernels' — lane q adds the deltas of its
// traversals k = q, q + 64, q + 128, ... one after the other, from 0.0 — so the result is bit-identical; what changes is the
// traffic: the records of the K traversals (tens of bytes each) instead of K rows of E doubles.  One block per lane keeps that
// lane's partial row in shared memory; the records of one traversal go to distinct entries and are added in parallel,
// traversals are separated by a barrier.  The chain over a lane's K / 64 traversals is sequential by definition, so the
// loads run kMcPrefetch traversals ahead of the adds (a register ring) to keep the chain at barrier + shared-memory speed.
// `width` = entries per partial row (E, or 2E for outcome sampling: regret deltas then average-policy deltas).
constexpr int kMcPrefetch = 16, kMcLogThreads = 256;
__global__ void __launch_bounds__(kMcLogThreads) k_mccfr_partial_log(int K, int lane_begin, int L, McLog lg, int width, double* __restrict__ partials) {
  extern __shared__ double mc_part[];
  const int ql = blockIdx.x, q = lane_begin + ql, tid = threadIdx.x;
  for (int e = tid; e < width; e += kMcLogThreads) mc_part[e] = 0.0;
  __syncthreads();
  const int nj = q < K ? (K - q + 63) / 64 : 0;          // traversal j of this lane is k = q + 64 j, held by thread row ql + L j
  int n[kMcPrefetch];
  int4 rec[kMcPrefetch];
  // the record is loaded whether or not slot `tid` is in use (validity is decided at the add, from the count): a load that
  // waited for the count would stall the in-order warp for a full memory latency per traversal and undo the prefetch
  auto fetch = [&](int j, int& nn, int4& r) {
    nn = 0;
    if (j < nj) {
      const size_t row = (size_t)ql + (size_t)L * j;
      nn = lg.counts[row];
      if (tid < lg.cap) r = lg.rec[row * lg.cap + tid];
    }
  };
  auto add = [&](const int4& r) {
    const double v = __longlong_as_double((long long)(((u64)(u32)r.w << 32) | (u32)r.z));
    mc_part[r.x] = __dadd_rn(mc_part[r.x], v);
  };
#pragma unroll
  for (int u = 0; u < kMcPrefetch; ++u) fetch(u, n[u], rec[u]);
  for (int j0 = 0; j0 < nj; j0 += kMcPrefetch) {
#pragma unroll
    for (int u = 0; u < kMcPrefetch; ++u) {
      const int j = j0 + u;
      if (j < nj) {                                      // uniform over the block
        if (tid < n[u]) add(rec[u]);
        if (n[u] > kMcLogThreads) {
          const size_t row = (size_t)ql + (size_t)L * j;
          for (int i = tid + kMcLogThreads; i < n[u]; i += kMcLogThreads) add(lg.rec[row * lg.cap + i]);
        }
        __syncthreads();
      }
      fetch(j + kMcPrefetch, n[u], rec[u]);
    }
  }
  for (int e = tid; e < width; e += kMcLogThreads) partials[(size_t)q * width + e] = mc_part[e];
}

// Log -> dense rows: one thread per record slot.  The traversal kernels are latency chains (a few thousand threads walking a
// tree); letting them also read-modify-write dense delta rows lengthens those chains, whereas scattering the same records
// from a kernel of its own is a few microseconds of fully parallel stores.  Entries are distinct within a traversal and the
// rows are zero between phases (k_mccfr_apply and k_mccfr_partial re-zero what they read), so a plain store suffices.
__global__ void __launch_bounds__(256) k_mccfr_scatter(McLog lg, long long slots, int stride, double* __restrict__ rows) {
  const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= slots) return;
  const long long t = g / lg.cap;
  const int j = (int)(g - t * lg.cap);
  if (j >= lg.counts[t]) return;
  const int4 r = lg.rec[g];
  rows[(size_t)t * stride + r.x] = __longlong_as_double((long long)(((u64)(u32)r.w << 32) | (u32)r.z));
}

// step 2 (after the lanes of all ranks have been gathered): the tree over the 64 lanes, then table += partial[0].
// `partials` = [64][stride]; mode as in k_mccfr_apply (0: by the entry's player, 1: regrets, 2: cumulative policy).
__global__ void __launch_bounds__(kMcLanes * kMcTile) k_mccfr_combine(CfrDev d, int p, const double* __restrict__ partials, int stride, int mode) {
  __shared__ double part[kMcLanes][kMcTile + 1];
  const int E = d.n_entries;
  const int ex = threadIdx.x, q = threadIdx.y;
  const int e = blockIdx.x * kMcTile + ex;
  part[q][ex] = e < E ? partials[(size_t)q * stride + e] : 0.0;
  mc_add_lanes(d, p, mode, part, q, ex, e);
}

// ---- AverageType::kFull of external sampling (external_sampling_mccfr.cc:188-230) ------------------------------------------
// Once per iteration, after both players' traversals: regret matching for every information state, players' reach
// probabilities down the whole tree (chance nodes pass them through), then every information state adds
// reach[its player](h) * policy[a] for its histories h in DFS order — the order the reference's post-order recursion
// produces for the (same-depth, disjoint) histories of one information state.  The reference prunes subtrees whose reach
// vector is all zero; their contributions would be +0.0 to tables that are never -0.0, so nothing changes.
__global__ void __launch_bounds__(1024) k_mccfr_full_average(CfrDev d) {
  const int tid = threadIdx.x, nt = blockDim.x;
  for (int I = tid; I < d.n_infosets; I += nt) {
    int off = d.is_off[I], na = d.is_off[I + 1] - off;
    regret_matching(d.regrets + off, d.cur_policy + off, na);
  }
  __syncthreads();
  cfr_level_passes(d, tid, nt);
  for (int I = tid; I < d.n_infosets; I += nt) {
    const int off = d.is_off[I], na = d.is_off[I + 1] - off, pl = d.is_player[I];
    for (int hh = d.hist_off[I]; hh < d.hist_off[I + 1]; ++hh) {
      const double r = d.reach[2 * d.hist[hh] + pl];
      for (int a = 0; a < na; ++a) d.cum_policy[off + a] = __dadd_rn(d.cum_policy[off + a], __dmul_rn(r, d.cur_policy[off + a]));
    }
  }
}

// ---- outcome-sampling MCCFR (outcome_sampling_mccfr.cc, default uniform policy, no baseline) ---------------------------------
// One thread = one SampleEpisode (:150-247) of update player p: a single sampled path to a terminal node (epsilon-on-policy
// at p's nodes :139-147, on-policy elsewhere, chance by its distribution), then the importance-weighted value estimates are
// unwound and every node of p on the path contributes regret and average-policy deltas to log k (entries of a [2E] row:
// regret deltas, then average-policy deltas), which the reduction kernels add in their fixed order.  Tables are read-only here.
// u(node, redraw) = U53(Philox(seed; h + 0x632BE59BD9B4E019 redraw, phase, k)); a draw is lo + u (hi - lo), redrawn while it
// rounds up to hi — the stream and the two samplers oracle/algorithms/os_mccfr.cc (rng_mode 1) restates.
__device__ __forceinline__ double os_real(u64 seed, u64 h, u32 phase, u32 k, double lo, double hi) {
  for (u32 redraw = 0;; ++redraw) {
    double u = mc_uniform(seed, h + 0x632BE59BD9B4E019ull * (u64)redraw, phase, k);
    double r = __dadd_rn(lo, __dmul_rn(u, __dsub_rn(hi, lo)));
    if (r < hi || lo == hi) return r;
  }
}

__global__ void __launch_bounds__(128) k_mccfr_os(CfrDev d, int p, u32 phase, u64 seed, int K, double epsilon, McLog lg, int* __restrict__ err) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= K) return;
  const int E = d.n_entries;
  int cnt = 0;
  struct Frame { int off, n, sampled, actor; double my_reach, opp_reach, sample_reach, sample_prob; double sig[kMcMaxActions]; };
  Frame st[kMcMaxDepth];
  int sp = 0, node = 0;
  u64 h = 0;
  double my_reach = 1.0, opp_reach = 1.0, sample_reach = 1.0, value;
  for (;;) {
    const int4 rec = __ldg(d.mc_node + node);
    const int kind = rec.z & 0xff, actor = (rec.z >> 8) & 0xff, n = rec.z >> 16, fc = rec.x;
    if (kind == 0) { value = d.ret[2 * node + p]; break; }
    if (kind == 1) {
      const int chosen = mc_chance_outcome(d.chance_prob + fc, n, os_real(seed, h, phase, (u32)k, 0.0, 1.0), err);
      const double prob = d.chance_prob[fc + chosen];
      opp_reach = __dmul_rn(prob, opp_reach);
      sample_reach = __dmul_rn(prob, sample_reach);
      h = mc_child_hash(h, chosen);
      node = fc + chosen;
      continue;
    }
    Frame& f = st[sp++];
    f.off = rec.y; f.n = n; f.actor = actor;
    f.my_reach = my_reach; f.opp_reach = opp_reach; f.sample_reach = sample_reach;
    regret_matching(d.regrets + f.off, f.sig, n);       // info_state_copy.ApplyRegretMatching()
    double sp_a[kMcMaxActions], total = 0.0;             // SamplePolicy (:139-147) / the current policy; discrete_distribution
    for (int a = 0; a < n; ++a) {
      sp_a[a] = actor == p ? __dadd_rn(__ddiv_rn(__dmul_rn(epsilon, 1.0), (double)n), __dmul_rn(__dsub_rn(1.0, epsilon), f.sig[a])) : f.sig[a];
      total = __dadd_rn(total, sp_a[a]);
    }
    const double u = os_real(seed, h, phase, (u32)k, 0.0, total);
    int sampled = n - 1;
    double acc = 0.0;
    for (int a = 0; a < n; ++a) { acc = __dadd_rn(acc, sp_a[a]); if (u < acc) { sampled = a; break; } }
    f.sampled = sampled; f.sample_prob = sp_a[sampled];
    if (actor == p) my_reach = __dmul_rn(my_reach, f.sig[sampled]); else opp_reach = __dmul_rn(opp_reach, f.sig[sampled]);
    sample_reach = __dmul_rn(sample_reach, sp_a[sampled]);
    h = mc_child_hash(h, sampled);
    node = fc + sampled;
  }
  // ---- unwind: child values, value estimates, updates at the update player's nodes (:206-245) ----
  while (sp > 0) {
    const Frame& f = st[--sp];
    double value_estimate = 0.0, cv_sampled = __dadd_rn(0.0, __ddiv_rn(__dsub_rn(value, 0.0), f.sample_prob));
    for (int a = 0; a < f.n; ++a) value_estimate = __dadd_rn(value_estimate, __dmul_rn(f.sig[a], a == f.sampled ? cv_sampled : 0.0));
    if (f.actor == p) {
      const double cf_value = __ddiv_rn(__dmul_rn(value_estimate, f.opp_reach), f.sample_reach);
      for (int a = 0; a < f.n; ++a) {
        const double cv = a == f.sampled ? cv_sampled : 0.0;
        const double cf_action_value = __ddiv_rn(__dmul_rn(cv, f.opp_reach), f.sample_reach);
        mc_log_append(lg, k, cnt, f.off + a, __dsub_rn(cf_action_value, cf_value), err);
        mc_log_append(lg, k, cnt, E + f.off + a, __ddiv_rn(__dmul_rn(f.my_reach, f.sig[a]), f.sample_reach), err);
      }
    }
    value = value_estimate;
  }
  lg.counts[k] = cnt;
}

// How the K traversals' deltas reach the tables (both add the same numbers in the same order; the GPU suite compares them
// bit for bit):
//   kMcScatter (default)  k_mccfr_scatter expands the logs into dense [K][width] rows, k_mccfr_apply streams the rows
//                         (coalesced, at HBM speed) — the fastest when the rows fit comfortably in HBM;
//   kMcLanes64            k_mccfr_partial_log adds the logs lane by lane in shared memory: no [K][width] buffer at all (memory
//                         O(K x records) instead of O(K x table)), but each lane's K / 64 traversals are a sequential chain —
//                         chosen when the dense rows would exceed kMcScatterMaxBytes and a partial row fits shared memory.
// B2S_MCCFR_MODE=scatter|lanes forces one of them (lanes still only where a partial row fits), so the lanes path can be
// compared with the default at sizes where it would not be chosen.
enum McMode { kMcScatter = 0, kMcLanes64 = 1 };
constexpr size_t kMcLogMaxShared = 200 * 1024;
constexpr size_t kMcScatterMaxBytes = (size_t)8 << 30;
static McMode mccfr_mode(int rows, int width) {
  static const int forced = [] {
    const char* e = getenv("B2S_MCCFR_MODE");
    if (!e) return -1;
    if (!strcmp(e, "lanes")) return (int)kMcLanes64;
    if (!strcmp(e, "scatter")) return (int)kMcScatter;
    return -1;
  }();
  const bool lanes_fit = sizeof(double) * (size_t)width <= kMcLogMaxShared;
  if (forced == kMcLanes64 && lanes_fit) return kMcLanes64;
  if (forced == kMcScatter) return kMcScatter;
  const size_t dense_bytes = sizeof(double) * (size_t)width * (size_t)rows;
  return (dense_bytes > kMcScatterMaxBytes && lanes_fit) ? kMcLanes64 : kMcScatter;
}
static McLog mccfr_log(const CfrSolver* S) { return McLog{S->mc_log, S->mc_counts, S->mc_log_cap}; }

// rows_needed: traversal threads of one launch; width: entries per row (E, or 2E for outcome sampling); cap: records per
// traversal
static int mccfr_prepare(CfrSolver* S, int rows_needed, int width, int cap) {
  if (!S->mccfr_tables) return fail("mccfr: the solver was not created with B2S_CFR_MCCFR_TABLES");
  if (S->max_actions > kMcMaxActions || S->d.n_levels > kMcMaxDepth) return fail("mccfr: game tree too wide / deep for the device traversal");
  B2S_CU(cudaSetDevice(S->device));
  const int E = S->d.n_entries;
  if (!S->mc_err) {
    B2S_CU(cudaMalloc((void**)&S->mc_err, sizeof(int)));
    B2S_CU(cudaMemset(S->mc_err, 0, sizeof(int)));
  }
  if (S->mc_log_rows < rows_needed || S->mc_log_cap < cap) {
    if (S->mc_log) cudaFree(S->mc_log);
    if (S->mc_counts) cudaFree(S->mc_counts);
    const int rows = std::max(rows_needed, S->mc_log_rows), c = std::max(cap, S->mc_log_cap);
    S->mc_log = nullptr; S->mc_counts = nullptr; S->mc_log_rows = 0;
    B2S_CU(cudaMalloc((void**)&S->mc_log, sizeof(int4) * (size_t)rows * (size_t)c));
    B2S_CU(cudaMalloc((void**)&S->mc_counts, sizeof(int) * (size_t)rows));
    B2S_CU(cudaMemset(S->mc_counts, 0, sizeof(int) * (size_t)rows));
    S->mc_log_rows = rows; S->mc_log_cap = c;
  }
  if (mccfr_mode(rows_needed, width) == kMcLanes64) {
    if (!S->mc_partials) {
      B2S_CU(cudaMalloc((void**)&S->mc_partials, sizeof(double) * (size_t)kMcLanes * 2 * (size_t)E));
      B2S_CU(cudaFuncSetAttribute(k_mccfr_partial_log, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kMcLogMaxShared));
    }
    return 0;
  }
  rows_needed *= width / E;                              // dense rows are allocated in units of E doubles
  if (S->mc_rows_k < rows_needed) {
    if (S->mc_rows) cudaFree(S->mc_rows);
    S->mc_rows = nullptr; S->mc_rows_k = 0;
    B2S_CU(cudaMalloc((void**)&S->mc_rows, sizeof(double) * (size_t)E * (size_t)rows_needed));
    B2S_CU(cudaMemset(S->mc_rows, 0, sizeof(double) * (size_t)E * (size_t)rows_needed));
    S->mc_rows_k = rows_needed;
  }
  return 0;
}

// The traversals of one phase: thread t < n_threads runs traversal k = lane_begin + t mod L + 64 (t div L) of K.  On one GPU
// every lane is local (lane_begin = 0, L = 64, n_threads = K, so k = t).
struct McLanes { int K, lane_begin, L, n_threads; };

// Phase step 1: player p's traversals into the delta logs — external sampling (k_mccfr_es), or outcome sampling with
// exploration epsilon (k_mccfr_os, one GPU only).
static void mccfr_traverse(CfrSolver* S, int p, u64 seed, const McLanes& ln, bool outcome, double epsilon, int simple_average,
                           cudaStream_t st) {
  const u32 phase = (u32)(S->iteration * 2 + p);
  const unsigned grid = (unsigned)((ln.n_threads + 127) / 128);
  if (outcome) k_mccfr_os<<<grid, 128, 0, st>>>(S->d, p, phase, seed, ln.K, epsilon, mccfr_log(S), S->mc_err);
  else k_mccfr_es<<<grid, 128, 0, st>>>(S->d, p, phase, seed, ln.K, ln.lane_begin, ln.L, ln.n_threads, mccfr_log(S), S->mc_err, simple_average);
  ++g_launches;
}

// Phase step 2: the logs, `width` entries per row (E: by the entry's player; 2E: regret, then average-policy deltas), in the fixed
// order into player p's tables, or into lane_partials [64][E] for the lanes this rank owns (sharded external sampling).
static void mccfr_reduce(CfrSolver* S, int p, const McLanes& ln, int width, double* lane_partials, cudaStream_t st) {
  const int E = S->d.n_entries;
  const dim3 ablock(kMcTile, kMcLanes);
  const unsigned agrid = (unsigned)((E + kMcTile - 1) / kMcTile);
  const bool lanes = mccfr_mode(ln.n_threads, width) == kMcLanes64;
  if (lanes) {
    k_mccfr_partial_log<<<ln.L, kMcLogThreads, sizeof(double) * (size_t)width, st>>>(ln.K, ln.lane_begin, ln.L, mccfr_log(S), width,
                                                                                   lane_partials ? lane_partials : S->mc_partials);
  } else {
    const long long slots = (long long)ln.n_threads * S->mc_log_cap;
    k_mccfr_scatter<<<(unsigned)((slots + 255) / 256), 256, 0, st>>>(mccfr_log(S), slots, width, S->mc_rows);
    if (lane_partials) {
      k_mccfr_partial<<<agrid, ablock, 0, st>>>(S->d, ln.K, ln.lane_begin, ln.L, S->mc_rows, lane_partials);
      ++g_launches;
    }
  }
  ++g_launches;
  if (lane_partials) return;
  for (int half = 0; half < width; half += E) {          // mode 0: by the entry's player (width E); 1: regrets, 2: cumulative policy
    const int mode = width == E ? 0 : 1 + half / E;
    if (lanes) k_mccfr_combine<<<agrid, ablock, 0, st>>>(S->d, p, S->mc_partials + half, width, mode);
    else k_mccfr_apply<<<agrid, ablock, 0, st>>>(S->d, p, ln.K, S->mc_rows + half, width, mode);
    ++g_launches;
  }
}

static int mccfr_check_errors(CfrSolver* S, cudaStream_t st) {
  if (int r = launch_status("k_mccfr launch")) return r;
  int bad = 0;
  B2S_CU(cudaMemcpyAsync(&bad, S->mc_err, sizeof(int), cudaMemcpyDeviceToHost, st));
  B2S_CU(cudaStreamSynchronize(st));
  if (bad) return fail("mccfr: a sampling step found sum of probabilities <= z (SampleActionIndex, cfr.cc:617-628)");
  return 0;
}

// `iters` iterations of K traversals (external sampling) or K episodes (outcome sampling, rows [K][2E]) per player phase on
// one GPU; full: AverageType::kFull of external sampling (RunIteration, external_sampling_mccfr.cc:76-79).
static int mccfr_iterate(CfrSolver* S, int iters, int K, u64 seed, bool outcome, double epsilon, int full, cudaStream_t st) {
  const int width = outcome ? 2 * S->d.n_entries : S->d.n_entries;
  if (int r = mccfr_prepare(S, K, width, outcome ? S->mc_cap_os : S->mc_cap_es)) return r;
  const McLanes ln{K, 0, kMcLanes, K};
  for (int it = 0; it < iters; ++it) {
    for (int p = 0; p < 2; ++p) {
      mccfr_traverse(S, p, seed, ln, outcome, epsilon, full ? 0 : 1, st);
      mccfr_reduce(S, p, ln, width, nullptr, st);
    }
    if (full) { k_mccfr_full_average<<<1, 1024, 0, st>>>(S->d); ++g_launches; }
    ++S->iteration;
  }
  return mccfr_check_errors(S, st);
}

}  // namespace b2s

using namespace b2s;

extern "C" {

int b2s_mccfr_traverse_lanes(void* solver, int player, int traversals_per_update, uint64_t seed, int lane_begin, int lane_end,
                             double* partials_d, void* stream) {
  if (!solver || !partials_d) return fail("mccfr: null argument");
  CfrSolver* S = (CfrSolver*)solver;
  if (player < 0 || player > 1 || traversals_per_update < 1) return fail("mccfr: bad player / traversals_per_update");
  if (lane_begin < 0 || lane_end > kMcLanes || lane_begin >= lane_end) return fail("mccfr: lane range must lie within [0, 64)");
  const int K = traversals_per_update, L = lane_end - lane_begin, E = S->d.n_entries;
  const McLanes ln{K, lane_begin, L, L * ((K + 63) / 64)};
  if (int r = mccfr_prepare(S, ln.n_threads, E, S->mc_cap_es)) return r;
  cudaStream_t st = (cudaStream_t)stream;
  mccfr_traverse(S, player, seed, ln, false, 0.0, 1, st);
  mccfr_reduce(S, player, ln, E, partials_d, st);
  return launch_status("k_mccfr launch");
}

int b2s_mccfr_apply_partials(void* solver, int player, const double* partials_d, void* stream) {
  if (!solver || !partials_d) return fail("mccfr: null argument");
  CfrSolver* S = (CfrSolver*)solver;
  if (player < 0 || player > 1) return fail("mccfr: bad player");
  if (int r = mccfr_prepare(S, 1, S->d.n_entries, S->mc_cap_es)) return r;
  cudaStream_t st = (cudaStream_t)stream;
  const int E = S->d.n_entries;
  k_mccfr_combine<<<(E + kMcTile - 1) / kMcTile, dim3(kMcTile, kMcLanes), 0, st>>>(S->d, player, partials_d, E, 0);
  ++g_launches;
  if (player == 1) ++S->iteration;
  return mccfr_check_errors(S, st);
}

int b2s_mccfr_external_iterate_ex(void* solver, int iters, int traversals_per_update, uint64_t seed, int flags, void* stream) {
  if (!solver) return fail("mccfr: null solver");
  if (iters < 0 || traversals_per_update < 1) return fail("mccfr: iters >= 0 and traversals_per_update >= 1 required");
  const int full = (flags & B2S_MCCFR_FULL_AVERAGE) ? 1 : 0;
  return mccfr_iterate((CfrSolver*)solver, iters, traversals_per_update, seed, false, 0.0, full, (cudaStream_t)stream);
}

int b2s_mccfr_external_iterate(void* solver, int iters, int traversals_per_update, uint64_t seed, void* stream) {
  return b2s_mccfr_external_iterate_ex(solver, iters, traversals_per_update, seed, 0, stream);
}

int b2s_mccfr_outcome_iterate(void* solver, int iters, int trajectories_per_update, uint64_t seed, double epsilon, void* stream) {
  if (!solver) return fail("mccfr: null solver");
  if (iters < 0 || trajectories_per_update < 1) return fail("mccfr: iters >= 0 and trajectories_per_update >= 1 required");
  if (!(epsilon >= 0.0 && epsilon <= 1.0)) return fail("mccfr: epsilon must lie in [0, 1]");
  return mccfr_iterate((CfrSolver*)solver, iters, trajectories_per_update, seed, true, epsilon, 0, (cudaStream_t)stream);
}

}  // extern "C"
