// Device-resident tabular CFR.  Semantics: reference open_spiel/algorithms/cfr.cc — CFRSolverBase::
// EvaluateAndUpdatePolicy :263-282 (alternating updates: one full traversal + regret matching per player),
// ComputeCounterFactualRegret :331-408 and ...ForActionProbs :443-469 (state values, counterfactual regrets,
// average-policy accumulation), CounterFactualReachProb :309-318, CFRInfoStateValues::ApplyRegretMatching
// :596-615, ApplyRegretMatchingPlusReset :683-691.
//
// The reference walks the game tree recursively, cloning a State per edge and looking every information
// state up by string.  Here the tree is expanded ONCE, level by level, with the batched device kernels
// (b2s_status / b2s_legal_mask / b2s_information_state / b2s_gather_states / b2s_apply_actions — the C ABI,
// no CPU rule code), flattened into level-ordered SoA arrays, and every iteration runs inside one persistent
// kernel: a top-down pass for reach probabilities, a bottom-up pass for state values, one thread per
// information state for the regret / average-policy update, then regret matching, with block barriers
// between tree levels.  The current policy is frozen during a traversal in the reference too, so the
// traversal is a pure tree reduction.
//
// Floating point: FP64 throughout, every product and sum written as an explicitly rounded operation (no FMA
// contraction), children combined in action order from 0.0, an information state's histories accumulated in
// the reference's DFS order, the chance player's reach kept as the last factor — the same operations in the
// same order as the reference, so tables are reproduced bit for bit (north-star tolerance: 1e-6).
// The reference prunes decision nodes where every player's reach is 0 and returns zeros (cfr.cc:350-355);
// we reproduce the returned zeros; the skipped updates below such a node add +-0 and change nothing.
#include <math.h>
#include <string.h>

#include <algorithm>
#include <string>
#include <unordered_map>
#include <vector>

#include "../../include/b2s.h"
#include "common.cuh"
#include "errors.h"
#include "nccl_dyn.h"

namespace b2s {
extern long long g_launches;

struct CfrDev {
  int n_nodes, n_levels, n_infosets, n_entries;
  const int* level_off;        // [n_levels + 1]
  const int* parent;           // [n]
  const signed char* kind;     // 0 terminal, 1 chance, 2 decision
  const signed char* actor;    // 0/1 = player to move, 2 = chance
  const int* first_child;      // [n]
  const signed char* nchild;   // [n]
  const signed char* aidx;     // index of this node among its parent's children
  const double* chance_prob;   // [n] probability of the edge into n when the parent is a chance node
  const double* ret;           // [n][2] terminal returns
  const int* infoset;          // [n] (decision nodes)
  const int* is_player;        // [I]
  const int* is_off;           // [I + 1] offsets into the per-action tables
  const int* hist_off;         // [I + 1] offsets into hist
  const int* hist;             // decision nodes of each information state in DFS order
  const int* is_level;         // [I] tree level of the information state's histories
  const int* policy_index;     // [n] index into cur_policy of the edge into n (-1 when the parent is a chance node)
  const signed char* par_actor;// [n] actor of the parent (0/1 player, 2 chance)
  const double* chance_reach;  // [n] the chance player's reach of n (product of chance probabilities along the path)
  double* reach;               // [n][3]  (player 0, player 1, chance)
  double* edge_prob;           // [n]
  double* value;               // [n][2]
  double* regrets;             // [E]
  double* cum_policy;          // [E]
  double* cur_policy;          // [E]
  double* delta;               // [2C]: per-(history, action) regret contributions, then average-policy contributions, of one sharded traversal
  const int* hist_entry_off;   // [n_hist + 1] offset of history slot hh in the contribution buffer (prefix sum of its action count)
  const int* hist_is;          // [n_hist] information state of history slot hh
  int n_hist, n_contrib;       // history slots (= decision nodes), C = sum of their action counts
  int* iter_d;                 // device iteration counter for graph-captured sharded iterations
  const signed char* entry_player;   // [E] the player an entry's information state belongs to
  const int4* mc_node;         // [n] MCCFR traversal record: {first_child, table offset of the information state, kind | actor << 8 | nchild << 16, 0}
};

// One traversal's tree passes, shared by the single-GPU kernel and the sharded one: (1) edge probabilities from the frozen
// policy, (2) L level steps in which the reach probabilities move one level DOWN while the state values move one level UP.
__device__ __forceinline__ void cfr_level_passes(const CfrDev& d, int tid, int nt) {
  const int L = d.n_levels;
  for (int n = 1 + tid; n < d.n_nodes; n += nt) {
    int pi = d.policy_index[n];
    d.edge_prob[n] = pi >= 0 ? d.cur_policy[pi] : d.chance_prob[n];
  }
  if (tid == 0) { d.reach[0] = 1.0; d.reach[1] = 1.0; }
  __syncthreads();
  for (int k = 0; k < L; ++k) {
    int ld = k + 1;                       // reach: new_reach_probabilities[current_player] *= prob (cfr.cc:457)
    if (ld < L) {
      for (int n = d.level_off[ld] + tid; n < d.level_off[ld + 1]; n += nt) {
        int par = d.parent[n];
        double r0 = d.reach[2 * par], r1 = d.reach[2 * par + 1];
        int a = d.par_actor[n];
        if (a == 0) r0 = __dmul_rn(r0, d.edge_prob[n]); else if (a == 1) r1 = __dmul_rn(r1, d.edge_prob[n]);
        d.reach[2 * n] = r0; d.reach[2 * n + 1] = r1;
      }
    }
    int lu = L - 1 - k;                   // values: state_value[i] += prob * child_value[i] (cfr.cc:461-463)
    for (int n = d.level_off[lu] + tid; n < d.level_off[lu + 1]; n += nt) {
      double v0, v1;
      if (d.kind[n] == 0) { v0 = d.ret[2 * n]; v1 = d.ret[2 * n + 1]; }
      else {
        v0 = 0.0; v1 = 0.0;
        int fc = d.first_child[n];
        for (int c = 0; c < d.nchild[n]; ++c) {
          double pr = d.edge_prob[fc + c];
          v0 = __dadd_rn(v0, __dmul_rn(pr, d.value[2 * (fc + c)]));
          v1 = __dadd_rn(v1, __dmul_rn(pr, d.value[2 * (fc + c) + 1]));
        }
      }
      d.value[2 * n] = v0; d.value[2 * n + 1] = v1;
    }
    __syncthreads();
  }
}

__global__ void __launch_bounds__(1024) k_cfr(CfrDev d, int iters, int iteration0, int linear_averaging, int rm_plus) {
  // One traversal = (1) edge probabilities from the frozen policy, (2) L level steps in which the reach
  // probabilities move one level DOWN while the state values move one level UP (the two sweeps are independent:
  // the reference's all-zero-reach pruning, cfr.cc:350-355, only ever replaces values that are multiplied by a zero
  // probability before they are used, so it cannot change any table entry), (3) one thread per information state of
  // the updating player: regrets and average policy over its histories in DFS order, then regret matching.
  // Regret matching of the other player's information states (cfr.cc:693-697 sweeps the whole table) would recompute
  // the same policy from unchanged regrets, so it is skipped.
  // One CTA on purpose: the same kernel as an 8-CTA thread-block cluster (cluster.sync() = barrier.cluster + MEMBAR.GPU +
  // L1 invalidate per level step, arrays in global memory) was no faster on Leduc and slower on Kuhn — the level steps are
  // latency-bound, and the cluster barrier costs what the extra threads save.
  const int tid = threadIdx.x, nt = blockDim.x;
  const int L = d.n_levels;
  for (int it = 0; it < iters; ++it) {
    const double iteration = (double)(iteration0 + it + 1);          // ++iteration_ (cfr.cc:264)
    for (int p = 0; p < 2; ++p) {
      cfr_level_passes(d, tid, nt);
      // regret / average-policy update (cfr.cc:379-405) + regret matching (cfr.cc:596-615) for player p
      for (int I = tid; I < d.n_infosets; I += nt) {
        if (d.is_player[I] != p) continue;
        int off = d.is_off[I], na = d.is_off[I + 1] - off;
        for (int hh = d.hist_off[I]; hh < d.hist_off[I + 1]; ++hh) {
          int h = d.hist[hh];
          double self_reach = d.reach[2 * h + p];
          // CounterFactualReachProb: 1.0 * reach[other player] * reach[chance], in index order
          double cfr_reach = __dmul_rn(__dmul_rn(1.0, d.reach[2 * h + (1 - p)]), d.chance_reach[h]);
          double vh = d.value[2 * h + p];
          int fc = d.first_child[h];
          for (int a = 0; a < na; ++a) {
            double regret = __dmul_rn(cfr_reach, __dsub_rn(d.value[2 * (fc + a) + p], vh));
            d.regrets[off + a] = __dadd_rn(d.regrets[off + a], regret);
            double pol = d.cur_policy[off + a];
            double inc = linear_averaging ? __dmul_rn(__dmul_rn(iteration, self_reach), pol) : __dmul_rn(self_reach, pol);
            d.cum_policy[off + a] = __dadd_rn(d.cum_policy[off + a], inc);
          }
        }
        double sum = 0.0;
        for (int a = 0; a < na; ++a) {
          double r = d.regrets[off + a];
          if (rm_plus && r < 0) { r = 0; d.regrets[off + a] = 0; }
          if (r > 0) sum = __dadd_rn(sum, r);
        }
        for (int a = 0; a < na; ++a) {
          double r = d.regrets[off + a];
          d.cur_policy[off + a] = sum > 0 ? (r > 0 ? __ddiv_rn(r, sum) : 0.0) : __ddiv_rn(1.0, (double)na);
        }
      }
      __syncthreads();
    }
  }
}

// ---- multi-GPU variant: one traversal split into "my shard's contributions" / all-reduce / "apply in order" ---------
// Every rank runs the level passes of the whole (tiny) tree; history slot hh's regret and average-policy contributions
// (one pair per action, the very expressions of k_cfr above) are written by rank (hh mod num_shards) into the
// contribution buffer `delta` and as 0.0 by every other rank, the ranks all-reduce the buffer (NCCL sum over NVLink, 2C
// doubles — x + 0 + ... + 0 is exact in any order), then every rank adds the contributions to its tables in the
// reference's DFS order and runs regret matching.  The tables therefore stay BIT-IDENTICAL to the single-GPU kernel and
// to the reference, whatever the number of ranks; the price is a 2C- instead of a 2E-double message (Leduc: 150 KB
// instead of 45 KB — still latency-, not bandwidth-sized on NVLink).
// iteration: CFRSolverBase::iteration_ of this traversal (1-based) — from `iteration`, or, when d.iter_d is used
// (graph-captured loops), from the device counter, which player 0's traversal advances.
__global__ void __launch_bounds__(1024) k_cfr_traverse(CfrDev d, int p, int iteration, int use_counter, int linear_averaging, int shard, int num_shards) {
  const int tid = threadIdx.x, nt = blockDim.x;
  if (use_counter) iteration = *d.iter_d + (p == 0 ? 1 : 0);
  cfr_level_passes(d, tid, nt);
  const double iter = (double)iteration;
  const int C = d.n_contrib;
  for (int hh = tid; hh < d.n_hist; hh += nt) {
    const int I = d.hist_is[hh];
    if (d.is_player[I] != p) continue;
    const int off = d.is_off[I], na = d.is_off[I + 1] - off, co = d.hist_entry_off[hh];
    if (hh % num_shards != shard) {
      for (int a = 0; a < na; ++a) { d.delta[co + a] = 0.0; d.delta[C + co + a] = 0.0; }
      continue;
    }
    const int h = d.hist[hh];
    double self_reach = d.reach[2 * h + p];
    double cfr_reach = __dmul_rn(__dmul_rn(1.0, d.reach[2 * h + (1 - p)]), d.chance_reach[h]);
    double vh = d.value[2 * h + p];
    int fc = d.first_child[h];
    for (int a = 0; a < na; ++a) {
      d.delta[co + a] = __dmul_rn(cfr_reach, __dsub_rn(d.value[2 * (fc + a) + p], vh));
      double pol = d.cur_policy[off + a];
      d.delta[C + co + a] = linear_averaging ? __dmul_rn(__dmul_rn(iter, self_reach), pol) : __dmul_rn(self_reach, pol);
    }
  }
  __syncthreads();
  if (use_counter && p == 0 && tid == 0) *d.iter_d = iteration;
}

__global__ void __launch_bounds__(1024) k_cfr_apply(CfrDev d, int p, int rm_plus) {
  const int tid = threadIdx.x, nt = blockDim.x;
  const int C = d.n_contrib;
  for (int I = tid; I < d.n_infosets; I += nt) {
    if (d.is_player[I] != p) continue;
    int off = d.is_off[I], na = d.is_off[I + 1] - off;
    for (int hh = d.hist_off[I]; hh < d.hist_off[I + 1]; ++hh) {      // the reference's DFS order (cfr.cc:387-401)
      const int co = d.hist_entry_off[hh];
      for (int a = 0; a < na; ++a) {
        d.regrets[off + a] = __dadd_rn(d.regrets[off + a], d.delta[co + a]);
        d.cum_policy[off + a] = __dadd_rn(d.cum_policy[off + a], d.delta[C + co + a]);
      }
    }
    double sum = 0.0;
    for (int a = 0; a < na; ++a) {
      double r = d.regrets[off + a];
      if (rm_plus && r < 0) { r = 0; d.regrets[off + a] = 0; }
      if (r > 0) sum = __dadd_rn(sum, r);
    }
    for (int a = 0; a < na; ++a) {
      double r = d.regrets[off + a];
      d.cur_policy[off + a] = sum > 0 ? (r > 0 ? __ddiv_rn(r, sum) : 0.0) : __ddiv_rn(1.0, (double)na);
    }
  }
}

// ---- NashConv / exploitability of the average (or current) policy on the same flattened tree -------------------
// Semantics: reference algorithms/tabular_exploitability.cc (NashConv = sum_p [BR_p(pi_-p) - v_p(pi)],
// Exploitability = NashConv / num_players) with best responses as in algorithms/best_response.cc: at the
// responder's information states the action maximising sum_h cf_reach(h) * value(child) is taken at every history.
// out[0..1] = best-response values of players 0/1 at the root, out[2..3] = on-policy root values.
__global__ void __launch_bounds__(1024) k_cfr_nashconv(CfrDev d, int use_average, double* pol, int* best, double* out) {
  const int tid = threadIdx.x, nt = blockDim.x;
  // the policy being evaluated (CFRAveragePolicy, cfr.cc:104-125: uniform where nothing was accumulated)
  for (int I = tid; I < d.n_infosets; I += nt) {
    int off = d.is_off[I], na = d.is_off[I + 1] - off;
    if (use_average) {
      double sum = 0.0;
      for (int a = 0; a < na; ++a) sum += d.cum_policy[off + a];
      for (int a = 0; a < na; ++a) pol[off + a] = sum == 0.0 ? 1.0 / na : d.cum_policy[off + a] / sum;
    } else {
      for (int a = 0; a < na; ++a) pol[off + a] = d.cur_policy[off + a];
    }
  }
  __syncthreads();
  // edge probabilities under the evaluated policy
  for (int n = 1 + tid; n < d.n_nodes; n += nt) {
    int par = d.parent[n];
    d.edge_prob[n] = d.kind[par] == 1 ? d.chance_prob[n] : pol[d.is_off[d.infoset[par]] + d.aidx[n]];
  }
  __syncthreads();
  // on-policy values
  for (int l = d.n_levels - 1; l >= 0; --l) {
    for (int n = d.level_off[l] + tid; n < d.level_off[l + 1]; n += nt) {
      double v0, v1;
      if (d.kind[n] == 0) { v0 = d.ret[2 * n]; v1 = d.ret[2 * n + 1]; }
      else {
        v0 = 0.0; v1 = 0.0;
        int fc = d.first_child[n];
        for (int c = 0; c < d.nchild[n]; ++c) { v0 += d.edge_prob[fc + c] * d.value[2 * (fc + c)]; v1 += d.edge_prob[fc + c] * d.value[2 * (fc + c) + 1]; }
      }
      d.value[2 * n] = v0; d.value[2 * n + 1] = v1;
    }
    __syncthreads();
  }
  if (tid == 0) { out[2] = d.value[0]; out[3] = d.value[1]; }
  __syncthreads();
  for (int b = 0; b < 2; ++b) {
    // counterfactual reach of every node for responder b: opponents' and chance's probabilities only
    if (tid == 0) d.reach[0] = 1.0;
    __syncthreads();
    for (int l = 1; l < d.n_levels; ++l) {
      for (int n = d.level_off[l] + tid; n < d.level_off[l + 1]; n += nt) {
        int par = d.parent[n];
        double r = d.reach[3 * par];
        if (!(d.kind[par] == 2 && d.actor[par] == b)) r *= d.edge_prob[n];
        d.reach[3 * n] = r;
      }
      __syncthreads();
    }
    // best-response values bottom-up; value slot 0 is reused for V_b
    for (int l = d.n_levels - 1; l >= 0; --l) {
      // responder's information states at this level choose their action from their children's values
      for (int I = tid; I < d.n_infosets; I += nt) {
        if (d.is_player[I] != b || d.is_level[I] != l) continue;
        int off = d.is_off[I], na = d.is_off[I + 1] - off;
        int arg = 0;
        double bestq = 0.0;
        for (int a = 0; a < na; ++a) {
          double q = 0.0;
          for (int hh = d.hist_off[I]; hh < d.hist_off[I + 1]; ++hh) {
            int h = d.hist[hh];
            q += d.reach[3 * h] * d.value[2 * (d.first_child[h] + a)];
          }
          if (a == 0 || q > bestq) { bestq = q; arg = a; }
        }
        best[I] = arg;
      }
      __syncthreads();
      for (int n = d.level_off[l] + tid; n < d.level_off[l + 1]; n += nt) {
        double v;
        if (d.kind[n] == 0) v = d.ret[2 * n + b];
        else if (d.kind[n] == 2 && d.actor[n] == b) v = d.value[2 * (d.first_child[n] + best[d.infoset[n]])];
        else {
          v = 0.0;
          int fc = d.first_child[n];
          for (int c = 0; c < d.nchild[n]; ++c) v += d.edge_prob[fc + c] * d.value[2 * (fc + c)];
        }
        d.value[2 * n] = v;
      }
      __syncthreads();
    }
    if (tid == 0) out[b] = d.value[0];
    __syncthreads();
    // restore nothing: value/reach/edge_prob are scratch, rewritten by the next traversal
  }
}

// ---- external-sampling MCCFR (external_sampling_mccfr.cc) ----------------------------------------------------
// One thread = one UpdateRegrets traversal (:124-186) of traverser p over the flattened tree, as an explicit-stack
// DFS: chance and opponent nodes are sampled and followed (no frame), the traverser's decision nodes keep a frame
// (policy, child values) until all actions are explored.  Tables are read-only here; each traversal owns row k of
// `rows` ([K][E]: in phase p an entry of player p receives a regret delta, an entry of the other player an
// average-policy delta, so one row serves both), which k_mccfr_apply adds in a fixed order.
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

// Sharding: the rank that owns reduction lanes [lane_begin, lane_begin + L) runs the traversals k with k mod 64 in
// that range; thread t is traversal k = lane_begin + t mod L + 64 (t div L) and owns row t.  One GPU: L = 64, k = t.
//
// Where a traversal's deltas go (template LOG):
//   false: row t of `rows` ([threads][E] doubles, dense, zero except for the cells this traversal touches);
//   true:  a delta log, log[t][0 .. counts[t]) of {table entry, value} records (McLog).  A traversal touches an entry at most
//          once (perfect recall: the information states on the paths of one traversal differ in the traverser's own
//          actions), so a log holds the same numbers as the row's non-zero cells — a few dozen records instead of E cells.
struct McLog {
  int4* rec;      // [threads][cap]: {entry, 0, value bits lo, value bits hi}
  int* counts;    // [threads]
  int cap;        // records per traversal: an exact upper bound from the tree (mccfr_log_capacity)
};
__device__ __forceinline__ void mc_log_append(const McLog& lg, int t, int& cnt, int entry, double v, int* err) {
  if (v == 0.0) return;                                  // the dense rows cannot tell a zero delta from an untouched cell either
  if (cnt >= lg.cap) { atomicAdd(err, 1); return; }
  const long long bits = __double_as_longlong(v);
  lg.rec[(size_t)t * lg.cap + cnt++] = make_int4(entry, 0, (int)(u32)bits, (int)(u32)((u64)bits >> 32));
}

template <bool LOG>
__global__ void __launch_bounds__(128) k_mccfr_es(CfrDev d, int p, u32 phase, u64 seed, int K, int lane_begin, int L, int n_threads,
                                                   double* __restrict__ rows, McLog lg, int* __restrict__ err, int simple_average) {
  int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n_threads) return;
  int k = lane_begin + t % L + 64 * (t / L);
  if (k >= K) { if (LOG) lg.counts[t] = 0; return; }
  const int E = d.n_entries;
  double* reg_row = LOG ? nullptr : rows + (size_t)t * E;
  double* avg_row = reg_row;
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
      if (kind == 1) {                                   // SampleAction(ChanceOutcomes(), z), spiel.cc:372-409
        double z = mc_uniform(seed, h, phase, (u32)k);
        int chosen = -1;
        if (n == 1) chosen = 0;
        else {
          double sum = 0.0;
          for (int c = 0; c < n; ++c) {
            double prob = d.chance_prob[fc + c];
            if (sum <= z && z < __dadd_rn(sum, prob)) { chosen = c; break; }
            sum = __dadd_rn(sum, prob);
          }
        }
        if (chosen < 0) { atomicAdd(err, 1); chosen = n - 1; }
        h = mc_child_hash(h, chosen);
        node = fc + chosen;
        continue;
      }
      const int off = rec.y;
      double sig[kMcMaxActions];
      {                                                  // ApplyRegretMatching on a copy, cfr.cc:596-615
        double sum_pos = 0.0;
        for (int a = 0; a < n; ++a) { double rg = d.regrets[off + a]; if (rg > 0) sum_pos = __dadd_rn(sum_pos, rg); }
        for (int a = 0; a < n; ++a) {
          double rg = d.regrets[off + a];
          sig[a] = sum_pos > 0 ? (rg > 0 ? __ddiv_rn(rg, sum_pos) : 0.0) : __ddiv_rn(1.0, (double)n);
        }
      }
      if (actor != p) {                                  // opponent: SampleActionIndex(0, z), cfr.cc:617-628
        double z = mc_uniform(seed, h, phase, (u32)k);
        int aidx = -1;
        double sum = 0.0;
        for (int a = 0; a < n; ++a) {
          if (z >= sum && z < __dadd_rn(sum, sig[a])) { aidx = a; break; }
          sum = __dadd_rn(sum, sig[a]);
        }
        if (aidx < 0) { atomicAdd(err, 1); aidx = n - 1; }
        if (simple_average && actor == ((p + 1) & 1)) {  // simple averaging at the next player's nodes (:176-183)
          for (int a = 0; a < n; ++a) {
            if (LOG) mc_log_append(lg, t, cnt, off + a, sig[a], err);
            else avg_row[off + a] = __dadd_rn(avg_row[off + a], sig[a]);
          }
        }
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
      for (int a = 0; a < f.n; ++a) {                    // regret += child value - node value (:168-172)
        if (LOG) mc_log_append(lg, t, cnt, f.off + a, __dsub_rn(f.cv[a], f.v), err);
        else reg_row[f.off + a] = __dadd_rn(reg_row[f.off + a], __dsub_rn(f.cv[a], f.v));
      }
      r = f.v;
      --sp;
    }
    if (done) break;
  }
  if (LOG) lg.counts[t] = cnt;
}

// tables += the sum of the K traversal rows, in a FIXED order so the result is reproducible (and restated by the
// oracle): 64 partial sums, partial[q] = delta[q] + delta[q+64] + delta[q+128] + ... (sequential, from 0.0), combined
// by the tree partial[q] += partial[q+s], s = 32, 16, 8, 4, 2, 1; table += partial[0].  With K = 1 this is
// table += delta[0].  A block owns 16 consecutive table entries (x) and the 64 partial lanes (y): every row is read
// in 128-byte coalesced segments, 8 independent loads in flight per thread.  Touched cells are re-zeroed for the
// next phase.
constexpr int kMcLanes = 64, kMcTile = 16;
// `stride` = doubles per row (E for external sampling, 2E for outcome sampling); mode 0: an entry of player p receives a regret
// delta, an entry of the other player an average-policy delta (external sampling); mode 1: every entry -> regrets; mode 2:
// every entry -> cumulative policy (outcome sampling: two passes over the two halves of its rows).
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
  __syncthreads();
  for (int s = kMcLanes / 2; s >= 1; s >>= 1) {
    if (q < s) part[q][ex] = __dadd_rn(part[q][ex], part[q + s][ex]);
    __syncthreads();
  }
  if (q == 0 && e < E) {
    double* dst = mode == 0 ? (d.entry_player[e] == p ? d.regrets + e : d.cum_policy + e) : (mode == 1 ? d.regrets + e : d.cum_policy + e);
    *dst = __dadd_rn(*dst, part[0][ex]);
  }
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
// The same partial sums from delta logs.  The order is the dense kernels' — lane q adds the deltas of its traversals
// k = q, q + 64, q + 128, ... one after the other, from 0.0 — so the result is bit-identical; what changes is the traffic:
// the records of the K traversals (tens of bytes each) instead of K rows of E doubles.  One block per lane keeps that
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
// tree); letting them also read-modify-write their dense delta rows lengthens those chains, whereas scattering the same
// records from a kernel of its own is a few microseconds of fully parallel stores.  Entries are distinct within a traversal and the rows are zero between phases
// (k_mccfr_apply re-zeroes what it reads), so a plain store reproduces the dense path's cell exactly.
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
  __syncthreads();
  for (int s = kMcLanes / 2; s >= 1; s >>= 1) {
    if (q < s) part[q][ex] = __dadd_rn(part[q][ex], part[q + s][ex]);
    __syncthreads();
  }
  if (q == 0 && e < E) {
    double* dst = mode == 0 ? (d.entry_player[e] == p ? d.regrets + e : d.cum_policy + e) : (mode == 1 ? d.regrets + e : d.cum_policy + e);
    *dst = __dadd_rn(*dst, part[0][ex]);
  }
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
    double sum = 0.0;
    for (int a = 0; a < na; ++a) { double r = d.regrets[off + a]; if (r > 0) sum = __dadd_rn(sum, r); }
    for (int a = 0; a < na; ++a) {
      double r = d.regrets[off + a];
      d.cur_policy[off + a] = sum > 0 ? (r > 0 ? __ddiv_rn(r, sum) : 0.0) : __ddiv_rn(1.0, (double)na);
    }
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
// unwound and every node of p on the path contributes regret and average-policy deltas to row k of `rows` ([K][2E]: regret
// deltas, then average-policy deltas), which k_mccfr_apply adds in its fixed order.  Tables are read-only here.
// u(node, redraw) = U53(Philox(seed; h + 0x632BE59BD9B4E019 redraw, phase, k)); a draw is lo + u (hi - lo), redrawn while it
// rounds up to hi — the stream and the two samplers oracle/algorithms/os_mccfr.cc (rng_mode 1) restates.
__device__ __forceinline__ double os_real(u64 seed, u64 h, u32 phase, u32 k, double lo, double hi) {
  for (u32 redraw = 0;; ++redraw) {
    double u = mc_uniform(seed, h + 0x632BE59BD9B4E019ull * (u64)redraw, phase, k);
    double r = __dadd_rn(lo, __dmul_rn(u, __dsub_rn(hi, lo)));
    if (r < hi || lo == hi) return r;
  }
}

template <bool LOG>
__global__ void __launch_bounds__(128) k_mccfr_os(CfrDev d, int p, u32 phase, u64 seed, int K, double epsilon, double* __restrict__ rows,
                                                   McLog lg, int* __restrict__ err) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= K) return;
  const int E = d.n_entries;
  double* reg_row = LOG ? nullptr : rows + (size_t)k * 2 * E;
  double* pol_row = LOG ? nullptr : reg_row + E;
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
    if (kind == 1) {                                     // SampleAction(ChanceOutcomes(), z), spiel.cc:372-409
      double z = os_real(seed, h, phase, (u32)k, 0.0, 1.0);
      int chosen = -1;
      double sum = 0.0;
      for (int c = 0; c < n; ++c) {
        double prob = d.chance_prob[fc + c];
        if (sum <= z && z < __dadd_rn(sum, prob)) { chosen = c; break; }
        sum = __dadd_rn(sum, prob);
      }
      if (chosen < 0) { atomicAdd(err, 1); chosen = n - 1; }
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
    {                                                    // info_state_copy.ApplyRegretMatching(), cfr.cc:596-615
      double sum_pos = 0.0;
      for (int a = 0; a < n; ++a) { double rg = d.regrets[f.off + a]; if (rg > 0) sum_pos = __dadd_rn(sum_pos, rg); }
      for (int a = 0; a < n; ++a) {
        double rg = d.regrets[f.off + a];
        f.sig[a] = sum_pos > 0 ? (rg > 0 ? __ddiv_rn(rg, sum_pos) : 0.0) : __ddiv_rn(1.0, (double)n);
      }
    }
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
        const double dr = __dsub_rn(cf_action_value, cf_value), dp = __ddiv_rn(__dmul_rn(f.my_reach, f.sig[a]), f.sample_reach);
        if (LOG) {
          mc_log_append(lg, k, cnt, f.off + a, dr, err);
          mc_log_append(lg, k, cnt, E + f.off + a, dp, err);
        } else {
          reg_row[f.off + a] = dr;
          pol_row[f.off + a] = dp;
        }
      }
    }
    value = value_estimate;
  }
  if (LOG) lg.counts[k] = cnt;
}

struct CfrSolver {
  // multi-GPU: communicator (owned or adopted), private stream + a CUDA graph of kGraphIters sharded iterations
  ncclComm_t comm = nullptr; bool comm_owned = false; int rank = 0, world = 1;
  cudaStream_t dist_stream = nullptr; cudaEvent_t dist_ev = nullptr;
  cudaGraphExec_t dist_graph = nullptr;
  int last_shard_player = 0;
  int mccfr_tables = 0;
  double* mc_rows = nullptr; int mc_rows_k = 0;              // dense delta rows (B2S_MCCFR_DENSE=1, or tables too wide for the log path)
  int4* mc_log = nullptr; int* mc_counts = nullptr;          // delta logs [mc_log_rows][mc_log_cap] + record counts
  int mc_log_rows = 0, mc_log_cap = 0;
  double* mc_partials = nullptr;                             // [64][2E] lane partial sums of the log path
  int mc_cap_es = 0, mc_cap_os = 0;                          // most records one traversal / one episode can write (from the tree)
  int* mc_err = nullptr;
  int max_actions = 0;
  int device = 0;
  int game_id = 0;
  int iteration = 0;
  int linear_averaging = 0, rm_plus = 0;
  int tensor_size = 0;
  CfrDev d;
  std::vector<void*> allocs;
  // host copies of the structure (export)
  std::vector<int> is_player, is_off, legal_actions, node_counts;    // node_counts = {chance, decision, terminal}
  std::vector<float> keys;                                           // [I][tensor_size] information-state tensors
  ~CfrSolver() {
    if (dist_graph) cudaGraphExecDestroy(dist_graph);
    if (comm && comm_owned && nccl_api().ok()) nccl_api().CommDestroy(comm);
    if (dist_ev) cudaEventDestroy(dist_ev);
    if (dist_stream) cudaStreamDestroy(dist_stream);
    for (void* p : allocs) cudaFree(p);
    if (mc_rows) cudaFree(mc_rows);
    if (mc_log) cudaFree(mc_log);
    if (mc_counts) cudaFree(mc_counts);
    if (mc_partials) cudaFree(mc_partials);
    if (mc_err) cudaFree(mc_err);
  }
};

template <typename T>
static int upload(CfrSolver* s, const std::vector<T>& v, const T** out) {
  void* p = nullptr;
  B2S_CU(cudaMalloc(&p, sizeof(T) * (v.empty() ? 1 : v.size())));
  s->allocs.push_back(p);
  if (!v.empty()) B2S_CU(cudaMemcpy(p, v.data(), sizeof(T) * v.size(), cudaMemcpyHostToDevice));
  *out = (const T*)p;
  return 0;
}
static int alloc_d(CfrSolver* s, size_t n, double** out) {
  void* p = nullptr;
  B2S_CU(cudaMalloc(&p, sizeof(double) * (n ? n : 1)));
  B2S_CU(cudaMemset(p, 0, sizeof(double) * (n ? n : 1)));
  s->allocs.push_back(p);
  *out = (double*)p;
  return 0;
}

}  // namespace b2s

using namespace b2s;

#define CK(x) do { int _r = (x); if (_r) { if (level) b2s_batch_destroy(level); if (next) b2s_batch_destroy(next); delete S; return _r; } } while (0)

extern "C" {

int b2s_cfr_create(int game_id, const b2s_params* params, int flags, int device, void** out_solver) {
  if (!out_solver) return fail("cfr: null out_solver");
  *out_solver = nullptr;
  if (b2s_device_count() <= 0) return fail("no CUDA device: the b2s device path has no CPU fallback");
  b2s_game_info gi;
  if (int r = b2s_game_info_get(game_id, params, &gi)) return r;
  if (gi.num_players != 2) return fail("cfr: two-player games only");
  if (gi.information_state_tensor_size <= 0)
    return fail("cfr: the game provides no information-state tensor (device CFR keys information states by it)");
  CfrSolver* S = new CfrSolver;
  S->device = device; S->game_id = game_id; S->tensor_size = gi.information_state_tensor_size;
  S->linear_averaging = (flags & B2S_CFR_LINEAR_AVERAGING) ? 1 : 0;
  S->rm_plus = (flags & B2S_CFR_REGRET_MATCHING_PLUS) ? 1 : 0;
  S->mccfr_tables = (flags & B2S_CFR_MCCFR_TABLES) ? 1 : 0;
  void* level = nullptr;
  void* next = nullptr;
  const int T = gi.information_state_tensor_size, MW = gi.mask_words;
  std::vector<int> parent, first_child, infoset, level_off;
  std::vector<signed char> kind, actor, nchild, aidx;
  std::vector<double> chance_prob, ret;
  std::unordered_map<std::string, int> key_to_is;
  std::vector<int> is_nact;
  int counts[3] = {0, 0, 0};
  // level 0 = the initial state
  CK(b2s_batch_create(game_id, params, 1, device, &level));
  long long n = 1;
  parent.push_back(-1); aidx.push_back(0); chance_prob.push_back(1.0);
  level_off.push_back(0);
  long long base = 0;                       // node id of lane 0 of the current level
  for (int depth = 0; n > 0; ++depth) {
    if (depth > 4096 || base + n > 50000000LL) CK(fail("cfr: game tree too large for the device solver"));
    // per-lane facts of this level, computed by the batched kernels
    signed char* cur_d; unsigned char* term_d; float* rets_d; uint32_t* mask_d; float* tens_d;
    CK(b2s_device_alloc(device, (void**)&cur_d, n));
    CK(b2s_device_alloc(device, (void**)&term_d, n));
    CK(b2s_device_alloc(device, (void**)&rets_d, sizeof(float) * 2 * n));
    CK(b2s_device_alloc(device, (void**)&mask_d, sizeof(uint32_t) * MW * n));
    CK(b2s_device_alloc(device, (void**)&tens_d, sizeof(float) * (size_t)T * n));
    CK(b2s_status(level, (int8_t*)cur_d, term_d, rets_d, n, nullptr));
    CK(b2s_legal_mask(level, mask_d, n, nullptr));
    CK(b2s_information_state(level, -1, tens_d, n, nullptr));
    std::vector<signed char> cur(n); std::vector<unsigned char> term(n); std::vector<float> rets(2 * n), tens((size_t)T * n);
    std::vector<uint32_t> mask((size_t)MW * n);
    CK(b2s_memcpy_d2h(device, cur.data(), cur_d, n, nullptr));
    CK(b2s_memcpy_d2h(device, term.data(), term_d, n, nullptr));
    CK(b2s_memcpy_d2h(device, rets.data(), rets_d, sizeof(float) * 2 * n, nullptr));
    CK(b2s_memcpy_d2h(device, mask.data(), mask_d, sizeof(uint32_t) * MW * n, nullptr));
    CK(b2s_memcpy_d2h(device, tens.data(), tens_d, sizeof(float) * (size_t)T * n, nullptr));
    CK(b2s_stream_synchronize(device, nullptr));
    b2s_device_free(device, cur_d); b2s_device_free(device, term_d); b2s_device_free(device, rets_d);
    b2s_device_free(device, mask_d); b2s_device_free(device, tens_d);
    // node records + the child list of the next level
    std::vector<long long> src_lanes;
    std::vector<int32_t> actions;
    kind.resize(base + n); actor.resize(base + n); nchild.resize(base + n); first_child.resize(base + n);
    infoset.resize(base + n, -1); ret.resize(2 * (base + n), 0.0);
    long long next_base = base + n;
    for (long long i = 0; i < n; ++i) {
      long long id = base + i;
      first_child[id] = (int)(next_base + (long long)src_lanes.size());
      if (term[i]) {
        kind[id] = 0; actor[id] = 0; nchild[id] = 0;
        ret[2 * id] = (double)rets[2 * i]; ret[2 * id + 1] = (double)rets[2 * i + 1];
        counts[2]++;
        continue;
      }
      std::vector<int> acts;
      for (int w = 0; w < MW; ++w)
        for (int b = 0; b < 32; ++b) if ((mask[(size_t)i * MW + w] >> b) & 1u) acts.push_back(w * 32 + b);
      if (acts.empty() || acts.size() > 120) CK(fail("cfr: unexpected legal-action count"));
      nchild[id] = (signed char)acts.size();
      if (cur[i] == -1) {                                    // chance: uniform over the available outcomes
        kind[id] = 1; actor[id] = 2; counts[0]++;            // (kuhn_poker.cc:329-337, leduc_poker.cc:546-571)
      } else {
        kind[id] = 2; actor[id] = cur[i]; counts[1]++;
        std::string key((const char*)&tens[(size_t)i * T], sizeof(float) * T);
        auto itk = key_to_is.find(key);
        int is;
        if (itk == key_to_is.end()) {
          is = (int)key_to_is.size();
          key_to_is.emplace(key, is);
          S->is_player.push_back(cur[i]);
          is_nact.push_back((int)acts.size());
          S->keys.insert(S->keys.end(), tens.begin() + (size_t)i * T, tens.begin() + (size_t)(i + 1) * T);
          S->is_off.push_back((int)S->legal_actions.size());
          for (int a : acts) S->legal_actions.push_back(a);
        } else {
          is = itk->second;
          if (is_nact[is] != (int)acts.size()) CK(fail("cfr: information state with inconsistent legal actions"));
        }
        infoset[id] = is;
      }
      for (size_t k = 0; k < acts.size(); ++k) {
        src_lanes.push_back(i);
        actions.push_back(acts[k]);
        parent.push_back((int)id);
        aidx.push_back((signed char)k);
        chance_prob.push_back(cur[i] == -1 ? 1.0 / (double)acts.size() : 0.0);
      }
    }
    level_off.push_back((int)(base + n));
    long long m = (long long)src_lanes.size();
    if (m == 0) break;
    // next level = clone of each parent lane, then the child action applied
    CK(b2s_batch_create(game_id, params, m, device, &next));
    long long* lanes_d; int32_t* act_d;
    CK(b2s_device_alloc(device, (void**)&lanes_d, sizeof(long long) * m));
    CK(b2s_device_alloc(device, (void**)&act_d, sizeof(int32_t) * m));
    CK(b2s_memcpy_h2d(device, lanes_d, src_lanes.data(), sizeof(long long) * m, nullptr));
    CK(b2s_memcpy_h2d(device, act_d, actions.data(), sizeof(int32_t) * m, nullptr));
    CK(b2s_gather_states(next, level, (const int64_t*)lanes_d, m, nullptr));
    CK(b2s_apply_actions(next, act_d, m, nullptr));
    int64_t bad = 0;
    CK(b2s_error_count(next, &bad, nullptr, nullptr));
    b2s_device_free(device, lanes_d); b2s_device_free(device, act_d);
    if (bad) CK(fail("cfr: tree expansion applied an illegal action"));
    b2s_batch_destroy(level);
    level = next; next = nullptr;
    base += n; n = m;
  }
  if (level) { b2s_batch_destroy(level); level = nullptr; }
  const int N = (int)kind.size(), I = (int)S->is_player.size();
  S->is_off.push_back((int)S->legal_actions.size());
  const int E = (int)S->legal_actions.size();
  // histories of each information state in the reference's DFS order (children in action order)
  std::vector<std::vector<int>> by_is(I);
  {
    std::vector<int> stack = {0};
    while (!stack.empty()) {
      int v = stack.back(); stack.pop_back();
      if (kind[v] == 2) by_is[infoset[v]].push_back(v);
      for (int c = nchild[v] - 1; c >= 0; --c) stack.push_back(first_child[v] + c);
    }
  }
  std::vector<int> hist_off(1, 0), hist;
  for (int i = 0; i < I; ++i) { hist.insert(hist.end(), by_is[i].begin(), by_is[i].end()); hist_off.push_back((int)hist.size()); }
  S->node_counts = {counts[0], counts[1], counts[2]};
  // upload
  B2S_CU(cudaSetDevice(device));
  CfrDev& d = S->d;
  memset(&d, 0, sizeof d);
  d.n_nodes = N; d.n_levels = (int)level_off.size() - 1; d.n_infosets = I; d.n_entries = E;
  CK(upload(S, level_off, &d.level_off)); CK(upload(S, parent, &d.parent)); CK(upload(S, kind, &d.kind));
  CK(upload(S, actor, &d.actor)); CK(upload(S, first_child, &d.first_child)); CK(upload(S, nchild, &d.nchild));
  CK(upload(S, aidx, &d.aidx)); CK(upload(S, chance_prob, &d.chance_prob)); CK(upload(S, ret, &d.ret));
  CK(upload(S, infoset, &d.infoset)); CK(upload(S, S->is_player, &d.is_player)); CK(upload(S, S->is_off, &d.is_off));
  CK(upload(S, hist_off, &d.hist_off)); CK(upload(S, hist, &d.hist));
  {
    std::vector<int> hist_is(hist.size(), 0), hist_entry_off(1, 0);
    for (int i = 0; i < I; ++i)
      for (int hh = hist_off[i]; hh < hist_off[i + 1]; ++hh) {
        hist_is[hh] = i;
        hist_entry_off.push_back(hist_entry_off.back() + (S->is_off[i + 1] - S->is_off[i]));
      }
    d.n_hist = (int)hist.size();
    d.n_contrib = hist_entry_off.back();
    CK(upload(S, hist_is, &d.hist_is)); CK(upload(S, hist_entry_off, &d.hist_entry_off));
  }
  {
    std::vector<int> policy_index(N, -1);
    std::vector<signed char> par_actor(N, 2);
    std::vector<double> chance_reach(N, 1.0);
    for (int v = 1; v < N; ++v) {
      int par = parent[v];
      par_actor[v] = actor[par];
      if (kind[par] == 2) policy_index[v] = S->is_off[infoset[par]] + aidx[v];
      chance_reach[v] = kind[par] == 1 ? chance_reach[par] * chance_prob[v] : chance_reach[par];   // parents precede children
    }
    std::vector<int4> mc(N);
    for (int v = 0; v < N; ++v)
      mc[v] = make_int4(first_child[v], kind[v] == 2 ? S->is_off[infoset[v]] : -1,
                        (int)kind[v] | ((int)(actor[v] & 0xff) << 8) | ((int)nchild[v] << 16), 0);
    CK(upload(S, mc, &d.mc_node));
    {
      // Most delta records one sampled traversal can produce, exactly, from the tree (children follow their parents in the node
      // order, so one backward sweep suffices).  External sampling (UpdateRegrets): the traverser's nodes explore every action and
      // write one regret delta per action; the other player's nodes follow one action and write one average-policy delta per
      // action; chance nodes follow one outcome.  Outcome sampling: one path, two deltas per action at the update player's nodes.
      int cap_es = 0, cap_os = 0;
      std::vector<int> es(N), os(N);
      for (int pl = 0; pl < 2; ++pl) {
        for (int v = N - 1; v >= 0; --v) {
          int sum_es = 0, max_es = 0, max_os = 0;
          for (int c = 0; c < nchild[v]; ++c) {
            const int w = first_child[v] + c;
            sum_es += es[w]; max_es = std::max(max_es, es[w]); max_os = std::max(max_os, os[w]);
          }
          if (kind[v] == 2) {
            es[v] = nchild[v] + (actor[v] == pl ? sum_es : max_es);
            os[v] = (actor[v] == pl ? 2 * nchild[v] : 0) + max_os;
          } else {
            es[v] = max_es; os[v] = max_os;                 // chance (one outcome followed) or terminal (no children)
          }
        }
        cap_es = std::max(cap_es, es[0]); cap_os = std::max(cap_os, os[0]);
      }
      S->mc_cap_es = std::max(cap_es, 1); S->mc_cap_os = std::max(cap_os, 1);
    }
    std::vector<signed char> entry_player(S->legal_actions.size(), 0);
    for (int i = 0; i < I; ++i)
      for (int k = S->is_off[i]; k < S->is_off[i + 1]; ++k) entry_player[k] = (signed char)S->is_player[i];
    CK(upload(S, entry_player, &d.entry_player));
    CK(upload(S, policy_index, &d.policy_index)); CK(upload(S, par_actor, &d.par_actor));
    CK(upload(S, chance_reach, &d.chance_reach));
  }
  {
    std::vector<int> node_level(N, 0), is_level(I, 0);
    for (int l = 0; l + 1 < (int)level_off.size(); ++l)
      for (int v = level_off[l]; v < level_off[l + 1]; ++v) node_level[v] = l;
    for (int i = 0; i < I; ++i) {
      is_level[i] = node_level[by_is[i][0]];
      for (int v : by_is[i]) if (node_level[v] != is_level[i]) CK(fail("cfr: information state spans tree levels"));
    }
    CK(upload(S, is_level, &d.is_level));
  }
  CK(alloc_d(S, 3 * (size_t)N, &d.reach)); CK(alloc_d(S, N, &d.edge_prob)); CK(alloc_d(S, 2 * (size_t)N, &d.value));
  CK(alloc_d(S, E, &d.regrets)); CK(alloc_d(S, E, &d.cum_policy)); CK(alloc_d(S, E, &d.cur_policy));
  CK(alloc_d(S, 2 * (size_t)d.n_contrib, &d.delta));
  {
    void* it = nullptr;
    B2S_CU(cudaMalloc(&it, sizeof(int)));
    B2S_CU(cudaMemset(it, 0, sizeof(int)));
    S->allocs.push_back(it);
    d.iter_d = (int*)it;
  }
  // CFRInfoStateValues(legal_actions): regrets 0, cumulative policy 0, current policy uniform (cfr.h:42-98)
  std::vector<double> uni(E);
  for (int i = 0; i < I; ++i)
    for (int k = S->is_off[i]; k < S->is_off[i + 1]; ++k) uni[k] = 1.0 / (double)(S->is_off[i + 1] - S->is_off[i]);
  B2S_CU(cudaMemcpy(d.cur_policy, uni.data(), sizeof(double) * E, cudaMemcpyHostToDevice));
  for (int i = 0; i < I; ++i) S->max_actions = std::max(S->max_actions, S->is_off[i + 1] - S->is_off[i]);
  if (S->mccfr_tables) {     // CFRInfoStateValues(legal_actions, kInitialTableValues), external_sampling_mccfr.cc:143
    std::vector<double> init(E, 0.000001);
    B2S_CU(cudaMemcpy(d.regrets, init.data(), sizeof(double) * E, cudaMemcpyHostToDevice));
    B2S_CU(cudaMemcpy(d.cum_policy, init.data(), sizeof(double) * E, cudaMemcpyHostToDevice));
  }
  *out_solver = S;
  return 0;
}

void b2s_cfr_destroy(void* solver) {
  if (!solver) return;
  CfrSolver* S = (CfrSolver*)solver;
  cudaSetDevice(S->device);
  delete S;
}

int b2s_cfr_iterate(void* solver, int iters, void* stream) {
  if (!solver) return fail("cfr: null solver");
  if (iters < 0) return fail("cfr: negative iteration count");
  CfrSolver* S = (CfrSolver*)solver;
  B2S_CU(cudaSetDevice(S->device));
  if (iters == 0) return 0;
  k_cfr<<<1, 1024, 0, (cudaStream_t)stream>>>(S->d, iters, S->iteration, S->linear_averaging, S->rm_plus);
  ++g_launches;
  S->iteration += iters;
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return cuda_fail(e, "k_cfr launch");
  return 0;
}

// How the K traversals' deltas reach the tables (all three add the same numbers in the same order; the GPU suite compares them
// bit for bit):
//   kMcScatter (default)  traversals write delta logs, k_mccfr_scatter expands them into the dense [K][width] rows, k_mccfr_apply
//                         streams the rows (coalesced, at HBM speed) — the fastest when the rows fit comfortably in HBM;
//   kMcLanes64            traversals write delta logs, k_mccfr_partial_log adds them lane by lane in shared memory: no [K][width]
//                         buffer at all (memory O(K x records) instead of O(K x table)), but each lane's K / 64 traversals are a
//                         sequential chain — chosen when the dense rows would exceed kMcDenseMaxBytes (or B2S_MCCFR_MODE=lanes);
//   kMcDense              round 1's path: the traversals read-modify-write their dense rows themselves (B2S_MCCFR_MODE=dense, or
//                         B2S_MCCFR_DENSE=1; kept for the before / after measurement, and when a partial row does not fit shared memory).
enum McMode { kMcScatter = 0, kMcLanes64 = 1, kMcDense = 2 };
constexpr size_t kMcLogMaxShared = 200 * 1024;
constexpr size_t kMcDenseMaxBytes = (size_t)8 << 30;
static McMode mccfr_mode(const CfrSolver*, int rows, int width) {
  static const int forced = [] {
    if (const char* d = getenv("B2S_MCCFR_DENSE")) if (atoi(d) != 0) return (int)kMcDense;
    const char* e = getenv("B2S_MCCFR_MODE");
    if (!e) return -1;
    if (!strcmp(e, "dense")) return (int)kMcDense;
    if (!strcmp(e, "lanes")) return (int)kMcLanes64;
    if (!strcmp(e, "scatter")) return (int)kMcScatter;
    return -1;
  }();
  const bool lanes_fit = sizeof(double) * (size_t)width <= kMcLogMaxShared;
  if (forced == kMcLanes64 && lanes_fit) return kMcLanes64;
  if (forced == kMcDense || forced == kMcScatter) return (McMode)forced;
  const size_t dense_bytes = sizeof(double) * (size_t)width * (size_t)rows;
  return (dense_bytes > kMcDenseMaxBytes && lanes_fit) ? kMcLanes64 : kMcScatter;
}
static McLog mccfr_log(const CfrSolver* S) { return McLog{S->mc_log, S->mc_counts, S->mc_log_cap}; }

// rows_needed: traversal threads of one launch; width: entries per row (E, or 2E for outcome sampling); cap: records per
// traversal when the log path is taken
static int mccfr_prepare(CfrSolver* S, int rows_needed, int width, int cap) {
  if (!S->mccfr_tables) return fail("mccfr: the solver was not created with B2S_CFR_MCCFR_TABLES");
  if (S->max_actions > kMcMaxActions || S->d.n_levels > kMcMaxDepth) return fail("mccfr: game tree too wide / deep for the device traversal");
  B2S_CU(cudaSetDevice(S->device));
  const int E = S->d.n_entries;
  if (!S->mc_err) {
    B2S_CU(cudaMalloc((void**)&S->mc_err, sizeof(int)));
    B2S_CU(cudaMemset(S->mc_err, 0, sizeof(int)));
  }
  const McMode mode = mccfr_mode(S, rows_needed, width);
  if (mode != kMcDense) {
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
    if (mode == kMcLanes64 && !S->mc_partials) {
      B2S_CU(cudaMalloc((void**)&S->mc_partials, sizeof(double) * (size_t)kMcLanes * 2 * (size_t)E));
      static bool attr = false;
      if (!attr) {
        B2S_CU(cudaFuncSetAttribute(k_mccfr_partial_log, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kMcLogMaxShared));
        attr = true;
      }
    }
    if (mode == kMcLanes64) return 0;
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

int b2s_mccfr_traverse_lanes(void* solver, int player, int traversals_per_update, uint64_t seed, int lane_begin, int lane_end,
                             double* partials_d, void* stream) {
  if (!solver || !partials_d) return fail("mccfr: null argument");
  CfrSolver* S = (CfrSolver*)solver;
  if (player < 0 || player > 1 || traversals_per_update < 1) return fail("mccfr: bad player / traversals_per_update");
  if (lane_begin < 0 || lane_end > kMcLanes || lane_begin >= lane_end) return fail("mccfr: lane range must lie within [0, 64)");
  const int K = traversals_per_update, L = lane_end - lane_begin, E = S->d.n_entries;
  const int n_threads = L * ((K + 63) / 64);
  if (int r = mccfr_prepare(S, n_threads, E, S->mc_cap_es)) return r;
  cudaStream_t st = (cudaStream_t)stream;
  unsigned phase = (unsigned)(S->iteration * 2 + player);
  const McMode mode = mccfr_mode(S, n_threads, E);
  if (mode == kMcLanes64) {
    k_mccfr_es<true><<<(n_threads + 127) / 128, 128, 0, st>>>(S->d, player, phase, seed, K, lane_begin, L, n_threads, nullptr, mccfr_log(S), S->mc_err, 1);
    k_mccfr_partial_log<<<L, kMcLogThreads, sizeof(double) * (size_t)E, st>>>(K, lane_begin, L, mccfr_log(S), E, partials_d);
  } else {
    if (mode == kMcScatter) {
      const long long slots = (long long)n_threads * S->mc_log_cap;
      k_mccfr_es<true><<<(n_threads + 127) / 128, 128, 0, st>>>(S->d, player, phase, seed, K, lane_begin, L, n_threads, nullptr, mccfr_log(S), S->mc_err, 1);
      k_mccfr_scatter<<<(unsigned)((slots + 255) / 256), 256, 0, st>>>(mccfr_log(S), slots, E, S->mc_rows);
      ++g_launches;
    } else {
      k_mccfr_es<false><<<(n_threads + 127) / 128, 128, 0, st>>>(S->d, player, phase, seed, K, lane_begin, L, n_threads, S->mc_rows, McLog{}, S->mc_err, 1);
    }
    k_mccfr_partial<<<(E + kMcTile - 1) / kMcTile, dim3(kMcTile, kMcLanes), 0, st>>>(S->d, K, lane_begin, L, S->mc_rows, partials_d);
  }
  g_launches += 2;
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return cuda_fail(e, "k_mccfr launch");
  return 0;
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
  int bad = 0;
  B2S_CU(cudaMemcpyAsync(&bad, S->mc_err, sizeof(int), cudaMemcpyDeviceToHost, st));
  B2S_CU(cudaStreamSynchronize(st));
  if (bad) return fail("mccfr: a sampling step found sum of probabilities <= z (SampleActionIndex, cfr.cc:617-628)");
  return 0;
}

static int mccfr_check_errors(CfrSolver* S, cudaStream_t st) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return cuda_fail(e, "k_mccfr launch");
  int bad = 0;
  B2S_CU(cudaMemcpyAsync(&bad, S->mc_err, sizeof(int), cudaMemcpyDeviceToHost, st));
  B2S_CU(cudaStreamSynchronize(st));
  if (bad) return fail("mccfr: a sampling step found sum of probabilities <= z (SampleActionIndex, cfr.cc:617-628)");
  return 0;
}

int b2s_mccfr_external_iterate_ex(void* solver, int iters, int traversals_per_update, uint64_t seed, int flags, void* stream) {
  if (!solver) return fail("mccfr: null solver");
  CfrSolver* S = (CfrSolver*)solver;
  if (iters < 0 || traversals_per_update < 1) return fail("mccfr: iters >= 0 and traversals_per_update >= 1 required");
  if (int r = mccfr_prepare(S, traversals_per_update, S->d.n_entries, S->mc_cap_es)) return r;
  cudaStream_t st = (cudaStream_t)stream;
  const int K = traversals_per_update, E = S->d.n_entries;
  const int full = (flags & B2S_MCCFR_FULL_AVERAGE) ? 1 : 0;
  const McMode mode = mccfr_mode(S, K, E);
  const dim3 ablock(kMcTile, kMcLanes);
  const unsigned agrid = (unsigned)((E + kMcTile - 1) / kMcTile);
  const long long slots = (long long)K * S->mc_log_cap;
  for (int it = 0; it < iters; ++it) {
    for (int p = 0; p < 2; ++p) {
      unsigned phase = (unsigned)(S->iteration * 2 + p);
      if (mode == kMcLanes64) {
        k_mccfr_es<true><<<(K + 127) / 128, 128, 0, st>>>(S->d, p, phase, seed, K, 0, kMcLanes, K, nullptr, mccfr_log(S), S->mc_err, full ? 0 : 1);
        k_mccfr_partial_log<<<kMcLanes, kMcLogThreads, sizeof(double) * (size_t)E, st>>>(K, 0, kMcLanes, mccfr_log(S), E, S->mc_partials);
        k_mccfr_combine<<<agrid, ablock, 0, st>>>(S->d, p, S->mc_partials, E, 0);
        g_launches += 3;
      } else if (mode == kMcScatter) {
        k_mccfr_es<true><<<(K + 127) / 128, 128, 0, st>>>(S->d, p, phase, seed, K, 0, kMcLanes, K, nullptr, mccfr_log(S), S->mc_err, full ? 0 : 1);
        k_mccfr_scatter<<<(unsigned)((slots + 255) / 256), 256, 0, st>>>(mccfr_log(S), slots, E, S->mc_rows);
        k_mccfr_apply<<<agrid, ablock, 0, st>>>(S->d, p, K, S->mc_rows, E, 0);
        g_launches += 3;
      } else {
        k_mccfr_es<false><<<(K + 127) / 128, 128, 0, st>>>(S->d, p, phase, seed, K, 0, kMcLanes, K, S->mc_rows, McLog{}, S->mc_err, full ? 0 : 1);
        k_mccfr_apply<<<agrid, ablock, 0, st>>>(S->d, p, K, S->mc_rows, E, 0);
        g_launches += 2;
      }
    }
    if (full) { k_mccfr_full_average<<<1, 1024, 0, st>>>(S->d); ++g_launches; }     // RunIteration, external_sampling_mccfr.cc:76-79
    ++S->iteration;
  }
  return mccfr_check_errors(S, st);
}

int b2s_mccfr_external_iterate(void* solver, int iters, int traversals_per_update, uint64_t seed, void* stream) {
  return b2s_mccfr_external_iterate_ex(solver, iters, traversals_per_update, seed, 0, stream);
}

int b2s_mccfr_outcome_iterate(void* solver, int iters, int trajectories_per_update, uint64_t seed, double epsilon, void* stream) {
  if (!solver) return fail("mccfr: null solver");
  CfrSolver* S = (CfrSolver*)solver;
  if (iters < 0 || trajectories_per_update < 1) return fail("mccfr: iters >= 0 and trajectories_per_update >= 1 required");
  if (!(epsilon >= 0.0 && epsilon <= 1.0)) return fail("mccfr: epsilon must lie in [0, 1]");
  if (int r = mccfr_prepare(S, trajectories_per_update, 2 * S->d.n_entries, S->mc_cap_os)) return r;       // rows are [K][2E]
  cudaStream_t st = (cudaStream_t)stream;
  const int K = trajectories_per_update, E = S->d.n_entries;
  const dim3 ablock(kMcTile, kMcLanes);
  const unsigned agrid = (unsigned)((E + kMcTile - 1) / kMcTile);
  const McMode mode = mccfr_mode(S, K, 2 * E);
  const long long slots = (long long)K * S->mc_log_cap;
  for (int it = 0; it < iters; ++it) {
    for (int p = 0; p < 2; ++p) {
      unsigned phase = (unsigned)(S->iteration * 2 + p);
      if (mode == kMcScatter) {
        k_mccfr_os<true><<<(K + 127) / 128, 128, 0, st>>>(S->d, p, phase, seed, K, epsilon, nullptr, mccfr_log(S), S->mc_err);
        k_mccfr_scatter<<<(unsigned)((slots + 255) / 256), 256, 0, st>>>(mccfr_log(S), slots, 2 * E, S->mc_rows);
        k_mccfr_apply<<<agrid, ablock, 0, st>>>(S->d, p, K, S->mc_rows, 2 * E, 1);
        k_mccfr_apply<<<agrid, ablock, 0, st>>>(S->d, p, K, S->mc_rows + E, 2 * E, 2);
        g_launches += 4;
      } else if (mode == kMcLanes64) {
        k_mccfr_os<true><<<(K + 127) / 128, 128, 0, st>>>(S->d, p, phase, seed, K, epsilon, nullptr, mccfr_log(S), S->mc_err);
        k_mccfr_partial_log<<<kMcLanes, kMcLogThreads, sizeof(double) * 2 * (size_t)E, st>>>(K, 0, kMcLanes, mccfr_log(S), 2 * E, S->mc_partials);
        k_mccfr_combine<<<agrid, ablock, 0, st>>>(S->d, p, S->mc_partials, 2 * E, 1);
        k_mccfr_combine<<<agrid, ablock, 0, st>>>(S->d, p, S->mc_partials + E, 2 * E, 2);
        g_launches += 4;
      } else {
        k_mccfr_os<false><<<(K + 127) / 128, 128, 0, st>>>(S->d, p, phase, seed, K, epsilon, S->mc_rows, McLog{}, S->mc_err);
        k_mccfr_apply<<<agrid, ablock, 0, st>>>(S->d, p, K, S->mc_rows, 2 * E, 1);
        k_mccfr_apply<<<agrid, ablock, 0, st>>>(S->d, p, K, S->mc_rows + E, 2 * E, 2);
        g_launches += 3;
      }
    }
    ++S->iteration;
  }
  return mccfr_check_errors(S, st);
}

int b2s_cfr_info_get(void* solver, b2s_cfr_info* out) {
  if (!solver || !out) return fail("cfr: null argument");
  CfrSolver* S = (CfrSolver*)solver;
  out->num_nodes = S->d.n_nodes; out->num_levels = S->d.n_levels; out->num_infosets = S->d.n_infosets;
  out->num_entries = S->d.n_entries; out->key_floats = S->tensor_size; out->iteration = S->iteration;
  out->chance_nodes = S->node_counts[0]; out->decision_nodes = S->node_counts[1]; out->terminal_nodes = S->node_counts[2];
  return 0;
}

int b2s_cfr_export(void* solver, double* regrets_h, double* cum_policy_h, double* cur_policy_h, int32_t* offsets_h,
                   int32_t* legal_actions_h, int32_t* players_h, float* keys_h, void* stream) {
  if (!solver) return fail("cfr: null solver");
  CfrSolver* S = (CfrSolver*)solver;
  B2S_CU(cudaSetDevice(S->device));
  cudaStream_t st = (cudaStream_t)stream;
  size_t eb = sizeof(double) * S->d.n_entries;
  if (regrets_h) B2S_CU(cudaMemcpyAsync(regrets_h, S->d.regrets, eb, cudaMemcpyDeviceToHost, st));
  if (cum_policy_h) B2S_CU(cudaMemcpyAsync(cum_policy_h, S->d.cum_policy, eb, cudaMemcpyDeviceToHost, st));
  if (cur_policy_h) B2S_CU(cudaMemcpyAsync(cur_policy_h, S->d.cur_policy, eb, cudaMemcpyDeviceToHost, st));
  B2S_CU(cudaStreamSynchronize(st));
  if (offsets_h) memcpy(offsets_h, S->is_off.data(), sizeof(int) * S->is_off.size());
  if (legal_actions_h) memcpy(legal_actions_h, S->legal_actions.data(), sizeof(int) * S->legal_actions.size());
  if (players_h) memcpy(players_h, S->is_player.data(), sizeof(int) * S->is_player.size());
  if (keys_h) memcpy(keys_h, S->keys.data(), sizeof(float) * S->keys.size());
  return 0;
}

int b2s_cfr_import(void* solver, const double* regrets_h, const double* cum_policy_h, const double* cur_policy_h,
                   int iteration, void* stream) {
  if (!solver) return fail("cfr: null solver");
  CfrSolver* S = (CfrSolver*)solver;
  B2S_CU(cudaSetDevice(S->device));
  cudaStream_t st = (cudaStream_t)stream;
  size_t eb = sizeof(double) * S->d.n_entries;
  if (regrets_h) B2S_CU(cudaMemcpyAsync(S->d.regrets, regrets_h, eb, cudaMemcpyHostToDevice, st));
  if (cum_policy_h) B2S_CU(cudaMemcpyAsync(S->d.cum_policy, cum_policy_h, eb, cudaMemcpyHostToDevice, st));
  if (cur_policy_h) B2S_CU(cudaMemcpyAsync(S->d.cur_policy, cur_policy_h, eb, cudaMemcpyHostToDevice, st));
  B2S_CU(cudaStreamSynchronize(st));
  if (iteration >= 0) S->iteration = iteration;
  return 0;
}

// Multi-GPU step 1 of 2 for one player's traversal of iteration `iteration` (1-based, as CFRSolverBase::iteration_):
// reach + value passes, then this shard's regret / average-policy deltas into the delta buffer.
int b2s_cfr_traverse_shard(void* solver, int player, int iteration, int shard, int num_shards, void* stream) {
  if (!solver) return fail("cfr: null solver");
  if (player < 0 || player > 1 || num_shards < 1 || shard < 0 || shard >= num_shards) return fail("cfr: bad shard arguments");
  CfrSolver* S = (CfrSolver*)solver;
  B2S_CU(cudaSetDevice(S->device));
  k_cfr_traverse<<<1, 1024, 0, (cudaStream_t)stream>>>(S->d, player, iteration, 0, S->linear_averaging, shard, num_shards);
  ++g_launches;
  S->last_shard_player = player;
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return cuda_fail(e, "k_cfr_traverse launch");
  return 0;
}
// Step 2 of 2 (after the caller all-reduced the contribution buffer): tables += contributions in the reference's order,
// RM+ reset, regret matching — for the player of the preceding b2s_cfr_traverse_shard.
int b2s_cfr_apply_deltas(void* solver, void* stream) {
  if (!solver) return fail("cfr: null solver");
  CfrSolver* S = (CfrSolver*)solver;
  B2S_CU(cudaSetDevice(S->device));
  k_cfr_apply<<<1, 1024, 0, (cudaStream_t)stream>>>(S->d, S->last_shard_player, S->rm_plus);
  ++g_launches;
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return cuda_fail(e, "k_cfr_apply launch");
  return 0;
}
int b2s_cfr_delta_count(void* solver, int64_t* count) {
  if (!solver || !count) return fail("cfr: null argument");
  *count = 2 * (int64_t)((CfrSolver*)solver)->d.n_contrib;
  return 0;
}

// ---- in-library NCCL: the whole sharded iteration loop enqueued by the library, no host code between the steps -----
#define B2S_NCCL(x) do { ncclResult_t _r = (x); if (_r != ncclSuccess) return fail(std::string("nccl: ") + #x + ": " + nccl_api().GetErrorString(_r)); } while (0)

int b2s_nccl_unique_id(void* id128) {
  if (!id128) return fail("nccl: null id");
  const NcclApi& N = nccl_api();
  if (!N.ok()) return fail(N.error);
  ncclUniqueId id;
  B2S_NCCL(N.GetUniqueId(&id));
  static_assert(sizeof(ncclUniqueId) == 128, "ncclUniqueId is 128 bytes");
  memcpy(id128, &id, sizeof id);
  return 0;
}

static int dist_prepare(CfrSolver* S) {
  if (!S->dist_stream) B2S_CU(cudaStreamCreateWithFlags(&S->dist_stream, cudaStreamNonBlocking));
  if (!S->dist_ev) B2S_CU(cudaEventCreateWithFlags(&S->dist_ev, cudaEventDisableTiming));
  return 0;
}

int b2s_cfr_comm_init(void* solver, const void* id128, int rank, int world) {
  if (!solver || !id128) return fail("cfr: null argument");
  if (world < 1 || rank < 0 || rank >= world) return fail("cfr: bad rank / world");
  CfrSolver* S = (CfrSolver*)solver;
  const NcclApi& N = nccl_api();
  if (!N.ok()) return fail(N.error);
  B2S_CU(cudaSetDevice(S->device));
  if (S->comm && S->comm_owned) N.CommDestroy(S->comm);
  S->comm = nullptr;
  ncclUniqueId id;
  memcpy(&id, id128, sizeof id);
  B2S_NCCL(N.CommInitRank(&S->comm, world, id, rank));
  S->comm_owned = true; S->rank = rank; S->world = world;
  if (S->dist_graph) { cudaGraphExecDestroy(S->dist_graph); S->dist_graph = nullptr; }
  return dist_prepare(S);
}

int b2s_cfr_comm_adopt(void* solver, void* nccl_comm, int rank, int world) {
  if (!solver || !nccl_comm) return fail("cfr: null argument");
  if (world < 1 || rank < 0 || rank >= world) return fail("cfr: bad rank / world");
  CfrSolver* S = (CfrSolver*)solver;
  const NcclApi& N = nccl_api();
  if (!N.ok()) return fail(N.error);
  if (S->comm && S->comm_owned) N.CommDestroy(S->comm);
  S->comm = (ncclComm_t)nccl_comm; S->comm_owned = false; S->rank = rank; S->world = world;
  if (S->dist_graph) { cudaGraphExecDestroy(S->dist_graph); S->dist_graph = nullptr; }
  B2S_CU(cudaSetDevice(S->device));
  return dist_prepare(S);
}

constexpr int kGraphIters = 16;     // sharded iterations per CUDA-graph launch

// one EvaluateAndUpdatePolicy (cfr.cc:263-282), sharded: per player traverse -> all-reduce -> apply, all on `st`
static int enqueue_sharded_iteration(CfrSolver* S, cudaStream_t st) {
  const NcclApi& N = nccl_api();
  for (int p = 0; p < 2; ++p) {
    k_cfr_traverse<<<1, 1024, 0, st>>>(S->d, p, 0, 1, S->linear_averaging, S->rank, S->world);
    B2S_NCCL(N.AllReduce(S->d.delta, S->d.delta, 2 * (size_t)S->d.n_contrib, ncclDouble, ncclSum, S->comm, st));
    k_cfr_apply<<<1, 1024, 0, st>>>(S->d, p, S->rm_plus);
    g_launches += 2;
  }
  return 0;
}

int b2s_cfr_iterate_sharded(void* solver, int iters, void* stream) {
  if (!solver) return fail("cfr: null solver");
  if (iters < 0) return fail("cfr: negative iteration count");
  CfrSolver* S = (CfrSolver*)solver;
  if (!S->comm) return fail("cfr: no communicator (b2s_cfr_comm_init / b2s_cfr_comm_adopt first)");
  B2S_CU(cudaSetDevice(S->device));
  if (iters == 0) return 0;
  cudaStream_t user = (cudaStream_t)stream, st = S->dist_stream;
  // order after the caller's stream, run on the solver's own stream (graphs cannot be captured on the legacy stream)
  B2S_CU(cudaEventRecord(S->dist_ev, user));
  B2S_CU(cudaStreamWaitEvent(st, S->dist_ev, 0));
  B2S_CU(cudaMemcpyAsync(S->d.iter_d, &S->iteration, sizeof(int), cudaMemcpyHostToDevice, st));
  B2S_CU(cudaStreamSynchronize(st));          // the source of the copy above is a host field that changes below
  int left = iters;
  if (left >= kGraphIters) {
    if (!S->dist_graph) {
      cudaGraph_t g = nullptr;
      B2S_CU(cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal));
      int rc = 0;
      for (int i = 0; i < kGraphIters && !rc; ++i) rc = enqueue_sharded_iteration(S, st);
      cudaError_t ce = cudaStreamEndCapture(st, &g);
      if (rc) { if (g) cudaGraphDestroy(g); return rc; }
      if (ce != cudaSuccess) return cuda_fail(ce, "cfr: graph capture");
      ce = cudaGraphInstantiate(&S->dist_graph, g, 0);
      cudaGraphDestroy(g);
      if (ce != cudaSuccess) return cuda_fail(ce, "cfr: graph instantiate");
    }
    for (; left >= kGraphIters; left -= kGraphIters) B2S_CU(cudaGraphLaunch(S->dist_graph, st));
  }
  for (; left > 0; --left) if (int rc = enqueue_sharded_iteration(S, st)) return rc;
  S->iteration += iters;
  B2S_CU(cudaEventRecord(S->dist_ev, st));
  B2S_CU(cudaStreamWaitEvent(user, S->dist_ev, 0));
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return cuda_fail(e, "cfr: sharded iteration");
  return 0;
}

// Latency floor of the exchange alone: `count` back-to-back all-reduces of the contribution buffer on the solver's stream
// (what two of them per iteration cost however fast the kernels are).  Synchronous; *seconds = elapsed device time.
int b2s_cfr_allreduce_probe(void* solver, int count, double* seconds) {
  if (!solver || !seconds || count < 1) return fail("cfr: bad probe arguments");
  CfrSolver* S = (CfrSolver*)solver;
  if (!S->comm) return fail("cfr: no communicator");
  const NcclApi& N = nccl_api();
  B2S_CU(cudaSetDevice(S->device));
  cudaStream_t st = S->dist_stream;
  cudaEvent_t e0, e1;
  B2S_CU(cudaEventCreate(&e0)); B2S_CU(cudaEventCreate(&e1));
  cudaGraph_t g = nullptr; cudaGraphExec_t ge = nullptr;
  B2S_CU(cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal));
  ncclResult_t nr = ncclSuccess;
  for (int i = 0; i < count && nr == ncclSuccess; ++i)
    nr = N.AllReduce(S->d.delta, S->d.delta, 2 * (size_t)S->d.n_contrib, ncclDouble, ncclSum, S->comm, st);
  cudaError_t ce = cudaStreamEndCapture(st, &g);
  if (nr != ncclSuccess) return fail(std::string("nccl: ") + N.GetErrorString(nr));
  if (ce != cudaSuccess) return cuda_fail(ce, "probe capture");
  B2S_CU(cudaGraphInstantiate(&ge, g, 0));
  B2S_CU(cudaGraphLaunch(ge, st));            // warm-up
  B2S_CU(cudaStreamSynchronize(st));
  B2S_CU(cudaEventRecord(e0, st));
  B2S_CU(cudaGraphLaunch(ge, st));
  B2S_CU(cudaEventRecord(e1, st));
  B2S_CU(cudaStreamSynchronize(st));
  float ms = 0;
  B2S_CU(cudaEventElapsedTime(&ms, e0, e1));
  *seconds = ms * 1e-3;
  cudaGraphExecDestroy(ge); cudaGraphDestroy(g);
  cudaEventDestroy(e0); cudaEventDestroy(e1);
  return 0;
}

// The contribution buffer: b2s_cfr_delta_count doubles (regret contributions, then average-policy contributions), device pointer.
int b2s_cfr_delta_buffer(void* solver, double** delta_d) {
  if (!solver || !delta_d) return fail("cfr: null argument");
  *delta_d = ((CfrSolver*)solver)->d.delta;
  return 0;
}
int b2s_cfr_set_iteration(void* solver, int iteration) {
  if (!solver) return fail("cfr: null solver");
  ((CfrSolver*)solver)->iteration = iteration;
  return 0;
}

// NashConv of the average policy (use_average != 0) or of the current policy; exploitability = nash_conv / 2.
// values_out (nullable, 4 doubles): best-response values of players 0 and 1, on-policy values of players 0 and 1.
// best_h (nullable, num_infosets ints): the best responder's choice at each of ITS information states, as an index into the
// state's legal actions (TabularBestResponse::BestResponseAction, best_response.cc:194-228: first maximum).
static int cfr_best_response_impl(void* solver, int use_average, double* nash_conv_out, double* values_out, int32_t* best_h, void* stream) {
  if (!solver) return fail("cfr: null argument");
  CfrSolver* S = (CfrSolver*)solver;
  B2S_CU(cudaSetDevice(S->device));
  cudaStream_t st = (cudaStream_t)stream;
  double* pol = nullptr; int* best = nullptr; double* out = nullptr;
  B2S_CU(cudaMalloc((void**)&pol, sizeof(double) * (S->d.n_entries + 1)));
  B2S_CU(cudaMalloc((void**)&best, sizeof(int) * (S->d.n_infosets + 1)));
  B2S_CU(cudaMalloc((void**)&out, sizeof(double) * 4));
  k_cfr_nashconv<<<1, 1024, 0, st>>>(S->d, use_average, pol, best, out);
  ++g_launches;
  double h[4];
  cudaError_t e = cudaMemcpyAsync(h, out, sizeof h, cudaMemcpyDeviceToHost, st);
  if (e == cudaSuccess && best_h) e = cudaMemcpyAsync(best_h, best, sizeof(int) * S->d.n_infosets, cudaMemcpyDeviceToHost, st);
  if (e == cudaSuccess) e = cudaStreamSynchronize(st);
  cudaFree(pol); cudaFree(best); cudaFree(out);
  if (e != cudaSuccess) return cuda_fail(e, "k_cfr_nashconv");
  if (nash_conv_out) *nash_conv_out = (h[0] - h[2]) + (h[1] - h[3]);
  if (values_out) memcpy(values_out, h, sizeof h);
  return 0;
}
int b2s_cfr_nash_conv(void* solver, int use_average, double* nash_conv_out, double* values_out, void* stream) {
  if (!nash_conv_out) return fail("cfr: null argument");
  return cfr_best_response_impl(solver, use_average, nash_conv_out, values_out, nullptr, stream);
}
int b2s_cfr_best_response(void* solver, int use_average, int32_t* best_action_index_h, double* values_out, void* stream) {
  if (!best_action_index_h) return fail("cfr: null argument");
  return cfr_best_response_impl(solver, use_average, nullptr, values_out, best_action_index_h, stream);
}

// Device pointers of the per-action tables (regrets, cumulative policy, current policy; num_entries doubles
// each) so a caller can all-reduce them in place (NCCL) between b2s_cfr_iterate calls.
int b2s_cfr_tables(void* solver, double** regrets_d, double** cum_policy_d, double** cur_policy_d) {
  if (!solver) return fail("cfr: null solver");
  CfrSolver* S = (CfrSolver*)solver;
  if (regrets_d) *regrets_d = S->d.regrets;
  if (cum_policy_d) *cum_policy_d = S->d.cum_policy;
  if (cur_policy_d) *cur_policy_d = S->d.cur_policy;
  return 0;
}

}  // extern "C"
