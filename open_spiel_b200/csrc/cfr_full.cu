// Full-width CFR (single-GPU persistent kernel and the sharded / NCCL iteration) and NashConv / best response on the
// flattened tree of cfr_tree.cu.  Floating-point conventions: cfr.cuh.
#include <float.h>
#include <limits.h>
#include <string.h>

#include <algorithm>
#include <cmath>

#include "cfr.cuh"

namespace b2s {

// The contribution of history h to the regrets and average policy of player p's information state at table offset `off`
// with `na` actions (cfr.cc:379-405), action by action: regret_out(a, regret), then avg_out(a, average-policy increment).
template <class RegretOut, class AvgOut>
__device__ __forceinline__ void cfr_contribution(const CfrDev& d, int h, int p, int off, int na, int linear_averaging, double iteration,
                                                 RegretOut regret_out, AvgOut avg_out) {
  const double self_reach = d.reach[2 * h + p];
  // CounterFactualReachProb: 1.0 * reach[other player] * reach[chance], in index order
  const double cfr_reach = __dmul_rn(__dmul_rn(1.0, d.reach[2 * h + (1 - p)]), d.chance_reach[h]);
  const double vh = d.value[2 * h + p];
  const int fc = d.first_child[h];
  for (int a = 0; a < na; ++a) {
    regret_out(a, __dmul_rn(cfr_reach, __dsub_rn(d.value[2 * (fc + a) + p], vh)));
    const double pol = d.cur_policy[off + a];
    avg_out(a, linear_averaging ? __dmul_rn(__dmul_rn(iteration, self_reach), pol) : __dmul_rn(self_reach, pol));
  }
}

// ApplyRegretMatchingPlusReset (cfr.cc:683-691) when rm_plus, then regret matching.  A reset regret is 0, which regret
// matching leaves out of the positive sum anyway.
__device__ __forceinline__ void cfr_update_policy(const CfrDev& d, int off, int na, int rm_plus) {
  if (rm_plus)
    for (int a = 0; a < na; ++a) if (d.regrets[off + a] < 0) d.regrets[off + a] = 0;
  regret_matching(d.regrets + off, d.cur_policy + off, na);
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
  for (int it = 0; it < iters; ++it) {
    const double iteration = (double)(iteration0 + it + 1);          // ++iteration_ (cfr.cc:264)
    for (int p = 0; p < 2; ++p) {
      cfr_level_passes(d, tid, nt);
      // regret / average-policy update (cfr.cc:379-405) + regret matching (cfr.cc:596-615) for player p
      for (int I = tid; I < d.n_infosets; I += nt) {
        if (d.is_player[I] != p) continue;
        int off = d.is_off[I], na = d.is_off[I + 1] - off;
        for (int hh = d.hist_off[I]; hh < d.hist_off[I + 1]; ++hh)
          cfr_contribution(d, d.hist[hh], p, off, na, linear_averaging, iteration,
                           [&](int a, double regret) { d.regrets[off + a] = __dadd_rn(d.regrets[off + a], regret); },
                           [&](int a, double inc) { d.cum_policy[off + a] = __dadd_rn(d.cum_policy[off + a], inc); });
        cfr_update_policy(d, off, na, rm_plus);
      }
      __syncthreads();
    }
  }
}

// ---- CFR-BR (algorithms/cfr_br.cc:50-82, CFRBRSolver::EvaluateAndUpdatePolicy) ------------------------------------
// Per iteration: (1) the pure best response BR_b of each player b to the current policy (the uniform policy on iteration 1,
// when the reference's best-response computers still hold the UniformPolicy they were built with); (2) for p = 0, 1 the
// traversal ComputeCounterFactualRegret(root, p) with the other player replaced by its best response as a 1.0 / 0.0 policy,
// updating p's regrets and (plain) average policy; (3) regret matching of the whole table.  Both best responses answer the
// same frozen policy and neither traversal reads what the other writes, so both responders share one bottom-up sweep and
// both traversals one set of level steps (cfr_level_passes<2>): L + (L + 1) + 1 barriers per iteration, where k_cfr has
// 2 (L + 2).
//
// The best response follows TabularBestResponse (best_response.cc:79-228, history_tree.cc:160-240; prob_cut_threshold and
// action_value_tolerance at their defaults of -1) operation for operation, every product and sum explicitly rounded:
//   counterfactual reach of a history h of responder b (DecisionNodes): formed from h UPWARD, acc = q * acc from 1.0, with
//     q = the chance probability, the evaluated policy at the other player's nodes, nothing (1.0) at b's own nodes;
//   action value at an information state: sum over its histories in DFS order (GetAllInfoSets) of cf_reach * V(child), from
//     0.0; the choice is the first strict maximum over ascending actions, from lowest();
//   node values from 0.0 in child order: terminal = return of b; chance and other player: sum of prob * V(child);
//     b's own node: sum over ALL children of V(child) * (1.0 at the chosen action, else 0.0).
// The evaluated policy at a decision edge with table index pi below a node with na children.
__device__ __forceinline__ double cfr_br_evaluated(const CfrDev& d, int pi, int na, bool uniform) {
  return uniform ? __ddiv_rn(1.0, (double)na) : d.cur_policy[pi];
}

__global__ void __launch_bounds__(1024) k_cfr_br(CfrDev d, CfrBrDev br, int iters, int iteration0) {
  const int tid = threadIdx.x, nt = blockDim.x, N = d.n_nodes, L = d.n_levels;
  for (int it = 0; it < iters; ++it) {
    const double iteration = (double)(iteration0 + it + 1);          // ++iteration_ (cfr_br.cc:51)
    const bool uniform = iteration0 + it == 0;                        // SetPolicy is skipped while iteration_ == 1
    // (1a) counterfactual reach of every history for the player acting there.  The deepest level holds terminals only, so
    // the barrier closing its level step below orders these writes before the first read.
    for (int hh = tid; hh < d.n_hist; hh += nt) {
      const int h = d.hist[hh], b = d.actor[h];
      double acc = 1.0;
      for (int n = h; n > 0; n = d.parent[n]) {
        const int pi = d.policy_index[n];
        if (pi < 0) acc = __dmul_rn(d.chance_prob[n], acc);
        else if (d.par_actor[n] != b) acc = __dmul_rn(cfr_br_evaluated(d, pi, d.nchild[d.parent[n]], uniform), acc);
      }
      br.cf_reach[hh] = acc;
    }
    // (1b) both best responses, bottom-up, one level step each: a responder's node gets its value from the thread of its
    // information state, which first chooses the action from the children's values; every other node from its children.
    for (int l = L - 1; l >= 0; --l) {
      for (int n = d.level_off[l] + tid; n < d.level_off[l + 1]; n += nt) {
        const int kind = d.kind[n], fc = d.first_child[n], nc = d.nchild[n];
        for (int b = 0; b < 2; ++b) {
          if (kind == 2 && d.actor[n] == b) continue;
          const double* V = br.value + b * N;
          double v;
          if (kind == 0) v = d.ret[2 * n + b];
          else {
            v = 0.0;
            for (int c = 0; c < nc; ++c) {
              const double pr = kind == 1 ? d.chance_prob[fc + c] : cfr_br_evaluated(d, d.policy_index[fc + c], nc, uniform);
              v = __dadd_rn(v, __dmul_rn(pr, V[fc + c]));
            }
          }
          br.value[b * N + n] = v;
        }
      }
      for (int I = tid; I < d.n_infosets; I += nt) {
        if (d.is_level[I] != l) continue;
        const int b = d.is_player[I], na = d.is_off[I + 1] - d.is_off[I], h0 = d.hist_off[I], h1 = d.hist_off[I + 1];
        double* V = br.value + b * N;
        int arg = 0;
        double best_value = -DBL_MAX;
        for (int a = 0; a < na; ++a) {
          double q = 0.0;
          for (int hh = h0; hh < h1; ++hh) q = __dadd_rn(q, __dmul_rn(br.cf_reach[hh], V[d.first_child[d.hist[hh]] + a]));
          if (q > best_value) { best_value = q; arg = a; }
        }
        br.best[I] = arg;
        for (int hh = h0; hh < h1; ++hh) {
          const int h = d.hist[hh], fc = d.first_child[h];
          double v = 0.0;
          for (int a = 0; a < na; ++a) v = __dadd_rn(v, __dmul_rn(V[fc + a], a == arg ? 1.0 : 0.0));
          V[h] = v;
        }
      }
      __syncthreads();
    }
    // (2) traversal t = p: p follows the current policy, the other player its best response (cfr.cc:371-377 overrides).
    cfr_level_passes<2>(d, tid, nt, [&](const CfrDev& g, int n, int t) {
      const int pi = g.policy_index[n];
      if (pi < 0) return g.chance_prob[n];
      if (g.par_actor[n] == t) return g.cur_policy[pi];
      return br.best[g.infoset[g.parent[n]]] == g.aidx[n] ? 1.0 : 0.0;
    });
    // (3) each information state's update from its player's traversal, then regret matching (ApplyRegretMatching after both
    // traversals: every read of the current policy above is behind the last level step's barrier).
    for (int I = tid; I < d.n_infosets; I += nt) {
      const int p = d.is_player[I], off = d.is_off[I], na = d.is_off[I + 1] - off;
      CfrDev dp = d;
      dp.reach += 2 * p * N; dp.value += 2 * p * N;
      for (int hh = d.hist_off[I]; hh < d.hist_off[I + 1]; ++hh)
        cfr_contribution(dp, d.hist[hh], p, off, na, 0, iteration,
                         [&](int a, double regret) { d.regrets[off + a] = __dadd_rn(d.regrets[off + a], regret); },
                         [&](int a, double inc) { d.cum_policy[off + a] = __dadd_rn(d.cum_policy[off + a], inc); });
      cfr_update_policy(d, off, na, 0);
    }
    __syncthreads();
  }
}

// ---- Discounted CFR (python/algorithms/discounted_cfr.py:190-209, _DCFRSolver.evaluate_and_update_policy) -----------
// Per iteration t, for p = 0, 1: (1) player p's traversal (:93-188): cfr.py's values, reach and regrets, the average-policy
// increment (reach * pi) * w_t (:181-184); (2) every regret of p's information states multiplied by pos_t where it is >= 0
// (so -0.0 too) and by neg_t elsewhere (:199-209); (3) regret matching of the whole table (cfr.py:78-98), which player 1's
// traversal then follows.  factors[3 k ...] = (pos_t, neg_t, w_t) of iteration t = base + 1 + k, computed on the host
// (dcfr_factors).
//
// The reference prunes decision nodes no player reaches (:132-133): it returns zeros there and updates nothing below.
// Under DCFR that decides bits: a regret left alone by ~1,075 halvings of beta = 0 is -0.0, and adding the +0.0 or -0.0 of
// a zero-reach contribution flips it or not.  So k_dcfr adds nothing at such histories and takes every other
// contribution, 0 * (V(child) - v) included, from the reference's pruned values.  Those need each node's reach before its
// value: the reach sweep runs to the bottom first, then the value sweep (2L - 1 level steps where cfr_level_passes takes
// L).  Only nodes no player reaches get other values than the fused sweep's; they sit below a zero-probability edge, which
// wipes the difference out of every value above them.
__global__ void __launch_bounds__(1024) k_dcfr(CfrDev d, const double* factors, int iters, int iteration0, int base) {
  const int tid = threadIdx.x, nt = blockDim.x, L = d.n_levels, N = d.n_nodes;
  for (int it = 0; it < iters; ++it) {
    const double* f = factors + 3 * ((size_t)(iteration0 - base) + it);   // t = iteration0 + it + 1: self._iteration += 1 (:192)
    const double pos = f[0], neg = f[1], w = f[2];
    for (int p = 0; p < 2; ++p) {
      for (int n = 1 + tid; n < N; n += nt) d.edge_prob[n] = CurrentPolicyEdge{}(d, n, 0);
      if (tid == 0) { d.reach[0] = 1.0; d.reach[1] = 1.0; }
      __syncthreads();
      for (int l = 1; l < L; ++l) {
        for (int n = d.level_off[l] + tid; n < d.level_off[l + 1]; n += nt) cfr_reach_step<1>(d, N, n);
        __syncthreads();
      }
      for (int l = L - 1; l >= 0; --l) {
        for (int n = d.level_off[l] + tid; n < d.level_off[l + 1]; n += nt) cfr_value_step<1, true>(d, N, n);
        __syncthreads();
      }
      for (int I = tid; I < d.n_infosets; I += nt) {
        const int off = d.is_off[I], na = d.is_off[I + 1] - off;
        if (d.is_player[I] == p) {
          for (int hh = d.hist_off[I]; hh < d.hist_off[I + 1]; ++hh) {
            const int h = d.hist[hh];
            if (d.reach[2 * h] == 0.0 && d.reach[2 * h + 1] == 0.0) continue;
            cfr_contribution(d, h, p, off, na, 0, 0.0,
                             [&](int a, double regret) { d.regrets[off + a] = __dadd_rn(d.regrets[off + a], regret); },
                             [&](int a, double inc) { d.cum_policy[off + a] = __dadd_rn(d.cum_policy[off + a], __dmul_rn(inc, w)); });
          }
          for (int a = 0; a < na; ++a) {
            const double r = d.regrets[off + a];
            d.regrets[off + a] = __dmul_rn(r, r >= 0 ? pos : neg);
          }
        }
        regret_matching(d.regrets + off, d.cur_policy + off, na);
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
    cfr_contribution(d, d.hist[hh], p, off, na, linear_averaging, iter, [&](int a, double regret) { d.delta[co + a] = regret; },
                     [&](int a, double inc) { d.delta[C + co + a] = inc; });
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
    cfr_update_policy(d, off, na, rm_plus);
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
        double r = d.reach[2 * par];
        if (!(d.kind[par] == 2 && d.actor[par] == b)) r *= d.edge_prob[n];
        d.reach[2 * n] = r;
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
            q += d.reach[2 * h] * d.value[2 * (d.first_child[h] + a)];
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

}  // namespace b2s

using namespace b2s;

static const char kNoShardedCfrBr[] = "cfr: a CFR-BR solver (B2S_CFR_BEST_RESPONSE_OPPONENTS) has no sharded iteration";
static const char kNoShardedDcfr[] = "cfr: a DCFR solver (b2s_dcfr_create) has no sharded iteration";

constexpr int kDcfrLaunch = 1 << 20;     // most iterations one k_dcfr launch runs: bounds the factor window
constexpr int kDcfrWindow = 1 << 16;     // fewest iterations a factor window covers

// Makes S->dcfr_factors cover iterations first + 1 .. first + n: (t**alpha / (t**alpha + 1), t**beta / (t**beta + 1),
// t**gamma) as discounted_cfr.py computes them, std::pow being glibc's pow as CPython's float ** is.  A window that does
// not cover them is replaced by one starting at first + 1, of max(n, kDcfrWindow) entries (at most 24 MiB), allocated,
// filled and the old one freed in the order of `st`: launches that read the old window were enqueued before this call,
// and calls on one solver are ordered (b2s.h), so none of them can still be reading it when it is freed.
static int dcfr_factors(CfrSolver* S, int first, int n, cudaStream_t st) {
  if (S->dcfr_factors && first >= S->dcfr_base && (long long)first + n <= (long long)S->dcfr_base + S->dcfr_capacity) return 0;
  const int cap = std::max(n, kDcfrWindow);
  std::vector<double> h(3 * (size_t)cap);
  for (long long k = 0; k < cap; ++k) {
    const double t = (double)(first + 1 + k);
    const double ta = std::pow(t, S->dcfr_alpha), tb = std::pow(t, S->dcfr_beta);
    h[3 * k] = ta / (ta + 1.0);
    h[3 * k + 1] = tb / (tb + 1.0);
    h[3 * k + 2] = std::pow(t, S->dcfr_gamma);
  }
  void* p = nullptr;
  B2S_CU(cudaMallocAsync(&p, sizeof(double) * h.size(), st));
  const cudaError_t e = cudaMemcpyAsync(p, h.data(), sizeof(double) * h.size(), cudaMemcpyHostToDevice, st);  // pageable: staged before return
  if (e != cudaSuccess) { cudaFreeAsync(p, st); return cuda_fail(e, "dcfr: factor window"); }
  if (S->dcfr_factors) B2S_CU(cudaFreeAsync(S->dcfr_factors, st));
  S->dcfr_factors = (double*)p;
  S->dcfr_base = first;
  S->dcfr_capacity = cap;
  return 0;
}

extern "C" {

int b2s_cfr_iterate(void* solver, int iters, void* stream) {
  if (!solver) return fail("cfr: null solver");
  if (iters < 0) return fail("cfr: negative iteration count");
  CfrSolver* S = (CfrSolver*)solver;
  B2S_CU(cudaSetDevice(S->device));
  if (iters == 0) return 0;
  if (S->dcfr) {
    if (S->iteration < 0 || iters > INT_MAX - S->iteration)
      return fail("dcfr: the iteration counter must stay within [0, INT_MAX]");
    for (int left = iters; left > 0;) {
      const int n = std::min(left, kDcfrLaunch);
      if (int r = dcfr_factors(S, S->iteration, n, (cudaStream_t)stream)) return r;
      k_dcfr<<<1, 1024, 0, (cudaStream_t)stream>>>(S->d, S->dcfr_factors, n, S->iteration, S->dcfr_base);
      ++g_launches;
      if (int r = launch_status("k_dcfr launch")) return r;
      S->iteration += n;
      left -= n;
    }
    return 0;
  }
  if (S->best_response_opponents) {
    k_cfr_br<<<1, 1024, 0, (cudaStream_t)stream>>>(S->d, S->br, iters, S->iteration);
    ++g_launches;
    S->iteration += iters;
    return launch_status("k_cfr_br launch");
  }
  k_cfr<<<1, 1024, 0, (cudaStream_t)stream>>>(S->d, iters, S->iteration, S->linear_averaging, S->rm_plus);
  ++g_launches;
  S->iteration += iters;
  return launch_status("k_cfr launch");
}

// Multi-GPU step 1 of 2 for one player's traversal of iteration `iteration` (1-based, as CFRSolverBase::iteration_):
// reach + value passes, then this shard's regret / average-policy deltas into the delta buffer.
int b2s_cfr_traverse_shard(void* solver, int player, int iteration, int shard, int num_shards, void* stream) {
  if (!solver) return fail("cfr: null solver");
  if (player < 0 || player > 1 || num_shards < 1 || shard < 0 || shard >= num_shards) return fail("cfr: bad shard arguments");
  CfrSolver* S = (CfrSolver*)solver;
  if (S->best_response_opponents) return fail(kNoShardedCfrBr);
  if (S->dcfr) return fail(kNoShardedDcfr);
  B2S_CU(cudaSetDevice(S->device));
  k_cfr_traverse<<<1, 1024, 0, (cudaStream_t)stream>>>(S->d, player, iteration, 0, S->linear_averaging, shard, num_shards);
  ++g_launches;
  S->last_shard_player = player;
  return launch_status("k_cfr_traverse launch");
}
// Step 2 of 2 (after the caller all-reduced the contribution buffer): tables += contributions in the reference's order,
// RM+ reset, regret matching — for the player of the preceding b2s_cfr_traverse_shard.
int b2s_cfr_apply_deltas(void* solver, void* stream) {
  if (!solver) return fail("cfr: null solver");
  CfrSolver* S = (CfrSolver*)solver;
  if (S->best_response_opponents) return fail(kNoShardedCfrBr);
  if (S->dcfr) return fail(kNoShardedDcfr);
  B2S_CU(cudaSetDevice(S->device));
  k_cfr_apply<<<1, 1024, 0, (cudaStream_t)stream>>>(S->d, S->last_shard_player, S->rm_plus);
  ++g_launches;
  return launch_status("k_cfr_apply launch");
}
int b2s_cfr_delta_count(void* solver, int64_t* count) {
  if (!solver || !count) return fail("cfr: null argument");
  *count = 2 * (int64_t)((CfrSolver*)solver)->d.n_contrib;
  return 0;
}
// The contribution buffer: b2s_cfr_delta_count doubles (regret contributions, then average-policy contributions), device pointer.
int b2s_cfr_delta_buffer(void* solver, double** delta_d) {
  if (!solver || !delta_d) return fail("cfr: null argument");
  *delta_d = ((CfrSolver*)solver)->d.delta;
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
  if (S->best_response_opponents) return fail(kNoShardedCfrBr);
  if (S->dcfr) return fail(kNoShardedDcfr);
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
  return launch_status("cfr: sharded iteration");
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
  cudaEvent_t e0 = nullptr, e1 = nullptr;
  cudaGraph_t g = nullptr; cudaGraphExec_t ge = nullptr;
  const ScopeExit release{[&] { if (ge) cudaGraphExecDestroy(ge); if (g) cudaGraphDestroy(g); if (e0) cudaEventDestroy(e0); if (e1) cudaEventDestroy(e1); }};
  B2S_CU(cudaEventCreate(&e0)); B2S_CU(cudaEventCreate(&e1));
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
  const ScopeExit release{[&] { cudaFree(pol); cudaFree(best); cudaFree(out); }};
  B2S_CU(cudaMalloc((void**)&pol, sizeof(double) * (S->d.n_entries + 1)));
  B2S_CU(cudaMalloc((void**)&best, sizeof(int) * (S->d.n_infosets + 1)));
  B2S_CU(cudaMalloc((void**)&out, sizeof(double) * 4));
  k_cfr_nashconv<<<1, 1024, 0, st>>>(S->d, use_average, pol, best, out);
  ++g_launches;
  double h[4];
  cudaError_t e = cudaMemcpyAsync(h, out, sizeof h, cudaMemcpyDeviceToHost, st);
  if (e == cudaSuccess && best_h) e = cudaMemcpyAsync(best_h, best, sizeof(int) * S->d.n_infosets, cudaMemcpyDeviceToHost, st);
  if (e == cudaSuccess) e = cudaStreamSynchronize(st);
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

}  // extern "C"
