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
// we reproduce the returned zeros; the skipped updates below such a node add +-0 and change nothing, because CFR's
// regrets are never -0.0.  Discounted CFR's can be (k_dcfr, cfr_full.cu), so k_dcfr prunes exactly as the reference does.
//
// Files: cfr_tree.cu (tree construction, solver lifetime), cfr_full.cu (full-width CFR, CFR-BR, DCFR, NashConv / best response,
// sharded NCCL path), cfr_mccfr.cu (external- and outcome-sampling MCCFR).
#pragma once
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
  double* reach;               // [n][2]  (player 0, player 1); NashConv keeps the responder's counterfactual reach in slot 0;
                               // [2][n][2] on a CFR-BR solver (one [n][2] block per traversal, cfr_level_passes<2>)
  double* edge_prob;           // [n]; [2][n] on a CFR-BR solver
  double* value;               // [n][2]; [2][n][2] on a CFR-BR solver
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

// ApplyRegretMatching (cfr.cc:596-615): the policy of an information state with n actions from its regrets — positive
// regrets normalised by their sum (added in action order), uniform when no regret is positive.  The unroll factors keep each
// kernel that calls this at or below the registers, stack and spills of its former open-coded loops (ptxas -v, sm_90a).
__device__ __forceinline__ void regret_matching(const double* regrets, double* policy, int n) {
  double sum = 0.0;
#pragma unroll 2
  for (int a = 0; a < n; ++a) { double r = regrets[a]; if (r > 0) sum = __dadd_rn(sum, r); }
#pragma unroll 1
  for (int a = 0; a < n; ++a) {
    double r = regrets[a];
    policy[a] = sum > 0 ? (r > 0 ? __ddiv_rn(r, sum) : 0.0) : __ddiv_rn(1.0, (double)n);
  }
}

// The probability of the edge into node n under the frozen current policy: the policy at decision nodes, the chance
// probability below chance nodes.  Traversal index t is unused: every traversal of plain CFR follows the same policy.
struct CurrentPolicyEdge {
  __device__ __forceinline__ double operator()(const CfrDev& d, int n, int) const {
    int pi = d.policy_index[n];
    return pi >= 0 ? d.cur_policy[pi] : d.chance_prob[n];
  }
};

// The reach probabilities of node n (not the root) in each of T traversals, from its parent's:
// new_reach_probabilities[current_player] *= prob (cfr.cc:457).
template <int T>
__device__ __forceinline__ void cfr_reach_step(const CfrDev& d, int N, int n) {
  int par = d.parent[n];
  int a = d.par_actor[n];
#pragma unroll
  for (int t = 0; t < T; ++t) {
    double* reach = d.reach + 2 * t * N;
    double r0 = reach[2 * par], r1 = reach[2 * par + 1];
    if (a == 0) r0 = __dmul_rn(r0, d.edge_prob[t * N + n]); else if (a == 1) r1 = __dmul_rn(r1, d.edge_prob[t * N + n]);
    reach[2 * n] = r0; reach[2 * n + 1] = r1;
  }
}

// The state values of node n in each of T traversals, from its children's: state_value[i] += prob * child_value[i]
// (cfr.cc:461-463).  Prune: a decision node that no player reaches is worth zeros, as the reference returns there
// (cfr.cc:350-355, discounted_cfr.py:132-133); its reach must already be in place.
template <int T, bool Prune = false>
__device__ __forceinline__ void cfr_value_step(const CfrDev& d, int N, int n) {
#pragma unroll
  for (int t = 0; t < T; ++t) {
    double* value = d.value + 2 * t * N;
    const double* edge_prob = d.edge_prob + t * N;
    double v0, v1;
    if (d.kind[n] == 0) { v0 = d.ret[2 * n]; v1 = d.ret[2 * n + 1]; }
    else {
      v0 = 0.0; v1 = 0.0;
      if (!Prune || d.kind[n] != 2 || d.reach[2 * t * N + 2 * n] != 0.0 || d.reach[2 * t * N + 2 * n + 1] != 0.0) {
        int fc = d.first_child[n];
        for (int c = 0; c < d.nchild[n]; ++c) {
          double pr = edge_prob[fc + c];
          v0 = __dadd_rn(v0, __dmul_rn(pr, value[2 * (fc + c)]));
          v1 = __dadd_rn(v1, __dmul_rn(pr, value[2 * (fc + c) + 1]));
        }
      }
    }
    value[2 * n] = v0; value[2 * n + 1] = v1;
  }
}

// T traversals' tree passes, shared by the single-GPU kernel, the sharded one, MCCFR's full averaging (T = 1) and CFR-BR
// (T = 2): (1) edge probabilities edge(d, n, t) from the frozen policies, (2) L level steps in which the reach probabilities
// move one level DOWN while the state values move one level UP.  Traversal t keeps its edge probabilities at
// edge_prob[t * n ...], its reach and values at reach / value[2 * t * n ...] (n = number of nodes).
template <int T = 1, class EdgeProb = CurrentPolicyEdge>
__device__ __forceinline__ void cfr_level_passes(const CfrDev& d, int tid, int nt, EdgeProb edge = {}) {
  const int L = d.n_levels, N = d.n_nodes;
  for (int n = 1 + tid; n < N; n += nt) {
#pragma unroll
    for (int t = 0; t < T; ++t) d.edge_prob[t * N + n] = edge(d, n, t);
  }
  if (tid == 0) {
#pragma unroll
    for (int t = 0; t < T; ++t) { d.reach[2 * t * N] = 1.0; d.reach[2 * t * N + 1] = 1.0; }
  }
  __syncthreads();
  for (int k = 0; k < L; ++k) {
    int ld = k + 1;
    if (ld < L)
      for (int n = d.level_off[ld] + tid; n < d.level_off[ld + 1]; n += nt) cfr_reach_step<T>(d, N, n);
    int lu = L - 1 - k;
    for (int n = d.level_off[lu] + tid; n < d.level_off[lu + 1]; n += nt) cfr_value_step<T>(d, N, n);
    __syncthreads();
  }
}

// CFR-BR's best-response scratch (a kernel argument of k_cfr_br only, so CfrDev and the other kernels stay as they are).
struct CfrBrDev {
  int* best;                   // [I] the pure best response at information state I, as an index into its legal actions
  double* cf_reach;            // [n_hist] counterfactual reach of history slot hh for the player acting there
  double* value;               // [2][n] best-response value of every node for responder 0, then responder 1
};

struct CfrSolver {
  // multi-GPU: communicator (owned or adopted), private stream + a CUDA graph of kGraphIters sharded iterations
  ncclComm_t comm = nullptr; bool comm_owned = false; int rank = 0, world = 1;
  cudaStream_t dist_stream = nullptr; cudaEvent_t dist_ev = nullptr;
  cudaGraphExec_t dist_graph = nullptr;
  int last_shard_player = 0;
  int mccfr_tables = 0;
  double* mc_rows = nullptr; int mc_rows_k = 0;              // [rows][E] dense delta rows the scatter path expands the logs into
  int4* mc_log = nullptr; int* mc_counts = nullptr;          // delta logs [mc_log_rows][mc_log_cap] + record counts
  int mc_log_rows = 0, mc_log_cap = 0;
  double* mc_partials = nullptr;                             // [64][2E] lane partial sums of the lanes path
  int mc_cap_es = 0, mc_cap_os = 0;                          // most records one traversal / one episode can write (from the tree)
  int* mc_err = nullptr;
  int max_actions = 0;
  int device = 0;
  int game_id = 0;
  int iteration = 0;
  int linear_averaging = 0, rm_plus = 0;
  int best_response_opponents = 0;                           // CFR-BR (B2S_CFR_BEST_RESPONSE_OPPONENTS): k_cfr_br, br scratch
  CfrBrDev br{};
  int dcfr = 0;                                              // Discounted CFR (b2s_dcfr_create): k_dcfr, factor table
  double dcfr_alpha = 0, dcfr_beta = 0, dcfr_gamma = 0;
  double* dcfr_factors = nullptr;                            // [dcfr_capacity][3]: (pos_t, neg_t, w_t) of t = dcfr_base + 1 + k
  int dcfr_base = 0, dcfr_capacity = 0;
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
    if (dcfr_factors) cudaFree(dcfr_factors);
  }
};

// Status of the kernel launches just enqueued: 0, or "<what>: <cuda error>".
inline int launch_status(const char* what) {
  const cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? 0 : cuda_fail(e, what);
}

// Runs f when the scope ends, on every return path (device buffers, events and graphs of one call).
template <class F> struct ScopeExit {
  F f;
  ~ScopeExit() { f(); }
};
template <class F> ScopeExit(F) -> ScopeExit<F>;

}  // namespace b2s
