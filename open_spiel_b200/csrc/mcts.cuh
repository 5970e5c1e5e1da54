// Device-resident MCTS: one search tree per thread (root parallelism), every tree in its own node arena.
// Semantics: reference open_spiel/algorithms/mcts.cc — ApplyTreePolicy :273-351 (expand on the second visit,
// children in a random order, first-max UCT / PUCT selection), RandomRolloutEvaluator::Evaluate :43-72, MCTSearch
// :353-467 (backup from the point of view of the player who chose each node, MCTS-Solver propagation, early exit when
// the root is proven or has a single child, node budget + GarbageCollect :441-482, wall-clock budget :362-365),
// BestChild / CompareFinal :114-143.
// A single tree is inherently sequential (every simulation sees the statistics of all earlier ones), so one
// thread runs one tree exactly in the reference's order and throughput comes from running thousands of
// independent roots per GPU.  Random decisions are an explicit function of (seed, tree, simulation, position)
// through Philox (common.cuh), the same function oracle/algorithms/mcts.cc uses, so trees match bit for bit:
//   expansion #e:  Fisher-Yates over the ascending legal list, j = rng(key, e, i, 1, i+1) for i = n-1..1
//   simulation #t, rollout #r, ply p:  k = shared(key, t, p + 4096 q, 2+r, C) over the C playout candidates
//     (the legal actions; for go: empty non-ko points + pass), q = 0,1,.. until the candidate is legal; shared(.., b, ..)
//     is word (b & 3) of the Philox block of (t, b >> 2, 2+r) — four consecutive plies share one block (PlayoutRng)
// UCT arithmetic is done with explicitly rounded double operations (no FMA contraction) and log(N_parent)
// comes from a table the HOST fills with std::log, so values equal the CPU's to the last bit.
//
// Memory.  The reference's SearchNode is 80 bytes + heap vectors; a 100k-simulation go tree has ~5e5 of them.  Here a
// node is 16 bytes (MctsNodeC): visits, an INTEGER reward numerator (returns of the five board games are -1 / 0 / +1, so
// with n_rollouts a power of two the reference's double total_reward is exactly numerator / n_rollouts), the index of
// its children block inside the tree's arena, and a packed word (action, #children, player, proven outcome).  Searches
// whose n_rollouts is not a power of two use 24-byte nodes with the reference's double accumulator (MctsNodeW).
// Every tree owns a contiguous arena of `nodes_per_tree` slots: children blocks are bump-allocated, and blocks released
// by the garbage collector go to per-size free lists (exact fit first, then the bump pointer, then splitting a larger
// free block).  The reference's `nodes_` accounting (+= children.capacity() on expansion, -= on collection) is kept
// as a separate logical counter, so collections happen after exactly the same simulations as in the reference.
//
// Selection is the reference's first-maximum scan in FP64 (an unvisited child is +infinity, so the first unvisited child ends
// the scan).  A float32 pre-selection with a proven error margin (FP64 only for children whose estimate could still win) was
// tried and removed.
// Not implemented here: chance nodes in the tree.  Custom evaluators and Dirichlet noise are the caller-evaluated search of
// mcts_eval.cuh (b2s_mcts_eval_*); the host adapters still route MCTSBots with per-state evaluators to the stock MCTSBot.
#pragma once
#include <type_traits>

#include "common.cuh"

namespace b2s {

// meta word of a node: action (10 bits) | number of children (9) | player who chose the action (1) | proven (1) | outcome (2);
// bits 23-31 are free.  Nine child-count bits hold go 19x19's 362 children.
// outcome: 0 = draw {0,0}, 1 = player 0 won {+1,-1}, 2 = player 1 won {-1,+1}
constexpr int kMetaMaxChildren = 511;
__host__ __device__ __forceinline__ u32 mcts_meta(int action, int nchild, int player, int proven, int outcome) {
  return (u32)(action & 1023) | (u32)nchild << 10 | (u32)player << 19 | (u32)proven << 20 | (u32)outcome << 21;
}
__host__ __device__ __forceinline__ int meta_action(u32 m) { return (int)(m & 1023); }
__host__ __device__ __forceinline__ int meta_nchild(u32 m) { return (int)((m >> 10) & 511); }
__host__ __device__ __forceinline__ int meta_player(u32 m) { return (int)((m >> 19) & 1); }
__host__ __device__ __forceinline__ int meta_proven(u32 m) { return (int)((m >> 20) & 1); }
__host__ __device__ __forceinline__ int meta_outcome(u32 m) { return (int)((m >> 21) & 3); }
// the same word with `n` children / proven with outcome `code`
__host__ __device__ __forceinline__ u32 meta_set_nchild(u32 m, int n) { return (m & ~(511u << 10)) | (u32)n << 10; }
__host__ __device__ __forceinline__ u32 meta_set_proven(u32 m, int code) { return (m & ~(7u << 20)) | 1u << 20 | (u32)code << 21; }
// child cursor of the collector's depth-first walk: one byte per stack level unless a node can have more than 255 children
template <int KMAX> using GcCursor = typename std::conditional<(KMAX > 255), unsigned short, unsigned char>::type;
// value of a proven outcome for player p: +1 / -1 / 0
__host__ __device__ __forceinline__ int outcome_value(int code, int p) { return code == 0 ? 0 : ((code == 1) == (p == 0) ? 1 : -1); }

struct __align__(16) MctsNodeC {    // compact: 16 B
  int reward;                       // sum over simulations of (sum over rollouts of returns[player]); total_reward = reward / n_rollouts
  u32 visits;                       // explore_count
  u32 first_child;                  // arena index (within the tree) of the first child; children are contiguous; 0 = none
  u32 meta;
};
struct __align__(8) MctsNodeW {     // wide: 24 B, the reference's double accumulator (n_rollouts not a power of two)
  double reward;
  u32 visits;
  u32 first_child;
  u32 meta;
  u32 pad;
};
struct __align__(16) MctsNodeE {    // caller-evaluated search (mcts_eval.cuh): 32 B, evaluator values are arbitrary doubles
  double reward;                    // total_reward
  double prior;                     // SearchNode::prior
  u32 visits;                       // explore_count
  u32 first_child;                  // children block; while unexpanded (#children 0) the cached-prior block if ncache > 0
  u32 meta;                         // mcts_meta
  u32 ncache;                       // size of the cached-prior block at first_child, 0 = none
};

struct MctsArgs {
  int sims, n_rollouts, solve, num_actions, mask_words, max_plies, puct;
  int max_nodes;                    // MCTSBot::max_nodes_: collect when the logical node count reaches it; <= 1: never
  double uct_c, max_utility, max_seconds;   // max_seconds > 0: stop starting simulations after this much wall clock (mcts.cc:362-365)
  u64 seed;
  long long tree_offset;
  const double* log_table;          // log_table[k] = std::log((double)k), k <= sims (host-computed)
  void* pool;                       // n_trees arenas of nodes_per_tree nodes (MctsNodeC or MctsNodeW)
  unsigned long long nodes_per_tree;
  unsigned long long* nodes_used;   // [1] sum over trees of the arena high-water marks, for b2s_mcts_nodes_used
  int compact;                      // host-side: 16-byte nodes (StatsC) or 24-byte nodes (StatsW)
  int tuning;                       // measurement switch (env B2S_MCTS_TUNING): 1 = no history filter
  int* visits_out;                  // [n][A]
  double* reward_out;               // [n][A]
  float* outcome_out;               // [n][A] (NaN = unproven), nullable
  int* best_out;                    // [n]
  int* sims_out;                    // [n], nullable
  int* gc_out;                      // [n] garbage collections performed, nullable
  ErrBuf* err;
};

// nanosecond wall clock (%globaltimer on the device) for the max_wall_clock_time budget
__device__ __forceinline__ unsigned long long mcts_now_ns() {
#ifdef __CUDA_ARCH__
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
#else
  return 0ull;                      // host builds (tests/host_emul, adapter) never set a time budget
#endif
}

__device__ __forceinline__ u32 rng_uniform(u64 key, u32 a, u32 b, u32 c, u32 n) {
  return philox_uniform(key, (u64)a | ((u64)b << 32), c, n);
}

// Playout draws (oracle/algorithms/philox.h RngUniformShared): draw number b of simulation `sim`, rollout domain `dom`, uses
// word (b & 3) of the Philox block keyed by (sim, b >> 2, dom), so the first tries of four consecutive plies cost one block
// (the block is kept in registers; retries, b >= 4096, compute theirs).  A rejected word falls back to streams 4 s + (b & 3).
struct PlayoutRng {
  u64 key;
  u32 sim, dom, id;
  u32 blk[4];
};
__device__ __forceinline__ u32 playout_draw(PlayoutRng& g, u32 b, u32 n) {
  const u32 id = b >> 2, wi = b & 3u;
  const u64 lane = (u64)g.sim | ((u64)id << 32);
  u32 w;
  if (b < 4096u) {
    if (id != g.id) { philox4(g.key, lane, g.dom, 0u, g.blk); g.id = id; }
    w = wi == 0 ? g.blk[0] : (wi == 1 ? g.blk[1] : (wi == 2 ? g.blk[2] : g.blk[3]));
  } else {
    u32 t[4];
    philox4(g.key, lane, g.dom, 0u, t);
    w = wi == 0 ? t[0] : (wi == 1 ? t[1] : (wi == 2 ? t[2] : t[3]));
  }
  u64 m = (u64)w * n;
  if ((u32)m >= n || (u32)m >= (u32)(0u - n) % n) return (u32)(m >> 32);
  const u32 thresh = (u32)(0u - n) % n;
  for (u32 s = 1;; ++s) {
    u32 t[4];
    philox4(g.key, lane, g.dom, 4u * s + wi, t);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      m = (u64)t[j] * n;
      if ((u32)m >= thresh) return (u32)(m >> 32);
    }
  }
}

// ---- per-representation statistics -----------------------------------------------------------------------------
struct SimReturn { int num[2]; double val[2]; };   // per simulation: integer numerators (StatsC only) and the reference's doubles

// puct_cp: the PUCT numerator (uct_c * prior) * sqrt(N_parent).  Nodes without a prior have the rollout evaluator's uniform
// prior 1/|children| (RandomRolloutEvaluator::Prior, mcts.cc:74-87), so theirs is the parent's `cp`, computed once per parent.
struct StatsC {
  typedef MctsNodeC Node;
  __device__ static __forceinline__ void zero(Node& n) { n.reward = 0; }
  __device__ static __forceinline__ void add(Node& n, int player, const SimReturn& r) { n.reward += r.num[player]; }
  __device__ static __forceinline__ double total(const Node& n, double inv_rollouts) { return __dmul_rn((double)n.reward, inv_rollouts); }
  __device__ static __forceinline__ double puct_cp(const Node&, double cp, double, double) { return cp; }
};
struct StatsW {
  typedef MctsNodeW Node;
  __device__ static __forceinline__ void zero(Node& n) { n.reward = 0.0; n.pad = 0; }
  __device__ static __forceinline__ void add(Node& n, int player, const SimReturn& r) { n.reward = __dadd_rn(n.reward, r.val[player]); }
  __device__ static __forceinline__ double total(const Node& n, double) { return n.reward; }
  __device__ static __forceinline__ double puct_cp(const Node&, double cp, double, double) { return cp; }
};
struct StatsE {
  typedef MctsNodeE Node;
  __device__ static __forceinline__ void zero(Node& n) { n.reward = 0.0; }
  __device__ static __forceinline__ void add(Node& n, int player, const SimReturn& r) { n.reward = __dadd_rn(n.reward, r.val[player]); }
  __device__ static __forceinline__ double total(const Node& n, double) { return n.reward; }
  __device__ static __forceinline__ double puct_cp(const Node& n, double, double uct_c, double sqrt_parent) {
    return __dmul_rn(__dmul_rn(uct_c, n.prior), sqrt_parent);
  }
};

// ---- the tree routines of both searches (k_mcts below, k_mcts_eval_step / k_mcts_eval_report in mcts_eval.cuh) ----------
// Args is MctsArgs or MctsEvalArgs.  Every routine is inlined into a kernel that sits at its register cap: arrays and counters
// are passed by reference, so no call copies the path, the collector's cursors or the free-list heads.

// ascending legal actions of a non-terminal state; returns the count (may exceed R::kMaxLegal: the caller checks).  `m` is
// scratch for the legal mask; the caller declares it, so that it keeps its place in k_mcts's local-memory frame.
template <class R>
__device__ __forceinline__ int mcts_legal_list(const typename R::S& s, const typename R::Cfg& cfg, int mask_words, u32 (&m)[R::kMaskWords],
                                               unsigned short* acts) {
  R::legal_nonterminal(s, cfg, m);
  int n = 0;
  for (int w = 0; w < mask_words; ++w) {
    u32 bits = m[w];
    while (bits) {
      const int b = __ffs(bits) - 1;
      bits &= bits - 1;
      if (n < R::kMaxLegal) acts[n] = (unsigned short)(w * 32 + b);
      ++n;
    }
  }
  return n;
}

// UCTValue (mcts.cc:90-101) / PUCTValue (:103-112), in the reference's left-to-right order
template <class NS, class Args>
__device__ __forceinline__ double mcts_child_value(const typename NS::Node& ch, double log_parent, double cp, double sqrt_parent,
                                                   const Args& P, double inv_rollouts) {
  if (meta_proven(ch.meta)) return (double)outcome_value(meta_outcome(ch.meta), meta_player(ch.meta));
  if (P.puct) {
    const double q = ch.visits ? __ddiv_rn(NS::total(ch, inv_rollouts), (double)ch.visits) : 0.0;
    return __dadd_rn(q, __ddiv_rn(NS::puct_cp(ch, cp, P.uct_c, sqrt_parent), (double)(ch.visits + 1u)));
  }
  if (ch.visits == 0) return __longlong_as_double(0x7ff0000000000000LL);
  const double n = (double)ch.visits;
  const double q = __ddiv_rn(NS::total(ch, inv_rollouts), n);
  const double u = __dsqrt_rn(__ddiv_rn(log_parent, n));
  return __dadd_rn(q, __dmul_rn(P.uct_c, u));
}

// the first-maximum scan over the children of the expanded node `nd` (mcts.cc:318-339); returns the chosen child's index
template <class NS, class Args>
__device__ __forceinline__ u32 mcts_select(const typename NS::Node* pool, const typename NS::Node& nd, int nch, const Args& P,
                                           double inv_rollouts) {
  const u32 first = nd.first_child, pv = nd.visits;
  const double log_parent = P.puct ? 0.0 : P.log_table[pv];
  const double cp = P.puct ? __dmul_rn(__dmul_rn(P.uct_c, __ddiv_rn(1.0, (double)nch)), __dsqrt_rn((double)pv)) : 0.0;
  const double sqrt_parent = P.puct ? __dsqrt_rn((double)pv) : 0.0;
  double best = __longlong_as_double(0xfff0000000000000LL);
  u32 chosen = first;
  for (int i = 0; i < nch; ++i) {
    const typename NS::Node ch = pool[first + i];
    if (!meta_proven(ch.meta) && ch.visits == 0 && !P.puct) {   // +infinity: the first unvisited child wins (every earlier value is finite)
      chosen = first + i;
      break;                                                     // nothing later can exceed +infinity
    }
    const double v = mcts_child_value<NS>(ch, log_parent, cp, sqrt_parent, P, inv_rollouts);
    if (v > best) { best = v; chosen = first + i; }
  }
  return chosen;
}

// backup and MCTS-Solver propagation (mcts.cc:384-434) along path(0) .. path(depth - 1); `path` reads the caller's stack
template <class NS, class Path>
__device__ __forceinline__ void mcts_backup(typename NS::Node* pool, const Path& path, int depth, const SimReturn& ret, bool solved,
                                            double max_utility) {
  while (depth > 0) {
    const u32 ni = path(--depth);
    typename NS::Node nd = pool[ni];
    NS::add(nd, meta_player(nd.meta), ret);
    nd.visits += 1;
    const int nch = meta_nchild(nd.meta);
    if (solved && nch > 0) {
      const int player = meta_player(pool[nd.first_child].meta);
      int best = -1, best_v = 0, best_code = 0;
      bool all_solved = true;
      for (int i = 0; i < nch; ++i) {
        const u32 cm = pool[nd.first_child + i].meta;
        if (!meta_proven(cm)) all_solved = false;
        else {
          const int v = outcome_value(meta_outcome(cm), player);
          if (best < 0 || v > best_v) { best = i; best_v = v; best_code = meta_outcome(cm); }
        }
      }
      if (best >= 0 && (all_solved || (double)best_v == max_utility)) nd.meta = meta_set_proven(nd.meta, best_code);
      else solved = false;
    }
    pool[ni] = nd;
  }
}
// MCTSearch's early exit (mcts.cc:437-440): the root is proven or has a single child.  `|` rather than `||`: with `||`, nvcc
// 12.9 lays out k_mcts's simulation loop differently (same registers and stack, about 1,200 SASS lines moved for go).
template <class Node>
__device__ __forceinline__ bool mcts_root_settled(const Node* pool) {
  const u32 rm = pool[0].meta;
  return meta_proven(rm) | (meta_nchild(rm) == 1);
}
// Children block allocator of one tree (thread-private): exact-size free list, else bump, else split a larger free block.
// Heads: the free-list heads, in registers / local memory (k_mcts) or a u32* into global memory (k_mcts_eval_step, whose
// trees outlive a launch).
template <class Node, int KMAX, class Heads = u32[KMAX + 1]>
struct TreeArena {
  Node* pool;
  u32 cap, top;
  Heads free_head;                  // free_head[k]: first free block of exactly k nodes (chained through first_child), 0 = none
  __device__ __forceinline__ void init(Node* p, u32 capacity) {
    pool = p; cap = capacity; top = 1;
    for (int k = 0; k <= KMAX; ++k) free_head[k] = 0;
  }
  __device__ __forceinline__ u32 alloc(int n) {
    u32 b = free_head[n];
    if (b) { free_head[n] = pool[b].first_child; return b; }
    if ((unsigned long long)top + (unsigned)n <= cap) { b = top; top += (u32)n; return b; }
    for (int m = n + 1; m <= KMAX; ++m) {
      b = free_head[m];
      if (!b) continue;
      free_head[m] = pool[b].first_child;
      release(b + (u32)n, m - n);
      return b;
    }
    return 0;
  }
  __device__ __forceinline__ void release(u32 b, int n) {
    if (n <= 0) return;
    pool[b].first_child = free_head[n];
    free_head[n] = b;
  }
};

// Node budget (mcts.cc:441-463): GarbageCollect (:469-482) as an explicit-stack post-order walk over the caller's `stk` / `it`,
// then adapt gc_limit_.  Cached prior blocks (StatsE) of nodes without children are freed as the walk reaches them.
template <class NS, int KMAX, int MAXPATH, class Arena>
__device__ __forceinline__ void mcts_collect(typename NS::Node* pool, Arena& arena, u32 (&stk)[MAXPATH], GcCursor<KMAX> (&it)[MAXPATH], int& nodes, int& gc_limit,
                                             int& gc_runs, int max_nodes) {
  typedef typename NS::Node Node;
  int sp = 0;
  stk[0] = 0; it[0] = 0;
  while (sp >= 0) {
    const u32 ni = stk[sp];
    const Node nd = pool[ni];
    const int nch = meta_nchild(nd.meta);
    if ((int)it[sp] < nch) {                       // children first (post-order)
      const u32 ci = nd.first_child + it[sp]++;
      if (meta_nchild(pool[ci].meta) > 0) {
        if (sp + 1 < MAXPATH) { ++sp; stk[sp] = ci; it[sp] = 0; }
      } else if constexpr (std::is_same<Node, MctsNodeE>::value) {
        if (pool[ci].ncache) {
          arena.release(pool[ci].first_child, (int)pool[ci].ncache);
          pool[ci].first_child = 0;
          pool[ci].ncache = 0;
        }
      }
      continue;
    }
    if (nch > 0 && (int)nd.visits < gc_limit) {    // clear_children = explore_count < gc_limit_
      arena.release(nd.first_child, nch);
      nodes -= nch;
      pool[ni].first_child = 0;
      pool[ni].meta = meta_set_nchild(nd.meta, 0);
    }
    --sp;
  }
  ++gc_runs;
  gc_limit = (int)((double)gc_limit * (nodes > max_nodes / 2 ? 1.25 : 0.9));     // int gc_limit_ *= double
  gc_limit = gc_limit > 5 ? gc_limit : 5;
}

// The root's children by action id (visits, total reward, outcome for player 0 if proven) and BestChild / CompareFinal
// (mcts.cc:114-143) into `best_action`, which keeps its value when the root has no children.  The caller has zero-filled the
// outputs.
template <class NS, class Args>
__device__ __forceinline__ void mcts_report(const typename NS::Node* pool, const Args& P, long long tree, double inv_rollouts,
                                            int& best_action) {
  typedef typename NS::Node Node;
  const Node r = pool[0];
  const int rn = meta_nchild(r.meta);
  int best = -1;
  for (int i = 0; i < rn; ++i) {
    const Node ch = pool[r.first_child + i];
    const long long o = tree * P.num_actions + meta_action(ch.meta);
    P.visits_out[o] = (int)ch.visits;
    P.reward_out[o] = NS::total(ch, inv_rollouts);
    if (P.outcome_out && meta_proven(ch.meta)) P.outcome_out[o] = (float)outcome_value(meta_outcome(ch.meta), 0);
    if (best < 0) { best = i; continue; }
    const Node b = pool[r.first_child + best];              // CompareFinal(b, ch): is b "less than" ch?
    const double ob = meta_proven(b.meta) ? (double)outcome_value(meta_outcome(b.meta), meta_player(b.meta)) : 0.0;
    const double oc = meta_proven(ch.meta) ? (double)outcome_value(meta_outcome(ch.meta), meta_player(ch.meta)) : 0.0;
    const double tb = NS::total(b, inv_rollouts), tc = NS::total(ch, inv_rollouts);
    const bool less = ob != oc ? ob < oc : (b.visits != ch.visits ? b.visits < ch.visits : tb < tc);
    if (less) best = i;
  }
  if (best >= 0) best_action = meta_action(pool[r.first_child + best].meta);
}

// rootctx holds the roots in the lane-blob form (R::load: b2s_mcts_search hands over a converted copy of the batch)
template <class R, class NS, int MAXPATH, int MINBLOCKS>
__global__ void __launch_bounds__(128, MINBLOCKS) k_mcts(Ctx rootctx, Ctx workctx, typename R::Cfg cfg, MctsArgs P, long long n_trees) {
  typedef typename NS::Node Node;
  long long tree = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (tree >= n_trees) return;
  typename R::S root;
  R::load(root, rootctx, tree);
  const u64 key = P.seed + (u64)(tree + P.tree_offset) * 0x9E3779B97F4A7C15ull;
  for (int a = 0; a < P.num_actions; ++a) {
    P.visits_out[tree * P.num_actions + a] = 0;
    P.reward_out[tree * P.num_actions + a] = 0.0;
    if (P.outcome_out) P.outcome_out[tree * P.num_actions + a] = __int_as_float(0x7fc00000);
  }
  P.best_out[tree] = -1;
  if (P.sims_out) P.sims_out[tree] = 0;
  if (P.gc_out) P.gc_out[tree] = 0;
  if (R::terminal(root, cfg)) return;              // nothing to search (the reference would index returns[-4])
  TreeArena<Node, R::kMaxLegal> arena;
  arena.init(reinterpret_cast<Node*>(P.pool) + (unsigned long long)tree * P.nodes_per_tree, (u32)P.nodes_per_tree);
  Node* pool = arena.pool;
  {
    Node r;
    NS::zero(r);
    r.visits = 0; r.first_child = 0;
    r.meta = mcts_meta(0, 0, R::cur_player(root, cfg), 0, 0);
    pool[0] = r;
  }
  // optional per-lane history filter (go: Bloom filter over the superko hash history, rules_go.cuh): built once from the
  // root's history, copied at the start of every simulation, updated by the rule core along the descent and the playout
  constexpr int kFW = R::kFilterWords > 0 ? R::kFilterWords : 1;
  u32 root_filter[kFW], filter[kFW];
  if constexpr (R::kFilterWords > 0) {
    if (!(P.tuning & 1)) {
      R::filter_build(root_filter, workctx, tree, root);
      workctx.filter = filter;
    }
  }
  const double inv_rollouts = __ddiv_rn(1.0, (double)P.n_rollouts);
  u32 path[MAXPATH];
  GcCursor<R::kMaxLegal> gc_iter[MAXPATH];         // child cursor per stack level of the collector's depth-first walk
  u32 expansions = 0;
  int nodes = 1;                                   // MCTSBot::nodes_
  int gc_limit = 5, gc_runs = 0;                   // MCTSBot::gc_limit_ (MIN_GC_LIMIT, mcts.cc:37)
  int sim = 0;
  bool failed = false;
  const unsigned long long t_start = P.max_seconds > 0 ? mcts_now_ns() : 0ull;
  for (; sim < P.sims && !failed; ++sim) {
    if (P.max_seconds > 0 && (double)(mcts_now_ns() - t_start) * 1e-9 >= P.max_seconds) break;
    typename R::S s = root;
    if constexpr (R::kFilterWords > 0)
      for (int w = 0; w < kFW; ++w) filter[w] = root_filter[w];
    int depth = 0;
    u32 cur = 0;
    path[depth++] = cur;
    bool term = false;
    // ---- tree policy (mcts.cc:273-351) ----
    while (!term) {
      Node nd = pool[cur];
      if (nd.visits == 0) break;
      int nch = meta_nchild(nd.meta);
      if (nch == 0) {
        u32 m[R::kMaskWords];
        unsigned short acts[R::kMaxLegal];
        const int n = mcts_legal_list<R>(s, cfg, P.mask_words, m, acts);
        if (n > R::kMaxLegal || n > kMetaMaxChildren || depth >= MAXPATH - 1) { failed = true; break; }
        u32 base = arena.alloc(n);
        if (!base) { failed = true; break; }
        u32 e = expansions++;
        for (int i = n - 1; i >= 1; --i) {          // random child order (std::shuffle's role, mcts.cc:294)
          u32 j = rng_uniform(key, e, (u32)i, 1u, (u32)(i + 1));
          unsigned short t = acts[i]; acts[i] = acts[j]; acts[j] = t;
        }
        const int player = R::cur_player(s, cfg);
        for (int k = 0; k < n; ++k) {
          Node c;
          NS::zero(c);
          c.visits = 0; c.first_child = 0;
          c.meta = mcts_meta(acts[k], 0, player, 0, 0);
          pool[base + k] = c;
        }
        nd.first_child = base;
        nd.meta = meta_set_nchild(nd.meta, n);
        pool[cur].first_child = nd.first_child;
        pool[cur].meta = nd.meta;
        nodes += n;                                 // nodes_ += children.capacity()
        nch = n;
      }
      cur = mcts_select<NS>(pool, nd, nch, P, inv_rollouts);
      apply_known_legal<R>(s, meta_action(pool[cur].meta), cfg, workctx, tree);
      path[depth++] = cur;
      term = R::terminal(s, cfg);
    }
    if (failed) break;
    // ---- evaluate (mcts.cc:372-381) ----
    SimReturn ret;
    bool solved;
    if (term) {
      float r[2];
      R::returns(s, cfg, r);
      ret.val[0] = r[0]; ret.val[1] = r[1];
      ret.num[0] = (int)r[0] * P.n_rollouts; ret.num[1] = (int)r[1] * P.n_rollouts;
      const int code = r[0] > 0.f ? 1 : (r[0] < 0.f ? 2 : 0);
      pool[cur].meta = meta_set_proven(pool[cur].meta, code);
      solved = P.solve != 0;
    } else {
      ret.val[0] = 0; ret.val[1] = 0; ret.num[0] = 0; ret.num[1] = 0;
      for (int ro = 0; ro < P.n_rollouts; ++ro) {
        typename R::S w = s;
        u32 ply = 0;
        PlayoutRng rng;
        rng.key = key; rng.sim = (u32)sim; rng.dom = 2u + (u32)ro; rng.id = 0xffffffffu;
        auto draw = [&](u32 b, u32 n) { return playout_draw(rng, b, n); };
        while (!R::terminal(w, cfg) && (int)ply < P.max_plies) {
          playout_step<R>(w, cfg, workctx, tree, P.mask_words, draw, ply);
          ++ply;
        }
        float r[2];
        R::returns(w, cfg, r);
        ret.val[0] = __dadd_rn(ret.val[0], (double)r[0]);
        ret.val[1] = __dadd_rn(ret.val[1], (double)r[1]);
        ret.num[0] += (int)r[0]; ret.num[1] += (int)r[1];
      }
      ret.val[0] = __ddiv_rn(ret.val[0], (double)P.n_rollouts);
      ret.val[1] = __ddiv_rn(ret.val[1], (double)P.n_rollouts);
      solved = false;
    }
    mcts_backup<NS>(pool, [&](int d) { return path[d]; }, depth, ret, solved, P.max_utility);
    if (mcts_root_settled(pool)) { ++sim; break; }
    // the collector's stack reuses `path`: the simulation's path is no longer needed
    if (P.max_nodes > 1 && nodes >= P.max_nodes)
      mcts_collect<NS, R::kMaxLegal, MAXPATH>(pool, arena, path, gc_iter, nodes, gc_limit, gc_runs, P.max_nodes);
  }
  if (failed) { flag_error(P.err, tree); }
  if (P.nodes_used) atomicAdd(P.nodes_used, (unsigned long long)arena.top);
  mcts_report<NS>(pool, P, tree, inv_rollouts, P.best_out[tree]);
  if (P.sims_out) P.sims_out[tree] = sim;
  if (P.gc_out) P.gc_out[tree] = gc_runs;
}

}  // namespace b2s
