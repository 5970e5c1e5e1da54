// Device MCTS with a caller-supplied evaluator (b2s_mcts_eval_*): MCTSBot::MCTSearch (reference open_spiel/algorithms/mcts.cc
// :353-467) for an arbitrary Evaluator (mcts.h:83-92), one tree per thread, driven in rounds from the host.
// A step launch advances every live tree until it needs Evaluate (a non-terminal leaf's first visit, mcts.cc:379) or Prior (an
// expansion, :282) or finishes; simulations that end at terminal states need neither, so one step may run several.  A tree that
// needs an answer writes its working state into its lane of the caller's leaves batch, marks itself pending and stops; the next
// step reads values [n][num_players] and priors [n][A] (by action id) and resumes.  Resume context per tree in global memory:
// the path stack, the arena's free lists and MctsEvalTree (phase, depth, counters).
// Prior cache: the answer to a leaf's Evaluate request also carries the leaf's prior; it is stored at once as the node's future
// children block (ascending legal order), but the node stays unexpanded (meta #children = 0, ncache = block size) until its
// second visit, which applies the root's Dirichlet mix, shuffles the block and makes it the children.  So a caller runs one
// inference per new node.  The reference's logical `nodes_` grows at that expansion only, so collections happen after the same
// simulations as in the reference.  A collection frees every cached block it reaches (and the children of nodes visited fewer
// than gc_limit_ times, as MCTSBot::GarbageCollect); a node without children and without a cache asks for its prior again at its
// next expansion (a prior-only request: its value is ignored).  Caches take at most half of a tree's arena (cache_cap);
// a leaf that finds no room is not cached and asks again at its expansion as well.
// Same random decisions as k_mcts (expansion #e: Fisher-Yates j = rng(key, e, i, 1, i+1)); explicitly rounded FP64 throughout:
//   PUCT (mcts.cc:103-112): q + ((uct_c * prior) * sqrt(N)) / (n + 1);  UCT (:90-101) ignores the prior.
//   Dirichlet mix at the root's expansion (:284-292): (1 - eps) * p + eps * noise[a], noise given by the caller per tree.
// Node: MctsNodeE, 32 bytes (the reference's double total_reward and double prior), with StatsE.  Selection, backup, the
// collector and the report are mcts.cuh's, shared with k_mcts; this file holds the evaluator protocol.
#pragma once
#include "mcts.cuh"

namespace b2s {

enum { kEvalInit = 0, kEvalSim = 1, kEvalValue = 2, kEvalPrior = 3, kEvalDone = 4 };
struct MctsEvalTree {               // per-tree resume context
  int phase;                        // kEval*: kEvalValue / kEvalPrior = waiting for the caller's answer
  int depth;                        // path length of the simulation in progress
  int sim, nodes, gc_limit, gc_runs;   // simulations finished, MCTSBot::nodes_ / gc_limit_, collections
  u32 expansions, top;              // expansion counter (shuffle stream), arena bump pointer
  int prior_requests;               // prior-only requests (re-expansions after a collection / without a cache)
  int pad;
};

struct MctsEvalArgs {
  int sims, solve, num_actions, mask_words, puct;
  int max_nodes;                    // MCTSBot::max_nodes_ (<= 1: never collect)
  double uct_c, max_utility, epsilon;
  u64 seed;
  long long tree_offset;
  const double* log_table;          // log_table[k] = std::log((double)k), k <= sims (host-computed)
  MctsNodeE* pool;                  // n_trees arenas of nodes_per_tree nodes
  unsigned long long nodes_per_tree;
  u32 cache_cap;                    // prior caches only while the bump pointer stays below this
  MctsEvalTree* trees;              // [n]
  u32* free_heads;                  // [n][kMaxLegal + 1]
  u32* path;                        // [MAXPATH][n]
  const double* noise;              // [n][A] root Dirichlet noise, nullable
  const double* values;             // [n][num_players] the caller's answers (pending lanes only)
  const double* priors;             // [n][A]
  unsigned char* pending;           // [n] out: 1 = lane i of the leaves batch waits for an answer
  unsigned long long* n_pending;    // [1] out: number of pending lanes (zeroed by the host before the launch)
  ErrBuf* err;
  // report
  int* visits_out;                  // [n][A]
  double* reward_out;               // [n][A]
  float* outcome_out;               // [n][A], nullable
  int* best_out;                    // [n], nullable
  int* sims_out;                    // [n], nullable
  int* gc_out;                      // [n], nullable
  int* prior_requests_out;          // [n], nullable
};

// roots: the roots in the lane-blob form (R::load); leaves: the caller's leaves batch (its history column holds the roots'
// superko histories, the descent appends the path's)
template <class R, int MAXPATH>
__global__ void __launch_bounds__(128) k_mcts_eval_step(Ctx roots, Ctx leaves, typename R::Cfg cfg, MctsEvalArgs P, long long n_trees) {
  typedef StatsE NS;
  typedef MctsNodeE Node;
  const long long tree = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (tree >= n_trees) return;
  MctsEvalTree T = P.trees[tree];
  if (T.phase == kEvalDone) { P.pending[tree] = 0; return; }
  TreeArena<Node, R::kMaxLegal, u32*> arena;
  arena.pool = P.pool + (unsigned long long)tree * P.nodes_per_tree;
  arena.cap = (u32)P.nodes_per_tree;
  arena.top = T.top;
  arena.free_head = P.free_heads + tree * (R::kMaxLegal + 1);
  Node* pool = arena.pool;
  u32* path = P.path + tree;                       // path[d * n_trees]
  const u64 key = P.seed + (u64)(tree + P.tree_offset) * 0x9E3779B97F4A7C15ull;
  const int A = P.num_actions;
  typename R::S s;
  if (T.phase == kEvalInit) {
    R::load(s, roots, tree);
    if (R::terminal(s, cfg)) {                     // nothing to search
      T.phase = kEvalDone;
      P.trees[tree] = T;
      P.pending[tree] = 0;
      return;
    }
    for (int k = 0; k <= R::kMaxLegal; ++k) arena.free_head[k] = 0;
    arena.top = 1;
    Node r;
    r.reward = 0.0; r.prior = 1.0; r.visits = 0; r.first_child = 0; r.ncache = 0;
    r.meta = mcts_meta(0, 0, R::cur_player(s, cfg), 0, 0);
    pool[0] = r;
    T.depth = 0; T.sim = 0; T.nodes = 1; T.gc_limit = 5; T.gc_runs = 0; T.expansions = 0; T.prior_requests = 0;
    T.phase = kEvalSim;
  }
  int phase = T.phase;
  bool failed = false, request = false;
  u32 m[R::kMaskWords];
  unsigned short acts[R::kMaxLegal];
  while (!request && !failed) {
    int depth;
    u32 cur;
    bool answered = false;                         // the caller's answer for this lane is to be used
    SimReturn ret;                                 // val[] only: evaluator values are doubles
    ret.val[0] = 0.0; ret.val[1] = 0.0;
    bool solved = false;
    if (phase == kEvalSim) {
      if (T.sim >= P.sims) { phase = kEvalDone; break; }
      R::load(s, roots, tree);
      depth = 0; cur = 0;
      path[0] = 0; depth = 1;
    } else {                                       // resume: the lane holds the state the request was made in
      load_state<R>(s, cfg, leaves, tree);
      depth = T.depth;
      cur = path[(long long)(depth - 1) * n_trees];
      answered = true;
    }
    if (phase == kEvalValue) {
      // Evaluate at a leaf's first visit (mcts.cc:379): take the value, cache the prior as the future children block
      ret.val[0] = P.values[tree * 2]; ret.val[1] = P.values[tree * 2 + 1];
      const int n = mcts_legal_list<R>(s, cfg, P.mask_words, m, acts);
      if (n <= R::kMaxLegal) {
        const u32 b = arena.top + (u32)n <= P.cache_cap ? arena.alloc(n) : 0u;
        if (b) {
          const int player = R::cur_player(s, cfg);
          for (int k = 0; k < n; ++k) {
            Node c;
            c.reward = 0.0; c.prior = P.priors[tree * A + acts[k]];
            c.visits = 0; c.first_child = 0; c.ncache = 0;
            c.meta = mcts_meta(acts[k], 0, player, 0, 0);
            pool[b + k] = c;
          }
          pool[cur].first_child = b;
          pool[cur].ncache = (u32)n;
        }
      }
    } else {
      // ---- tree policy (mcts.cc:273-351) ----
      bool term = false;
      while (!term) {
        Node nd = pool[cur];
        if (nd.visits == 0) break;
        int nch = meta_nchild(nd.meta);
        if (nch == 0) {
          if (nd.ncache == 0 && !answered) {       // no cached prior: ask for it
            store_state<R>(s, cfg, leaves, tree);
            phase = kEvalPrior;
            ++T.prior_requests;
            request = true;
            break;
          }
          const int n = mcts_legal_list<R>(s, cfg, P.mask_words, m, acts);
          if (n > R::kMaxLegal || n > kMetaMaxChildren || depth >= MAXPATH - 1) { failed = true; break; }
          u32 base = nd.ncache ? nd.first_child : 0u;
          if (!base) {                             // Evaluator::Prior from this round's answer
            base = arena.alloc(n);
            if (!base) { failed = true; break; }
            const int player = R::cur_player(s, cfg);
            for (int k = 0; k < n; ++k) {
              Node c;
              c.reward = 0.0; c.prior = P.priors[tree * A + acts[k]];
              c.visits = 0; c.first_child = 0; c.ncache = 0;
              c.meta = mcts_meta(acts[k], 0, player, 0, 0);
              pool[base + k] = c;
            }
          }
          answered = false;
          if (cur == 0 && P.noise) {               // Dirichlet noise at the root (mcts.cc:284-292), before the shuffle
            const double keep = __dsub_rn(1.0, P.epsilon);
            for (int k = 0; k < n; ++k) {
              const double p = pool[base + k].prior;
              const double z = P.noise[tree * A + meta_action(pool[base + k].meta)];
              pool[base + k].prior = __dadd_rn(__dmul_rn(keep, p), __dmul_rn(P.epsilon, z));
            }
          }
          const u32 e = T.expansions++;
          for (int i = n - 1; i >= 1; --i) {       // random child order (std::shuffle's role, mcts.cc:294)
            const u32 j = rng_uniform(key, e, (u32)i, 1u, (u32)(i + 1));
            if (j != (u32)i) { const Node t = pool[base + i]; pool[base + i] = pool[base + j]; pool[base + j] = t; }
          }
          nd.first_child = base;
          nd.ncache = 0;
          nd.meta = meta_set_nchild(nd.meta, n);
          pool[cur].first_child = base;
          pool[cur].ncache = 0;
          pool[cur].meta = nd.meta;
          T.nodes += n;                            // nodes_ += children.capacity()
          nch = n;
        }
        cur = mcts_select<NS>(pool, nd, nch, P, 1.0);
        apply_known_legal<R>(s, meta_action(pool[cur].meta), cfg, leaves, tree);
        path[(long long)depth * n_trees] = cur;
        ++depth;
        term = R::terminal(s, cfg);
      }
      if (request || failed) { T.depth = depth; break; }
      if (term) {
        float r[2];
        R::returns(s, cfg, r);
        ret.val[0] = r[0]; ret.val[1] = r[1];
        const int code = r[0] > 0.f ? 1 : (r[0] < 0.f ? 2 : 0);
        pool[cur].meta = meta_set_proven(pool[cur].meta, code);
        solved = P.solve != 0;
      } else {                                     // a leaf's first visit: ask for Evaluate (and Prior)
        store_state<R>(s, cfg, leaves, tree);
        T.depth = depth;
        phase = kEvalValue;
        request = true;
        break;
      }
    }
    mcts_backup<NS>(pool, [&](int d) { return path[(long long)d * n_trees]; }, depth, ret, solved, P.max_utility);
    ++T.sim;
    phase = kEvalSim;
    if (mcts_root_settled(pool)) { phase = kEvalDone; break; }
    if (P.max_nodes > 1 && T.nodes >= P.max_nodes) {
      u32 stk[MAXPATH];
      GcCursor<R::kMaxLegal> it[MAXPATH];
      mcts_collect<NS, R::kMaxLegal, MAXPATH>(pool, arena, stk, it, T.nodes, T.gc_limit, T.gc_runs, P.max_nodes);
    }
  }
  if (failed) { flag_error(P.err, tree); phase = kEvalDone; request = false; }
  T.phase = phase;
  T.top = arena.top;
  P.trees[tree] = T;
  P.pending[tree] = request ? 1 : 0;
  if (request) atomicAdd(P.n_pending, 1ull);
}

// The root's children by action id and BestChild (mcts.cc:114-143), as k_mcts reports them; valid between steps.
template <class R>
__global__ void __launch_bounds__(128) k_mcts_eval_report(MctsEvalArgs P, long long n_trees) {
  const long long tree = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (tree >= n_trees) return;
  const int A = P.num_actions;
  for (int a = 0; a < A; ++a) {
    P.visits_out[tree * A + a] = 0;
    P.reward_out[tree * A + a] = 0.0;
    if (P.outcome_out) P.outcome_out[tree * A + a] = __int_as_float(0x7fc00000);
  }
  const MctsEvalTree T = P.trees[tree];
  const bool started = T.nodes > 0;                // root node written (not before the first step, never for terminal roots)
  int best = -1;
  if (started) mcts_report<StatsE>(P.pool + (unsigned long long)tree * P.nodes_per_tree, P, tree, 1.0, best);
  if (P.best_out) P.best_out[tree] = best;
  if (P.sims_out) P.sims_out[tree] = started ? T.sim : 0;
  if (P.gc_out) P.gc_out[tree] = started ? T.gc_runs : 0;
  if (P.prior_requests_out) P.prior_requests_out[tree] = started ? T.prior_requests : 0;
}

}  // namespace b2s
