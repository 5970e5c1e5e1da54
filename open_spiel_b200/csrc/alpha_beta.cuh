// Device-resident AlphaBetaSearch: one exact minimax search with alpha-beta pruning per root, one root at a time per thread.
// Semantics: reference open_spiel/algorithms/minimax.cc — _alpha_beta :49-137 (children in ascending action order, MAX keeps the
// first child whose value is strictly greater, MIN the first strictly smaller, alpha = max(alpha, value) / beta = min(beta, value)
// and a cut at alpha >= beta, a non-terminal node at depth 0 is SpielFatalError), AlphaBetaSearch :221-258 (the root searched
// from (-inf, +inf), kInvalidPlayer = the root's current player, best_action = kInvalidAction for a terminal root).
// The contract, including the node count and budget the device adds, is written out at b2s_alpha_beta_search in b2s.h.
//
// Values.  Every return of the served games is -1, 0 or +1, so alpha, beta and values are small integers with +-2 standing for
// +-infinity; the lane's result is converted to the reference's double at the end.
//
// Stack.  The search is depth-first with an explicit stack.  The current node lives in registers; descending into a non-terminal
// child pushes the parent's frame (state, the legal actions not yet searched, alpha, beta, value, MAX / MIN) to a library-owned
// buffer laid out [depth][thread], so the frames of neighbouring threads are adjacent.  A terminal child is evaluated in
// registers and never pushes anything.  Go's superko history: a root's column in the work lanes holds its history, and every
// child writes its hash at its ply index, as the MCTS work lanes do; a frame's state carries its ply, so returning to a frame
// simply makes the deeper entries dead, and the next child overwrites them.  The Bloom filter over the history (rules_go.cuh) is
// off here: it only grows along a path, so it would have to be saved per frame.
//
// Scheduling.  Per-root work is heavy-tailed (a few nodes to millions), so the grid is persistent: each thread takes the next
// root from a device counter, writes its outputs and takes another, instead of a warp waiting for its slowest static lane.
#pragma once
#include "common.cuh"

namespace b2s {

constexpr int kAbInf = 2;   // +-infinity among the integer values -1, 0, +1

// V: the value type; signed char for the exact search's integer values, double for the caller's values (k_alpha_beta_eval_step)
template <class R, class V = signed char>
struct AbFrame {
  typename R::S s;
  u32 rem[R::kMaskWords];        // legal actions of s not searched yet
  V alpha, beta, value;
  signed char max;
};

// Games whose frame stack fits B2S_ALPHA_BETA_THREAD_STACK_BYTES per thread: every deterministic game except go 10..19.
template <class R>
constexpr bool ab_served() {
  return R::kMaxPath > 0 && (unsigned long long)R::kMaxPath * sizeof(AbFrame<R>) <= B2S_ALPHA_BETA_THREAD_STACK_BYTES;
}

struct AlphaBetaArgs {
  int depth_limit, maximizing_player, mask_words;
  long long max_nodes;           // generated children per root; 0 = unlimited
  long long threads;             // frame d of thread t is stack[d * threads + t]
  void* stack;
  unsigned long long* next;      // the next root to take (zeroed on the stream before the launch)
  double* value;                 // outputs, nullable
  int* best_action;
  long long* nodes;
  unsigned char* status;
  ErrBuf* err;
};

struct AbResult {
  double value;
  int best_action, status;
  long long nodes;
};

// the lowest action left in `rem`, removed from it; -1 when none is left
template <class R>
__device__ __forceinline__ int ab_take_lowest(u32 (&rem)[R::kMaskWords]) {
  int a = -1;
#pragma unroll
  for (int w = 0; w < R::kMaskWords; ++w)
    if (a < 0 && rem[w]) { a = 32 * w + __ffs(rem[w]) - 1; rem[w] &= rem[w] - 1; }
  return a;
}

// minimax.cc:83-96 / 116-129: a finished child's value v updates its MAX / MIN parent (value, alpha, beta), strictly and with the
// operand order of std::max(alpha, value) / std::min(beta, value); `taken()` runs when v became the node's value (its action is
// the best so far).  For doubles these are IEEE comparisons: a NaN child is never taken, -0.0 and +0.0 tie.
template <class V, class Taken>
__device__ __forceinline__ void ab_update(bool is_max, V v, V& value, V& alpha, V& beta, Taken&& taken) {
  if (is_max) {
    if (v > value) { value = v; taken(); }
    alpha = alpha < value ? value : alpha;
  } else {
    if (v < value) { value = v; taken(); }
    beta = value < beta ? value : beta;
  }
}

// the cut after a child (minimax.cc:94, 127): the remaining children of a node are skipped once alpha >= beta
template <class V>
__device__ __forceinline__ bool ab_cut(V alpha, V beta) { return alpha >= beta; }

template <class R>
__device__ __forceinline__ void ab_legal(const typename R::S& s, const typename R::Cfg& cfg, int mask_words, u32 (&rem)[R::kMaskWords]) {
  R::legal_nonterminal(s, cfg, rem);
#pragma unroll
  for (int w = 0; w < R::kMaskWords; ++w)
    if (w >= mask_words) rem[w] = 0;
}

// AlphaBetaSearch from root i of `work` (lane-blob form; go: its history column is extended in place).  `stk` is this thread's
// frame 0; frame d is stk[d * P.threads].
template <class R>
__device__ __forceinline__ void alpha_beta_root(const Ctx& work, const typename R::Cfg& cfg, const AlphaBetaArgs& P, long long i,
                                                AbFrame<R>* stk, AbResult& out) {
  out.value = __longlong_as_double(0x7ff8000000000000LL);
  out.best_action = -1;
  out.status = 0;
  out.nodes = 0;
  typename R::S s;
  R::load(s, work, i);
  float r[R::kPlayers];
  if (R::terminal(s, cfg)) {
    // maximizing_player = kInvalidPlayer takes the terminal player id, which the reference indexes its returns with
    if (P.maximizing_player < 0) { out.status = 3; return; }
    R::returns(s, cfg, r);
    out.value = (double)r[P.maximizing_player];
    return;
  }
  if (P.depth_limit == 0) { out.status = 2; return; }
  const int maxp = P.maximizing_player >= 0 ? P.maximizing_player : R::cur_player(s, cfg);
  u32 rem[R::kMaskWords];
  ab_legal<R>(s, cfg, P.mask_words, rem);
  bool is_max = R::cur_player(s, cfg) == maxp;
  int alpha = -kAbInf, beta = kAbInf, value = is_max ? -kAbInf : kAbInf;
  int d = 0, root_action = -1, best = -1;
  long long nodes = 0;
  for (;;) {
    int v;                                       // the value of a finished child of the node in registers (depth d)
    const int a = !ab_cut(alpha, beta) ? ab_take_lowest<R>(rem) : -1;
    if (a >= 0) {
      if (P.max_nodes > 0 && nodes == P.max_nodes) { out.status = 1; out.nodes = nodes; return; }
      ++nodes;
      if (d == 0) root_action = a;
      typename R::S c = s;
      apply_known_legal<R>(c, a, cfg, work, i);
      if (R::terminal(c, cfg)) {
        R::returns(c, cfg, r);
        v = (int)r[maxp];
      } else if (d + 1 == P.depth_limit) {
        out.status = 2; out.nodes = nodes; return;
      } else {                                   // descend: push this node, open the child with the same alpha and beta
        AbFrame<R> f;
        f.s = s;
#pragma unroll
        for (int w = 0; w < R::kMaskWords; ++w) f.rem[w] = rem[w];
        f.alpha = (signed char)alpha; f.beta = (signed char)beta; f.value = (signed char)value; f.max = is_max;
        stk[(long long)d * P.threads] = f;
        ++d;
        s = c;
        ab_legal<R>(s, cfg, P.mask_words, rem);
        is_max = R::cur_player(s, cfg) == maxp;
        value = is_max ? -kAbInf : kAbInf;
        continue;
      }
    } else {                                     // every child searched, or cut: the node's value returns to its parent
      if (d == 0) break;
      v = value;
      --d;
      const AbFrame<R> f = stk[(long long)d * P.threads];
      s = f.s;
#pragma unroll
      for (int w = 0; w < R::kMaskWords; ++w) rem[w] = f.rem[w];
      alpha = f.alpha; beta = f.beta; value = f.value; is_max = f.max;
    }
    ab_update(is_max, v, value, alpha, beta, [&] { if (d == 0) best = root_action; });
  }
  out.value = value >= kAbInf ? __longlong_as_double(0x7ff0000000000000LL)
            : value <= -kAbInf ? __longlong_as_double(0xfff0000000000000LL) : (double)value;
  out.best_action = best;
  out.nodes = nodes;
}

// Persistent grid: P.threads threads take roots [0, n) from P.next until none is left.
template <class R>
__global__ void __launch_bounds__(128) k_alpha_beta(Ctx work, typename R::Cfg cfg, AlphaBetaArgs P, long long n) {
  AbFrame<R>* stk = reinterpret_cast<AbFrame<R>*>(P.stack) + ((long long)blockIdx.x * blockDim.x + threadIdx.x);
  for (;;) {
    const long long i = (long long)atomicAdd(P.next, 1ull);
    if (i >= n) return;
    AbResult res;
    alpha_beta_root<R>(work, cfg, P, i, stk, res);
    if (P.value) P.value[i] = res.value;
    if (P.best_action) P.best_action[i] = res.best_action;
    if (P.nodes) P.nodes[i] = res.nodes;
    if (P.status) P.status[i] = (unsigned char)res.status;
    if (res.status >= 2) flag_error(P.err, i);
  }
}

// ---- AlphaBetaSearch with a caller-supplied value function (b2s_alpha_beta_eval_*) ----------------------------------------------
// The same search to a depth limit, where a non-terminal state at depth 0 takes the caller's value instead of being an error.
// It runs in rounds: a step advances each live root until it needs one value or finishes.  Where k_alpha_beta would report
// status 2, the root saves the node in registers as frame d, writes the child into its lane of the leaves batch and stops; the
// next step reloads frame d and takes values[i][maxp] as that child's value.  One leaf per root and round, so the caller sees
// exactly the reference's value_function calls, in order.  Values are the caller's doubles, compared as IEEE doubles and never
// computed with, so the root's value is one of them (or a terminal return, or +-inf) bit for bit.  The frame stack lives in
// global memory laid out [depth][root]; between steps each root also keeps an AbEvalRoot.

enum { kAbEvalInit = 0, kAbEvalChild = 1, kAbEvalRoot = 2, kAbEvalDone = 3 };

struct AbEvalRoot {
  long long nodes, evals;        // child states generated, value-function calls
  int depth;                     // kAbEvalChild: the depth of the node whose child waits for its value (frame `depth`)
  int best, root_action, maxp, phase;
};

struct AlphaBetaEvalArgs {
  int depth_limit, maximizing_player, mask_words, num_players;
  long long max_nodes;           // generated children per root; 0 = unlimited
  void* stack;                   // AbFrame<R, double>: frame d of root i is stack[d * n + i]
  AbEvalRoot* roots;             // [n] the per-root context between steps
  const double* values;          // [n][num_players] the caller's answers (pending lanes only)
  unsigned char* pending;        // [n] out: 1 = lane i of the leaves batch waits for a value
  unsigned long long* n_pending; // [1] out: number of pending lanes (zeroed by the host before the launch)
  double* value;                 // [n] results, written when a root finishes
  int* best_action;
  long long* nodes;
  unsigned char* status;
  long long* evals;
  ErrBuf* err;                   // the leaves batch's
};

// One step of root i: true when it waits for the value of the state now in lane i of `leaves`, false when it finished (`out`).
// roots: the roots in the lane-blob form; leaves: the caller's leaves batch, whose history column (go) holds the root's superko
// history and is extended along the path, so a leaf lane is the real state for every batched kernel.
template <class R>
__device__ __forceinline__ bool alpha_beta_eval_advance(const Ctx& roots, const Ctx& leaves, const typename R::Cfg& cfg,
                                                        const AlphaBetaEvalArgs& P, long long i, long long n, AbEvalRoot& T,
                                                        AbResult& out) {
  const double inf = __longlong_as_double(0x7ff0000000000000LL);
  out.value = __longlong_as_double(0x7ff8000000000000LL);
  out.best_action = -1;
  out.status = 0;
  AbFrame<R, double>* stk = reinterpret_cast<AbFrame<R, double>*>(P.stack) + i;
  typename R::S s;
  u32 rem[R::kMaskWords];
  double alpha = -inf, beta = inf, value = 0.0, v = 0.0;
  bool is_max = false, resumed = false;
  int d = 0;
  float r[R::kPlayers];
  if (T.phase == kAbEvalInit) {
    R::load(s, roots, i);
    T.nodes = 0; T.evals = 0; T.depth = 0; T.best = -1; T.root_action = -1;
    if (R::terminal(s, cfg)) {
      out.nodes = 0;
      if (P.maximizing_player < 0) { out.status = 3; return false; }
      R::returns(s, cfg, r);
      out.value = (double)r[P.maximizing_player];
      return false;
    }
    T.maxp = P.maximizing_player >= 0 ? P.maximizing_player : R::cur_player(s, cfg);
    if (P.depth_limit == 0) {                    // a non-terminal root at depth 0: its own value
      store_state<R>(s, cfg, leaves, i);
      ++T.evals;
      T.phase = kAbEvalRoot;
      return true;
    }
    ab_legal<R>(s, cfg, P.mask_words, rem);
    is_max = R::cur_player(s, cfg) == T.maxp;
    value = is_max ? -inf : inf;
  } else if (T.phase == kAbEvalRoot) {
    out.value = P.values[i * P.num_players + T.maxp];
    out.nodes = 0;
    return false;
  } else {                                       // kAbEvalChild: frame d holds the node, values[i] its child's value
    d = T.depth;
    const AbFrame<R, double> f = stk[(long long)d * n];
    s = f.s;
#pragma unroll
    for (int w = 0; w < R::kMaskWords; ++w) rem[w] = f.rem[w];
    alpha = f.alpha; beta = f.beta; value = f.value; is_max = f.max;
    v = P.values[i * P.num_players + T.maxp];
    resumed = true;
  }
  long long nodes = T.nodes;
  for (;;) {
    if (resumed) {
      resumed = false;
    } else {
      const int a = !ab_cut(alpha, beta) ? ab_take_lowest<R>(rem) : -1;
      if (a >= 0) {
        if (P.max_nodes > 0 && nodes == P.max_nodes) { out.status = 1; out.nodes = nodes; return false; }
        ++nodes;
        if (d == 0) T.root_action = a;
        typename R::S c = s;
        apply_known_legal<R>(c, a, cfg, leaves, i);
        if (R::terminal(c, cfg)) {               // terminal before the depth test: never sent to the caller
          R::returns(c, cfg, r);
          v = (double)r[T.maxp];
        } else if (d + 1 == P.depth_limit) {     // the child is at depth 0: save this node and ask for the child's value
          AbFrame<R, double> f;
          f.s = s;
#pragma unroll
          for (int w = 0; w < R::kMaskWords; ++w) f.rem[w] = rem[w];
          f.alpha = alpha; f.beta = beta; f.value = value; f.max = is_max;
          stk[(long long)d * n] = f;
          store_state<R>(c, cfg, leaves, i);
          T.nodes = nodes; ++T.evals; T.depth = d; T.phase = kAbEvalChild;
          return true;
        } else {                                 // descend: push this node, open the child with the same alpha and beta
          AbFrame<R, double> f;
          f.s = s;
#pragma unroll
          for (int w = 0; w < R::kMaskWords; ++w) f.rem[w] = rem[w];
          f.alpha = alpha; f.beta = beta; f.value = value; f.max = is_max;
          stk[(long long)d * n] = f;
          ++d;
          s = c;
          ab_legal<R>(s, cfg, P.mask_words, rem);
          is_max = R::cur_player(s, cfg) == T.maxp;
          value = is_max ? -inf : inf;
          continue;
        }
      } else {                                   // every child searched, or cut: the node's value returns to its parent
        if (d == 0) break;
        v = value;
        --d;
        const AbFrame<R, double> f = stk[(long long)d * n];
        s = f.s;
#pragma unroll
        for (int w = 0; w < R::kMaskWords; ++w) rem[w] = f.rem[w];
        alpha = f.alpha; beta = f.beta; value = f.value; is_max = f.max;
      }
    }
    ab_update(is_max, v, value, alpha, beta, [&] { if (d == 0) T.best = T.root_action; });
  }
  out.value = value;
  out.best_action = T.best;
  out.nodes = nodes;
  return false;
}

// One thread per root; a finished root writes its results once and stays done.
template <class R>
__global__ void __launch_bounds__(128) k_alpha_beta_eval_step(Ctx roots, Ctx leaves, typename R::Cfg cfg, AlphaBetaEvalArgs P,
                                                              long long n) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  AbEvalRoot T = P.roots[i];
  if (T.phase == kAbEvalDone) { P.pending[i] = 0; return; }
  AbResult res;
  const bool request = alpha_beta_eval_advance<R>(roots, leaves, cfg, P, i, n, T, res);
  if (!request) {
    T.phase = kAbEvalDone;
    P.value[i] = res.value; P.best_action[i] = res.best_action; P.nodes[i] = res.nodes; P.status[i] = (unsigned char)res.status;
    P.evals[i] = T.evals;
    if (res.status >= 2) flag_error(P.err, i);
  }
  P.roots[i] = T;
  P.pending[i] = request ? 1 : 0;
  if (request) atomicAdd(P.n_pending, 1ull);
}

}  // namespace b2s
