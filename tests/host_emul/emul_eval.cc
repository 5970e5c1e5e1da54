// TEST INFRASTRUCTURE ONLY — never part of the product (libb2s.so has no CPU path and fails without a GPU).
//
// Host build of the caller-evaluated MCTS (open_spiel_b200/csrc/mcts_eval.cuh, b2s_mcts_eval_*): the PRODUCT's rule cores and
// the KERNEL BODIES k_mcts_eval_step / k_mcts_eval_report compiled with g++ (as tests/host_emul/emul.cc does for the other
// kernels), one "thread" at a time, so that tests/test_mcts_eval_host.py can run the search round by round in the CPU suite:
// the buffers and the argument block are set up as api.cu's b2s_mcts_eval_create does, and the caller's evaluator is computed
// on the host from the leaves lanes (their observation tensor and legal mask, read back through the rule cores).
// Roots: lanes [0, n) of a host batch reset to the initial state and advanced with emv_apply.
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>

#include <cmath>
#include <string>
#include <type_traits>
#include <vector>

#include "../../open_spiel_b200/csrc/host_compat.h"   // host definitions of the device intrinsics (product header)
// one "thread" at a time: the kernels index with blockIdx.x * blockDim.x + threadIdx.x
static struct { unsigned x, y, z; } blockIdx, blockDim = {1, 1, 1}, threadIdx;

#include "../../open_spiel_b200/csrc/common.cuh"
#include "../../open_spiel_b200/csrc/rules_tic_tac_toe.cuh"
#include "../../open_spiel_b200/csrc/rules_connect_four.cuh"
#include "../../open_spiel_b200/csrc/rules_breakthrough.cuh"
#include "../../open_spiel_b200/csrc/rules_hex.cuh"
#include "../../open_spiel_b200/csrc/rules_go.cuh"
#include "../../open_spiel_b200/csrc/rules_kuhn_poker.cuh"
#include "../../open_spiel_b200/csrc/rules_mnk.cuh"
#include "../../open_spiel_b200/csrc/rules_othello.cuh"
#include "../../open_spiel_b200/csrc/rules_y.cuh"
#include "../../open_spiel_b200/csrc/rules_havannah.cuh"
#include "../../open_spiel_b200/csrc/mcts_eval.cuh"

namespace {
using namespace b2s;

template <class R> auto call_init(int) -> decltype(R::device_init(), void()) { R::device_init(); }
template <class R> void call_init(long) {}

struct Emv {
  virtual ~Emv() {}
  virtual void apply(const int* a, long long n) = 0;
  virtual int eval_create(long long n, const b2s_mcts_eval_config& mc) = 0;
  virtual long long eval_step(const double* values, const double* priors, unsigned char* pending) = 0;
  virtual void eval_leaves(float* obs, u32* mask) = 0;
  virtual void eval_results(int* visits, double* reward, float* outcome, int* best, int* sims_run, int* gc_runs, int* prior_requests) = 0;
  b2s_game_info info;
  ErrBuf err;
};

template <class R>
struct EmvT : Emv {
  typename R::Cfg cfg;
  std::vector<char> planes;        // the roots batch, lane-blob form (R::load / R::store) as tests/host_emul/emul.cc keeps it
  std::vector<u64> hist;
  long long cap = 0;
  Ctx ctx() { Ctx c; c.planes = planes.data(); c.cap = cap; c.hist = hist.empty() ? nullptr : hist.data(); c.err = &err; return c; }
  const char* configure(const b2s_params& p, long long capacity) {
    memset(&info, 0, sizeof info);
    const char* e = R::make_cfg(p, cfg, info);
    if (e) return e;
    int width = info.num_distinct_actions > info.max_chance_outcomes ? info.num_distinct_actions : info.max_chance_outcomes;
    info.mask_words = (width + 31) / 32;                    // as GameOpsT<R>::configure (batch_kernels.cuh)
    if (info.mask_words > R::kMaskWords) return "action space too large for the device path";
    info.state_bytes = (int)(sizeof(typename R::Chunk) * R::kChunks);
    info.game_id = R::kGameId;
    cap = capacity;
    planes.assign(sizeof(typename R::Chunk) * R::kChunks * (size_t)cap, 0);
    if (info.history_bytes) hist.assign((size_t)info.history_bytes / sizeof(u64) * (size_t)cap, 0);
    call_init<R>(0);
    err.count = 0; err.first = 0x7fffffffffffffffLL;
    Ctx c = ctx();
    for (long long i = 0; i < cap; ++i) { typename R::S s; R::init(s, cfg, c, i); R::store(s, c, i); }   // k_reset
    return nullptr;
  }
  void apply(const int* a, long long n) override {                      // k_apply
    Ctx c = ctx();
    for (long long i = 0; i < n; ++i) {
      if (a[i] == -1) continue;
      typename R::S s;
      R::load(s, c, i);
      if (R::terminal(s, cfg) || !R::apply(s, a[i], cfg, c, i)) { flag_error(&err, i); continue; }
      R::store(s, c, i);
    }
  }
  // b2s_mcts_eval_*: buffers and argument block as api.cu sets them up; the KERNEL BODIES of mcts_eval.cuh run once per tree
  struct EvalRun {
    long long n = 0;
    std::vector<char> roots, leaves, pool;
    std::vector<u64> hist;
    std::vector<double> logt, noise;
    std::vector<MctsEvalTree> trees;
    std::vector<u32> heads, path;
    std::vector<unsigned char> pending;
    unsigned long long n_pending = 0;
    MctsEvalArgs a;
    Ctx rootctx, leafctx;
  } ev;
  int eval_create(long long n, const b2s_mcts_eval_config& mc) override {
    return eval_create_impl(n, mc, std::integral_constant<bool, (R::kMaxPath > 0)>());
  }
  int eval_create_impl(long long, const b2s_mcts_eval_config&, std::false_type) { return 1; }
  int eval_create_impl(long long n, const b2s_mcts_eval_config& mc, std::true_type) {
    if (info.max_game_length + 2 > R::kMaxPath) return 2;
    const size_t A = (size_t)info.num_distinct_actions;
    ev.n = n;
    ev.roots.assign((size_t)info.state_bytes * (size_t)n, 0);
    ev.leaves.assign(sizeof(StoredChunk<R>) * R::kChunks * (size_t)n, 0);
    ev.hist.assign(info.history_bytes ? (size_t)info.history_bytes / sizeof(u64) * (size_t)n : 0, 0);
    ev.rootctx.planes = ev.roots.data(); ev.rootctx.cap = n; ev.rootctx.hist = ev.hist.empty() ? nullptr : ev.hist.data(); ev.rootctx.err = &err;
    ev.leafctx = ev.rootctx;
    ev.leafctx.planes = ev.leaves.data();
    {                                                       // api.cu: B->ops->copy_to_blob(roots, batch, n) — k_copy_to_blob
      Ctx src = ctx();
      for (long long i = 0; i < n; ++i) {
        typename R::S s;
        R::load(s, src, i);
        R::store(s, ev.rootctx, i);
        R::copy_history(ev.rootctx, i, src, i, s, cfg);
      }
    }
    ev.logt.assign((size_t)mc.max_simulations + 2, 0.0);
    for (size_t k = 1; k < ev.logt.size(); ++k) ev.logt[k] = std::log((double)k);
    unsigned long long per_tree;                            // arena sizing as b2s_mcts_eval_create (without the free-memory cap)
    if (mc.max_nodes_total > 0) per_tree = (unsigned long long)mc.max_nodes_total / (unsigned long long)n;
    else {
      per_tree = 2ull + 2ull * (unsigned long long)mc.max_simulations * A;
      if (mc.max_nodes_per_tree > 1) {
        unsigned long long want = 4ull * (unsigned long long)mc.max_nodes_per_tree + 16 * A + 128;
        if (want < per_tree) per_tree = want;
      }
    }
    ev.pool.assign((size_t)per_tree * (size_t)n * sizeof(MctsNodeE) + 16, 0);
    ev.trees.assign((size_t)n, MctsEvalTree());
    memset(ev.trees.data(), 0, sizeof(MctsEvalTree) * (size_t)n);
    ev.heads.assign((size_t)(R::kMaxLegal + 1) * (size_t)n, 0);
    ev.path.assign((size_t)R::kMaxPath * (size_t)n, 0);
    ev.pending.assign((size_t)n, 0);
    if (mc.root_noise_d) ev.noise.assign(mc.root_noise_d, mc.root_noise_d + A * (size_t)n);
    else ev.noise.clear();
    MctsEvalArgs& a = ev.a;
    memset(&a, 0, sizeof a);
    a.sims = mc.max_simulations; a.solve = mc.solve; a.num_actions = (int)A; a.mask_words = info.mask_words;
    a.puct = mc.child_selection_policy == B2S_MCTS_PUCT; a.max_nodes = (int)mc.max_nodes_per_tree;
    a.uct_c = mc.uct_c; a.max_utility = info.max_utility; a.epsilon = mc.dirichlet_epsilon;
    a.seed = mc.seed; a.tree_offset = mc.tree_index_offset; a.log_table = ev.logt.data();
    a.pool = (MctsNodeE*)(((uintptr_t)ev.pool.data() + 15) & ~(uintptr_t)15); a.nodes_per_tree = per_tree; a.cache_cap = (u32)(per_tree / 2);
    a.trees = ev.trees.data(); a.free_heads = ev.heads.data(); a.path = ev.path.data(); a.noise = ev.noise.empty() ? nullptr : ev.noise.data();
    a.pending = ev.pending.data(); a.n_pending = &ev.n_pending; a.err = &err;
    return 0;
  }
  long long eval_step(const double* values, const double* priors, unsigned char* pending) override {
    return eval_step_impl(values, priors, pending, std::integral_constant<bool, (R::kMaxPath > 0)>());
  }
  long long eval_step_impl(const double*, const double*, unsigned char*, std::false_type) { return -1; }
  long long eval_step_impl(const double* values, const double* priors, unsigned char* pending, std::true_type) {
    MctsEvalArgs a = ev.a;
    a.values = values; a.priors = priors;
    ev.n_pending = 0;
    blockDim.x = 1; threadIdx.x = 0;
    for (long long t = 0; t < ev.n; ++t) {
      blockIdx.x = (unsigned)t;
      k_mcts_eval_step<R, R::kMaxPath>(ev.rootctx, ev.leafctx, cfg, a, ev.n);
    }
    memcpy(pending, ev.pending.data(), (size_t)ev.n);
    return (long long)ev.n_pending;
  }
  void eval_leaves(float* obs, u32* mask) override {        // b2s_observation(-1) / b2s_legal_mask on the leaves batch
    const int size = info.observation_tensor_size;
    for (long long i = 0; i < ev.n; ++i) {
      typename R::S s;
      load_state<R>(s, cfg, ev.leafctx, i);
      int pl = R::cur_player(s, cfg);
      if (pl < 0) pl = 0;
      typename R::ObsPack pk;
      R::obs_pack(s, cfg, pl, 0, pk);
      for (int e = 0; e < size; ++e) obs[i * size + e] = R::obs_elem(pk, cfg, e);
      u32 m[R::kMaskWords];
      R::legal(s, cfg, m);
      for (int w = 0; w < info.mask_words; ++w) mask[i * info.mask_words + w] = m[w];
    }
  }
  void eval_results(int* visits, double* reward, float* outcome, int* best, int* sims_run, int* gc_runs, int* prior_requests) override {
    eval_results_impl(visits, reward, outcome, best, sims_run, gc_runs, prior_requests, std::integral_constant<bool, (R::kMaxPath > 0)>());
  }
  void eval_results_impl(int*, double*, float*, int*, int*, int*, int*, std::false_type) {}
  void eval_results_impl(int* visits, double* reward, float* outcome, int* best, int* sims_run, int* gc_runs, int* prior_requests,
                         std::true_type) {
    MctsEvalArgs a = ev.a;
    a.visits_out = visits; a.reward_out = reward; a.outcome_out = outcome; a.best_out = best; a.sims_out = sims_run; a.gc_out = gc_runs;
    a.prior_requests_out = prior_requests;
    blockDim.x = 1; threadIdx.x = 0;
    for (long long t = 0; t < ev.n; ++t) {
      blockIdx.x = (unsigned)t;
      k_mcts_eval_report<R>(a, ev.n);
    }
  }
};

std::string g_err;
template <class R>
Emv* make(const b2s_params& p, long long cap) {
  auto* e = new EmvT<R>();
  const char* msg = e->configure(p, cap);
  if (msg) { g_err = msg; delete e; return nullptr; }
  return e;
}
}  // namespace

extern "C" {
const char* emv_last_error() { return g_err.c_str(); }
// a host batch of `cap` lanes at the initial state (game ids and parameters as b2s_batch_create)
void* emv_create(int game_id, const b2s_params* p, long long cap) {
  switch (game_id) {
    case B2S_TIC_TAC_TOE: return make<TicTacToeRules>(*p, cap);
    case B2S_CONNECT_FOUR: return make<ConnectFourRules>(*p, cap);
    case B2S_BREAKTHROUGH: return make<BreakthroughRules>(*p, cap);
    case B2S_HEX: return make<HexRules>(*p, cap);
    case B2S_GO: return make<GoRules>(*p, cap);
    case B2S_KUHN_POKER: return make<KuhnRules>(*p, cap);
    case B2S_MNK: return make<MnkRules>(*p, cap);
    case B2S_OTHELLO: return make<OthelloRules>(*p, cap);
    case B2S_Y: return make<YRules>(*p, cap);
    case B2S_HAVANNAH: return make<HavannahRules>(*p, cap);
  }
  g_err = "unknown game id";
  return nullptr;
}
void emv_destroy(void* h) { delete (Emv*)h; }
void emv_info(void* h, b2s_game_info* out) { *out = ((Emv*)h)->info; }
void emv_apply(void* h, const int* a, long long n) { ((Emv*)h)->apply(a, n); }
long long emv_error_count(void* h) { return (long long)((Emv*)h)->err.count; }
// 0 = ok, 1 = the game has no device MCTS, 2 = max_game_length too large for the path stack
int emv_mcts_eval_create(void* h, long long n, const b2s_mcts_eval_config* mc) { return ((Emv*)h)->eval_create(n, *mc); }
long long emv_mcts_eval_step(void* h, const double* values, const double* priors, unsigned char* pending) {
  return ((Emv*)h)->eval_step(values, priors, pending);
}
void emv_mcts_eval_leaves(void* h, float* obs, uint32_t* mask) { ((Emv*)h)->eval_leaves(obs, mask); }
void emv_mcts_eval_results(void* h, int* visits, double* reward, float* outcome, int* best, int* sims_run, int* gc_runs, int* prior_requests) {
  ((Emv*)h)->eval_results(visits, reward, outcome, best, sims_run, gc_runs, prior_requests);
}
}
