// TEST INFRASTRUCTURE ONLY — never part of the product (libb2s.so has no CPU path and fails without a GPU).
//
// Host build of AlphaBetaSearch with a caller-supplied value function (b2s_alpha_beta_eval_*): the PRODUCT's rule cores and the
// KERNEL BODY k_alpha_beta_eval_step (open_spiel_b200/csrc/alpha_beta.cuh) compiled with g++, one "thread" at a time, so that
// tests/test_alpha_beta_eval_host.py can run the search round by round in the CPU suite against tests/alpha_beta_lib.py.  The
// buffers and the argument block are set up as api.cu's b2s_alpha_beta_eval_create does; the caller's values are computed on the
// host from the leaves lanes (their observation tensor and legal mask, read back through the rule cores).
// Roots: lanes [0, n) of a host batch reset to the initial state and advanced with eab_apply.
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>

#include <string>
#include <vector>

#include "../../open_spiel_b200/csrc/host_compat.h"
// one "thread" at a time: the kernel indexes with blockIdx.x * blockDim.x + threadIdx.x
static struct { unsigned x, y, z; } blockIdx, blockDim = {1, 1, 1}, threadIdx;

#include "../../open_spiel_b200/csrc/common.cuh"
#include "../../open_spiel_b200/csrc/alpha_beta.cuh"
#include "../../open_spiel_b200/csrc/rules_tic_tac_toe.cuh"
#include "../../open_spiel_b200/csrc/rules_connect_four.cuh"
#include "../../open_spiel_b200/csrc/rules_breakthrough.cuh"
#include "../../open_spiel_b200/csrc/rules_hex.cuh"
#include "../../open_spiel_b200/csrc/rules_go.cuh"
#include "../../open_spiel_b200/csrc/rules_mnk.cuh"
#include "../../open_spiel_b200/csrc/rules_othello.cuh"
#include "../../open_spiel_b200/csrc/rules_y.cuh"
#include "../../open_spiel_b200/csrc/rules_havannah.cuh"

namespace {
using namespace b2s;

std::string g_err;

template <class R> auto call_init(int) -> decltype(R::device_init(), void()) { R::device_init(); }
template <class R> void call_init(long) {}

struct Eab {
  virtual ~Eab() {}
  virtual void apply(const int* a, long long n) = 0;
  virtual int search_create(long long n, int depth_limit, int maxp, long long max_nodes) = 0;
  virtual long long step(const double* values, unsigned char* pending) = 0;
  virtual void leaves(float* obs, u32* mask) = 0;
  virtual void results(double* value, int* best, long long* nodes, unsigned char* status, long long* evals) = 0;
  b2s_game_info info;
  ErrBuf err;
};

template <class R>
struct EabT : Eab {
  typename R::Cfg cfg;
  std::vector<char> planes;        // the roots batch, lane-blob form (R::load / R::store)
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
  // b2s_alpha_beta_eval_*: buffers and argument block as api.cu sets them up
  struct Run {
    long long n = 0;
    std::vector<char> roots, leaves, stack;
    std::vector<u64> hist;
    std::vector<AbEvalRoot> ctx;
    std::vector<unsigned char> pending, status;
    std::vector<double> value;
    std::vector<int> best;
    std::vector<long long> nodes, evals;
    unsigned long long n_pending = 0;
    AlphaBetaEvalArgs a;
    Ctx rootctx, leafctx;
  } ev;
  // 0 = ok, 1 = not served, 2 = the frame stack exceeds B2S_ALPHA_BETA_THREAD_STACK_BYTES
  int search_create(long long n, int depth_limit, int maxp, long long max_nodes) override {
    if constexpr (R::kMaxPath == 0) {
      return 1;
    } else {
      const long long len = info.max_game_length;
      const long long frames = depth_limit < 0 ? len + 2 : (depth_limit < len + 1 ? depth_limit : len + 1) + 1;
      const unsigned long long per_root = (unsigned long long)frames * sizeof(AbFrame<R, double>);
      if (per_root > B2S_ALPHA_BETA_THREAD_STACK_BYTES) return 2;
      ev.n = n;
      ev.roots.assign((size_t)info.state_bytes * (size_t)n, 0);
      ev.leaves.assign(sizeof(StoredChunk<R>) * R::kChunks * (size_t)n, 0);
      ev.hist.assign(info.history_bytes ? (size_t)info.history_bytes / sizeof(u64) * (size_t)n : 0, 0);
      ev.stack.assign((size_t)per_root * (size_t)n, 0);
      ev.ctx.assign((size_t)n, AbEvalRoot());
      memset(ev.ctx.data(), 0, sizeof(AbEvalRoot) * (size_t)n);
      ev.pending.assign((size_t)n, 0); ev.status.assign((size_t)n, 0); ev.value.assign((size_t)n, 0.0);
      ev.best.assign((size_t)n, 0); ev.nodes.assign((size_t)n, 0); ev.evals.assign((size_t)n, 0);
      ev.rootctx.planes = ev.roots.data(); ev.rootctx.cap = n; ev.rootctx.hist = ev.hist.empty() ? nullptr : ev.hist.data();
      ev.rootctx.err = &err;
      ev.leafctx = ev.rootctx;
      ev.leafctx.planes = ev.leaves.data();
      Ctx src = ctx();                                      // k_copy_to_blob
      for (long long i = 0; i < n; ++i) {
        typename R::S s;
        R::load(s, src, i);
        R::store(s, ev.rootctx, i);
        R::copy_history(ev.rootctx, i, src, i, s, cfg);
      }
      AlphaBetaEvalArgs& a = ev.a;
      memset(&a, 0, sizeof a);
      a.depth_limit = depth_limit; a.maximizing_player = maxp; a.max_nodes = max_nodes;
      a.mask_words = info.mask_words; a.num_players = info.num_players;
      a.stack = ev.stack.data(); a.roots = ev.ctx.data(); a.pending = ev.pending.data(); a.n_pending = &ev.n_pending;
      a.value = ev.value.data(); a.best_action = ev.best.data(); a.nodes = ev.nodes.data(); a.status = ev.status.data();
      a.evals = ev.evals.data(); a.err = &err;
      return 0;
    }
  }
  long long step(const double* values, unsigned char* pending) override {
    if constexpr (R::kMaxPath == 0) {
      return -1;
    } else {
      AlphaBetaEvalArgs a = ev.a;
      a.values = values;
      ev.n_pending = 0;
      blockDim.x = 1; threadIdx.x = 0;
      for (long long t = 0; t < ev.n; ++t) {
        blockIdx.x = (unsigned)t;
        k_alpha_beta_eval_step<R>(ev.rootctx, ev.leafctx, cfg, a, ev.n);
      }
      memcpy(pending, ev.pending.data(), (size_t)ev.n);
      return (long long)ev.n_pending;
    }
  }
  void leaves(float* obs, u32* mask) override {             // b2s_observation(-1) / b2s_legal_mask on the leaves batch
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
  void results(double* value, int* best, long long* nodes, unsigned char* status, long long* evals) override {
    const size_t n = (size_t)ev.n;
    memcpy(value, ev.value.data(), sizeof(double) * n);
    memcpy(best, ev.best.data(), sizeof(int) * n);
    memcpy(nodes, ev.nodes.data(), sizeof(long long) * n);
    memcpy(status, ev.status.data(), n);
    memcpy(evals, ev.evals.data(), sizeof(long long) * n);
  }
};

template <class R>
Eab* make(const b2s_params& p, long long cap) {
  auto* e = new EabT<R>();
  const char* msg = e->configure(p, cap);
  if (msg) { g_err = msg; delete e; return nullptr; }
  return e;
}
}  // namespace

extern "C" {
const char* eab_last_error() { return g_err.c_str(); }
// a host batch of `cap` lanes at the initial state (game ids and parameters as b2s_batch_create; rule core as make_ops)
void* eab_create(int game_id, const b2s_params* p, long long cap) {
  const bool c4_std = (p->rows < 0 || p->rows == 6) && (p->columns < 0 || p->columns == 7) && (p->x_in_row < 0 || p->x_in_row == 4);
  switch (game_id) {
    case B2S_TIC_TAC_TOE: return make<TicTacToeRules>(*p, cap);
    case B2S_CONNECT_FOUR: return c4_std ? make<ConnectFourStdRules>(*p, cap) : make<ConnectFourRules>(*p, cap);
    case B2S_BREAKTHROUGH: return make<BreakthroughRules>(*p, cap);
    case B2S_HEX: return make<HexRules>(*p, cap);
    case B2S_GO: return (p->board_size < 0 || p->board_size > 9) ? make<GoWideRules>(*p, cap) : make<GoRules>(*p, cap);
    case B2S_MNK: return make<MnkRules>(*p, cap);
    case B2S_OTHELLO: return make<OthelloRules>(*p, cap);
    case B2S_Y: return make<YRules>(*p, cap);
    case B2S_HAVANNAH: return make<HavannahRules>(*p, cap);
  }
  g_err = "unknown game id";
  return nullptr;
}
void eab_destroy(void* h) { delete (Eab*)h; }
void eab_info(void* h, b2s_game_info* out) { *out = ((Eab*)h)->info; }
void eab_apply(void* h, const int* a, long long n) { ((Eab*)h)->apply(a, n); }
long long eab_error_count(void* h) { return (long long)((Eab*)h)->err.count; }
int eab_search_create(void* h, long long n, int depth_limit, int maxp, long long max_nodes) {
  return ((Eab*)h)->search_create(n, depth_limit, maxp, max_nodes);
}
long long eab_step(void* h, const double* values, unsigned char* pending) { return ((Eab*)h)->step(values, pending); }
void eab_leaves(void* h, float* obs, uint32_t* mask) { ((Eab*)h)->leaves(obs, mask); }
void eab_results(void* h, double* value, int* best, long long* nodes, unsigned char* status, long long* evals) {
  ((Eab*)h)->results(value, best, nodes, status, evals);
}
}
