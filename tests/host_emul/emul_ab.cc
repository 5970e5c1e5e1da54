// TEST INFRASTRUCTURE ONLY — never part of the product (libb2s.so has no CPU path and fails without a GPU).
//
// Host build of AlphaBetaSearch: the PRODUCT's kernel body k_alpha_beta (open_spiel_b200/csrc/alpha_beta.cuh) over the product's
// rule cores, run as one thread on a one-root batch.  tests/test_alpha_beta_host.py
// compares it with the restatement in tests/alpha_beta_lib.py before any GPU time is spent; the persistent grid and the
// [depth][thread] stack layout are what the -m gpu tests are for.
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>

#include <string>
#include <vector>

#include "../../open_spiel_b200/csrc/host_compat.h"

// one "thread": the kernel indexes its frame stack with blockIdx.x * blockDim.x + threadIdx.x
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

// Root = the initial state after `actions`; the result as lane 0 of b2s_alpha_beta_search.  Returns 0, or 1 with g_err set.
template <class R>
int search(const b2s_params& p, const int* actions, int n_actions, int depth_limit, int maxp, long long max_nodes, AbResult& out) {
  if constexpr (!ab_served<R>()) {
    g_err = "not served";
    return 1;
  } else {
    typename R::Cfg cfg;
    b2s_game_info info;
    memset(&info, 0, sizeof info);
    if (const char* e = R::make_cfg(p, cfg, info)) { g_err = e; return 1; }
    const int width = info.num_distinct_actions > info.max_chance_outcomes ? info.num_distinct_actions : info.max_chance_outcomes;
    call_init<R>(0);
    std::vector<typename R::Chunk> planes(R::kChunks);
    std::vector<u64> hist(info.history_bytes ? info.history_bytes / sizeof(u64) : 0);
    ErrBuf err = {0, 0x7fffffffffffffffLL};
    Ctx c;
    c.planes = planes.data(); c.cap = 1; c.hist = hist.empty() ? nullptr : hist.data(); c.err = &err;
    typename R::S s;
    R::init(s, cfg, c, 0);
    for (int k = 0; k < n_actions; ++k)
      if (!R::apply(s, actions[k], cfg, c, 0)) { g_err = "illegal root action"; return 1; }
    R::store(s, c, 0);
    std::vector<AbFrame<R>> stack(info.max_game_length + 2);
    AlphaBetaArgs a;
    memset(&a, 0, sizeof a);
    a.depth_limit = depth_limit; a.maximizing_player = maxp; a.mask_words = (width + 31) / 32; a.max_nodes = max_nodes;
    unsigned long long next = 0;
    int best = 0;
    unsigned char status = 0;
    a.threads = 1; a.stack = stack.data(); a.next = &next; a.err = &err;
    a.value = &out.value; a.best_action = &best; a.nodes = &out.nodes; a.status = &status;
    k_alpha_beta<R>(c, cfg, a, 1);
    out.best_action = best; out.status = status;
    if ((err.count != 0) != (status >= 2)) { g_err = "error count disagrees with the status"; return 1; }
    return 0;
  }
}
}  // namespace

extern "C" {
const char* emu_ab_last_error() { return g_err.c_str(); }
int emu_ab_search(int game_id, const b2s_params* p, const int* actions, int n_actions, int depth_limit, int maxp, long long max_nodes,
                  double* value, int* best_action, long long* nodes, int* status) {
  AbResult r;
  int rc = 1;
  const bool c4_std = (p->rows < 0 || p->rows == 6) && (p->columns < 0 || p->columns == 7) && (p->x_in_row < 0 || p->x_in_row == 4);
  switch (game_id) {                                          // as make_ops (api.cu)
    case B2S_TIC_TAC_TOE: rc = search<TicTacToeRules>(*p, actions, n_actions, depth_limit, maxp, max_nodes, r); break;
    case B2S_CONNECT_FOUR:
      rc = c4_std ? search<ConnectFourStdRules>(*p, actions, n_actions, depth_limit, maxp, max_nodes, r)
                  : search<ConnectFourRules>(*p, actions, n_actions, depth_limit, maxp, max_nodes, r);
      break;
    case B2S_BREAKTHROUGH: rc = search<BreakthroughRules>(*p, actions, n_actions, depth_limit, maxp, max_nodes, r); break;
    case B2S_HEX: rc = search<HexRules>(*p, actions, n_actions, depth_limit, maxp, max_nodes, r); break;
    case B2S_GO:
      rc = (p->board_size < 0 || p->board_size > 9) ? search<GoWideRules>(*p, actions, n_actions, depth_limit, maxp, max_nodes, r)
                                                    : search<GoRules>(*p, actions, n_actions, depth_limit, maxp, max_nodes, r);
      break;
    case B2S_MNK: rc = search<MnkRules>(*p, actions, n_actions, depth_limit, maxp, max_nodes, r); break;
    case B2S_OTHELLO: rc = search<OthelloRules>(*p, actions, n_actions, depth_limit, maxp, max_nodes, r); break;
    case B2S_Y: rc = search<YRules>(*p, actions, n_actions, depth_limit, maxp, max_nodes, r); break;
    case B2S_HAVANNAH: rc = search<HavannahRules>(*p, actions, n_actions, depth_limit, maxp, max_nodes, r); break;
    default: g_err = "not served";
  }
  if (rc) return rc;
  *value = r.value; *best_action = r.best_action; *nodes = r.nodes; *status = r.status;
  return 0;
}
}
