// TEST INFRASTRUCTURE ONLY — never part of the product (libb2s.so has no CPU path and fails without a GPU).
//
// Host build of the RL environment step: the PRODUCT's per-lane body env_step_lane (open_spiel_b200/csrc/env_step.cuh, the
// source k_env_step is built from) over the product's rule cores, one lane at a time, with the outputs k_env_step and the
// k_obs rows of b2s_env_step write.  tests/test_env_host.py replays it against tests/env_lib.py before any GPU time is
// spent; launch geometry and the coalesced stores are what the -m gpu tests are for.
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>

#include <string>
#include <vector>

#include "../../open_spiel_b200/csrc/host_compat.h"

#include "../../open_spiel_b200/csrc/common.cuh"
#include "../../open_spiel_b200/csrc/env_step.cuh"
#include "../../open_spiel_b200/csrc/rules_tic_tac_toe.cuh"
#include "../../open_spiel_b200/csrc/rules_connect_four.cuh"
#include "../../open_spiel_b200/csrc/rules_breakthrough.cuh"
#include "../../open_spiel_b200/csrc/rules_hex.cuh"
#include "../../open_spiel_b200/csrc/rules_go.cuh"
#include "../../open_spiel_b200/csrc/rules_kuhn_poker.cuh"
#include "../../open_spiel_b200/csrc/rules_leduc_poker.cuh"
#include "../../open_spiel_b200/csrc/rules_leduc_poker_n.cuh"
#include "../../open_spiel_b200/csrc/rules_mnk.cuh"
#include "../../open_spiel_b200/csrc/rules_othello.cuh"
#include "../../open_spiel_b200/csrc/rules_y.cuh"
#include "../../open_spiel_b200/csrc/rules_havannah.cuh"

namespace {
using namespace b2s;

template <class R> auto call_init(int) -> decltype(R::device_init(), void()) { R::device_init(); }
template <class R> void call_init(long) {}

struct EnvEmu {
  virtual ~EnvEmu() {}
  // actions == nullptr: reset.  Outputs as b2s_env_out (observations player-major [P][n][F]).
  virtual void call(const int* actions, int reset_if_done, long long n, float* obs, uint32_t* mask, float* rewards, uint8_t* done,
                    uint8_t* step_type, int8_t* cur) = 0;
  b2s_game_info info;
  ErrBuf err;
};

template <class R>
struct EnvEmuT : EnvEmu {
  typename R::Cfg cfg;
  std::vector<char> planes;
  std::vector<u64> hist;
  long long cap = 0;
  u64 seed = 0;
  long long lane_offset = 0;
  int which = 0;
  unsigned long long counter = 0;
  Ctx ctx() { Ctx c; c.planes = planes.data(); c.cap = cap; c.hist = hist.empty() ? nullptr : hist.data(); c.err = &err; return c; }
  const char* configure(const b2s_params& p, long long capacity, u64 sd, long long off, int observation) {
    memset(&info, 0, sizeof info);
    if (const char* e = R::make_cfg(p, cfg, info)) return e;
    int width = info.num_distinct_actions > info.max_chance_outcomes ? info.num_distinct_actions : info.max_chance_outcomes;
    info.mask_words = (width + 31) / 32;                      // as GameOpsT<R>::configure
    cap = capacity; seed = sd; lane_offset = off;
    which = observation < 0 ? (info.information_state_tensor_size > 0 ? 1 : 0) : observation;   // as b2s_env_create
    if (which == 1 && !R::kHasInfoState) return "no information state tensor";
    planes.assign(sizeof(StoredChunk<R>) * R::kChunks * (size_t)cap, 0);
    if (info.history_bytes) hist.assign((size_t)info.history_bytes / sizeof(u64) * (size_t)cap, 0);
    err.count = 0; err.first = 0x7fffffffffffffffLL;
    call_init<R>(0);
    return nullptr;
  }
  void call(const int* actions, int reset_if_done, long long n, float* obs, uint32_t* mask, float* rewards, uint8_t* done,
            uint8_t* step_type, int8_t* cur) override {
    Ctx c = ctx();
    const u32 b0 = env_block(counter);
    const int P = info.num_players, W = info.mask_words;
    for (long long i = 0; i < n; ++i) {                       // k_env_step, one lane per "thread"
      typename R::S s;
      if (actions) load_state<R>(s, cfg, c, i);
      const u64 g = (u64)(i + lane_offset);
      auto draw = [=](u32 b, u32 k) { return philox_uniform(seed, g, b, k); };
      float r[R::kPlayers];
      unsigned char d;
      bool changed;
      step_type[i] = env_step_lane<R>(s, actions ? actions[i] : -1, actions == nullptr, reset_if_done != 0, cfg, c, i, W, draw, b0, r, d,
                                      changed);
      if (changed) store_state<R>(s, cfg, c, i);
      done[i] = d;
      for (int p = 0; p < P; ++p) rewards[i * P + p] = r[p];
      const int cp = R::cur_player(s, cfg);
      cur[i] = (int8_t)cp;
      u32 m[R::kMaskWords];
      if (cp == kTerminalPlayerId) { for (int w = 0; w < R::kMaskWords; ++w) m[w] = 0; }
      else R::legal_nonterminal(s, cfg, m);
      for (int w = 0; w < W; ++w) mask[i * W + w] = m[w];
    }
    const int F = which ? info.information_state_tensor_size : info.observation_tensor_size;
    for (int p = 0; p < P; ++p)                               // k_obs(player = p) into row p
      for (long long i = 0; i < n; ++i) {
        typename R::S s;
        load_state<R>(s, cfg, c, i);
        typename R::ObsPack pk;
        R::obs_pack(s, cfg, p, which, pk);
        for (int e = 0; e < F; ++e) obs[((size_t)p * n + i) * F + e] = R::obs_elem(pk, cfg, e);
      }
    ++counter;                                                // k_env_tick
  }
};

std::string g_err;
template <class R>
EnvEmu* make(const b2s_params& p, long long cap, u64 seed, long long off, int observation) {
  auto* e = new EnvEmuT<R>();
  if (const char* msg = e->configure(p, cap, seed, off, observation)) { g_err = msg; delete e; return nullptr; }
  return e;
}
}  // namespace

extern "C" {
const char* emu_env_last_error() { return g_err.c_str(); }
void* emu_env_create(int game_id, const b2s_params* p, long long cap, unsigned long long seed, long long lane_offset, int observation) {
  const bool c4_std = (p->rows < 0 || p->rows == 6) && (p->columns < 0 || p->columns == 7) && (p->x_in_row < 0 || p->x_in_row == 4);
  switch (game_id) {                                          // as make_ops (api.cu)
    case B2S_TIC_TAC_TOE: return make<TicTacToeRules>(*p, cap, seed, lane_offset, observation);
    case B2S_CONNECT_FOUR:
      return c4_std ? make<ConnectFourStdRules>(*p, cap, seed, lane_offset, observation) : make<ConnectFourRules>(*p, cap, seed, lane_offset, observation);
    case B2S_BREAKTHROUGH: return make<BreakthroughRules>(*p, cap, seed, lane_offset, observation);
    case B2S_HEX: return make<HexRules>(*p, cap, seed, lane_offset, observation);
    case B2S_GO: return (p->board_size < 0 || p->board_size > 9) ? make<GoWideRules>(*p, cap, seed, lane_offset, observation)
                                                                 : make<GoRules>(*p, cap, seed, lane_offset, observation);
    case B2S_KUHN_POKER: return make<KuhnRules>(*p, cap, seed, lane_offset, observation);
    case B2S_MNK: return make<MnkRules>(*p, cap, seed, lane_offset, observation);
    case B2S_OTHELLO: return make<OthelloRules>(*p, cap, seed, lane_offset, observation);
    case B2S_Y: return make<YRules>(*p, cap, seed, lane_offset, observation);
    case B2S_HAVANNAH: return make<HavannahRules>(*p, cap, seed, lane_offset, observation);
    case B2S_LEDUC_POKER: return p->players > 2 ? make<LeducNRules>(*p, cap, seed, lane_offset, observation)
                                                : make<LeducRules>(*p, cap, seed, lane_offset, observation);
  }
  g_err = "unknown game id";
  return nullptr;
}
void emu_env_destroy(void* h) { delete (EnvEmu*)h; }
void emu_env_info(void* h, b2s_game_info* out) { *out = ((EnvEmu*)h)->info; }
void emu_env_call(void* h, const int* actions, int reset_if_done, long long n, float* obs, uint32_t* mask, float* rewards, uint8_t* done,
                  uint8_t* step_type, int8_t* cur) {
  ((EnvEmu*)h)->call(actions, reset_if_done, n, obs, mask, rewards, done, step_type, cur);
}
long long emu_env_error_count(void* h) { return (long long)((EnvEmu*)h)->err.count; }
}
