// Host instantiation of the b2s rule cores for the scalar State adapter (see host_rules.h).
// Everything game-specific below is a call into open_spiel_b200/csrc/rules_<game>.cuh — the source the sm_90a kernels
// are instantiated from — through the one-lane Ctx the kernels use (cap = 1: the SoA planes of a single lane are
// contiguous, which is exactly the b2s_state_get blob layout).
#include "host_rules.h"

// The rule cores live in namespace b2s and define globals there (go's Zobrist table).  libb2s.so carries host-side shadow
// symbols of the same names for its __device__ globals, and an executable that links both would interpose them (the
// library's cudaMemcpyToSymbol would then be handed this file's array as the symbol).  The host build therefore compiles
// the cores in a namespace of its own.
#define b2s b2s_hostcore

#include "../csrc/host_compat.h"   // host definitions of the device intrinsics; must precede the rule cores

#include "../csrc/common.cuh"
#include "../csrc/rules_tic_tac_toe.cuh"
#include "../csrc/rules_connect_four.cuh"
#include "../csrc/rules_breakthrough.cuh"
#include "../csrc/rules_hex.cuh"
#include "../csrc/rules_go.cuh"
#include "../csrc/rules_kuhn_poker.cuh"
#include "../csrc/rules_leduc_poker.cuh"
#include "../csrc/rules_leduc_poker_n.cuh"
#include "../csrc/rules_mnk.cuh"
#include "../csrc/rules_othello.cuh"
#include "../csrc/rules_y.cuh"
#include "../csrc/rules_havannah.cuh"

namespace b2s_host {
namespace {
using namespace b2s;

template <class R> auto call_init(int) -> decltype(R::device_init(), void()) { R::device_init(); }   // go: Zobrist table
template <class R> void call_init(long) {}

// per-game decode of the unpacked state S into the game-independent Decoded view
void decode(const TicTacToeRules::S& s, const TicTacToeRules::Cfg&, Decoded* d) {
  d->cells.assign(9, 0);
  for (int c = 0; c < 9; ++c) d->cells[c] = ((s.b >> c) & 1u) ? 1 : (((s.b >> (9 + c)) & 1u) ? 2 : 0);
  d->to_play = TicTacToeRules::mover(s);
}
void decode(const ConnectFourRules::S& s, const ConnectFourRules::Cfg& c, Decoded* d) {
  d->cells.assign((size_t)c.rows * c.cols, 0);
  const u64 x = ConnectFourRules::xs(s, c);
  for (int r = 0; r < c.rows; ++r)
    for (int col = 0; col < c.cols; ++col) {
      const int bit = col * c.h1 + r;
      d->cells[(size_t)r * c.cols + col] = ((x >> bit) & 1ull) ? 1 : (((s.o >> bit) & 1ull) ? 2 : 0);
    }
  d->to_play = ConnectFourRules::mover(s, c);
}
void decode(const BreakthroughRules::S& s, const BreakthroughRules::Cfg& c, Decoded* d) {
  d->cells.assign((size_t)c.cells, 0);
  const u64 white = s.w & c.board;
  for (int cell = 0; cell < c.cells; ++cell)
    d->cells[cell] = ((s.b >> cell) & 1ull) ? 1 : (((white >> cell) & 1ull) ? 2 : 0);
  d->to_play = s.mover;
}
void decode(const HexRules::S& s, const HexRules::Cfg& c, Decoded* d) {
  d->cells.assign((size_t)c.cells, 0);
  for (int cell = 0; cell < c.cells; ++cell) {
    const bool bl = b_test(s.black, cell), wh = b_test(s.white, cell);
    if (!bl && !wh) continue;
    const int lab = (b_test(s.la, cell) ? 1 : 0) | (b_test(s.lb, cell) ? 2 : 0);   // 1 = edge A, 2 = edge B, 3 = both (win)
    static const int8_t kBlack[4] = {1, 2, 3, 4}, kWhite[4] = {5, 6, 7, 8};
    d->cells[cell] = bl ? kBlack[lab] : kWhite[lab];
  }
  d->to_play = s.mover;
}
void decode(const GoRules::S& s, const GoRules::Cfg& c, Decoded* d) {
  d->cells.assign((size_t)c.cells, 0);
  for (int r = 0; r < c.n; ++r)
    for (int col = 0; col < c.n; ++col) {
      const int p = r * GoRules::kStride + col;
      d->cells[(size_t)r * c.n + col] = b_test(s.black, p) ? 1 : (b_test(s.white, p) ? 2 : 0);
    }
  d->to_play = s.to_play;
}
void decode(const MnkRules::S& s, const MnkRules::Cfg& c, Decoded* d) {
  d->cells.assign((size_t)c.cells, 0);
  for (int r = 0; r < c.rows; ++r)
    for (int col = 0; col < c.cols; ++col) {
      const int bit = r * MnkRules::kStride + col;
      d->cells[(size_t)r * c.cols + col] = q_test(s.x, bit) ? 1 : (q_test(s.o, bit) ? 2 : 0);
    }
  d->to_play = MnkRules::mover(s);
}
void decode(const OthelloRules::S& s, const OthelloRules::Cfg&, Decoded* d) {
  d->cells.assign(64, 0);
  for (int c = 0; c < 64; ++c) d->cells[c] = ((s.b >> c) & 1ull) ? 1 : (((s.w >> c) & 1ull) ? 2 : 0);
  d->to_play = s.mover;
}
void decode(const YRules::S& s, const YRules::Cfg& c, Decoded* d) {
  d->cells.assign((size_t)c.cells, 0);
  for (int cell = 0; cell < c.cells; ++cell) d->cells[cell] = b_test(s.p1, cell) ? 1 : (b_test(s.p2, cell) ? 2 : 0);
  d->to_play = s.mover;
  d->last_move = s.last == YRules::kNoMove ? -1 : s.last;
}
void decode(const HavannahRules::S& s, const HavannahRules::Cfg& c, Decoded* d) {
  d->cells.assign((size_t)c.cells, 0);
  for (int cell = 0; cell < c.cells; ++cell) d->cells[cell] = q_test(s.p1, cell) ? 1 : (q_test(s.p2, cell) ? 2 : 0);
  d->to_play = s.mover;
  d->last_move = s.last == HavannahRules::kNoMove ? -1 : s.last;
}
void decode(const KuhnRules::S& s, const KuhnRules::Cfg& c, Decoded* d) {   // the packed kuhn state is its action history
  d->num_players = c.n;
  const int len = KuhnRules::len(s);
  for (int p = 0; p < c.n; ++p) d->private_card[p] = p < len ? KuhnRules::card(s, p) : -1;
  d->round1.clear();
  for (int k = 0; k < KuhnRules::num_bet_actions(s, c); ++k) d->round1.push_back(KuhnRules::bet(s, k));
}
void decode(const LeducRules::S& s, const LeducRules::Cfg&, Decoded* d) {
  typedef LeducRules L;
  d->round = L::round2(s) ? 2 : 1;
  d->cur_player = L::cur(s) == L::kChance ? -1 : L::cur(s);
  d->public_card = L::pub(s) == L::kNone ? -1 : L::pub(s);
  for (int p = 0; p < 2; ++p) {
    d->private_card[p] = L::priv_of(s, p) == L::kNone ? -1 : L::priv_of(s, p);
    d->ante[p] = L::ante_of(s, p);
    d->folded[p] = L::folded_of(s, p);
  }
  d->round1.clear(); d->round2.clear();
  for (int i = 0; i < L::seq_len(s, 0); ++i) d->round1.push_back((L::seq(s, 0) >> (2 * i)) & 3);
  for (int i = 0; i < L::seq_len(s, 1); ++i) d->round2.push_back((L::seq(s, 1) >> (2 * i)) & 3);
}

void decode(const LeducNRules::S& s, const LeducNRules::Cfg& c, Decoded* d) {
  d->round = s.round2 ? 2 : 1;
  d->cur_player = s.cur == LeducNRules::kChance ? -1 : s.cur;
  d->public_card = s.pub == LeducNRules::kNone ? -1 : s.pub;
  d->num_players = c.n;
  for (int p = 0; p < c.n; ++p) {
    d->private_card[p] = s.priv[p] == LeducNRules::kNone ? -1 : s.priv[p];
    d->ante[p] = s.ante[p];
    d->folded[p] = (s.folded >> p) & 1;
  }
  d->round1.clear(); d->round2.clear();
  for (int i = 0; i < s.r1len; ++i) d->round1.push_back((int)((s.r1seq >> (2 * i)) & 3u));
  for (int i = 0; i < s.r2len; ++i) d->round2.push_back((int)((s.r2seq >> (2 * i)) & 3u));
}

template <class R>
class RulesT final : public Rules {
 public:
  const char* Configure(const b2s_params& p) {
    memset(&info_, 0, sizeof info_);
    const char* e = R::make_cfg(p, cfg_, info_);
    if (e) return e;
    const int width = info_.num_distinct_actions > info_.max_chance_outcomes ? info_.num_distinct_actions : info_.max_chance_outcomes;
    info_.mask_words = (width + 31) / 32;                       // as GameOpsT<R>::configure (csrc/batch_kernels.cuh)
    if (info_.mask_words > R::kMaskWords) return "action space too large for the packed layout";
    info_.state_bytes = (int)(sizeof(typename R::Chunk) * R::kChunks);
    info_.game_id = R::kGameId;
    call_init<R>(0);
    return nullptr;
  }
  // one-lane view over a blob: planes = blob, history column right behind the state chunks
  Ctx ctx(void* blob) const {
    Ctx c;
    c.planes = blob; c.cap = 1;
    c.hist = info_.history_bytes ? reinterpret_cast<u64*>(static_cast<char*>(blob) + info_.state_bytes) : nullptr;
    c.err = nullptr;
    return c;
  }
  void load(typename R::S& s, const void* blob) const { R::load(s, ctx(const_cast<void*>(blob)), 0); }

  void Init(void* blob) const override {
    memset(blob, 0, blob_bytes());
    Ctx c = ctx(blob);
    typename R::S s;
    R::init(s, cfg_, c, 0);
    R::store(s, c, 0);
  }
  bool Apply(void* blob, int action) const override {
    Ctx c = ctx(blob);
    typename R::S s;
    R::load(s, c, 0);
    if (R::terminal(s, cfg_) || !R::apply(s, action, cfg_, c, 0)) return false;
    R::store(s, c, 0);
    return true;
  }
  int CurrentPlayer(const void* blob) const override {
    typename R::S s;
    load(s, blob);
    return R::cur_player(s, cfg_);
  }
  void Returns(const void* blob, float* out) const override {
    typename R::S s;
    load(s, blob);
    R::returns(s, cfg_, out);
  }
  void LegalMask(const void* blob, uint32_t* words) const override {
    typename R::S s;
    load(s, blob);
    u32 m[R::kMaskWords];
    R::legal(s, cfg_, m);
    for (int w = 0; w < info_.mask_words; ++w) words[w] = m[w];
  }
  bool Tensor(const void* blob, int player, int which, float* out) const override {
    const int size = which == 0 ? info_.observation_tensor_size : info_.information_state_tensor_size;
    if (size <= 0 || (which == 1 && !R::kHasInfoState)) return false;
    typename R::S s;
    load(s, blob);
    typename R::ObsPack pk;
    R::obs_pack(s, cfg_, player, which, pk);
    for (int e = 0; e < size; ++e) out[e] = R::obs_elem(pk, cfg_, e);
    return true;
  }
  void Decode(const void* blob, Decoded* out) const override {
    typename R::S s;
    load(s, blob);
    decode(s, cfg_, out);
  }

 private:
  typename R::Cfg cfg_;
};

template <class R>
std::unique_ptr<Rules> make(const b2s_params& p, std::string* error) {
  auto r = std::make_unique<RulesT<R>>();
  if (const char* e = r->Configure(p)) { if (error) *error = e; return nullptr; }
  return r;
}

}  // namespace

std::unique_ptr<Rules> Rules::Create(int game_id, const b2s_params& p, std::string* error) {
  switch (game_id) {
    case B2S_TIC_TAC_TOE: return make<TicTacToeRules>(p, error);
    case B2S_CONNECT_FOUR: return make<ConnectFourRules>(p, error);
    case B2S_BREAKTHROUGH: return make<BreakthroughRules>(p, error);
    case B2S_HEX: return make<HexRules>(p, error);
    case B2S_GO: return make<GoRules>(p, error);
    case B2S_KUHN_POKER: return make<KuhnRules>(p, error);
    case B2S_MNK: return make<MnkRules>(p, error);
    case B2S_OTHELLO: return make<OthelloRules>(p, error);
    case B2S_Y: return make<YRules>(p, error);
    case B2S_HAVANNAH: return make<HavannahRules>(p, error);
    case B2S_LEDUC_POKER: return p.players > 2 ? make<LeducNRules>(p, error) : make<LeducRules>(p, error);
  }
  if (error) *error = "unknown game id";
  return nullptr;
}

}  // namespace b2s_host
