// breakthrough rule core on bitboards.  Semantics: reference open_spiel/games/breakthrough/breakthrough.cc
// (ctor :121-144, DoApplyAction :154-194, LegalActions :219-258, IsTerminal :308-310, Returns :312-320,
// ObservationTensor :286-342).  Packed: two 64-bit boards (black = player 0, moving to higher rows; white =
// player 1), bit = row*cols+col, 16 B per state.  Action id = ((r*cols+c)*6+dir)*2+capture (mixed-base rank
// over {rows, cols, 6, 2}, spiel_utils.cc:50-63).
#pragma once
#include "common.cuh"

namespace b2s {

struct BreakthroughRules {
  static constexpr int kGameId = B2S_BREAKTHROUGH;
  typedef uint4 Chunk;                 // {black.lo, black.hi, white.lo, white.hi}
  static constexpr int kChunks = 1;
  static constexpr int kMaskWords = 24;   // 64 cells * 12
  static constexpr int kObsWords = 3;
  static constexpr int kPlayers = 2;
  static constexpr int kMaxPath = 224;   // MCTS path stack (>= max_game_length + 2); 0 = no device MCTS
  static constexpr int kMaxLegal = 96;   // most legal actions any state can have (MCTS children block size)
  static constexpr int kFilterWords = 0;   // no per-lane history filter (see rules_go.cuh)
  static constexpr int kIlp = 2;      // lanes per thread in the streaming kernels
  static constexpr int kMinBlocks = 4;
  static constexpr bool kHasInfoState = false;

  struct Cfg {
    int rows, cols, cells;
    u64 board, last_row, first_row, not_col0, not_collast;
    u64 init_black, init_white;
  };
  // The player to move is not derivable from the position (captures change the piece counts) and an 8x8
  // board uses all 64 bits of both words, so the mover is folded into the stored pair: the white word is
  // stored complemented when player 1 is to move.  Boards are disjoint, so (black & stored_white) == 0 means
  // player 0 to move; otherwise black & ~white == black != 0 (black only runs out of pieces on white's
  // capture, after which player 0 is to move and the game is over anyway).
  struct S { u64 b, w; int mover; };

  static __host__ const char* make_cfg(const b2s_params& p, Cfg& c, b2s_game_info& gi) {
    c.rows = p.rows >= 0 ? p.rows : 8;     // breakthrough.h:41-42
    c.cols = p.columns >= 0 ? p.columns : 8;
    if (c.rows < 2 || c.cols < 2) return "breakthrough: rows, columns must be > 1";
    if (c.rows * c.cols > 64) return "breakthrough: rows*columns must fit 64 bits for the device path";
    c.cells = c.rows * c.cols;
    c.board = c.cells == 64 ? ~0ull : ((1ull << c.cells) - 1);
    u64 row0 = (c.cols == 64 ? ~0ull : ((1ull << c.cols) - 1));
    c.first_row = row0;
    c.last_row = row0 << ((c.rows - 1) * c.cols);
    c.not_col0 = 0; c.not_collast = 0;
    for (int r = 0; r < c.rows; ++r)
      for (int col = 0; col < c.cols; ++col) {
        if (col != 0) c.not_col0 |= 1ull << (r * c.cols + col);
        if (col != c.cols - 1) c.not_collast |= 1ull << (r * c.cols + col);
      }
    c.init_black = row0; c.init_white = c.last_row;
    if (c.rows >= 6) { c.init_black |= row0 << c.cols; c.init_white |= row0 << ((c.rows - 2) * c.cols); }
    gi.num_players = 2;
    gi.num_distinct_actions = c.cells * 12;                       // breakthrough.cc:388-390
    gi.max_game_length = 2 * (2 * c.rows - 3) * c.cols + 1;       // breakthrough.h:118-120
    gi.observation_tensor_size = 3 * c.cells;
    gi.obs_shape[0] = 3; gi.obs_shape[1] = c.rows; gi.obs_shape[2] = c.cols;
    gi.min_utility = -1; gi.max_utility = 1;
    return nullptr;
  }
  __device__ static __forceinline__ void load(S& s, const Ctx& ctx, long long i) {
    ulonglong2 v = reinterpret_cast<const ulonglong2*>(ctx.planes)[i];   // one 128-bit load
    s.b = v.x;
    u64 w = v.y;
    s.mover = (s.b & w) != 0 ? 1 : 0;
    s.w = s.mover ? ~w : w;
  }
  __device__ static __forceinline__ void store(const S& s, const Ctx& ctx, long long i) {
    u64 w = s.mover ? ~s.w : s.w;
    reinterpret_cast<ulonglong2*>(ctx.planes)[i] = make_ulonglong2(s.b, w);
  }
  __device__ static __forceinline__ void init(S& s, const Cfg& c, const Ctx&, long long) { s.b = c.init_black; s.w = c.init_white; s.mover = 0; }
  __device__ static __forceinline__ void copy_history(const Ctx&, long long, const Ctx&, long long, const S&, const Cfg&) {}

  // winner: 0 / 1 / -1
  __device__ static __forceinline__ int winner(const S& s, const Cfg& c) {
    u64 w = s.w & c.board;
    if ((s.b & c.last_row) || w == 0) return 0;
    if ((w & c.first_row) || s.b == 0) return 1;
    return -1;
  }
  __device__ static __forceinline__ bool terminal(const S& s, const Cfg& c) { return winner(s, c) >= 0; }
  __device__ static __forceinline__ int cur_player(const S& s, const Cfg& c) { return terminal(s, c) ? kTerminalPlayerId : s.mover; }
  __device__ static __forceinline__ void returns(const S& s, const Cfg& c, float* r) {
    int w = winner(s, c);
    r[0] = w == 0 ? 1.f : w == 1 ? -1.f : 0.f;
    r[1] = w == 1 ? 1.f : w == 0 ? -1.f : 0.f;
  }
  // Legal-action mask, bit-parallel.  Action id = (cell * 6 + dir) * 2 + capture with dir = mover * 3 + o, o = 0 / 1 / 2 for
  // the left / straight / right forward neighbour (breakthrough.cc:163-208, 289-337): every cell owns a 12-bit group, of
  // which the mover can set five bits (2o + capture, + 6 for player 1).  The five move kinds are computed for all cells at
  // once as bitboards of FROM cells; what remains is a bit permutation, byte t of each bitboard (cells 8t..8t+7) -> mask
  // words 3t..3t+2 at stride 12.  Multiplying a byte by a sum of 2^(11 j) puts bit j of its j-th copy at position 12 j
  // (copies are 11 apart, a byte is 8 wide: no carries), so a byte spreads with two 64-bit multiplies and two masks:
  //   cells 0..4 of the byte -> bits 12 j + k (j <= 4) of the 96-bit group triple, held in `lo`
  //   cells 5..7             -> bits 60 + k, 72 + k, 84 + k, held in `hi` relative to bit 32
  // No loop over pieces, no indexed local array: straight-line code, identical for every lane of a warp.
#ifndef B2S_BREAKTHROUGH_LEGAL_LOOP
  template <int K>
  __device__ static __forceinline__ void spread(u64 board, int t, u64& lo, u64& hi) {
    constexpr u64 kMulLo = (1ull | 1ull << 11 | 1ull << 22 | 1ull << 33 | 1ull << 44) << K;
    constexpr u64 kBitLo = (1ull | 1ull << 12 | 1ull << 24 | 1ull << 36 | 1ull << 48) << K;
    constexpr u64 kMulHi = (1ull << 23 | 1ull << 34 | 1ull << 45) << K;
    constexpr u64 kBitHi = (1ull << 28 | 1ull << 40 | 1ull << 52) << K;
    const u32 byte = __byte_perm((u32)(board >> (32 * (t >> 2))), 0u, 0x4440u | (u32)(t & 3));      // byte t, one PRMT
    lo |= mul_byte(byte, kMulLo) & kBitLo;
    hi |= mul_byte(byte, kMulHi) & kBitHi;
  }
  // byte * k for a byte < 256 and a 64-bit constant: one widening multiply-add per half (a plain u64 * u64 costs twice that)
  __device__ static __forceinline__ u64 mul_byte(u32 byte, u64 k) {
    return (u64)byte * (u32)k + ((u64)(byte * (u32)(k >> 32)) << 32);
  }
  __device__ static __forceinline__ void legal_nonterminal(const S& s, const Cfg& c, u32* m) {
    const u64 white = s.w & c.board;
    const u64 mine = s.mover == 0 ? s.b : white, theirs = s.mover == 0 ? white : s.b;
    const u64 empty = ~(s.b | white) & c.board;
    // target sets shifted back onto the FROM cell; player 0 moves up the board (r + 1), player 1 down (r - 1);
    // 2 <= cols <= 32, so every shift count is in 1..33
    u64 e_l, e_s, e_r, t_l, t_r;                 // empty / enemy target at the left, straight, right forward neighbour
    if (s.mover == 0) {
      e_l = empty >> (c.cols - 1); e_s = empty >> c.cols; e_r = empty >> (c.cols + 1);
      t_l = theirs >> (c.cols - 1); t_r = theirs >> (c.cols + 1);
    } else {
      e_l = empty << (c.cols + 1); e_s = empty << c.cols; e_r = empty << (c.cols - 1);
      t_l = theirs << (c.cols + 1); t_r = theirs << (c.cols - 1);
    }
    const u64 from_l = mine & c.not_col0, from_r = mine & c.not_collast;
    const u64 p0 = from_l & e_l, c0 = from_l & t_l, p1 = mine & e_s, p2 = from_r & e_r, c2 = from_r & t_r;
    const int sh = 6 * s.mover;
#pragma unroll
    for (int t = 0; t < 8; ++t) {
      u64 lo = 0, hi = 0;
      spread<0>(p0, t, lo, hi);
      spread<1>(c0, t, lo, hi);
      spread<2>(p1, t, lo, hi);
      spread<4>(p2, t, lo, hi);
      spread<5>(c2, t, lo, hi);
      lo <<= sh; hi <<= sh;                    // player 1's directions are 3..5: six bits further up in every group
      m[3 * t] = (u32)lo;
      m[3 * t + 1] = (u32)(lo >> 32) | (u32)hi;
      m[3 * t + 2] = (u32)(hi >> 32);
    }
  }
#else
  // the first version (a loop over the mover's pieces setting bits in an indexed local array), kept for before / after
  // measurements: build a second library with -DB2S_BREAKTHROUGH_LEGAL_LOOP and load it through B2S_LIBRARY
  __device__ static __forceinline__ void legal_nonterminal(const S& s, const Cfg& c, u32* m) {
    for (int i = 0; i < kMaskWords; ++i) m[i] = 0;
    u64 white = s.w & c.board;
    u64 mine = s.mover == 0 ? s.b : white, theirs = s.mover == 0 ? white : s.b;
    u64 empty = ~(s.b | white) & c.board;
    u64 pcs = mine;
    while (pcs) {
      int cell = __ffsll((long long)pcs) - 1;
      pcs &= pcs - 1;
      int r = cell / c.cols, col = cell - r * c.cols;
      int rp = s.mover == 0 ? r + 1 : r - 1;
      if (rp < 0 || rp >= c.rows) continue;
#pragma unroll
      for (int o = 0; o < 3; ++o) {
        int cp = col + o - 1;
        if (cp < 0 || cp >= c.cols) continue;
        u64 tb = 1ull << (rp * c.cols + cp);
        int dir = s.mover * 3 + o;
        int a = (cell * 6 + dir) * 2;
        if (empty & tb) m[a >> 5] |= 1u << (a & 31);
        else if (o != 1 && (theirs & tb)) { a += 1; m[a >> 5] |= 1u << (a & 31); }
      }
    }
  }
#endif
  __device__ static __forceinline__ void legal(const S& s, const Cfg& c, u32* m) {
    if (terminal(s, c)) { for (int i = 0; i < kMaskWords; ++i) m[i] = 0; return; }
    legal_nonterminal(s, c, m);
  }
  __device__ static __forceinline__ bool apply(S& s, int a, const Cfg& c, const Ctx&, long long) {
    if (a < 0 || a >= c.cells * 12) return false;
    int cap = a & 1, dir = (a >> 1) % 6, cell = a / 12;
    if (dir / 3 != s.mover) return false;
    int r = cell / c.cols, col = cell - r * c.cols;
    int rp = dir < 3 ? r + 1 : r - 1, cp = col + (dir % 3) - 1;
    if (rp < 0 || rp >= c.rows || cp < 0 || cp >= c.cols) return false;
    u64 from = 1ull << cell, to = 1ull << (rp * c.cols + cp);
    u64 white = s.w & c.board;
    u64 mine = s.mover == 0 ? s.b : white, theirs = s.mover == 0 ? white : s.b;
    if (!(mine & from)) return false;
    bool target_enemy = (theirs & to) != 0, target_empty = ((s.b | white) & to) == 0;
    if (cap) { if (!target_enemy || (dir % 3) == 1) return false; }
    else if (!target_empty) return false;
    mine = (mine & ~from) | to;
    theirs &= ~to;
    if (s.mover == 0) { s.b = mine; s.w = theirs; } else { s.w = mine; s.b = theirs; }
    s.mover ^= 1;
    return true;
  }
  static constexpr bool kObsBitPacked = true;   // ObsPack = the tensor as a flat bit string in output order
  // playout candidates: piece k/3 (ascending cell order) moving in direction k%3; -1 when it leaves the board,
  // the capture id when a diagonal lands on an enemy piece, else the plain-move id (apply() rejects blocked moves)
  __device__ static __forceinline__ int num_candidates(const S& s, const Cfg& c) {
    return 3 * __popcll(s.mover == 0 ? s.b : (s.w & c.board));
  }
  __device__ static __forceinline__ int candidate(const S& s, const Cfg& c, int k) {
    u64 white = s.w & c.board;
    u64 mine = s.mover == 0 ? s.b : white, theirs = s.mover == 0 ? white : s.b;
    int pi = k / 3, o = k - 3 * pi;
    int c0 = __popc((u32)mine);
    int cell = pi < c0 ? (int)__fns((u32)mine, 0, pi + 1) : 32 + (int)__fns((u32)(mine >> 32), 0, pi - c0 + 1);
    int r = cell / c.cols, col = cell - r * c.cols;
    int rp = s.mover == 0 ? r + 1 : r - 1, cp = col + o - 1;
    if (rp < 0 || rp >= c.rows || cp < 0 || cp >= c.cols) return -1;
    int dir = s.mover * 3 + o;
    int cap = (o != 1 && ((theirs >> (rp * c.cols + cp)) & 1ull)) ? 1 : 0;
    return (cell * 6 + dir) * 2 + cap;
  }
  __device__ static __forceinline__ bool play_candidate(S& s, int a, const Cfg& c, const Ctx& ctx, long long lane) {
    return a >= 0 && apply(s, a, c, ctx, lane);
  }
  struct ObsPack { u64 w[kObsWords]; };
  // planes 0 = black, 1 = white, 2 = empty; [plane][r][c] — breakthrough.cc:286-342
  __device__ static __forceinline__ void obs_pack(const S& s, const Cfg& c, int, int, ObsPack& p) {
    u64 pl[3] = {s.b, s.w & c.board, ~(s.b | s.w) & c.board};
    p.w[0] = p.w[1] = p.w[2] = 0;
    if (c.cells == 64) { p.w[0] = pl[0]; p.w[1] = pl[1]; p.w[2] = pl[2]; return; }
    int e = 0;
    for (int k = 0; k < 3; ++k)
      for (int cell = 0; cell < c.cells; ++cell, ++e) p.w[e >> 6] |= ((pl[k] >> cell) & 1ull) << (e & 63);
  }
  __device__ static __forceinline__ float obs_elem(const ObsPack& p, const Cfg&, int e) {
    return (float)((p.w[e >> 6] >> (e & 63)) & 1ull);
  }
};

}  // namespace b2s
