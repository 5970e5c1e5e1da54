// hex rule core on 128-bit bitboards.  Semantics: reference open_spiel/games/hex/hex.cc
// (PlayerAndActionToState :108-171, DoApplyAction :229-278 incl. the swap branch and the edge-label flood
// fill, LegalActions :280-293, AdjacentCells :316-329, IsTerminal :361, Returns :363-365 with its -0.0,
// ObservationTensor :379-398).  The reference keeps one of nine labels per cell (hex.h:68-78); we keep four
// 128-bit sets — black stones, white stones, labelA (BlackNorth | WhiteWest), labelB (BlackSouth | WhiteEast);
// a cell in both label sets is the winning stone (BlackWin / WhiteWin).  64 B per state as four 16-byte SoA
// planes.  The player to move sits in bit 127 of the black plane (boards have at most 121 cells).
#pragma once
#include "common.cuh"

namespace b2s {

struct HexRules {
  static constexpr int kGameId = B2S_HEX;
  typedef uint4 Chunk;
  static constexpr int kChunks = 4;
  static constexpr int kMaskWords = 4;     // up to 121 cells + swap
  static constexpr int kPlayers = 2;
  static constexpr int kMaxPath = 128;   // MCTS path stack (>= max_game_length + 2); 0 = no device MCTS
  static constexpr int kMaxLegal = 122;   // most legal actions any state can have (MCTS children block size)
  static constexpr int kFilterWords = 0;   // no per-lane history filter (see rules_go.cuh)
  static constexpr int kIlp = 1;
  static constexpr int kMinBlocks = 4;
  static constexpr bool kHasInfoState = false;

  struct Cfg {
    int cols, rows, cells, swap, plain;
    B128 board, not_west, not_east, row_first, row_last, col_first, col_last;
    u32 cells_magic;       // floor(e * magic >> 32) == e / cells for e < 9*cells
  };
  struct S { B128 black, white, la, lb; int mover; };

  static __host__ const char* make_cfg(const b2s_params& p, Cfg& c, b2s_game_info& gi) {
    int bs = p.board_size >= 0 ? p.board_size : 11;           // hex.h:41-44
    c.cols = p.columns >= 0 ? p.columns : bs;
    c.rows = p.rows >= 0 ? p.rows : bs;
    c.swap = p.swap > 0 ? 1 : 0;
    c.plain = p.plain_obs_tensor > 0 ? 1 : 0;
    // one row or one column: the reference's edge tests (hex.cc:122-126, 146-150) give a stone on both edges only one of them,
    // so no game ever ends and a full board is a non-terminal state with no legal action
    if (c.cols < 2 || c.rows < 2) return "hex: board too small (num_rows and num_cols must be at least 2)";
    if (c.cols * c.rows > 121 || c.cols > 63) return "hex: at most 121 cells on the device path";
    if (c.plain && c.cols < c.rows) return "hex: plain_obs_tensor with num_cols < num_rows is not supported (the reference indexes out of its plane)";
    if (c.swap && c.cols > c.rows)
      return "hex: swap with num_cols > num_rows is not supported (the reference mirrors the first stone outside the board, hex.cc:238)";
    c.cells = c.cols * c.rows;
    B128 z = {0, 0};
    c.board = c.not_west = c.not_east = c.row_first = c.row_last = c.col_first = c.col_last = z;
    for (int cell = 0; cell < c.cells; ++cell) {
      B128 b = b_bit(cell);
      int col = cell % c.cols, row = cell / c.cols;
      c.board = b_or(c.board, b);
      if (col != 0) c.not_west = b_or(c.not_west, b); else c.col_first = b_or(c.col_first, b);
      if (col != c.cols - 1) c.not_east = b_or(c.not_east, b); else c.col_last = b_or(c.col_last, b);
      if (row == 0) c.row_first = b_or(c.row_first, b);
      if (row == c.rows - 1) c.row_last = b_or(c.row_last, b);
    }
    if (!make_magic(c.cells, 9 * c.cells + 1, &c.cells_magic)) return "hex: internal magic";
    gi.num_players = 2;
    gi.num_distinct_actions = c.cells + c.swap;         // hex.h:135-137
    gi.max_game_length = c.cells;                       // hex.h:147
    gi.observation_tensor_size = (c.plain ? 3 : 9) * c.cells;
    gi.obs_shape[0] = c.plain ? 3 : 9; gi.obs_shape[1] = c.cols; gi.obs_shape[2] = c.rows;
    gi.min_utility = -1; gi.max_utility = 1;
    return nullptr;
  }
  static bool make_magic(int d, int limit, u32* out) {
    u64 M = ((1ull << 32) + d - 1) / d;
    for (int e = 0; e < limit; ++e) if ((int)(((u64)e * M) >> 32) != e / d) return false;
    *out = (u32)M;
    return true;
  }

  __device__ static __forceinline__ B128 ld(const Ctx& ctx, int plane, long long i) {
    ulonglong2 v = reinterpret_cast<const ulonglong2*>(ctx.planes)[(long long)plane * ctx.cap + i];
    return {v.x, v.y};
  }
  __device__ static __forceinline__ void st(const Ctx& ctx, int plane, long long i, B128 b) {
    reinterpret_cast<ulonglong2*>(ctx.planes)[(long long)plane * ctx.cap + i] = make_ulonglong2(b.lo, b.hi);
  }
  __device__ static __forceinline__ void load(S& s, const Ctx& ctx, long long i) {
    s.black = ld(ctx, 0, i); s.white = ld(ctx, 1, i); s.la = ld(ctx, 2, i); s.lb = ld(ctx, 3, i);
    s.mover = (int)(s.black.hi >> 63);
    s.black.hi &= ~(1ull << 63);
  }
  __device__ static __forceinline__ void store(const S& s, const Ctx& ctx, long long i) {
    B128 b = s.black;
    b.hi |= (u64)s.mover << 63;
    st(ctx, 0, i, b); st(ctx, 1, i, s.white); st(ctx, 2, i, s.la); st(ctx, 3, i, s.lb);
  }
  __device__ static __forceinline__ void init(S& s, const Cfg&, const Ctx&, long long) {
    B128 z = {0, 0};
    s.black = s.white = s.la = s.lb = z;
    s.mover = 0;
  }
  __device__ static __forceinline__ void copy_history(const Ctx&, long long, const Ctx&, long long, const S&, const Cfg&) {}

  // All cells adjacent to a cell of x (N, NE, E, S, SW, W — hex.cc:316-329; adjacency is symmetric).
  __device__ static __forceinline__ B128 neighbours(B128 x, const Cfg& c) {
    B128 xe = b_and(x, c.not_east), xw = b_and(x, c.not_west);
    B128 r = b_or(b_shr(x, c.cols), b_shl(x, c.cols));          // N, S
    r = b_or(r, b_or(b_shl(xe, 1), b_shr(xw, 1)));              // E, W
    if (c.cols > 1) r = b_or(r, b_or(b_shr(xe, c.cols - 1), b_shl(xw, c.cols - 1)));   // NE, SW
    return b_and(r, c.board);
  }
  // result from black's perspective: +1 / -1 / 0
  __device__ static __forceinline__ int result(const S& s) {
    B128 win = b_and(s.la, s.lb);
    if (!b_any(win)) return 0;
    return b_any(b_and(win, s.black)) ? 1 : -1;
  }
  __device__ static __forceinline__ bool terminal(const S& s, const Cfg&) { return result(s) != 0; }
  __device__ static __forceinline__ int cur_player(const S& s, const Cfg& c) { return terminal(s, c) ? kTerminalPlayerId : s.mover; }
  __device__ static __forceinline__ void returns(const S& s, const Cfg&, float* r) {
    float v = (float)result(s);
    r[0] = v; r[1] = -v;              // {r, -r}: non-terminal gives {0, -0}, as the reference does
  }
  __device__ static __forceinline__ bool swap_available(const S& s, const Cfg& c) {
    return c.swap && s.mover == 1 && !b_any(s.white) && b_popc(s.black) == 1;     // history_.size() == 1
  }
  __device__ static __forceinline__ void legal_nonterminal(const S& s, const Cfg& c, u32* m) {
    B128 e = b_andn(c.board, b_or(s.black, s.white));
    m[0] = (u32)e.lo; m[1] = (u32)(e.lo >> 32); m[2] = (u32)e.hi; m[3] = (u32)(e.hi >> 32);
    if (swap_available(s, c)) m[c.cells >> 5] |= 1u << (c.cells & 31);
  }
  __device__ static __forceinline__ void legal(const S& s, const Cfg& c, u32* m) {
    if (terminal(s, c)) { m[0] = m[1] = m[2] = m[3] = 0; return; }
    legal_nonterminal(s, c, m);
  }
  // Label of a new stone (hex.cc:108-171): bit0 = edge A (north / west), bit1 = edge B (south / east).
  __device__ static __forceinline__ int label_for(const S& s, const Cfg& c, int player, int move) {
    B128 mb = b_bit(move), nb = neighbours(mb, c);
    bool a, b;
    B128 own = player == 0 ? s.black : s.white;
    if (player == 0) {
      a = b_any(b_and(mb, c.row_first));
      b = !a && b_any(b_and(mb, c.row_last));        // `else if`: first row wins over last row
    } else {
      a = b_any(b_and(mb, c.col_first));
      b = !a && b_any(b_and(mb, c.col_last));
    }
    B128 onlyA = b_and(own, b_andn(s.la, s.lb)), onlyB = b_and(own, b_andn(s.lb, s.la));
    if (b_any(b_and(nb, onlyA))) a = true;
    if (b_any(b_and(nb, onlyB))) b = true;
    return (a ? 1 : 0) | (b ? 2 : 0);
  }
  __device__ static __forceinline__ bool apply(S& s, int a, const Cfg& c, const Ctx&, long long) {
    if (c.swap && a == c.cells) {
      if (!swap_available(s, c)) return false;
      int first = b_ffs(s.black);
      int r = first / c.cols, col = first - r * c.cols;
      int mirrored = col * c.cols + r;                 // hex.cc:238 (assumes a square board, as the reference does)
      if (mirrored >= c.cells) return false;
      B128 z = {0, 0};
      s.black = z; s.la = z; s.lb = z;
      int lab = label_for(s, c, 1, mirrored);
      B128 mb = b_bit(mirrored);
      s.white = mb;
      if (lab & 1) s.la = mb;
      if (lab & 2) s.lb = mb;
      s.mover = 0;
      return true;
    }
    if (a < 0 || a >= c.cells) return false;
    B128 mb = b_bit(a);
    if (b_any(b_and(mb, b_or(s.black, s.white)))) return false;
    int lab = label_for(s, c, s.mover, a);
    if (s.mover == 0) s.black = b_or(s.black, mb); else s.white = b_or(s.white, mb);
    if (lab & 1) s.la = b_or(s.la, mb);
    if (lab & 2) s.lb = b_or(s.lb, mb);
    if (lab == 1 || lab == 2) {
      // flood fill: plain stones of the mover connected to the new stone take its label (hex.cc:250-275)
      B128 own = s.mover == 0 ? s.black : s.white;
      B128 plain = b_andn(b_andn(own, s.la), s.lb);
      B128 frontier = mb, grown = {0, 0};
      while (true) {
        B128 g = b_and(neighbours(frontier, c), plain);
        if (!b_any(g)) break;
        plain = b_andn(plain, g);
        grown = b_or(grown, g);
        frontier = g;
      }
      if (lab == 1) s.la = b_or(s.la, grown); else s.lb = b_or(s.lb, grown);
    }
    s.mover ^= 1;
    return true;
  }
  // Observation planes by label value + 4 (hex.h:68-78, hex.cc:392-396):
  // 0 WhiteWin, 1 WhiteWest, 2 WhiteEast, 3 White, 4 Empty, 5 Black, 6 BlackSouth, 7 BlackNorth, 8 BlackWin.
  static constexpr bool kObsBitPacked = true;   // ObsPack = the tensor as a flat bit string in output order
  struct ObsPack { u64 w[18]; };      // up to 9 * 121 = 1089 bits
  // OR the low `cells` bits of v into the flat string at bit offset `off`
  __device__ static __forceinline__ void put_flat(ObsPack& p, int off, B128 v) {
    int i = off >> 6, sh = off & 63;
    p.w[i] |= v.lo << sh;
    u64 c1 = sh ? (v.lo >> (64 - sh)) : 0ull;
    if (i + 1 < 18) p.w[i + 1] |= c1 | (v.hi << sh);
    if (i + 2 < 18 && sh) p.w[i + 2] |= v.hi >> (64 - sh);
  }
  __device__ static __forceinline__ void obs_pack(const S& s, const Cfg& c, int, int, ObsPack& p) {
    B128 both = b_and(s.la, s.lb), onlyA = b_andn(s.la, s.lb), onlyB = b_andn(s.lb, s.la), any = b_or(s.la, s.lb);
    B128 empty = b_andn(c.board, b_or(s.black, s.white));
    for (int k = 0; k < 18; ++k) p.w[k] = 0;
    if (c.plain) {            // CellStateToPlainPlane, hex.cc:76-93: 0 black, 1 white, 2 empty
      B128 pl[3] = {s.black, s.white, empty};
      if (c.cols == c.rows) {
        for (int k = 0; k < 3; ++k) put_flat(p, k * c.cells, pl[k]);
      } else {
        // TensorView<3>{3, num_cols, num_rows} indexed {plane, cell / num_cols, cell % num_cols} (hex.cc:383-388):
        // offset = plane*cells + a*num_rows + b with a = cell / num_cols, b = cell % num_cols; on non-square boards
        // several cells alias one offset and the reference stores 1.0 for each, i.e. the bits are OR-ed.
        for (int k = 0; k < 3; ++k)
          for (int cell = 0; cell < c.cells; ++cell)
            if (b_test(pl[k], cell)) {
              int e = k * c.cells + (cell / c.cols) * c.rows + (cell % c.cols);
              p.w[e >> 6] |= 1ull << (e & 63);
            }
      }
      return;
    }
    // planes by label value + 4 (hex.h:68-78, hex.cc:392-396):
    // 0 WhiteWin, 1 WhiteWest, 2 WhiteEast, 3 White, 4 Empty, 5 Black, 6 BlackSouth, 7 BlackNorth, 8 BlackWin
    put_flat(p, 0 * c.cells, b_and(s.white, both));
    put_flat(p, 1 * c.cells, b_and(s.white, onlyA));
    put_flat(p, 2 * c.cells, b_and(s.white, onlyB));
    put_flat(p, 3 * c.cells, b_andn(s.white, any));
    put_flat(p, 4 * c.cells, empty);
    put_flat(p, 5 * c.cells, b_andn(s.black, any));
    put_flat(p, 6 * c.cells, b_and(s.black, onlyB));
    put_flat(p, 7 * c.cells, b_and(s.black, onlyA));
    put_flat(p, 8 * c.cells, b_and(s.black, both));
  }
  __device__ static __forceinline__ float obs_elem(const ObsPack& p, const Cfg&, int e) {
    return (float)((p.w[e >> 6] >> (e & 63)) & 1ull);
  }
};

}  // namespace b2s
