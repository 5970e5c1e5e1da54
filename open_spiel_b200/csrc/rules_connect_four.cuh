// connect_four rule core on bitboards.  Semantics: reference open_spiel/games/connect_four/connect_four.cc
// (DoApplyAction :130-145, LegalActions :147-156, HasLine :163-196, IsTerminal :277-279, Returns :281-285,
// ObservationTensor :299-328).  Representation is ours: in registers (S), two 64-bit boards, column-major with one
// sentinel bit above every column (bit = col*(rows+1)+row, row 0 = bottom) so the four line directions are plain
// shifts with no wrap-around.
// In a device batch a state is ONE 64-bit key (Packed), 8 B per state: stones only ever sit on a column's bottom rows, so
// each column's h1 = rows+1 bits hold, below a marker bit at the column's height, who owns each stone (1 = player 0), and
// zeros above the marker (a full column has its marker on the sentinel row):  key = x | (occ + bottom).  One key per
// position; pack() encodes it, unpack() decodes it.  The lane blob of b2s_state_get / b2s_state_set and of host States
// (Chunk, load() / store()) is the decoded pair {x, o}, 16 B, which needs no configuration to read.
// When the board leaves two spare bits (every size up to (rows+1)*cols <= 62, including the default 6x7) the
// outcome_ of the reference (connect_four.h:58-63) is cached in bits 62-63 of the key, exactly as the
// reference caches it in `outcome_`: a step then costs ONE line test (for the stone just dropped) instead of
// re-deriving the outcome before and after.  Larger boards derive it on load.
// Two instantiations of one source: ConnectFourCore<true> is the default board (6x7, four in a row) with every size a
// compile-time constant, so the kernels' shifts by rows+1, rows and columns are immediates instead of 64-bit shifts by a
// run-time amount (the batched ApplyAction of the default board is an HBM stream whose integer work otherwise shows);
// ConnectFourCore<false> (ConnectFourRules) reads the sizes from the configuration and serves every other board and the
// host tools.
#pragma once
#include "common.cuh"

namespace b2s {

template <bool kStd>
struct ConnectFourCore {
  static constexpr int kGameId = B2S_CONNECT_FOUR;
  typedef uint4 Chunk;                 // the lane blob: {x, o}
  typedef u64 Packed;                  // a lane in a device batch: the key
  static constexpr int kChunks = 1;
  static constexpr int kMaskWords = 1;
  static constexpr int kObsWords = 3;  // 3*rows*cols <= 189 bits
  static constexpr int kPlayers = 2;
  static constexpr int kMaxPath = 72;   // MCTS path stack (>= max_game_length + 2); 0 = no device MCTS
  static constexpr int kMaxLegal = 32;   // most legal actions any state can have (MCTS children block size)
  static constexpr int kFilterWords = 0;   // no per-lane history filter (see rules_go.cuh)
  static constexpr int kIlp = 4;      // lanes per thread in the streaming kernels (8 was measured slower with 8-byte lanes: k_step_fused then needs 58 registers)
  static constexpr int kMinBlocks = 6;   // <= 42 registers (capping k_apply at 32 registers to fit the 1M-lane grid in one wave spills and was measured 20 % slower)
  static constexpr bool kHasInfoState = false;
  static constexpr int kStdRows = 6, kStdCols = 7, kStdK = 4;   // connect_four.h:45-50 defaults

  struct Cfg {
    int rows, cols, k, ego;
    int h1;            // rows + 1
    int meta;          // 1: outcome cached in bits 62-63 of the key
    int gather;        // 1: legal mask by multiply-gather (verified exhaustively on the host)
    u32 gmul_lo, gmul_hi;   // per-32-bit-half gather multipliers
    int gsh_lo, gsh_hi, cols_lo;
    int rgather;       // 1: row extraction (bits c*h1 -> bits 0..cols-1) by multiply-gather, verified on the host
    u32 rmul_lo, rmul_hi;
    int rsh_lo, rsh_hi, rcols_lo, rfirst_hi;
    int line4;         // 1: has_line's four-in-a-row fast path (k == 4, every shift below 64); sits in padding before top
    u64 top;           // top playable cell of every column
    u64 board;         // all playable cells
    u64 bottom;        // bit c*h1 of every column (row 0)
    u64 fill[6];       // fill[j]: rows < h1 - 2^j of every column (0 when 2^j >= h1), so a shift down by 2^j masked with it
                       // moves no bit into the column below
  };
  // x keeps the key's player 0 stones plus (when cfg.meta) the cached outcome in bits 62-63, stored
  // as outcome ^ 2 so that "unknown" is all-zero.  outcome: 0 = player 0 won, 1 = player 1 won, 2 = unknown,
  // 3 = draw (connect_four.h:58-63).
  struct S { u64 x, o; };   // player 0 ("x", kCross) / player 1 ("o", kNought) stones
  // the sizes as the device code reads them: constants on the default board
  __host__ __device__ static __forceinline__ int ROWS(const Cfg& c) { return kStd ? kStdRows : c.rows; }
  __host__ __device__ static __forceinline__ int COLS(const Cfg& c) { return kStd ? kStdCols : c.cols; }
  __host__ __device__ static __forceinline__ int H1(const Cfg& c) { return kStd ? kStdRows + 1 : c.h1; }
  __host__ __device__ static __forceinline__ int K(const Cfg& c) { return kStd ? kStdK : c.k; }
  __host__ __device__ static __forceinline__ bool META(const Cfg& c) { return kStd ? true : c.meta != 0; }

  static __host__ const char* make_cfg(const b2s_params& p, Cfg& c, b2s_game_info& gi) {
    c.rows = p.rows >= 0 ? p.rows : 6;            // connect_four.h:45-50 defaults
    c.cols = p.columns >= 0 ? p.columns : 7;
    c.k = p.x_in_row >= 0 ? p.x_in_row : 4;
    c.ego = p.egocentric_obs_tensor > 0 ? 1 : 0;
    if (c.rows < 1 || c.cols < 1 || c.k < 1) return "connect_four: rows, columns, x_in_row must be positive";
    if ((c.rows + 1) * c.cols > 64 || c.cols > 32)
      return "connect_four: (rows+1)*columns must fit 64 bits for the device path";
    if (kStd && (c.rows != kStdRows || c.cols != kStdCols || c.k != kStdK)) return "connect_four: not the default board";
    c.h1 = c.rows + 1;
    c.meta = (c.rows + 1) * c.cols <= 62 ? 1 : 0;
    c.line4 = c.k == 4 && 2 * (c.h1 + 1) < 64 ? 1 : 0;
    c.top = 0; c.board = 0; c.bottom = 0;
    for (int col = 0; col < c.cols; ++col) {
      c.top |= 1ull << (col * c.h1 + c.rows - 1);
      c.board |= ((1ull << c.rows) - 1) << (col * c.h1);
      c.bottom |= 1ull << (col * c.h1);
    }
    for (int j = 0; j < 6; ++j) c.fill[j] = (1 << j) < c.h1 ? c.bottom * ((1ull << (c.h1 - (1 << j))) - 1) : 0;
    make_gather(c);
    make_row_gather(c);
    gi.num_players = 2;
    gi.num_distinct_actions = c.cols;              // connect_four.h:179
    gi.max_game_length = c.rows * c.cols;          // connect_four.h:200
    gi.max_chance_outcomes = 0;
    gi.observation_tensor_size = 3 * c.rows * c.cols;
    gi.obs_shape[0] = 3; gi.obs_shape[1] = c.rows; gi.obs_shape[2] = c.cols;
    gi.information_state_tensor_size = 0;
    gi.min_utility = -1; gi.max_utility = 1;
    return nullptr;
  }
  // Legal mask = the free top cells (bits c*h1 + rows-1) gathered into bits 0..cols-1.  The top bits are split
  // at bit 32 into two 32-bit words; within a word the bits sit h1 apart, and one 32-bit multiply whose
  // partial products cannot collide packs them contiguously.  Checked for every column subset below.
  static __host__ u32 gather_word(int n, int h1, u32* mul, int* sh) {
    // n bits sitting h1 apart (at j*h1 after the shift) -> multiplier sum_j 2^{(h1-1)*(n-1-j)} packs them at *sh
    u32 m = 0;
    for (int j = 0; j < n; ++j) {
      int e = (h1 - 1) * (n - 1 - j);
      if (e >= 32) return 0;
      m |= 1u << e;
    }
    *mul = m; *sh = (h1 - 1) * (n - 1);
    return 1;
  }
  static __host__ u32 gather_eval(const Cfg& c, u64 free_top) {
    u32 lo = (u32)free_top, hi = (u32)(free_top >> 32);
    int p0 = c.rows - 1;
    u32 out = 0;
    if (c.cols_lo > 0) out |= (((lo >> p0) * c.gmul_lo) >> c.gsh_lo) & ((1u << c.cols_lo) - 1);
    if (c.cols_lo < c.cols) {
      int first_hi = c.cols_lo * c.h1 + c.rows - 1 - 32;
      out |= ((((hi >> first_hi) * c.gmul_hi) >> c.gsh_hi) & ((1u << (c.cols - c.cols_lo)) - 1)) << c.cols_lo;
    }
    return out;
  }
  static __host__ void make_gather(Cfg& c) {
    c.gather = 0; c.gmul_lo = c.gmul_hi = 0; c.gsh_lo = c.gsh_hi = 0;
    c.cols_lo = 0;
    while (c.cols_lo < c.cols && c.cols_lo * c.h1 + c.rows - 1 < 32) ++c.cols_lo;
    if (c.cols > 24) return;
    u32 ok = 1;
    if (c.cols_lo > 0) ok &= gather_word(c.cols_lo, c.h1, &c.gmul_lo, &c.gsh_lo);
    if (c.cols_lo < c.cols) ok &= gather_word(c.cols - c.cols_lo, c.h1, &c.gmul_hi, &c.gsh_hi);
    if (!ok) return;
    for (u32 subset = 0; subset < (1u << c.cols); ++subset) {       // exhaustive check of the multiply trick
      u64 ft = 0;
      for (int col = 0; col < c.cols; ++col) if ((subset >> col) & 1u) ft |= 1ull << (col * c.h1 + c.rows - 1);
      if (gather_eval(c, ft) != subset) return;
    }
    c.gather = 1;
  }

  // Row r of a column-major board = bits r + c*h1.  After shifting by r they sit at c*h1; the same verified
  // multiply-gather as the legal mask packs them into bits 0..cols-1 (used by the observation tensor).
  static __host__ __device__ __forceinline__ u32 row_gather_eval(const Cfg& c, u64 t) {
    u32 lo = (u32)t, hi = (u32)(t >> 32);
    u32 out = ((lo * c.rmul_lo) >> c.rsh_lo) & ((1u << c.rcols_lo) - 1);
    if (c.rcols_lo < c.cols) out |= ((((hi >> c.rfirst_hi) * c.rmul_hi) >> c.rsh_hi) & ((1u << (c.cols - c.rcols_lo)) - 1)) << c.rcols_lo;
    return out;
  }
  static __host__ void make_row_gather(Cfg& c) {
    c.rgather = 0; c.rmul_lo = c.rmul_hi = 0; c.rsh_lo = c.rsh_hi = 0; c.rfirst_hi = 0;
    c.rcols_lo = 0;
    while (c.rcols_lo < c.cols && c.rcols_lo * c.h1 < 32) ++c.rcols_lo;
    if (c.cols > 24) return;
    u32 ok = 1;
    if (c.rcols_lo > 0) ok &= gather_word(c.rcols_lo, c.h1, &c.rmul_lo, &c.rsh_lo);
    if (c.rcols_lo < c.cols) { ok &= gather_word(c.cols - c.rcols_lo, c.h1, &c.rmul_hi, &c.rsh_hi); c.rfirst_hi = c.rcols_lo * c.h1 - 32; }
    if (!ok) return;
    u64 colbits = 0;
    for (int col = 0; col < c.cols; ++col) colbits |= 1ull << (col * c.h1);
    for (u32 subset = 0; subset < (1u << c.cols); ++subset) {       // exhaustive check, with every other bit set as noise
      u64 t = 0;
      for (int col = 0; col < c.cols; ++col) if ((subset >> col) & 1u) t |= 1ull << (col * c.h1);
      if (row_gather_eval(c, t) != subset) return;
    }
    c.rgather = 1;
    (void)colbits;
  }

  __device__ static __forceinline__ bool has_line(u64 b, const Cfg& c) {
    // four in a row by three shift-and-steps; its largest shift, 2 * (h1 + 1), must stay below 64 (a shift by 64 or more is
    // undefined in C++: the host build gives wrong lines there), so boards of 30 rows and more take the guarded loop
    if (kStd || c.line4) {
      const int d1 = H1(c), d2 = H1(c) + 1, d3 = H1(c) - 1;
      u64 m1 = b & (b >> 1), m2 = b & (b >> d1), m3 = b & (b >> d2), m4 = b & (b >> d3);
      u64 any = (m1 & (m1 >> 2)) | (m2 & (m2 >> (2 * d1))) | (m3 & (m3 >> (2 * d2))) | (m4 & (m4 >> (2 * d3)));
      return any != 0;
    }
    const int d[4] = {1, H1(c), H1(c) + 1, H1(c) - 1};
    for (int j = 0; j < 4; ++j) {
      u64 m = b;
      bool ok = true;
      for (int i = 1; i < K(c); ++i) {
        int sh = i * d[j];
        if (sh >= 64) { ok = false; break; }
        m &= b >> sh;
      }
      if (ok && m) return true;
    }
    return false;
  }
  __host__ __device__ static __forceinline__ u64 xs(const S& s, const Cfg& c) { return META(c) ? (s.x & ~(3ull << 62)) : s.x; }
  __device__ static __forceinline__ int mover(const S& s, const Cfg& c) { return __popcll(xs(s, c) | s.o) & 1; }
  __device__ static __forceinline__ int derive_outcome(u64 x, u64 o, const Cfg& c) {
    int last = 1 - (__popcll(x | o) & 1);            // only the player who just moved can have completed a line
    if (has_line(last == 0 ? x : o, c)) return last;
    if (((x | o) & c.top) == c.top) return 3;
    return 2;
  }
  __device__ static __forceinline__ int outcome(const S& s, const Cfg& c) {
    return META(c) ? ((int)(s.x >> 62) ^ 2) : derive_outcome(s.x, s.o, c);
  }

  __host__ __device__ static __forceinline__ void load(S& s, const Ctx& ctx, long long i) {
    ulonglong2 v = reinterpret_cast<const ulonglong2*>(ctx.planes)[i];
    s.x = v.x;
    s.o = v.y;
  }
  __host__ __device__ static __forceinline__ void store(const S& s, const Ctx& ctx, long long i) {
    reinterpret_cast<ulonglong2*>(ctx.planes)[i] = make_ulonglong2(s.x, s.o);
  }
  __host__ __device__ static __forceinline__ void unpack(S& s, u64 key, const Cfg& c) {
    // fill every column from its marker down (the outcome bits never reach a column: fill[] covers none of their shifts);
    // fill[j] = 0 where 2^j >= h1, and past j = 2 only boards taller than 7 rows have any
    u64 f = key;
    f |= (f >> 1) & c.fill[0];
    f |= (f >> 2) & c.fill[1];
    f |= (f >> 4) & c.fill[2];
    if (H1(c) > 8) {
      f |= (f >> 8) & c.fill[3];
      f |= (f >> 16) & c.fill[4];
      f |= (f >> 32) & c.fill[5];
    }
    const u64 occ = (f >> 1) & c.fill[0];           // the rows below each marker
    s.x = key & (occ | (META(c) ? 3ull << 62 : 0ull));
    s.o = occ & ~key;
  }
  // occ + bottom carries every column's stone stack into its marker bit
  __host__ __device__ static __forceinline__ u64 pack(const S& s, const Cfg& c) { return s.x | ((xs(s, c) | s.o) + c.bottom); }
  __device__ static __forceinline__ void init(S& s, const Cfg&, const Ctx&, long long) { s.x = 0; s.o = 0; }
  __device__ static __forceinline__ void copy_history(const Ctx&, long long, const Ctx&, long long, const S&, const Cfg&) {}

  __device__ static __forceinline__ bool terminal(const S& s, const Cfg& c) { return outcome(s, c) != 2; }
  __device__ static __forceinline__ int cur_player(const S& s, const Cfg& c) {
    return terminal(s, c) ? kTerminalPlayerId : mover(s, c);
  }
  __device__ static __forceinline__ void returns(const S& s, const Cfg& c, float* r) {
    int oc = outcome(s, c);
    r[0] = oc == 0 ? 1.f : oc == 1 ? -1.f : 0.f;
    r[1] = oc == 1 ? 1.f : oc == 0 ? -1.f : 0.f;
  }
  // Legal columns of a NON-terminal state.
  __device__ static __forceinline__ void legal_nonterminal(const S& s, const Cfg& c, u32* m) {
    u64 free_top = ~(xs(s, c) | s.o) & c.top;
    if (c.gather) {
      u32 lo = (u32)free_top, hi = (u32)(free_top >> 32);
      u32 out = (((lo >> (ROWS(c) - 1)) * c.gmul_lo) >> c.gsh_lo) & ((1u << c.cols_lo) - 1);
      if (c.cols_lo < COLS(c)) {
        int first_hi = c.cols_lo * H1(c) + ROWS(c) - 1 - 32;
        out |= ((((hi >> first_hi) * c.gmul_hi) >> c.gsh_hi) & ((1u << (COLS(c) - c.cols_lo)) - 1)) << c.cols_lo;
      }
      m[0] = out;
      return;
    }
    u32 out = 0;
    for (int col = 0; col < COLS(c); ++col) out |= (u32)((free_top >> (col * H1(c) + ROWS(c) - 1)) & 1ull) << col;
    m[0] = out;
  }
  __device__ static __forceinline__ void legal(const S& s, const Cfg& c, u32* m) {
    if (terminal(s, c)) { m[0] = 0; return; }
    legal_nonterminal(s, c, m);
  }
  // Apply to a NON-terminal state; false = illegal (state untouched).
  __device__ static __forceinline__ bool apply(S& s, int a, const Cfg& c, const Ctx&, long long) {
    if (a < 0 || a >= COLS(c)) return false;
    u64 x = xs(s, c);
    u64 occ = x | s.o;
    int base = a * H1(c);
    if ((occ >> (base + ROWS(c) - 1)) & 1ull) return false;
    u64 colmask = ((1ull << ROWS(c)) - 1) << base;
    u64 bit = (occ & colmask) + (1ull << base);
    int mv = __popcll(occ) & 1;
    u64 mine = (mv == 0 ? x : s.o) | bit;
    if (mv == 0) x = mine; else s.o = mine;
    if (META(c)) {
      // outcome_ after the move (connect_four.cc:139-143): a line for the mover, else a full board
      int oc = has_line(mine, c) ? mv : (((occ | bit) & c.top) == c.top ? 3 : 2);
      x |= (u64)(oc ^ 2) << 62;
    }
    s.x = x;
    return true;
  }

  // Observation tensor as a packed bit string in output (CHW) order.
  static constexpr bool kObsBitPacked = true;   // ObsPack = the tensor as a flat bit string in output order
  struct ObsPack { u64 w[kObsWords]; };
  __device__ static __forceinline__ void obs_pack(const S& s, const Cfg& c, int player, int /*which*/, ObsPack& p) {
    u64 planes[3];
    if (c.ego) {                         // PlayerRelative, connect_four.cc:299-310
      planes[0] = player == 0 ? s.o : xs(s, c);
      planes[1] = player == 0 ? xs(s, c) : s.o;
    } else {                             // StateToPlayer, connect_four.cc:75-86
      planes[0] = xs(s, c); planes[1] = s.o;
    }
    planes[2] = ~(xs(s, c) | s.o) & c.board;
    p.w[0] = p.w[1] = p.w[2] = 0;
    if (c.rgather) {
      u64 colbits = c.board & ~(c.board << 1);             // bit c*h1 of every column
      int e = 0;
#pragma unroll
      for (int pl = 0; pl < 3; ++pl)
        for (int r = 0; r < ROWS(c); ++r, e += COLS(c)) {
          u64 row = (u64)row_gather_eval(c, (planes[pl] >> r) & colbits);
          p.w[e >> 6] |= row << (e & 63);
          if ((e & 63) + COLS(c) > 64) p.w[(e >> 6) + 1] |= row >> (64 - (e & 63));
        }
      return;
    }
    int e = 0;
#pragma unroll
    for (int pl = 0; pl < 3; ++pl)
      for (int r = 0; r < ROWS(c); ++r)
        for (int col = 0; col < COLS(c); ++col, ++e) {
          u64 bit = (planes[pl] >> (col * H1(c) + r)) & 1ull;
          p.w[e >> 6] |= bit << (e & 63);
        }
  }
  __device__ static __forceinline__ float obs_elem(const ObsPack& p, const Cfg&, int e) {
    return (float)((p.w[e >> 6] >> (e & 63)) & 1ull);
  }
};

typedef ConnectFourCore<false> ConnectFourRules;   // every board; the host tools' core
typedef ConnectFourCore<true> ConnectFourStdRules;  // the default 6x7 board, four in a row

}  // namespace b2s
