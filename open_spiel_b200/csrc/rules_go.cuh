// go (board_size <= 9) rule core on 128-bit bitboards.  Semantics: reference open_spiel/games/go/go.cc
// (LegalActions :160-170, IsTerminal :225-230, Returns :232-258, DoApplyAction :275-285, ObservationTensor
// :138-158) and go_board.cc (IsLegalMove :481-506, PlayMove :299-336 with its ko rule :313-331,
// CaptureDeadChains :423-439, Zobrist SetStone :355-364, TrompTaylorScore :612-683).
// The reference keeps linked-list chains with pseudo-liberty counters on a 21x21 guarded board; here a state
// is two stone sets (bit = row*10 + col: nine rows with a one-column guard so E/W shifts cannot wrap) and
// chains / liberties are recomputed on demand by bitboard flood fill.  "In atari" (go_board.h:243-248: all
// pseudo-liberties are one point) is exactly "the chain has one liberty", which is what we count.
// Packed state, 32 B as two 16-byte SoA planes: {black.lo, black.hi | meta << 32}, {white.lo, white.hi};
// meta = ko+1 (7 bits) | to_play (1) | pass_run (2) | superko (1) | ply (10) | cap_ply (10), where cap_ply is the
// index of the position produced by the most recent capturing move: a position can only recur if stones were
// removed in between, so the superko scan needs the history before cap_ply only.
// Positional superko (go.cc:280-285) needs every earlier position: an extra per-lane column of Zobrist hashes
// hist[k][lane], k = 0..max_game_length, holds the same hash values the reference computes
// (chess_common.h:129-170 table, seed 2765481), so repetition is detected on identical 64-bit keys.
#pragma once
#include <random>

#include "common.cuh"

namespace b2s {

__device__ u64 g_go_zobrist[2][96];     // [colour][row*10+col]; filled by GoRules::device_init()

struct GoRules {
  static constexpr int kGameId = B2S_GO;
  typedef uint4 Chunk;
  static constexpr int kChunks = 2;
  static constexpr int kMaskWords = 3;     // 81 points + pass
  static constexpr int kPlayers = 2;
  static constexpr int kMaxPath = 176;   // MCTS path stack (>= max_game_length + 2); 0 = no device MCTS
  static constexpr int kMaxLegal = 82;   // most legal actions any state can have (MCTS children block size)
  // Positional superko needs "has this hash occurred before?" after every stone placement that follows a capture: a scan of up
  // to `ply` history entries per move, which in a random playout is most of the work.  Searches that replay one lane many
  // times (MCTS) therefore carry a thread-private Bloom filter over the lane's history hashes (1024 bits, two probes from
  // independent hash bits): a miss proves the position is new and skips the scan; a hit (a repeat, or ~3 % false positives at
  // 100 entries) runs the exact scan as before.  Results are identical by construction; only the scan count changes.
  static constexpr int kFilterWords = 32;
  static constexpr int kIlp = 1;
  static constexpr int kMinBlocks = 4;
  static constexpr bool kHasInfoState = false;
  static constexpr int kStride = 10;

  struct Cfg {
    int n, cells, max_len, handicap;
    float komi;
    B128 board;
    u64 rowmask;          // n low bits
  };
  struct S {
    B128 black, white;
    int ko;               // bit index of the ko point, -1 none
    int to_play;          // 0 black, 1 white
    int pass_run;         // consecutive passes ending at the last move (capped at 2)
    int superko;
    int ply;              // history_.size()
    int cap_ply;          // index of the position created by the latest capture (0 = no capture yet)
  };

  __device__ static __forceinline__ bool filter_test_and_set(u32* f, u64 h) {
    const u32 b0 = (u32)h & 1023u, b1 = (u32)(h >> 10) & 1023u;
    const u32 w0 = f[b0 >> 5], w1 = f[b1 >> 5];
    const bool hit = ((w0 >> (b0 & 31)) & (w1 >> (b1 & 31)) & 1u) != 0;
    f[b0 >> 5] = w0 | 1u << (b0 & 31);
    f[b1 >> 5] |= 1u << (b1 & 31);
    return hit;
  }
  // filter over hist[0 .. ply] of `lane`
  __device__ static __forceinline__ void filter_build(u32* f, const Ctx& ctx, long long lane, const S& s) {
    for (int w = 0; w < kFilterWords; ++w) f[w] = 0;
    for (int k = 0; k <= s.ply; ++k) filter_test_and_set(f, ctx.hist[(long long)k * ctx.cap + lane]);
  }

  static __host__ const char* make_cfg(const b2s_params& p, Cfg& c, b2s_game_info& gi) {
    c.n = p.board_size >= 0 ? p.board_size : 19;                 // go.h:47-49 (default 19 is not a device size)
    if (c.n < 2 || c.n > 9) return "go: the device path supports board_size 2..9";
    c.komi = p.komi == p.komi ? (float)p.komi : 7.5f;
    c.handicap = p.handicap >= 0 ? p.handicap : 0;
    if (c.handicap >= 2) return "go: handicap stones use 19x19 coordinates (go.cc:72-93); unsupported on the device path";
    c.cells = c.n * c.n;
    c.max_len = p.max_game_length >= 0 ? p.max_game_length : 2 * c.cells;    // go.h:68-70
    if (c.max_len > 1000) return "go: max_game_length too large for the device path";
    c.board = {0, 0};
    for (int r = 0; r < c.n; ++r)
      for (int col = 0; col < c.n; ++col) c.board = b_or(c.board, b_bit(r * kStride + col));
    c.rowmask = (1ull << c.n) - 1;
    gi.num_players = 2;
    gi.num_distinct_actions = c.cells + 1;                       // go.h:61-63
    gi.max_game_length = c.max_len;
    gi.observation_tensor_size = 4 * c.cells;                    // go.h:175-179
    gi.obs_shape[0] = 4; gi.obs_shape[1] = c.n; gi.obs_shape[2] = c.n;
    // a game is never terminal before ply 2 (go.cc:225-230), so max_game_length 0 / 1 still plays two moves
    gi.history_bytes = 8 * ((c.max_len > 2 ? c.max_len : 2) + 1);
    gi.min_utility = -1; gi.max_utility = 1;
    return nullptr;
  }
  // ZobristTable<uint64_t, 441, 2>(2765481) restricted to the board points (go_board.cc:356-361).
  static __host__ void device_init() {
    static u64 host[2][96];
    static bool done = false;
    if (!done) {
      std::mt19937_64 outer(2765481);
      for (int vp = 0; vp < 21 * 21; ++vp) {
        std::mt19937_64 inner(outer());
        u64 v0 = inner(), v1 = inner();
        int vr = vp / 21 - 1, vc = vp % 21 - 1;               // virtual point -> board coordinates
        if (vr >= 0 && vr < 9 && vc >= 0 && vc < 9) { host[0][vr * kStride + vc] = v0; host[1][vr * kStride + vc] = v1; }
      }
      done = true;
    }
    cudaMemcpyToSymbol(g_go_zobrist, host, sizeof host);
  }

  __device__ static __forceinline__ void load(S& s, const Ctx& ctx, long long i) {
    const ulonglong2* pl = reinterpret_cast<const ulonglong2*>(ctx.planes);
    ulonglong2 b = pl[i], w = pl[ctx.cap + i];
    u32 meta = (u32)(b.y >> 32);
    s.black = {b.x, b.y & 0xffffffffull};
    s.white = {w.x, w.y};
    s.ko = (int)(meta & 127) - 1;
    s.to_play = (meta >> 7) & 1;
    s.pass_run = (meta >> 8) & 3;
    s.superko = (meta >> 10) & 1;
    s.ply = (meta >> 11) & 1023;
    s.cap_ply = (meta >> 21) & 1023;
  }
  __device__ static __forceinline__ void store(const S& s, const Ctx& ctx, long long i) {
    ulonglong2* pl = reinterpret_cast<ulonglong2*>(ctx.planes);
    u32 meta = (u32)(s.ko + 1) | (u32)s.to_play << 7 | (u32)s.pass_run << 8 | (u32)s.superko << 10 | (u32)s.ply << 11 |
               (u32)s.cap_ply << 21;
    pl[i] = make_ulonglong2(s.black.lo, s.black.hi | ((u64)meta << 32));
    pl[ctx.cap + i] = make_ulonglong2(s.white.lo, s.white.hi);
  }
  __device__ static __forceinline__ void init(S& s, const Cfg&, const Ctx& ctx, long long i) {
    s.black = {0, 0}; s.white = {0, 0};
    s.ko = -1; s.to_play = 0; s.pass_run = 0; s.superko = 0; s.ply = 0; s.cap_ply = 0;
    ctx.hist[i] = 0;                      // repetitions_ starts with the empty-board hash (go.cc:298-299)
  }
  __device__ static __forceinline__ void copy_history(const Ctx& dst, long long di, const Ctx& src, long long si, const S& s, const Cfg&) {
    for (int k = 0; k <= s.ply; ++k) dst.hist[(long long)k * dst.cap + di] = src.hist[(long long)k * src.cap + si];
  }

  __device__ static __forceinline__ B128 nb4(B128 x, const Cfg& c) {
    B128 r = b_or(b_or(b_shl(x, 1), b_shr(x, 1)), b_or(b_shl(x, kStride), b_shr(x, kStride)));
    return b_and(r, c.board);
  }
  // connected component(s) of `seed` inside `mask`
  __device__ static __forceinline__ B128 flood(B128 seed, B128 mask, const Cfg& c) {
    B128 cur = b_and(seed, mask);
    while (true) {
      B128 nx = b_and(b_or(cur, nb4(cur, c)), mask);
      if (nx.lo == cur.lo && nx.hi == cur.hi) return cur;
      cur = nx;
    }
  }
  // Does the connected component of `seed` inside `mask` touch `libs`?  Grows the component one step at a time like flood()
  // but stops at the first liberty: most chains have one within a step or two, and the full chain is only needed when the
  // answer is no (a capture).  *component receives the component when the answer is no (it is complete then).
  __device__ static __forceinline__ bool flood_finds(B128 seed, B128 mask, B128 libs, const Cfg& c, B128* component) {
    B128 cur = b_and(seed, mask);
    while (true) {
      B128 n4 = nb4(cur, c);
      if (b_any(b_and(n4, libs))) return true;
      B128 nx = b_and(b_or(cur, n4), mask);
      if (nx.lo == cur.lo && nx.hi == cur.hi) { *component = cur; return false; }
      cur = nx;
    }
  }
  __device__ static __forceinline__ u64 hash_of(B128 black, B128 white) {
    u64 h = 0;
    while (b_any(black)) { int p = b_ffs(black); black = b_andn(black, b_bit(p)); h ^= g_go_zobrist[0][p]; }
    while (b_any(white)) { int p = b_ffs(white); white = b_andn(white, b_bit(p)); h ^= g_go_zobrist[1][p]; }
    return h;
  }

  __device__ static __forceinline__ bool terminal(const S& s, const Cfg& c) {
    if (s.ply < 2) return false;
    return s.ply >= c.max_len || s.superko || s.pass_run >= 2;
  }
  __device__ static __forceinline__ int cur_player(const S& s, const Cfg& c) { return terminal(s, c) ? kTerminalPlayerId : s.to_play; }

  // Tromp-Taylor area score from black's side minus komi (go_board.cc:641-683): an empty region counts for a colour iff it
  // borders only that colour.  Instead of flooding the regions one by one, flood the empty points reachable from black
  // stones and those reachable from white stones (two floods, the same work in every lane): a region bordering only black is
  // exactly the set of empty points reachable from black and not from white.
  __device__ static __forceinline__ float score(const S& s, const Cfg& c) {
    int delta = b_popc(s.black) - b_popc(s.white);
    B128 empty = b_andn(c.board, b_or(s.black, s.white));
    if (b_any(empty)) {
      B128 rb = flood(nb4(s.black, c), empty, c), rw = flood(nb4(s.white, c), empty, c);
      delta += b_popc(b_andn(rb, rw)) - b_popc(b_andn(rw, rb));
    }
    return (float)delta - c.komi;
  }
  __device__ static __forceinline__ void returns(const S& s, const Cfg& c, float* r) {
    r[0] = 0.f; r[1] = 0.f;
    if (!terminal(s, c) || s.superko) return;
    float sc = score(s, c);
    if (sc > 0) { r[0] = 1.f; r[1] = -1.f; }
    else if (sc < 0) { r[0] = -1.f; r[1] = 1.f; }
  }

  // Stones (either colour) adjacent to `pts` that belong to chains with exactly one liberty.
  // `pts` are empty points without empty neighbours.  A chain that touches an "open" empty point (one that has an
  // empty neighbour) keeps that liberty whichever point of `pts` is played, so when many chains border `pts`
  // those chains are found with one whole-board flood per colour and only the remaining chains — whose liberties
  // are all surrounded points — are examined one by one.
  __device__ static __forceinline__ B128 atari_chains_near(const S& s, const Cfg& c, B128 pts, B128 empty) {
    B128 atari = {0, 0};
    B128 todo = b_and(nb4(pts, c), b_or(s.black, s.white));
    if (b_popc(todo) > 4) {
      B128 open = b_and(empty, nb4(empty, c));
      B128 near_open = nb4(open, c);
      B128 safe = b_or(flood(b_and(s.black, near_open), s.black, c), flood(b_and(s.white, near_open), s.white, c));
      todo = b_andn(todo, safe);
    }
    while (b_any(todo)) {
      int p = b_ffs(todo);
      B128 pb = b_bit(p);
      B128 colour = b_any(b_and(pb, s.black)) ? s.black : s.white;
      B128 chain = flood(pb, colour, c);
      B128 libs = b_and(nb4(chain, c), empty);
      if (b_popc(libs) == 1) atari = b_or(atari, chain);
      todo = b_andn(todo, chain);
    }
    return atari;
  }
  // All legal board points for the player to move (IsLegalMove, go_board.cc:481-506), as a board bitset.
  __device__ static __forceinline__ B128 legal_points(const S& s, const Cfg& c) {
    B128 own = s.to_play == 0 ? s.black : s.white, opp = s.to_play == 0 ? s.white : s.black;
    B128 empty = b_andn(c.board, b_or(s.black, s.white));
    B128 open = b_and(empty, nb4(empty, c));           // has an empty neighbour
    B128 cand = b_andn(empty, open);                   // completely surrounded by stones / edges
    B128 legal = open;
    if (b_any(cand)) {
      B128 atari = atari_chains_near(s, c, cand, empty);
      legal = b_or(legal, b_and(cand, nb4(b_andn(own, atari), c)));   // joins a friendly chain that keeps a liberty
      legal = b_or(legal, b_and(cand, nb4(b_and(opp, atari), c)));    // captures an enemy chain in atari
    }
    if (s.ko >= 0) legal = b_andn(legal, b_bit(s.ko));
    return legal;
  }
  // Does the chain containing stone set `seed` (all of one colour `col`) have a liberty in `libs_allowed`?
  // Quick accept when a seed stone itself touches an allowed empty point; otherwise flood the chain.
  __device__ static __forceinline__ bool chain_has_liberty(B128 seed, B128 col, B128 libs_allowed, const Cfg& c) {
    B128 chain;
    return flood_finds(seed, col, libs_allowed, c, &chain);
  }
  __device__ static __forceinline__ bool legal_point(const S& s, const Cfg& c, int p) {
    B128 pb = b_bit(p);
    B128 empty = b_andn(c.board, b_or(s.black, s.white));
    if (!b_any(b_and(pb, empty)) || p == s.ko) return false;
    B128 nbp = nb4(pb, c);
    if (b_any(b_and(nbp, empty))) return true;
    B128 own = s.to_play == 0 ? s.black : s.white, opp = s.to_play == 0 ? s.white : s.black;
    B128 other = b_andn(empty, pb);                    // liberties other than p itself
    // joins a friendly chain that keeps a liberty (one flood covers every friendly neighbour chain)
    B128 mine = b_and(nbp, own);
    if (b_any(mine) && chain_has_liberty(mine, own, other, c)) return true;
    // captures an enemy chain whose only liberty is p; neighbours that touch another empty point themselves are safe at
    // once (one whole-board neighbourhood instead of one per stone), the rest need the chain search
    B128 todo = b_andn(b_and(nbp, opp), nb4(other, c));
    while (b_any(todo)) {
      B128 q = b_bit(b_ffs(todo));
      B128 chain;
      if (!flood_finds(q, opp, other, c, &chain)) return true;       // no liberty but p: playing p captures it
      todo = b_andn(todo, q);                                          // (another stone of the same chain just repeats the short search)
    }
    return false;
  }
  // playout candidates: empty points other than the ko point (ascending), then pass
  __device__ static __forceinline__ int num_candidates(const S& s, const Cfg& c) {
    B128 e = b_andn(c.board, b_or(s.black, s.white));
    if (s.ko >= 0) e = b_andn(e, b_bit(s.ko));
    return b_popc(e) + 1;
  }
  __device__ static __forceinline__ int candidate(const S& s, const Cfg& c, int k) {
    B128 e = b_andn(c.board, b_or(s.black, s.white));
    if (s.ko >= 0) e = b_andn(e, b_bit(s.ko));
    if (k >= b_popc(e)) return c.cells;
    int p = b_select(e, k);
    int r = p / kStride;
    return r * c.n + (p - r * kStride);
  }
  // board bitset (stride 10) -> action-ordered bits (row*n + col) appended into words at bit offset `off`
  __device__ static __forceinline__ void deposit_rows(B128 x, const Cfg& c, u64* words, int off) {
    for (int r = 0; r < c.n; ++r) {
      int sh = r * kStride;
      u64 row = (sh < 64 ? (x.lo >> sh) | (sh ? (x.hi << (64 - sh)) : 0) : (x.hi >> (sh - 64))) & c.rowmask;
      int pos = off + r * c.n;
      words[pos >> 6] |= row << (pos & 63);
      if ((pos & 63) + c.n > 64) words[(pos >> 6) + 1] |= row >> (64 - (pos & 63));
    }
  }
  __device__ static __forceinline__ void legal_nonterminal(const S& s, const Cfg& c, u32* m) {
    u64 w[2] = {0, 0};
    deposit_rows(legal_points(s, c), c, w, 0);
    w[c.cells >> 6] |= 1ull << (c.cells & 63);          // pass is always legal (go.cc:168)
    m[0] = (u32)w[0]; m[1] = (u32)(w[0] >> 32); m[2] = (u32)w[1];
  }
  __device__ static __forceinline__ void legal(const S& s, const Cfg& c, u32* m) {
    if (terminal(s, c)) { m[0] = m[1] = m[2] = 0; return; }
    legal_nonterminal(s, c, m);
  }

  // PlayMove + GoState::DoApplyAction.  `checked` = legality already established by the caller.
  __device__ static __forceinline__ bool apply_impl(S& s, int a, const Cfg& c, const Ctx& ctx, long long lane, bool checked) {
    if (a < 0 || a > c.cells) return false;
    u64 h = ctx.hist[(long long)s.ply * ctx.cap + lane];
    if (a == c.cells) {                                   // pass: clears the ko point; never a superko
      s.ko = -1;
      s.pass_run = s.pass_run < 2 ? s.pass_run + 1 : 2;
    } else {
      int r = a / c.n, col = a - r * c.n, p = r * kStride + col;
      if (!checked && !legal_point(s, c, p)) return false;
      B128 pb = b_bit(p);
      B128 own = s.to_play == 0 ? s.black : s.white, opp = s.to_play == 0 ? s.white : s.black;
      B128 empty = b_andn(c.board, b_or(s.black, s.white));
      B128 nbp = nb4(pb, c);
      bool in_enemy_eye = !b_any(b_and(nbp, b_or(own, empty)));
      own = b_or(own, pb);
      empty = b_andn(empty, pb);
      h ^= g_go_zobrist[s.to_play][p];
      // capture enemy chains left without liberties; neighbours that touch an empty point themselves are safe at once
      B128 todo = b_andn(b_and(nbp, opp), nb4(empty, c)), captured = {0, 0};
      while (b_any(todo)) {
        B128 q = b_bit(b_ffs(todo));
        B128 chain;
        if (flood_finds(q, opp, empty, c, &chain)) { todo = b_andn(todo, q); continue; }   // the chain still has a liberty
        captured = b_or(captured, chain);
        todo = b_andn(todo, chain);
      }
      int ncap = b_popc(captured);
      opp = b_andn(opp, captured);
      s.ko = (in_enemy_eye && ncap == 1) ? b_ffs(captured) : -1;
      while (b_any(captured)) { int q = b_ffs(captured); captured = b_andn(captured, b_bit(q)); h ^= g_go_zobrist[1 - s.to_play][q]; }
      if (s.to_play == 0) { s.black = own; s.white = opp; } else { s.white = own; s.black = opp; }
      s.pass_run = 0;
      // positional superko: has this position occurred before (including the initial one)?  Stones only leave the
      // board by capture, so an earlier equal position must precede the latest capture.
      if (ncap > 0) s.cap_ply = s.ply + 1;
      const bool maybe_seen = ctx.filter ? filter_test_and_set(ctx.filter, h) : true;
      if (maybe_seen)
        for (int k = 0; k < s.cap_ply; ++k)
          if (ctx.hist[(long long)k * ctx.cap + lane] == h) { s.superko = 1; break; }
    }
    s.to_play ^= 1;
    s.ply += 1;
    ctx.hist[(long long)s.ply * ctx.cap + lane] = h;
    return true;
  }
  __device__ static __forceinline__ bool apply(S& s, int a, const Cfg& c, const Ctx& ctx, long long lane) {
    return apply_impl(s, a, c, ctx, lane, false);
  }
  // the caller guarantees `a` came from this state's legal set (tree descent)
  __device__ static __forceinline__ bool apply_legal(S& s, int a, const Cfg& c, const Ctx& ctx, long long lane) {
    return apply_impl(s, a, c, ctx, lane, true);
  }
  // playout step: try a candidate (an empty non-ko point or pass); false = it was illegal, state untouched.
  // Two restructurings of this step were measured in the MCTS kernel and dropped: (i) replacing the per-chain walks by
  // two liberty-seeded whole-board floods per move (slower), (ii) one flattened loop over a per-move work list of chains
  // with early exit on the first liberty (slower: its extra registers cost a resident warp per scheduler).
  __device__ static __forceinline__ bool play_candidate(S& s, int a, const Cfg& c, const Ctx& ctx, long long lane) {
    if (a != c.cells) {
      int r = a / c.n;
      if (!legal_point(s, c, r * kStride + (a - r * c.n))) return false;
    }
    return apply_impl(s, a, c, ctx, lane, true);
  }

  // planes black, white, empty in board-point order, plane 3 = "white to play" (go.cc:138-158)
  static constexpr bool kObsBitPacked = true;   // ObsPack = the tensor as a flat bit string in output order
  struct ObsPack { u64 w[6]; };
  __device__ static __forceinline__ void obs_pack(const S& s, const Cfg& c, int, int, ObsPack& p) {
    for (int k = 0; k < 6; ++k) p.w[k] = 0;
    deposit_rows(s.black, c, p.w, 0);
    deposit_rows(s.white, c, p.w, c.cells);
    deposit_rows(b_andn(c.board, b_or(s.black, s.white)), c, p.w, 2 * c.cells);
    if (s.to_play == 1) deposit_rows(c.board, c, p.w, 3 * c.cells);
  }
  __device__ static __forceinline__ float obs_elem(const ObsPack& p, const Cfg&, int e) {
    return (float)((p.w[e >> 6] >> (e & 63)) & 1ull);
  }
};

}  // namespace b2s
