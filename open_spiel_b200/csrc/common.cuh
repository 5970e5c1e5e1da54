// Shared device/host helpers for the batched game kernels (sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/b2s.h"

namespace b2s {

typedef unsigned long long u64;
typedef unsigned int u32;

// Sentinels: reference open_spiel/spiel_globals.h:26-56,82.
constexpr int kChancePlayerId = -1;
constexpr int kTerminalPlayerId = -4;

// Per-batch error record written by kernels when an action is rejected.
struct ErrBuf {
  u64 count;        // lanes rejected since last reset
  long long first;  // a rejected lane index (min over racing writers), -1 if none
};

__device__ __forceinline__ void flag_error(ErrBuf* e, long long lane) {
  atomicAdd(&e->count, 1ull);
  atomicMin(&e->first, lane);
}

// Everything a kernel needs to find lane i's packed state.
struct Ctx {
  void* planes;       // kChunks planes of `cap` chunks each (SoA)
  long long cap;
  u64* hist;          // go: [max_len+1][cap] zobrist history, else nullptr
  ErrBuf* err;
  long long lane0 = 0;   // batch lane of this view's lane 0 (sub-range views: planes / hist are pre-offset, errors report lane0 + i)
  u32* filter = nullptr; // optional thread-private membership filter over this lane's history hashes (go superko, see rules_go.cuh)
};

// ---- Philox4x32-10 counter RNG (Salmon et al. 2011), key = seed, counter = (lane, ply) ----------
struct Philox {
  u32 c[4];
  u32 k[2];
};
__host__ __device__ __forceinline__ void philox_round(u32 (&c)[4], const u32 (&k)[2]) {
  const u32 M0 = 0xD2511F53u, M1 = 0xCD9E8D57u;
  u64 p0 = (u64)M0 * c[0], p1 = (u64)M1 * c[2];
  u32 hi0 = (u32)(p0 >> 32), lo0 = (u32)p0, hi1 = (u32)(p1 >> 32), lo1 = (u32)p1;
  u32 n0 = hi1 ^ c[1] ^ k[0], n1 = lo1, n2 = hi0 ^ c[3] ^ k[1], n3 = lo0;
  c[0] = n0; c[1] = n1; c[2] = n2; c[3] = n3;
}
// Four 32-bit words for (seed, lane, ply).
__host__ __device__ __forceinline__ void philox4(u64 seed, u64 lane, u32 ply, u32 stream, u32 (&out)[4]) {
  u32 c[4] = {(u32)lane, (u32)(lane >> 32), ply, stream};
  u32 k[2] = {(u32)seed, (u32)(seed >> 32)};
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    philox_round(c, k);
    k[0] += 0x9E3779B9u; k[1] += 0xBB67AE85u;
  }
  out[0] = c[0]; out[1] = c[1]; out[2] = c[2]; out[3] = c[3];
}
// Unbiased uniform integer in [0, n) from the (seed, lane, ply) block: Lemire's multiply-shift with
// rejection; the four words of the block are tried in order, then the block for stream+1, ...
__host__ __device__ __forceinline__ u32 philox_uniform(u64 seed, u64 lane, u32 ply, u32 n) {
  // a word is rejected iff the low half of word * n is below (2^32 - n) mod n; that threshold is < n, so the modulo is only
  // evaluated when the low half is below n (probability n / 2^32) — same accept / reject decisions, no division otherwise
  for (u32 stream = 0;; ++stream) {
    u32 r[4];
    philox4(seed, lane, ply, stream, r);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      u64 m = (u64)r[j] * n;
      if ((u32)m >= n || (u32)m >= (u32)(0u - n) % n) return (u32)(m >> 32);
    }
  }
}

// k-th (0-based) set bit position of a multi-word mask; returns -1 if fewer bits.
__device__ __forceinline__ int nth_set_bit(const u32* words, int nwords, int k) {
  for (int w = 0; w < nwords; ++w) {
    int c = __popc(words[w]);
    if (k < c) return w * 32 + (int)__fns(words[w], 0, k + 1);
    k -= c;
  }
  return -1;
}

// R::apply_legal(...) when the rule core offers a cheaper "already known legal" path, else R::apply(...)
template <class R, class S, class Cfg>
__device__ __forceinline__ auto apply_known_legal_impl(S& s, int a, const Cfg& c, const Ctx& ctx, long long lane, int)
    -> decltype(R::apply_legal(s, a, c, ctx, lane)) { return R::apply_legal(s, a, c, ctx, lane); }
template <class R, class S, class Cfg>
__device__ __forceinline__ bool apply_known_legal_impl(S& s, int a, const Cfg& c, const Ctx& ctx, long long lane, long) {
  return R::apply(s, a, c, ctx, lane);
}
template <class R, class S, class Cfg>
__device__ __forceinline__ bool apply_known_legal(S& s, int a, const Cfg& c, const Ctx& ctx, long long lane) {
  return apply_known_legal_impl<R>(s, a, c, ctx, lane, 0);
}

// Number of players of a configured game: R::num_players(cfg) when the rule core has a run-time count (kuhn_poker), else the
// compile-time R::kPlayers (which is always the size of the returns array a kernel keeps).
template <class R, class Cfg>
__device__ __forceinline__ auto rule_num_players_impl(const Cfg& c, int) -> decltype(R::num_players(c)) { return R::num_players(c); }
template <class R, class Cfg>
__device__ __forceinline__ int rule_num_players_impl(const Cfg&, long) { return R::kPlayers; }
template <class R, class Cfg>
__device__ __forceinline__ int rule_num_players(const Cfg& c) { return rule_num_players_impl<R>(c, 0); }

// One playout step: choose a uniformly random legal action and apply it; returns the action.
// Rule cores may expose a cheap candidate superset (R::num_candidates / R::candidate, e.g. go: empty non-ko points
// + pass) together with R::play_candidate, which applies the candidate or reports it illegal: a uniformly drawn
// candidate is kept iff legal (rejection sampling = uniform over the legal actions); retry q draws at ply + 4096 q.
// Otherwise the action is the k-th set bit of the legal mask.  `draw(b, n)` returns a uniform integer in [0, n).
template <class R, class S, class Cfg, class Draw>
__device__ __forceinline__ auto playout_step_impl(S& s, const Cfg& c, const Ctx& ctx, long long lane, int /*mask_words*/,
                                                  Draw& draw, u32 ply, int) -> decltype(R::num_candidates(s, c)) {
  int n = R::num_candidates(s, c);
  for (u32 retry = 0;; ++retry) {
    int a = R::candidate(s, c, (int)draw(ply + 4096u * retry, (u32)n));
    if (R::play_candidate(s, a, c, ctx, lane)) return a;
  }
}
template <class R, class S, class Cfg, class Draw>
__device__ __forceinline__ int playout_step_impl(S& s, const Cfg& c, const Ctx& ctx, long long lane, int mask_words,
                                                 Draw& draw, u32 ply, long) {
  u32 m[R::kMaskWords];
  R::legal_nonterminal(s, c, m);
  int cnt = 0;
  for (int w = 0; w < mask_words; ++w) cnt += __popc(m[w]);
  int a = nth_set_bit(m, mask_words, (int)draw(ply, (u32)cnt));
  apply_known_legal<R>(s, a, c, ctx, lane);
  return a;
}
template <class R, class S, class Cfg, class Draw>
__device__ __forceinline__ int playout_step(S& s, const Cfg& c, const Ctx& ctx, long long lane, int mask_words, Draw& draw, u32 ply) {
  return playout_step_impl<R>(s, c, ctx, lane, mask_words, draw, ply, 0);
}

// ---- 128-bit bitboards (hex: up to 121 cells; go: 9 rows x 10-bit stride) ------------------------------------
struct B128 {
  u64 lo, hi;
};
__host__ __device__ __forceinline__ B128 b_and(B128 a, B128 b) { return {a.lo & b.lo, a.hi & b.hi}; }
__host__ __device__ __forceinline__ B128 b_or(B128 a, B128 b) { return {a.lo | b.lo, a.hi | b.hi}; }
__host__ __device__ __forceinline__ B128 b_andn(B128 a, B128 b) { return {a.lo & ~b.lo, a.hi & ~b.hi}; }   // a & ~b
__host__ __device__ __forceinline__ bool b_any(B128 a) { return (a.lo | a.hi) != 0; }
__host__ __device__ __forceinline__ B128 b_shl(B128 a, int s) {   // 0 < s < 64
  return {a.lo << s, (a.hi << s) | (a.lo >> (64 - s))};
}
__host__ __device__ __forceinline__ B128 b_shr(B128 a, int s) {
  return {(a.lo >> s) | (a.hi << (64 - s)), a.hi >> s};
}
__host__ __device__ __forceinline__ B128 b_bit(int i) { return i < 64 ? B128{1ull << i, 0} : B128{0, 1ull << (i - 64)}; }
__host__ __device__ __forceinline__ bool b_test(B128 a, int i) { return i < 64 ? (a.lo >> i) & 1ull : (a.hi >> (i - 64)) & 1ull; }
__device__ __forceinline__ int b_popc(B128 a) { return __popcll(a.lo) + __popcll(a.hi); }
// position of the k-th (0-based) set bit; k < popcount
__device__ __forceinline__ int b_select(B128 a, int k) {
  int c0 = __popc((u32)a.lo), c1 = __popc((u32)(a.lo >> 32)), c2 = __popc((u32)a.hi);
  if (k < c0) return (int)__fns((u32)a.lo, 0, k + 1);
  k -= c0;
  if (k < c1) return 32 + (int)__fns((u32)(a.lo >> 32), 0, k + 1);
  k -= c1;
  if (k < c2) return 64 + (int)__fns((u32)a.hi, 0, k + 1);
  k -= c2;
  return 96 + (int)__fns((u32)(a.hi >> 32), 0, k + 1);
}
__device__ __forceinline__ int b_ffs(B128 a) { return a.lo ? __ffsll((long long)a.lo) - 1 : 64 + __ffsll((long long)a.hi) - 1; }

// ---- 256-bit bitboards (mnk: 15 rows x 16-bit stride; havannah: up to 15 x 15 cells) ---------------------------------
struct B256 {
  u64 w[4];
};
__host__ __device__ __forceinline__ B256 q_and(B256 a, B256 b) { return {{a.w[0] & b.w[0], a.w[1] & b.w[1], a.w[2] & b.w[2], a.w[3] & b.w[3]}}; }
__host__ __device__ __forceinline__ B256 q_or(B256 a, B256 b) { return {{a.w[0] | b.w[0], a.w[1] | b.w[1], a.w[2] | b.w[2], a.w[3] | b.w[3]}}; }
__host__ __device__ __forceinline__ B256 q_andn(B256 a, B256 b) { return {{a.w[0] & ~b.w[0], a.w[1] & ~b.w[1], a.w[2] & ~b.w[2], a.w[3] & ~b.w[3]}}; }   // a & ~b
__host__ __device__ __forceinline__ bool q_any(B256 a) { return (a.w[0] | a.w[1] | a.w[2] | a.w[3]) != 0; }
__host__ __device__ __forceinline__ B256 q_shr(B256 a, int s) {          // 0 < s < 256
  const int ws = s >> 6, bs = s & 63;
  B256 r;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int j = i + ws;
    u64 lo = j < 4 ? a.w[j] : 0ull, hi = j + 1 < 4 ? a.w[j + 1] : 0ull;
    r.w[i] = bs ? (lo >> bs) | (hi << (64 - bs)) : lo;
  }
  return r;
}
__host__ __device__ __forceinline__ B256 q_shl(B256 a, int s) {          // 0 < s < 64
  return {{a.w[0] << s, (a.w[1] << s) | (a.w[0] >> (64 - s)), (a.w[2] << s) | (a.w[1] >> (64 - s)), (a.w[3] << s) | (a.w[2] >> (64 - s))}};
}
__host__ __device__ __forceinline__ bool q_test(const B256& a, int i) { return (a.w[i >> 6] >> (i & 63)) & 1ull; }
__host__ __device__ __forceinline__ void q_set(B256& a, int i) { a.w[i >> 6] |= 1ull << (i & 63); }
__host__ __device__ __forceinline__ void q_clear(B256& a, int i) { a.w[i >> 6] &= ~(1ull << (i & 63)); }
__device__ __forceinline__ int q_popc(const B256& a) { return __popcll(a.w[0]) + __popcll(a.w[1]) + __popcll(a.w[2]) + __popcll(a.w[3]); }

}  // namespace b2s
