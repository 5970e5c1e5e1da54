// Host definitions of the few device intrinsics the per-game rule cores (rules_*.cuh) and mcts.cuh use, so that the SAME
// rule-core source the sm_90a kernels are built from also compiles with a plain host compiler (g++ + CUDA's
// cuda_runtime.h, whose host_defines.h makes __device__ / __forceinline__ harmless).
// Users: (1) open_spiel_b200/adapter/host_rules.cc — the scalar open_spiel::State adapter (SURVEY §8b: "scalar State
// methods run the same __host__ __device__ rule core on the CPU"); one State is one object, never a batch: every
// batched entry point lives in libb2s.so and is GPU-only; (2) tests/host_emul (CPU unit tests of the rule cores).
// Include this BEFORE common.cuh / rules_*.cuh, from host translation units only.
#pragma once
#ifdef __CUDACC__
#error "host_compat.h is for host compilers only (the device build uses the real intrinsics)"
#endif
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>

static inline int __popc(unsigned x) { return __builtin_popcount(x); }
static inline int __popcll(unsigned long long x) { return __builtin_popcountll(x); }
static inline int __ffs(int x) { return __builtin_ffs(x); }
static inline int __ffsll(long long x) { return __builtin_ffsll(x); }
// __fns(mask, base, offset > 0): position of the offset-th set bit of mask counting upwards from bit `base`
static inline unsigned __fns(unsigned mask, unsigned base, int offset) {
  for (unsigned b = base; b < 32; ++b)
    if ((mask >> b) & 1u) { if (--offset == 0) return b; }
  return 0xffffffffu;
}
static inline unsigned __funnelshift_r(unsigned lo, unsigned hi, unsigned sh) {
  unsigned long long v = ((unsigned long long)hi << 32) | lo;
  return (unsigned)(v >> (sh & 31));
}
// PRMT: result byte i = byte (selector nibble i) of the 8 bytes {x, y}; selector values 0-7 only (no sign replication)
static inline unsigned __byte_perm(unsigned x, unsigned y, unsigned sel) {
  const unsigned long long v = ((unsigned long long)y << 32) | x;
  unsigned r = 0;
  for (int i = 0; i < 4; ++i) r |= (unsigned)((v >> (8 * ((sel >> (4 * i)) & 7u))) & 0xffull) << (8 * i);
  return r;
}
template <typename T> static inline T __ldg(const T* p) { return *p; }
static inline unsigned long long atomicAdd(unsigned long long* p, unsigned long long v) { unsigned long long o = *p; *p += v; return o; }
static inline long long atomicMin(long long* p, long long v) { long long o = *p; if (v < o) *p = v; return o; }
// explicitly rounded FP64 operations (x86-64 g++ does not contract a*b+c into an FMA at -O2 without -ffast-math / -march flags)
static inline double __dadd_rn(double a, double b) { return a + b; }
static inline double __dsub_rn(double a, double b) { return a - b; }
static inline double __dmul_rn(double a, double b) { return a * b; }
static inline double __ddiv_rn(double a, double b) { return a / b; }
static inline double __dsqrt_rn(double a) { return __builtin_sqrt(a); }
static inline double __longlong_as_double(long long v) { double d; memcpy(&d, &v, 8); return d; }
static inline float __int_as_float(int v) { float f; memcpy(&f, &v, 4); return f; }
#define __launch_bounds__(...)
// GoRules::device_init uploads its Zobrist table with cudaMemcpyToSymbol; on the host the "symbol" is a plain array
#define cudaMemcpyToSymbol(sym, src, size) (memcpy((void*)&(sym), (src), (size)), cudaSuccess)
