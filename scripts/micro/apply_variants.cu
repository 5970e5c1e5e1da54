// Microbenchmark (development tool, not part of the library): connect_four ApplyAction kernel variants on
// rotating 1M-state batches inside a CUDA graph, to pick ILP / block size / launch attributes: the earlier 16-byte
// two-board lanes ({x, o}), the library's 8-byte lanes and 7-byte lanes in 32-lane tiles (measured, not adopted: DESIGN §3),
// each beside a pure copy kernel that moves the same bytes per lane (the ceiling an ApplyAction of that lane format is judged
// against).
// nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o apply_variants apply_variants.cu
#include <cstdio>
#include <cstdlib>
#include <vector>
#include <cuda_runtime.h>
typedef unsigned long long u64;
#define CK(x) do{cudaError_t e=(x); if(e!=cudaSuccess){printf("ERR %s line %d\n", cudaGetErrorString(e), __LINE__); exit(1);} }while(0)

__device__ __forceinline__ bool has_line(u64 b) {
  u64 m;
  m = b & (b >> 1);  if (m & (m >> 2)) return true;
  m = b & (b >> 7);  if (m & (m >> 14)) return true;
  m = b & (b >> 8);  if (m & (m >> 16)) return true;
  m = b & (b >> 6);  if (m & (m >> 12)) return true;
  return false;
}
__device__ __forceinline__ void step(ulonglong2& s, int a, unsigned long long* err) {
  const u64 TOP = 0x810204081020ull;   // bit col*7+5
  if (a == -1) return;
  u64 occ = s.x | s.y;
  int mover = __popcll(occ) & 1;
  bool term = has_line(mover ? s.x : s.y) || ((occ & TOP) == TOP);
  int base = a * 7;
  if (term || a < 0 || a >= 7 || ((occ >> (base + 5)) & 1)) { atomicAdd(err, 1ull); return; }
  u64 bit = (occ & (0x3full << base)) + (1ull << base);
  if (mover == 0) s.x |= bit; else s.y |= bit;
}

template <int ILP, int BLOCK, bool PDL>
__global__ void __launch_bounds__(BLOCK) k_apply(ulonglong2* st, const int* __restrict__ act, long long n, unsigned long long* err) {
  if (PDL) asm volatile("griddepcontrol.wait;" ::: "memory");
  long long base = (long long)blockIdx.x * (BLOCK * ILP) + threadIdx.x;
  int a[ILP]; ulonglong2 s[ILP];
#pragma unroll
  for (int j = 0; j < ILP; ++j) { long long i = base + (long long)j * BLOCK; a[j] = -1; if (i < n) { a[j] = __ldg(act + i); s[j] = st[i]; } }
  if (PDL) asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
#pragma unroll
  for (int j = 0; j < ILP; ++j) { long long i = base + (long long)j * BLOCK; if (i < n) { step(s[j], a[j], err); st[i] = s[j]; } }
}

// PDL launch WITHOUT griddepcontrol.wait: legal only when the step does not depend on the previous kernel in the stream
// (a different batch whose actions were ready earlier) — the regime of the bench (one batch per step).  Upper bound of
// what removing the grid-wide drain between steps can buy.
template <int ILP, int BLOCK>
__global__ void __launch_bounds__(BLOCK) k_apply_nowait(ulonglong2* st, const int* __restrict__ act, long long n, unsigned long long* err) {
  long long base = (long long)blockIdx.x * (BLOCK * ILP) + threadIdx.x;
  int a[ILP]; ulonglong2 s[ILP];
#pragma unroll
  for (int j = 0; j < ILP; ++j) { long long i = base + (long long)j * BLOCK; a[j] = -1; if (i < n) { a[j] = __ldg(act + i); s[j] = st[i]; } }
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
#pragma unroll
  for (int j = 0; j < ILP; ++j) { long long i = base + (long long)j * BLOCK; if (i < n) { step(s[j], a[j], err); st[i] = s[j]; } }
}

// Per-tile dependency for steps on the SAME batch: CTA b of step e waits until CTA b of step e-1 has released its tile
// (flags[b] == e), instead of waiting for the whole previous grid.  flags must be zero before step 0.
template <int ILP, int BLOCK>
__global__ void __launch_bounds__(BLOCK) k_apply_tileflags(ulonglong2* st, const int* __restrict__ act, long long n, unsigned long long* err,
                                                            unsigned* flags, unsigned epoch) {
  if (threadIdx.x == 0) {
    unsigned v;
    do { asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(flags + blockIdx.x) : "memory"); } while (v != epoch);
  }
  __syncthreads();
  long long base = (long long)blockIdx.x * (BLOCK * ILP) + threadIdx.x;
  int a[ILP]; ulonglong2 s[ILP];
#pragma unroll
  for (int j = 0; j < ILP; ++j) { long long i = base + (long long)j * BLOCK; a[j] = -1; if (i < n) { a[j] = __ldg(act + i); s[j] = st[i]; } }
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
#pragma unroll
  for (int j = 0; j < ILP; ++j) { long long i = base + (long long)j * BLOCK; if (i < n) { step(s[j], a[j], err); st[i] = s[j]; } }
  __syncthreads();
  if (threadIdx.x == 0) { __threadfence(); asm volatile("st.release.gpu.global.u32 [%0], %1;" :: "l"(flags + blockIdx.x), "r"(epoch + 1) : "memory"); }
}

// persistent grid-stride variant
template <int ILP, int BLOCK>
__global__ void __launch_bounds__(BLOCK) k_apply_gs(ulonglong2* st, const int* __restrict__ act, long long n, unsigned long long* err) {
  long long stride = (long long)gridDim.x * BLOCK * ILP;
  for (long long base = (long long)blockIdx.x * (BLOCK * ILP) + threadIdx.x; base < n; base += stride) {
    int a[ILP]; ulonglong2 s[ILP];
#pragma unroll
    for (int j = 0; j < ILP; ++j) { long long i = base + (long long)j * BLOCK; a[j] = -1; if (i < n) { a[j] = __ldg(act + i); s[j] = st[i]; } }
#pragma unroll
    for (int j = 0; j < ILP; ++j) { long long i = base + (long long)j * BLOCK; if (i < n) { step(s[j], a[j], err); st[i] = s[j]; } }
  }
}

// ---- 8-byte lanes: the library's connect_four layout (rules_connect_four.cuh) at the default 6x7 ------------------------
// key = x | (occ + BOTTOM): below a marker bit at its height, every column holds who owns each stone (1 = x); the cached
// outcome sits in bits 62-63 as outcome ^ 2 (0 = game running).
constexpr u64 BOTTOM = 0x40810204081ull;                                  // bit col*7
constexpr u64 L1 = BOTTOM * 0x3f, L2 = BOTTOM * 0x1f, L4 = BOTTOM * 0x7;   // in-column rows < 6, < 5, < 3
// MS: bit of the cached outcome (62: 8-byte key, 54: 7-byte key)
template <int MS = 62>
__device__ __forceinline__ bool step8(u64& key, int a, unsigned long long* err) {
  if (a == -1) return false;
  u64 s = key;
  s |= (s >> 1) & L1; s |= (s >> 2) & L2; s |= (s >> 4) & L4;          // every column filled up to its marker
  const u64 occ = (s >> 1) & L1;
  u64 x = key & occ, o = occ & ~key;
  if ((key >> MS) || a < 0 || a >= 7 || ((occ >> (a * 7 + 5)) & 1)) { atomicAdd(err, 1ull); return false; }
  const u64 bit = (occ & (0x3full << (a * 7))) + (1ull << (a * 7));
  const int mover = __popcll(occ) & 1;
  const u64 mine = (mover ? o : x) | bit;
  if (mover == 0) x = mine; else o = mine;
  const int oc = has_line(mine) ? mover : (((occ | bit) & (BOTTOM << 5)) == (BOTTOM << 5) ? 3 : 2);
  key = x | ((x | o) + BOTTOM) | ((u64)(oc ^ 2) << MS);
  return true;
}

// one lane per 8-byte load, ILP lanes per thread (block-strided), MINB = __launch_bounds__ min blocks per SM
template <int ILP, int BLOCK, int MINB>
__global__ void __launch_bounds__(BLOCK, MINB) k_apply8(u64* st, const int* __restrict__ act, long long n, unsigned long long* err) {
  asm volatile("griddepcontrol.wait;" ::: "memory");
  long long base = (long long)blockIdx.x * (BLOCK * ILP) + threadIdx.x;
  int a[ILP]; u64 s[ILP];
#pragma unroll
  for (int j = 0; j < ILP; ++j) { long long i = base + (long long)j * BLOCK; a[j] = -1; if (i < n) { a[j] = __ldg(act + i); s[j] = st[i]; } }
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
#pragma unroll
  for (int j = 0; j < ILP; ++j) { long long i = base + (long long)j * BLOCK; if (step8(s[j], a[j], err)) st[i] = s[j]; }
}

// two adjacent lanes per thread: one 16-byte state load / store and one 8-byte action load (n even)
template <int ILP, int BLOCK, int MINB>
__global__ void __launch_bounds__(BLOCK, MINB) k_apply8_pair(u64* st, const int* __restrict__ act, long long n, unsigned long long* err) {
  asm volatile("griddepcontrol.wait;" ::: "memory");
  long long base = (long long)blockIdx.x * (BLOCK * ILP) + threadIdx.x;
  int2 a[ILP]; ulonglong2 s[ILP];
#pragma unroll
  for (int j = 0; j < ILP; ++j) {
    long long p = base + (long long)j * BLOCK;
    a[j] = make_int2(-1, -1);
    if (p < n / 2) { a[j] = __ldg(reinterpret_cast<const int2*>(act) + p); s[j] = reinterpret_cast<const ulonglong2*>(st)[p]; }
  }
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
#pragma unroll
  for (int j = 0; j < ILP; ++j) {
    long long p = base + (long long)j * BLOCK;
    bool w0 = step8(s[j].x, a[j].x, err), w1 = step8(s[j].y, a[j].y, err);
    if (w0 || w1) reinterpret_cast<ulonglong2*>(st)[p] = s[j];
  }
}

// 7-byte keys in 32-lane tiles (common.cuh LaneTiles<4, 2, 1>): bytes 0-3 of the tile's 32 lanes, then bytes 4-5, then byte
// 6, 224 B per tile; the lanes of thread j are 8 j tiles past its first lane, at the same slot
__device__ __forceinline__ u64 tile7_get(const unsigned char* t, int slot) {
  return (u64)reinterpret_cast<const unsigned*>(t)[slot] | (u64)reinterpret_cast<const unsigned short*>(t + 128)[slot] << 32 |
         (u64)t[192 + slot] << 48;
}
__device__ __forceinline__ void tile7_set(unsigned char* t, int slot, u64 key) {
  reinterpret_cast<unsigned*>(t)[slot] = (unsigned)key;
  reinterpret_cast<unsigned short*>(t + 128)[slot] = (unsigned short)(key >> 32);
  t[192 + slot] = (unsigned char)(key >> 48);
}
template <int ILP, int BLOCK, int MINB>
__global__ void __launch_bounds__(BLOCK, MINB) k_apply7(unsigned char* st, const int* __restrict__ act, long long n, unsigned long long* err) {
  asm volatile("griddepcontrol.wait;" ::: "memory");
  long long base = (long long)blockIdx.x * (BLOCK * ILP) + threadIdx.x;
  unsigned char* t0 = st + (base >> 5) * 224;
  const int slot = threadIdx.x & 31;
  int a[ILP]; u64 s[ILP];
#pragma unroll
  for (int j = 0; j < ILP; ++j) { long long i = base + (long long)j * BLOCK; a[j] = -1; if (i < n) { a[j] = __ldg(act + i); s[j] = tile7_get(t0 + j * (BLOCK / 32) * 224, slot); } }
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
#pragma unroll
  for (int j = 0; j < ILP; ++j) if (step8<54>(s[j], a[j], err)) tile7_set(t0 + j * (BLOCK / 32) * 224, slot, s[j]);
}

// pure copies of the same traffic: lane state in, action in, state + action out (no game logic) — 8-byte lanes: 12 R / 8 W
// = 20 B, 7-byte tiled lanes: 11 R / 7 W = 18 B
template <int ILP, int BLOCK, int MINB>
__global__ void __launch_bounds__(BLOCK, MINB) k_copy8(u64* st, const int* __restrict__ act, long long n, unsigned long long*) {
  asm volatile("griddepcontrol.wait;" ::: "memory");
  long long base = (long long)blockIdx.x * (BLOCK * ILP) + threadIdx.x;
  int a[ILP]; u64 s[ILP];
#pragma unroll
  for (int j = 0; j < ILP; ++j) { long long i = base + (long long)j * BLOCK; a[j] = -1; if (i < n) { a[j] = __ldg(act + i); s[j] = st[i]; } }
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
#pragma unroll
  for (int j = 0; j < ILP; ++j) { long long i = base + (long long)j * BLOCK; if (a[j] != -1) st[i] = s[j] + (u64)a[j]; }
}
template <int ILP, int BLOCK, int MINB>
__global__ void __launch_bounds__(BLOCK, MINB) k_copy7(unsigned char* st, const int* __restrict__ act, long long n, unsigned long long*) {
  asm volatile("griddepcontrol.wait;" ::: "memory");
  long long base = (long long)blockIdx.x * (BLOCK * ILP) + threadIdx.x;
  unsigned char* t0 = st + (base >> 5) * 224;
  const int slot = threadIdx.x & 31;
  int a[ILP]; u64 s[ILP];
#pragma unroll
  for (int j = 0; j < ILP; ++j) { long long i = base + (long long)j * BLOCK; a[j] = -1; if (i < n) { a[j] = __ldg(act + i); s[j] = tile7_get(t0 + j * (BLOCK / 32) * 224, slot); } }
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
#pragma unroll
  for (int j = 0; j < ILP; ++j) if (a[j] != -1) tile7_set(t0 + j * (BLOCK / 32) * 224, slot, s[j] + (u64)a[j]);
}

template <int ILP, int BLOCK, int MINB, int KIND>   // KIND 2: apply7, 3: copy8, 4: copy7
void launch_k(void* st, const int* act, long long n, unsigned long long* err, cudaStream_t s) {
  unsigned grid = (unsigned)((n + (long long)BLOCK * ILP - 1) / ((long long)BLOCK * ILP));
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(grid); cfg.blockDim = dim3(BLOCK); cfg.stream = s;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization; at[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = at; cfg.numAttrs = 1;
  if (KIND == 2) CK(cudaLaunchKernelEx(&cfg, k_apply7<ILP, BLOCK, MINB>, (unsigned char*)st, act, n, err));
  else if (KIND == 3) CK(cudaLaunchKernelEx(&cfg, k_copy8<ILP, BLOCK, MINB>, (u64*)st, act, n, err));
  else CK(cudaLaunchKernelEx(&cfg, k_copy7<ILP, BLOCK, MINB>, (unsigned char*)st, act, n, err));
}

template <int ILP, int BLOCK, int MINB, bool PAIR>
void launch8(void* st, const int* act, long long n, unsigned long long* err, cudaStream_t s) {
  long long units = PAIR ? n / 2 : n;
  unsigned grid = (unsigned)((units + (long long)BLOCK * ILP - 1) / ((long long)BLOCK * ILP));
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(grid); cfg.blockDim = dim3(BLOCK); cfg.stream = s;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization; at[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = at; cfg.numAttrs = 1;
  if (PAIR) CK(cudaLaunchKernelEx(&cfg, k_apply8_pair<ILP, BLOCK, MINB>, (u64*)st, act, n, err));
  else CK(cudaLaunchKernelEx(&cfg, k_apply8<ILP, BLOCK, MINB>, (u64*)st, act, n, err));
}

struct Variant { const char* name; void (*launch)(ulonglong2*, const int*, long long, unsigned long long*, cudaStream_t); };
struct Variant8 { const char* name; void (*launch)(void*, const int*, long long, unsigned long long*, cudaStream_t); double bytes = 20; };

template <int ILP, int BLOCK, bool PDL>
void launch_v(ulonglong2* st, const int* act, long long n, unsigned long long* err, cudaStream_t s) {
  unsigned grid = (unsigned)((n + (long long)BLOCK * ILP - 1) / ((long long)BLOCK * ILP));
  if (!PDL) { k_apply<ILP, BLOCK, false><<<grid, BLOCK, 0, s>>>(st, act, n, err); return; }
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(grid); cfg.blockDim = dim3(BLOCK); cfg.stream = s;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization; at[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = at; cfg.numAttrs = 1;
  CK(cudaLaunchKernelEx(&cfg, k_apply<ILP, BLOCK, true>, st, act, n, err));
}
template <int ILP, int BLOCK>
void launch_nowait(ulonglong2* st, const int* act, long long n, unsigned long long* err, cudaStream_t s) {
  unsigned grid = (unsigned)((n + (long long)BLOCK * ILP - 1) / ((long long)BLOCK * ILP));
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(grid); cfg.blockDim = dim3(BLOCK); cfg.stream = s;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization; at[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = at; cfg.numAttrs = 1;
  CK(cudaLaunchKernelEx(&cfg, k_apply_nowait<ILP, BLOCK>, st, act, n, err));
}
static int g_sms = 0;   // SMs of the device (132 on an H100 SXM), read in main
template <int ILP, int BLOCK, int BPS>
void launch_gs(ulonglong2* st, const int* act, long long n, unsigned long long* err, cudaStream_t s) {
  k_apply_gs<ILP, BLOCK><<<g_sms * BPS, BLOCK, 0, s>>>(st, act, n, err);
}

int main(int argc, char** argv) {
  long long n = argc > 1 ? atoll(argv[1]) : (1 << 20);
  int K = argc > 2 ? atoi(argv[2]) : 200;
  int slots = K + 10;
  std::vector<ulonglong2*> st(slots); std::vector<int*> act(slots);
  unsigned long long* err; CK(cudaMalloc(&err, 8)); CK(cudaMemset(err, 0, 8));
  std::vector<int> ha(n); for (long long i = 0; i < n; ++i) ha[i] = (int)((i * 2654435761u >> 7) % 7);
  for (int k = 0; k < slots; ++k) {
    CK(cudaMalloc(&st[k], n * 16)); CK(cudaMalloc(&act[k], n * 4));
    CK(cudaMemcpy(act[k], ha.data(), n * 4, cudaMemcpyHostToDevice));
  }
  Variant vs[] = {
    {"ilp1_b256", launch_v<1, 256, false>}, {"ilp2_b256", launch_v<2, 256, false>}, {"ilp4_b256", launch_v<4, 256, false>},
    {"ilp8_b256", launch_v<8, 256, false>}, {"ilp4_b128", launch_v<4, 128, false>}, {"ilp8_b128", launch_v<8, 128, false>},
    {"ilp4_b512", launch_v<4, 512, false>}, {"ilp2_b1024", launch_v<2, 1024, false>},
    {"ilp4_b256_pdl", launch_v<4, 256, true>}, {"ilp8_b256_pdl", launch_v<8, 256, true>}, {"ilp2_b256_pdl", launch_v<2, 256, true>},
    {"ilp8_b128_pdl", launch_v<8, 128, true>},
    {"ilp4_b256_pdl_nowait", launch_nowait<4, 256>}, {"ilp2_b256_pdl_nowait", launch_nowait<2, 256>},
    {"gs_ilp4_b256_x4", launch_gs<4, 256, 4>}, {"gs_ilp4_b256_x8", launch_gs<4, 256, 8>}, {"gs_ilp2_b256_x8", launch_gs<2, 256, 8>},
    {"gs_ilp4_b512_x4", launch_gs<4, 512, 4>}, {"gs_ilp1_b256_x8", launch_gs<1, 256, 8>}, {"gs_ilp2_b1024_x2", launch_gs<2, 1024, 2>},
  };
  CK(cudaDeviceGetAttribute(&g_sms, cudaDevAttrMultiProcessorCount, 0));
  cudaStream_t s; CK(cudaStreamCreate(&s));
  cudaEvent_t e0, e1; CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
  for (auto& v : vs) {
    for (int k = 0; k < slots; ++k) CK(cudaMemsetAsync(st[k], 0, n * 16, s));
    cudaGraph_t g; cudaGraphExec_t ge;
    CK(cudaStreamBeginCapture(s, cudaStreamCaptureModeGlobal));
    for (int k = 10; k < slots; ++k) v.launch(st[k], act[k], n, err, s);
    CK(cudaStreamEndCapture(s, &g)); CK(cudaGraphInstantiate(&ge, g, 0));
    for (int k = 0; k < 10; ++k) v.launch(st[k], act[k], n, err, s);
    float best = 1e9;
    for (int rep = 0; rep < 3; ++rep) {
      CK(cudaStreamSynchronize(s));
      CK(cudaEventRecord(e0, s)); CK(cudaGraphLaunch(ge, s)); CK(cudaEventRecord(e1, s));
      CK(cudaStreamSynchronize(s));
      float ms; CK(cudaEventElapsedTime(&ms, e0, e1)); if (ms < best) best = ms;
    }
    double us = best * 1e3 / K;
    printf("%-20s n=%lld  %.2f us/step  %.1f GB/s (36 B/step)  %.3e steps/s\n", v.name, n, us, 36.0 * n / us / 1e3, n / us * 1e6);
    CK(cudaGraphExecDestroy(ge)); CK(cudaGraphDestroy(g));
  }
  // ---- 8-byte lanes, the K steps captured as one chain and as two parallel chains (step k on chain k mod 2, as bench.py) --
  Variant8 v8[] = {
    {"c8_ilp4_b256_m6", launch8<4, 256, 6, false>}, {"c8_ilp8_b256_m1", launch8<8, 256, 1, false>},
    {"c8_ilp8_b256_m4", launch8<8, 256, 4, false>}, {"c8_ilp8_b256_m6", launch8<8, 256, 6, false>},
    {"c8_ilp16_b256_m1", launch8<16, 256, 1, false>}, {"c8_ilp8_b128_m1", launch8<8, 128, 1, false>},
    {"c8_ilp4_b512_m1", launch8<4, 512, 1, false>},
    {"c8_pair2_b256_m6", launch8<2, 256, 6, true>}, {"c8_pair4_b256_m1", launch8<4, 256, 1, true>},
    {"c8_pair4_b256_m6", launch8<4, 256, 6, true>},
    {"copy8_ilp4_b256_m6", launch_k<4, 256, 6, 3>, 20},
    {"c7_ilp4_b256_m6", launch_k<4, 256, 6, 2>, 18}, {"copy7_ilp4_b256_m6", launch_k<4, 256, 6, 4>, 18},
  };
  cudaStream_t s2; CK(cudaStreamCreate(&s2));
  cudaEvent_t fork, join; CK(cudaEventCreateWithFlags(&fork, cudaEventDisableTiming)); CK(cudaEventCreateWithFlags(&join, cudaEventDisableTiming));
  for (int chains = 1; chains <= 2; ++chains) {
    for (auto& v : v8) {
      for (int k = 0; k < slots; ++k) CK(cudaMemsetAsync(st[k], 0, n * 8, s));    // all-zero keys decode to the empty board (n * 8 bytes hold n tiled 7-byte lanes for n % 32 == 0)
      cudaGraph_t g; cudaGraphExec_t ge;
      CK(cudaStreamBeginCapture(s, cudaStreamCaptureModeGlobal));
      if (chains == 2) { CK(cudaEventRecord(fork, s)); CK(cudaStreamWaitEvent(s2, fork, 0)); }
      for (int k = 10; k < slots; ++k) v.launch(st[k], act[k], n, err, (chains == 2 && (k & 1)) ? s2 : s);
      if (chains == 2) { CK(cudaEventRecord(join, s2)); CK(cudaStreamWaitEvent(s, join, 0)); }
      CK(cudaStreamEndCapture(s, &g)); CK(cudaGraphInstantiate(&ge, g, 0));
      for (int k = 0; k < 10; ++k) v.launch(st[k], act[k], n, err, s);
      float best = 1e9;
      for (int rep = 0; rep < 3; ++rep) {
        CK(cudaStreamSynchronize(s));
        CK(cudaEventRecord(e0, s)); CK(cudaGraphLaunch(ge, s)); CK(cudaEventRecord(e1, s));
        CK(cudaStreamSynchronize(s));
        float ms; CK(cudaEventElapsedTime(&ms, e0, e1)); if (ms < best) best = ms;
      }
      double us = best * 1e3 / K;
      printf("%-20s chains=%d n=%lld  %.2f us/step  %.1f GB/s (%.0f B/step)  %.3e steps/s\n", v.name, chains, n, us, v.bytes * n / us / 1e3, v.bytes, n / us * 1e6);
      CK(cudaGraphExecDestroy(ge)); CK(cudaGraphDestroy(g));
    }
  }
  // ---- dependent steps on ONE large batch (argv[3] lanes, default 16M): grid-wide PDL wait vs per-tile flags ----
  {
    long long nb = argc > 3 ? atoll(argv[3]) : (1 << 24);
    const int steps = 6;                         // connect_four columns hold 6 stones: 6 legal drops of the same column
    ulonglong2 *big, *ref; int* bact; unsigned* flags;
    CK(cudaMalloc(&big, nb * 16)); CK(cudaMalloc(&ref, nb * 16)); CK(cudaMalloc(&bact, nb * 4));
    std::vector<int> hb(nb); for (long long i = 0; i < nb; ++i) hb[i] = (int)((i * 2654435761u >> 7) % 7);
    CK(cudaMemcpy(bact, hb.data(), nb * 4, cudaMemcpyHostToDevice));
    unsigned grid = (unsigned)((nb + 1023) / 1024);
    CK(cudaMalloc(&flags, 4 * grid));
    auto run = [&](int mode, ulonglong2* dst) {
      CK(cudaMemsetAsync(dst, 0, nb * 16, s)); CK(cudaMemsetAsync(flags, 0, 4 * grid, s)); CK(cudaStreamSynchronize(s));
      CK(cudaEventRecord(e0, s));
      for (int ep = 0; ep < steps; ++ep) {
        cudaLaunchConfig_t cfg = {};
        cfg.gridDim = dim3(grid); cfg.blockDim = dim3(256); cfg.stream = s;
        cudaLaunchAttribute at[1];
        at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization; at[0].val.programmaticStreamSerializationAllowed = 1;
        cfg.attrs = at; cfg.numAttrs = 1;
        if (mode == 0) CK(cudaLaunchKernelEx(&cfg, k_apply<4, 256, true>, dst, (const int*)bact, nb, err));
        else CK(cudaLaunchKernelEx(&cfg, k_apply_tileflags<4, 256>, dst, (const int*)bact, nb, err, flags, (unsigned)ep));
      }
      CK(cudaEventRecord(e1, s)); CK(cudaStreamSynchronize(s));
      float ms; CK(cudaEventElapsedTime(&ms, e0, e1));
      return ms * 1e3 / steps;
    };
    run(0, ref); run(1, big);
    double us0 = run(0, ref), us1 = run(1, big);
    std::vector<ulonglong2> h0(1 << 16), h1(1 << 16);
    CK(cudaMemcpy(h0.data(), ref + (nb / 2), h0.size() * 16, cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(h1.data(), big + (nb / 2), h1.size() * 16, cudaMemcpyDeviceToHost));
    long bad = 0; for (size_t i = 0; i < h0.size(); ++i) bad += (h0[i].x != h1[i].x || h0[i].y != h1[i].y);
    printf("dependent steps, one batch of %lld lanes: pdl+grid wait %.2f us/step (%.1f GB/s), per-tile flags %.2f us/step (%.1f GB/s), mismatching lanes %ld\n",
           nb, us0, 36.0 * nb / us0 / 1e3, us1, 36.0 * nb / us1 / 1e3, bad);
  }
  unsigned long long herr; CK(cudaMemcpy(&herr, err, 8, cudaMemcpyDeviceToHost)); printf("err lanes (expected >0 after repeated reps): %llu\n", herr);
  return 0;
}
