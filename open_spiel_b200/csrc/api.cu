// extern "C" layer (include/b2s.h) over the per-game kernel tables.  Host logic only: argument checks,
// buffer ownership, stream plumbing.  No CPU fallback anywhere: without a CUDA device every call fails.
#include <ctype.h>
#include <math.h>
#include <sched.h>
#include <stdlib.h>
#include <stdio.h>
#include <string.h>

#include <mutex>
#include <string>
#include <vector>

#include "batch_kernels.cuh"
#include "errors.h"

namespace b2s {

long long g_launches = 0;
static thread_local std::string g_err;

int fail(const std::string& m) { g_err = m; return 1; }
int cuda_fail(cudaError_t e, const char* what) {
  g_err = std::string(what) + ": " + cudaGetErrorString(e);
  return 2;
}
#define CU(x) do { cudaError_t _e = (x); if (_e != cudaSuccess) return cuda_fail(_e, #x); } while (0)

constexpr int kMaxDevices = 64;
struct HostPipe {                 // per device: b2s_step_fused_host's upload+kernel stream, download stream, chunk events
  std::mutex mu;
  cudaStream_t hs = nullptr, hs2 = nullptr;
  cudaEvent_t ev[8] = {};
};
static HostPipe g_host_pipe[kMaxDevices];
constexpr int kHostChunks = 8, kHostChunksDefault = 2;   // B2S_HOST_CHUNKS overrides (scripts/e2e_chunks.py measures each)

struct Batch {
  GameOps* ops = nullptr;
  b2s_game_info info;
  long long cap = 0;
  int device = 0;
  void* planes = nullptr;
  u64* hist = nullptr;
  ErrBuf* err = nullptr;
  // staging for the *_host entry points
  int* act_d = nullptr; u32* mask_d = nullptr; unsigned char* term_d = nullptr; float* rets_d = nullptr;
  bool host_ready = false;                       // b2s_step_fused_host staging buffers allocated
  // b2s_step_fused_host*: instantiated CUDA graphs of the chunked upload -> kernel -> download pipeline, one per
  // (host buffers, lane count, entry point) the batch has been stepped with (step_host_impl)
  struct HostGraph {
    const void* actions; void* mask; void* term; void* rets; long long n; int action_bytes, compact;
    cudaGraphExec_t exec; unsigned long long stamp;
  };
  std::vector<HostGraph> host_graphs;
  unsigned long long host_graph_clock = 0;
  // MCTS scratch (b2s_mcts_search): work lanes, log table, node arena
  void* mcts_work = nullptr; u64* mcts_hist = nullptr; long long mcts_work_cap = 0;
  double* mcts_log = nullptr; int mcts_log_n = 0;
  void* mcts_pool = nullptr; unsigned long long mcts_pool_bytes = 0; unsigned long long* mcts_top = nullptr;
  Ctx ctx() const { Ctx c; c.planes = planes; c.cap = cap; c.hist = hist; c.err = err; return c; }
  ~Batch() {
    for (auto& g : host_graphs) if (g.exec) cudaGraphExecDestroy(g.exec);
    if (planes) cudaFree(planes);
    if (hist) cudaFree(hist);
    if (err) cudaFree(err);
    if (act_d) cudaFree(act_d);
    if (mask_d) cudaFree(mask_d);
    if (term_d) cudaFree(term_d);
    if (rets_d) cudaFree(rets_d);
    if (mcts_work) cudaFree(mcts_work);
    if (mcts_hist) cudaFree(mcts_hist);
    if (mcts_log) cudaFree(mcts_log);
    if (mcts_pool) cudaFree(mcts_pool);
    if (mcts_top) cudaFree(mcts_top);
    delete ops;
  }
};

static GameOps* make_ops(int id, const b2s_params* p) {
  switch (id) {
    case B2S_TIC_TAC_TOE: return make_ops_tic_tac_toe();
    case B2S_CONNECT_FOUR: return make_ops_connect_four();
    case B2S_BREAKTHROUGH: return make_ops_breakthrough();
    case B2S_HEX: return make_ops_hex();
    case B2S_GO: return make_ops_go();
    case B2S_KUHN_POKER: return make_ops_kuhn_poker();
    case B2S_MNK: return make_ops_mnk();
    case B2S_OTHELLO: return make_ops_othello();
    case B2S_Y: return make_ops_y();
    case B2S_HAVANNAH: return make_ops_havannah();
    case B2S_LEDUC_POKER: return (p && p->players > 2) ? make_ops_leduc_poker_n() : make_ops_leduc_poker();
  }
  return nullptr;
}

static int check(void* b, long long n) {
  if (!b) return fail("null batch");
  Batch* B = (Batch*)b;
  if (n < 0 || n > B->cap) return fail("n out of range for batch capacity");
  CU(cudaSetDevice(B->device));
  return 0;
}
static int post() {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return cuda_fail(e, "kernel launch");
  return 0;
}

}  // namespace b2s

using namespace b2s;

extern "C" {

const char* b2s_last_error(void) { return g_err.c_str(); }
const char* b2s_version(void) { return "b2s 0.1 (sm_90a)"; }
int64_t b2s_launch_count(void) { return g_launches; }
static int64_t g_host_graph_launches = 0, g_host_zero_copy_steps = 0;
int64_t b2s_host_graph_launches(void) { return g_host_graph_launches; }
int64_t b2s_host_zero_copy_steps(void) { return g_host_zero_copy_steps; }

int b2s_game_id(const char* name) {
  static const char* names[B2S_NUM_GAMES] = {"tic_tac_toe", "connect_four", "breakthrough", "hex", "go",
                                             "kuhn_poker", "leduc_poker", "mnk", "othello", "y", "havannah"};
  if (!name) return -1;
  for (int i = 0; i < B2S_NUM_GAMES; ++i) if (!strcmp(name, names[i])) return i;
  return -1;
}

void b2s_params_default(b2s_params* p) {
  memset(p, 0xff, sizeof *p);          // every int field = -1 ("unset")
  p->komi = NAN;
  for (double& d : p->reserved_d) d = NAN;
}

int b2s_game_info_get(int game_id, const b2s_params* params, b2s_game_info* out) {
  GameOps* ops = make_ops(game_id, params);
  if (!ops) return fail("unsupported game id");
  b2s_params p;
  if (params) p = *params; else b2s_params_default(&p);
  b2s_game_info gi;
  memset(&gi, 0, sizeof gi);
  const char* e = ops->configure(p, gi);
  delete ops;
  if (e) return fail(e);
  *out = gi;
  return 0;
}

// Pin the calling thread (and, by first touch, the pinned buffers it allocates afterwards) to the CPUs of the NUMA node
// the GPU hangs off: /sys/bus/pci/devices/<bus id>/local_cpulist.  Returns 0 and the number of CPUs in *n_cpus.
int b2s_bind_host_to_device(int device, int* n_cpus) {
  char bus[32] = {0};
  CU(cudaDeviceGetPCIBusId(bus, sizeof bus, device));
  for (char* q = bus; *q; ++q) *q = (char)tolower(*q);
  std::string path = std::string("/sys/bus/pci/devices/") + bus + "/local_cpulist";
  FILE* f = fopen(path.c_str(), "r");
  if (!f) return fail("bind: cannot read " + path);
  char line[4096] = {0};
  if (!fgets(line, sizeof line, f)) { fclose(f); return fail("bind: empty " + path); }
  fclose(f);
  cpu_set_t set;
  CPU_ZERO(&set);
  int count = 0;
  for (char* tok = strtok(line, ",\n"); tok; tok = strtok(nullptr, ",\n")) {
    int a = 0, b = 0;
    int k = sscanf(tok, "%d-%d", &a, &b);
    if (k == 1) b = a;
    if (k < 1) continue;
    for (int cpu = a; cpu <= b && cpu < CPU_SETSIZE; ++cpu) { CPU_SET(cpu, &set); ++count; }
  }
  if (count == 0) return fail("bind: no CPUs listed in " + path);
  if (sched_setaffinity(0, sizeof set, &set) != 0) return fail("bind: sched_setaffinity failed");
  if (n_cpus) *n_cpus = count;
  return 0;
}

int b2s_device_count(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
  return n;
}

int b2s_batch_create(int game_id, const b2s_params* params, int64_t capacity, int device, void** out_batch) {
  if (!out_batch) return fail("null out_batch");
  *out_batch = nullptr;
  if (capacity <= 0) return fail("capacity must be positive");
  if (b2s_device_count() <= 0) return fail("no CUDA device: the b2s device path has no CPU fallback");
  GameOps* ops = make_ops(game_id, params);
  if (!ops) return fail("unsupported game id");
  b2s_params p;
  if (params) p = *params; else b2s_params_default(&p);
  Batch* B = new Batch;
  B->ops = ops;
  memset(&B->info, 0, sizeof B->info);
  const char* e = ops->configure(p, B->info);
  if (e) { delete B; return fail(e); }
  B->cap = capacity;
  B->device = device;
  cudaError_t ce = cudaSetDevice(device);
  if (ce != cudaSuccess) { delete B; return cuda_fail(ce, "cudaSetDevice"); }
  ops->device_init();
  ce = cudaGetLastError();                       // e.g. go's Zobrist table upload (cudaMemcpyToSymbol)
  if (ce != cudaSuccess) { delete B; return cuda_fail(ce, "per-game device tables"); }
  size_t bytes = ops->chunk_bytes() * (size_t)ops->chunks() * (size_t)capacity;
  ce = cudaMalloc(&B->planes, bytes);
  if (ce != cudaSuccess) { delete B; return cuda_fail(ce, "cudaMalloc(state planes)"); }
  if (B->info.history_bytes > 0) {
    ce = cudaMalloc((void**)&B->hist, (size_t)B->info.history_bytes * (size_t)capacity);
    if (ce != cudaSuccess) { delete B; return cuda_fail(ce, "cudaMalloc(history)"); }
  }
  ce = cudaMalloc((void**)&B->err, sizeof(ErrBuf));
  if (ce != cudaSuccess) { delete B; return cuda_fail(ce, "cudaMalloc(err)"); }
  ops->reset(B->ctx(), capacity, 0);
  ce = cudaDeviceSynchronize();
  if (ce != cudaSuccess) { delete B; return cuda_fail(ce, "initial reset"); }
  *out_batch = B;
  return 0;
}

void b2s_batch_destroy(void* batch) {
  if (!batch) return;
  Batch* B = (Batch*)batch;
  cudaSetDevice(B->device);
  delete B;
}

int b2s_batch_info(void* batch, b2s_game_info* out) {
  if (!batch || !out) return fail("null argument");
  *out = ((Batch*)batch)->info;
  return 0;
}
int64_t b2s_batch_capacity(void* batch) { return batch ? ((Batch*)batch)->cap : 0; }

int b2s_reset(void* batch, int64_t n, void* stream) {
  if (int r = check(batch, n)) return r;
  Batch* B = (Batch*)batch;
  B->ops->reset(B->ctx(), n, (cudaStream_t)stream);
  return post();
}

int b2s_apply_actions(void* batch, const int32_t* actions_d, int64_t n, void* stream) {
  if (int r = check(batch, n)) return r;
  if (!actions_d) return fail("null actions");
  Batch* B = (Batch*)batch;
  B->ops->apply(B->ctx(), actions_d, n, (cudaStream_t)stream);
  return post();
}

int b2s_legal_mask(void* batch, uint32_t* mask_words_d, int64_t n, void* stream) {
  if (int r = check(batch, n)) return r;
  if (!mask_words_d) return fail("null mask");
  Batch* B = (Batch*)batch;
  B->ops->legal_mask(B->ctx(), mask_words_d, n, (cudaStream_t)stream);
  return post();
}

int b2s_legal_list(void* batch, int16_t* actions_d, int32_t* counts_d, int32_t stride, int64_t n, void* stream) {
  if (int r = check(batch, n)) return r;
  if (!actions_d || !counts_d || stride <= 0) return fail("bad legal_list arguments");
  Batch* B = (Batch*)batch;
  B->ops->legal_list(B->ctx(), actions_d, counts_d, stride, n, (cudaStream_t)stream);
  return post();
}

int b2s_status(void* batch, int8_t* cur_d, uint8_t* term_d, float* rets_d, int64_t n, void* stream) {
  if (int r = check(batch, n)) return r;
  Batch* B = (Batch*)batch;
  B->ops->status(B->ctx(), cur_d, term_d, rets_d, n, (cudaStream_t)stream);
  return post();
}

int b2s_observation(void* batch, int player, float* obs_d, int64_t n, void* stream) {
  if (int r = check(batch, n)) return r;
  Batch* B = (Batch*)batch;
  if (!obs_d) return fail("null obs");
  if ((uintptr_t)obs_d & 3u) return fail("observation: output pointer must be 4-byte aligned");
  if (player >= B->info.num_players) return fail("player out of range");
  const char* e = B->ops->obs(B->ctx(), player, 0, 0, obs_d, n, (cudaStream_t)stream);
  if (e) return fail(e);
  return post();
}

int b2s_information_state(void* batch, int player, float* out_d, int64_t n, void* stream) {
  if (int r = check(batch, n)) return r;
  Batch* B = (Batch*)batch;
  if (!out_d) return fail("null out");
  if ((uintptr_t)out_d & 3u) return fail("information_state: output pointer must be 4-byte aligned");
  if (player >= B->info.num_players) return fail("player out of range");
  const char* e = B->ops->obs(B->ctx(), player, 1, 0, out_d, n, (cudaStream_t)stream);
  if (e) return fail(e);
  return post();
}

int b2s_step_fused(void* batch, const int32_t* actions_d, uint32_t* mask_d, uint8_t* term_d, float* rets_d, int64_t n, void* stream) {
  if (int r = check(batch, n)) return r;
  if (!actions_d) return fail("null actions");
  Batch* B = (Batch*)batch;
  B->ops->step_fused(B->ctx(), actions_d, mask_d, term_d, rets_d, n, (cudaStream_t)stream);
  return post();
}

// Shared body of the *_host step entry points.  compact = 0: int32 actions in, mask words / terminal / float returns out
// (b2s_step_fused_host); compact = 1: `action_bytes`-wide actions in, one status byte (+ optional mask words) out.
constexpr size_t kHostGraphsPerBatch = 4;

// Chunked and double-streamed: the upload + kernel of chunk c+1 (stream hs) overlaps the download of chunk c (stream hs2) —
// PCIe is full duplex, so the step costs about max(H2D, D2H) instead of their sum.  join: hs finally waits for hs2 (needed
// when the sequence is being captured into a graph: every forked stream must rejoin the origin).
static int enqueue_host_step(Batch* B, HostPipe& pipe, const void* actions_h, int action_bytes, uint32_t* mask_h, uint8_t* term_or_status_h,
                             float* rets_h, int64_t n, int compact, int n_chunks, bool join) {
  cudaStream_t st = pipe.hs, st2 = pipe.hs2;
  const size_t W = (size_t)B->info.mask_words, P = (size_t)B->info.num_players, cb = B->ops->chunk_bytes();
  const size_t ab = (size_t)action_bytes;
  const int64_t chunk = n_chunks > 1 ? ((n + n_chunks - 1) / n_chunks + 1023) / 1024 * 1024 : n;
  int c = 0, rc = 0;
  cudaError_t e = cudaSuccess;
  for (int64_t lo = 0; lo < n && !rc; lo += chunk, ++c) {
    const int64_t len = n - lo < chunk ? n - lo : chunk;
    Ctx v = B->ctx();
    v.planes = (char*)v.planes + (size_t)lo * cb;
    if (v.hist) v.hist += lo;
    v.lane0 = lo;
    char* act_d = (char*)B->act_d + (size_t)lo * ab;
    e = cudaMemcpyAsync(act_d, (const char*)actions_h + (size_t)lo * ab, ab * len, cudaMemcpyHostToDevice, st);
    if (e != cudaSuccess) { rc = cuda_fail(e, "step_host: upload"); break; }
    if (compact)
      B->ops->step_compact(v, act_d, action_bytes, B->term_d + lo, mask_h ? B->mask_d + lo * W : nullptr, len, st);
    else
      B->ops->step_fused(v, (const int*)act_d, mask_h ? B->mask_d + lo * W : nullptr, term_or_status_h ? B->term_d + lo : nullptr,
                         rets_h ? B->rets_d + lo * P : nullptr, len, st);
    if ((rc = post())) break;
    cudaEvent_t ev = pipe.ev[c % kHostChunks];
    if ((e = cudaEventRecord(ev, st)) != cudaSuccess || (e = cudaStreamWaitEvent(st2, ev, 0)) != cudaSuccess) { rc = cuda_fail(e, "step_host: event"); break; }
    if (mask_h && (e = cudaMemcpyAsync(mask_h + lo * W, B->mask_d + lo * W, sizeof(u32) * W * len, cudaMemcpyDeviceToHost, st2)) != cudaSuccess) { rc = cuda_fail(e, "step_host: download"); break; }
    if (term_or_status_h && (e = cudaMemcpyAsync(term_or_status_h + lo, B->term_d + lo, len, cudaMemcpyDeviceToHost, st2)) != cudaSuccess) { rc = cuda_fail(e, "step_host: download"); break; }
    if (rets_h && (e = cudaMemcpyAsync(rets_h + lo * P, B->rets_d + lo * P, sizeof(float) * P * len, cudaMemcpyDeviceToHost, st2)) != cudaSuccess) { rc = cuda_fail(e, "step_host: download"); break; }
  }
  if (join && c > 0) {
    cudaEvent_t ev = pipe.ev[c % kHostChunks];
    if ((e = cudaEventRecord(ev, st2)) != cudaSuccess || (e = cudaStreamWaitEvent(st, ev, 0)) != cudaSuccess) { if (!rc) rc = cuda_fail(e, "step_host: join"); }
  }
  return rc;
}

static int step_host_impl(Batch* B, const void* actions_h, int action_bytes, uint32_t* mask_h, uint8_t* term_or_status_h,
                          float* rets_h, int64_t n, int compact) {
  // The two streams and the chunk events are shared by all batches of a device (a fresh stream / event costs tens of
  // microseconds on first use, which a per-batch pair would pay inside the first call on every batch); calls on one
  // device are serialised by the pipe's mutex — they are PCIe-bound anyway.
  if (B->device < 0 || B->device >= kMaxDevices) return fail("device index out of range");
  HostPipe& pipe = g_host_pipe[B->device];
  std::lock_guard<std::mutex> lock(pipe.mu);
  if (!pipe.hs) {
    // BLOCKING streams (cudaStreamDefault): they are implicitly ordered after work already enqueued on the legacy default
    // stream (NULL) — e.g. a b2s_reset / b2s_apply_actions(…, NULL) issued just before — and later NULL-stream work is
    // ordered after them.  Work the caller enqueued on OTHER streams must be synchronised by the caller (b2s.h).
    CU(cudaStreamCreateWithFlags(&pipe.hs, cudaStreamDefault));
    CU(cudaStreamCreateWithFlags(&pipe.hs2, cudaStreamDefault));
    for (int i = 0; i < kHostChunks; ++i) CU(cudaEventCreateWithFlags(&pipe.ev[i], cudaEventDisableTiming));
  }
  if (!B->host_ready) {
    CU(cudaMalloc((void**)&B->act_d, sizeof(int) * B->cap));
    CU(cudaMalloc((void**)&B->mask_d, sizeof(u32) * (size_t)B->info.mask_words * B->cap));
    CU(cudaMalloc((void**)&B->term_d, B->cap));
    CU(cudaMalloc((void**)&B->rets_d, sizeof(float) * (size_t)B->info.num_players * B->cap));
    B->host_ready = true;                        // only once every staging buffer exists
  }
  cudaStream_t st = pipe.hs, st2 = pipe.hs2;
  const size_t W = (size_t)B->info.mask_words, P = (size_t)B->info.num_players;
  const size_t bytes_per_lane = (size_t)action_bytes + (compact ? 1 : (term_or_status_h ? 1 : 0) + (rets_h ? sizeof(float) * P : 0)) + (mask_h ? sizeof(u32) * W : 0);
  static const int env_chunks = [] {               // B2S_HOST_CHUNKS=1..8 overrides the defaults (tuning knob)
    const char* e = getenv("B2S_HOST_CHUNKS");
    int v = e ? atoi(e) : 0;
    return v < 1 ? 0 : (v > kHostChunks ? kHostChunks : v);
  }();
  static const bool graphs_on = [] { const char* e = getenv("B2S_HOST_GRAPH"); return !e || atoi(e) != 0; }();

  // two chunks overlap the upload + kernel of one half with the download of the other; that only pays when the copies
  // are long compared with the fixed DMA set-up cost of a copy: below ~4 MiB of traffic the call runs as one chunk
  const int n_chunks = env_chunks ? env_chunks : kHostChunksDefault;
  const bool split = n_chunks > 1 && n >= (1 << 18) && (env_chunks || bytes_per_lane * (size_t)n >= (4u << 20));
  const int chunks = split ? n_chunks : 1;

  // ---- zero-copy path (byte-wide entry, pinned + device-mapped buffers): no DMA copies at all, see k_step_compact_zc ----------
  static const bool zero_copy_on = [] { const char* e = getenv("B2S_HOST_ZEROCOPY"); return !e || atoi(e) != 0; }();
  if (zero_copy_on && compact && action_bytes == 1 && !mask_h && n >= (1 << 12) &&
      ((uintptr_t)actions_h & 15) == 0 && ((uintptr_t)term_or_status_h & 15) == 0) {
    void *a_dev = nullptr, *s_dev = nullptr;
    cudaPointerAttributes pa, ps;
    if (cudaPointerGetAttributes(&pa, actions_h) == cudaSuccess && cudaPointerGetAttributes(&ps, term_or_status_h) == cudaSuccess &&
        pa.type == cudaMemoryTypeHost && ps.type == cudaMemoryTypeHost && pa.devicePointer && ps.devicePointer) {
      a_dev = pa.devicePointer; s_dev = ps.devicePointer;
      B->ops->step_compact_zero_copy(B->ctx(), (const unsigned char*)a_dev, (unsigned char*)s_dev, n, st);
      int rc = post();
      cudaError_t e1 = cudaStreamSynchronize(st);
      ++g_host_zero_copy_steps;
      if (rc) return rc;
      if (e1 != cudaSuccess) return cuda_fail(e1, "step_host: synchronize");
      return 0;
    }
    cudaGetLastError();
  }

  // ---- graph path: the pipeline is ONE cudaGraphLaunch -----------------------------------------------------------------
  // RL loops step the same batch with the same pinned buffers every time, so the upload -> kernel -> download sequence is
  // captured once per (batch, buffers, n) and replayed: one driver call instead of five per chunk, so the float entry's
  // 2-chunk overlap no longer pays ten driver calls.  Pageable buffers (a captured copy must be a real DMA) and small
  // batches take the plain stream path below.
  static bool graphs_broken = false;            // a capture / instantiate failure turns the graph path off for the process
  if (graphs_on && !graphs_broken && n >= (1 << 16)) {
    auto pinned = [](const void* p) {
      if (!p) return true;
      cudaPointerAttributes a;
      if (cudaPointerGetAttributes(&a, p) != cudaSuccess) { cudaGetLastError(); return false; }
      return a.type == cudaMemoryTypeHost;
    };
    if (pinned(actions_h) && pinned(mask_h) && pinned(term_or_status_h) && pinned(rets_h)) {
      Batch::HostGraph* hit = nullptr;
      for (auto& g : B->host_graphs)
        if (g.actions == actions_h && g.mask == mask_h && g.term == term_or_status_h && g.rets == rets_h && g.n == n &&
            g.action_bytes == action_bytes && g.compact == compact) { hit = &g; break; }
      if (!hit) {
        cudaGraph_t graph = nullptr;
        Batch::HostGraph g{actions_h, mask_h, term_or_status_h, rets_h, n, action_bytes, compact, nullptr, 0};
        cudaError_t e = cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal);
        if (e == cudaSuccess) {
          const int rc = enqueue_host_step(B, pipe, actions_h, action_bytes, mask_h, term_or_status_h, rets_h, n, compact, chunks, /*join=*/true);
          e = cudaStreamEndCapture(st, &graph);
          if (rc && e == cudaSuccess) e = cudaErrorUnknown;
        }
        if (e == cudaSuccess) e = cudaGraphInstantiate(&g.exec, graph, 0);
        if (graph) cudaGraphDestroy(graph);
        if (e != cudaSuccess) {                    // not capturable here: fall back to the plain stream path, for good
          cudaGetLastError();
          graphs_broken = true;
          goto stream_path;
        }
        if (B->host_graphs.size() >= kHostGraphsPerBatch) {                    // evict the least recently used
          size_t lru = 0;
          for (size_t i = 1; i < B->host_graphs.size(); ++i) if (B->host_graphs[i].stamp < B->host_graphs[lru].stamp) lru = i;
          cudaGraphExecDestroy(B->host_graphs[lru].exec);
          B->host_graphs[lru] = g;
          hit = &B->host_graphs[lru];
        } else {
          B->host_graphs.push_back(g);
          hit = &B->host_graphs.back();
        }
      }
      hit->stamp = ++B->host_graph_clock;
      cudaError_t e = cudaGraphLaunch(hit->exec, st);
      g_launches += 1;
      g_host_graph_launches += 1;
      cudaError_t e1 = cudaStreamSynchronize(st);
      if (e != cudaSuccess) return cuda_fail(e, "step_host: graph launch");
      if (e1 != cudaSuccess) return cuda_fail(e1, "step_host: synchronize");
      return 0;
    }
  }

stream_path:
  // ---- stream path ------------------------------------------------------------------------------------------------------
  int rc = enqueue_host_step(B, pipe, actions_h, action_bytes, mask_h, term_or_status_h, rets_h, n, compact, chunks, /*join=*/false);
  // always drain both streams, error or not: no copy into a caller's host buffer may stay in flight after the call
  cudaError_t e1 = cudaStreamSynchronize(st), e2 = cudaStreamSynchronize(st2);
  if (rc) return rc;
  if (e1 != cudaSuccess) return cuda_fail(e1, "step_host: synchronize");
  if (e2 != cudaSuccess) return cuda_fail(e2, "step_host: synchronize");
  return 0;
}

int b2s_step_fused_host(void* batch, const int32_t* actions_h, uint32_t* mask_h, uint8_t* term_h, float* rets_h, int64_t n) {
  if (int r = check(batch, n)) return r;
  if (!actions_h) return fail("null actions");
  return step_host_impl((Batch*)batch, actions_h, 4, mask_h, term_h, rets_h, n, 0);
}

int b2s_step_fused_host_compact(void* batch, const void* actions_h, int action_bytes, uint8_t* status_h, uint32_t* mask_h, int64_t n) {
  if (int r = check(batch, n)) return r;
  if (!actions_h || !status_h) return fail("null actions / status");
  Batch* B = (Batch*)batch;
  if (action_bytes != 1 && action_bytes != 4) return fail("step_compact: action_bytes must be 1 (uint8, 0xFF = skip) or 4 (int32, -1 = skip)");
  if (action_bytes == 1 && B->info.num_distinct_actions > 255) return fail("step_compact: uint8 actions need num_distinct_actions <= 255");
  if (B->info.min_utility != -1.0 || B->info.max_utility != 1.0 || B->info.max_chance_outcomes > 0)
    return fail("step_compact: the 2-bit outcome code needs a win / loss / draw game (use b2s_step_fused_host)");
  return step_host_impl(B, actions_h, action_bytes, mask_h, status_h, nullptr, n, 1);
}

int b2s_error_count(void* batch, int64_t* count, int64_t* first_bad_lane, void* stream) {
  if (int r = check(batch, 0)) return r;
  Batch* B = (Batch*)batch;
  ErrBuf e;
  CU(cudaMemcpyAsync(&e, B->err, sizeof e, cudaMemcpyDeviceToHost, (cudaStream_t)stream));
  CU(cudaStreamSynchronize((cudaStream_t)stream));
  if (count) *count = (int64_t)e.count;
  if (first_bad_lane) *first_bad_lane = e.count ? e.first : -1;
  return 0;
}

// Packed lane blob: the kChunks chunks in plane order, then (go) the history column.
int b2s_state_get(void* batch, int64_t idx, void* host_blob, size_t cap) {
  if (int r = check(batch, 0)) return r;
  Batch* B = (Batch*)batch;
  if (idx < 0 || idx >= B->cap) return fail("lane out of range");
  size_t cb = B->ops->chunk_bytes();
  size_t need = cb * B->ops->chunks() + B->info.history_bytes;
  if (cap < need) return fail("blob too small");
  CU(cudaDeviceSynchronize());
  char* out = (char*)host_blob;
  for (int k = 0; k < B->ops->chunks(); ++k)
    CU(cudaMemcpy(out + k * cb, (char*)B->planes + ((size_t)k * B->cap + idx) * cb, cb, cudaMemcpyDeviceToHost));
  if (B->info.history_bytes)
    CU(cudaMemcpy2D(out + cb * B->ops->chunks(), sizeof(u64), B->hist + idx, sizeof(u64) * B->cap, sizeof(u64),
                    B->info.history_bytes / sizeof(u64), cudaMemcpyDeviceToHost));
  return 0;
}
int b2s_state_set(void* batch, int64_t idx, const void* host_blob, size_t len) {
  if (int r = check(batch, 0)) return r;
  Batch* B = (Batch*)batch;
  if (idx < 0 || idx >= B->cap) return fail("lane out of range");
  size_t cb = B->ops->chunk_bytes();
  size_t need = cb * B->ops->chunks() + B->info.history_bytes;
  if (len != need) return fail("blob size mismatch");
  CU(cudaDeviceSynchronize());
  const char* in = (const char*)host_blob;
  for (int k = 0; k < B->ops->chunks(); ++k)
    CU(cudaMemcpy((char*)B->planes + ((size_t)k * B->cap + idx) * cb, in + k * cb, cb, cudaMemcpyHostToDevice));
  if (B->info.history_bytes)
    CU(cudaMemcpy2D(B->hist + idx, sizeof(u64) * B->cap, in + cb * B->ops->chunks(), sizeof(u64), sizeof(u64),
                    B->info.history_bytes / sizeof(u64), cudaMemcpyHostToDevice));
  return 0;
}

int b2s_broadcast_state(void* dst_batch, int64_t dst_begin, int64_t count, void* src_batch, int64_t src, void* stream) {
  if (int r = check(dst_batch, 0)) return r;
  if (!src_batch) return fail("null src batch");
  Batch* D = (Batch*)dst_batch;
  Batch* S = (Batch*)src_batch;
  if (D->info.game_id != S->info.game_id || D->device != S->device ||
      memcmp(&D->info, &S->info, sizeof(b2s_game_info)) != 0)
    return fail("broadcast: batches differ in game/params/device");
  if (dst_begin < 0 || count < 0 || dst_begin + count > D->cap || src < 0 || src >= S->cap) return fail("broadcast: range");
  D->ops->broadcast(D->ctx(), dst_begin, count, S->ctx(), src, (cudaStream_t)stream);
  return post();
}

int b2s_copy_states(void* dst_batch, int64_t dst_begin, void* src_batch, int64_t src_begin, int64_t count, void* stream) {
  if (int r = check(dst_batch, 0)) return r;
  if (!src_batch) return fail("null src batch");
  Batch* D = (Batch*)dst_batch;
  Batch* S = (Batch*)src_batch;
  if (D->device != S->device || memcmp(&D->info, &S->info, sizeof(b2s_game_info)) != 0)
    return fail("copy: batches differ in game/params/device");
  if (dst_begin < 0 || src_begin < 0 || count < 0 || dst_begin + count > D->cap || src_begin + count > S->cap)
    return fail("copy: range");
  D->ops->copy(D->ctx(), dst_begin, S->ctx(), src_begin, count, (cudaStream_t)stream);
  return post();
}

int b2s_rollout(void* batch, uint64_t seed, int64_t lane_offset, int64_t n, float* rets_d, int32_t* plies_d, void* stream) {
  if (int r = check(batch, n)) return r;
  Batch* B = (Batch*)batch;
  B->ops->rollout(B->ctx(), seed, lane_offset, rets_d, plies_d, n, (cudaStream_t)stream);
  return post();
}

int b2s_record_trajectories(void* batch, uint64_t seed, int64_t lane_offset, int64_t n, int32_t max_unroll_length,
                            const b2s_trajectory_out* out, void* stream) {
  if (int r = check(batch, n)) return r;
  if (!out) return fail("trajectories: null output descriptor");
  Batch* B = (Batch*)batch;
  cudaStream_t st = (cudaStream_t)stream;
  const int T = max_unroll_length > 0 ? max_unroll_length : B->info.max_game_length;
  const int which = B->info.information_state_tensor_size > 0 ? 1 : 0;
  const size_t F = (size_t)(which ? B->info.information_state_tensor_size : B->info.observation_tensor_size);
  const size_t W = (size_t)B->info.mask_words, N = (size_t)n;
  B->ops->traj_begin(B->ctx(), seed, lane_offset, out->lengths, n, st);
  for (int t = 0; t < T; ++t) {
    if (out->observations) {
      // tensor of the state the decision is taken in (acting player's view); zeros once the episode is over
      const char* e = B->ops->obs(B->ctx(), -1, which, 1, out->observations + (size_t)t * N * F, n, st);
      if (e) return fail(e);
    }
    TrajStepOut o;
    o.mask = out->legal_mask ? out->legal_mask + (size_t)t * N * W : nullptr;
    o.actions = out->actions ? out->actions + (size_t)t * N : nullptr;
    o.players = out->player_ids ? out->player_ids + (size_t)t * N : nullptr;
    o.valid = out->valid ? out->valid + (size_t)t * N : nullptr;
    o.next_is_terminal = out->next_is_terminal ? out->next_is_terminal + (size_t)t * N : nullptr;
    o.lengths = out->lengths;
    B->ops->traj_step(B->ctx(), seed, lane_offset, t, o, n, st);
  }
  B->ops->traj_finish(B->ctx(), out->rewards, n, st);
  return post();
}

int b2s_gather_states(void* dst_batch, void* src_batch, const int64_t* src_lanes_d, int64_t count, void* stream) {
  if (int r = check(dst_batch, count)) return r;
  if (!src_batch || !src_lanes_d) return fail("gather: null argument");
  Batch* D = (Batch*)dst_batch;
  Batch* S = (Batch*)src_batch;
  if (D->device != S->device || memcmp(&D->info, &S->info, sizeof(b2s_game_info)) != 0)
    return fail("gather: batches differ in game/params/device");
  D->ops->gather(D->ctx(), S->ctx(), (const long long*)src_lanes_d, count, (cudaStream_t)stream);
  return post();
}

// ---- MCTS ---------------------------------------------------------------------------------------------------
int b2s_mcts_search(void* roots_batch, int64_t n_trees, const b2s_mcts_config* cfg, int32_t* visit_counts_d,
                    double* total_reward_d, float* outcome_p0_d, int32_t* best_action_d, int32_t* sims_run_d,
                    void* stream) {
  if (int r = check(roots_batch, n_trees)) return r;
  if (!cfg || !visit_counts_d || !total_reward_d || !best_action_d) return fail("mcts: null argument");
  if (cfg->max_simulations < 1 || cfg->n_rollouts < 1) return fail("mcts: max_simulations and n_rollouts must be >= 1");
  if (cfg->max_wall_clock_time < 0 || cfg->max_nodes_per_tree < 0) return fail("mcts: negative budget");
  if (cfg->child_selection_policy != B2S_MCTS_UCT && cfg->child_selection_policy != B2S_MCTS_PUCT)
    return fail("mcts: unknown child_selection_policy");
  if (n_trees == 0) return 0;
  Batch* B = (Batch*)roots_batch;
  cudaStream_t st = (cudaStream_t)stream;
  // scratch lanes: same layout as the roots; only the per-lane history column (go) is ever written
  if (B->mcts_work_cap < n_trees) {
    if (B->mcts_work) cudaFree(B->mcts_work);
    if (B->mcts_hist) cudaFree(B->mcts_hist);
    B->mcts_work = nullptr; B->mcts_hist = nullptr; B->mcts_work_cap = 0;
    CU(cudaMalloc(&B->mcts_work, B->ops->chunk_bytes() * (size_t)B->ops->chunks() * (size_t)n_trees));
    if (B->info.history_bytes) CU(cudaMalloc((void**)&B->mcts_hist, (size_t)B->info.history_bytes * (size_t)n_trees));
    B->mcts_work_cap = n_trees;
  }
  Ctx work;
  work.planes = B->mcts_work; work.cap = B->mcts_work_cap; work.hist = B->mcts_hist; work.err = B->err;
  B->ops->copy(work, 0, B->ctx(), 0, n_trees, st);
  // log table filled by the host's std::log
  int need = cfg->max_simulations + 2;
  if (B->mcts_log_n < need) {
    if (B->mcts_log) cudaFree(B->mcts_log);
    B->mcts_log = nullptr; B->mcts_log_n = 0;
    std::vector<double> t(need);
    for (int k = 0; k < need; ++k) t[k] = std::log((double)k);
    CU(cudaMalloc((void**)&B->mcts_log, sizeof(double) * need));
    CU(cudaMemcpy(B->mcts_log, t.data(), sizeof(double) * need, cudaMemcpyHostToDevice));
    B->mcts_log_n = need;
  }
  // node arenas, one per tree (mcts.cuh): nodes_per_tree slots of 16 B (n_rollouts a power of two) or 24 B
  const unsigned long long A = (unsigned long long)B->info.num_distinct_actions;
  const long long work_units = (long long)cfg->max_simulations * cfg->n_rollouts;
  const int compact = (cfg->n_rollouts & (cfg->n_rollouts - 1)) == 0 && work_units < (1ll << 30);
  const size_t node_bytes = compact ? sizeof(MctsNodeC) : sizeof(MctsNodeW);
  unsigned long long per_tree;
  if (cfg->max_nodes_total > 0) {
    per_tree = (unsigned long long)cfg->max_nodes_total / (unsigned long long)n_trees;
  } else {
    const unsigned long long worst = 2ull + (unsigned long long)cfg->max_simulations * A;      // one expansion per simulation at most
    size_t free_b = 0, total_b = 0;
    CU(cudaMemGetInfo(&free_b, &total_b));
    const unsigned long long fit = (unsigned long long)((free_b + B->mcts_pool_bytes) * 0.6 / node_bytes) / (unsigned long long)n_trees;
    per_tree = worst < fit ? worst : fit;
    if (cfg->max_nodes_per_tree > 1) {
      // the budget is logical (MCTSBot::nodes_, live nodes <= budget + one expansion); blocks freed by the collector are reused
      // by exact size (a pruned node re-expands to the same number of children) or split, never coalesced, so the arena is
      // twice the budget; a tree that still cannot allocate stops and is reported by b2s_error_count
      const unsigned long long want = 2ull * (unsigned long long)cfg->max_nodes_per_tree + 8 * A + 64;
      if (want < per_tree) per_tree = want;
    }
  }
  if (per_tree > 0xffffffffull) per_tree = 0xffffffffull;
  if (per_tree < A + 2) return fail("mcts: node arena too small (max_nodes_total / free memory)");
  if (cfg->max_nodes_per_tree > 0x7fffffffll) return fail("mcts: max_nodes_per_tree out of range");
  const unsigned long long want_bytes = per_tree * (unsigned long long)n_trees * node_bytes;
  if (B->mcts_pool_bytes < want_bytes) {
    if (B->mcts_pool) cudaFree(B->mcts_pool);
    B->mcts_pool = nullptr; B->mcts_pool_bytes = 0;
    CU(cudaMalloc(&B->mcts_pool, want_bytes));
    B->mcts_pool_bytes = want_bytes;
  }
  if (!B->mcts_top) CU(cudaMalloc((void**)&B->mcts_top, sizeof(unsigned long long)));
  CU(cudaMemsetAsync(B->mcts_top, 0, sizeof(unsigned long long), st));
  MctsArgs a;
  memset(&a, 0, sizeof a);
  a.sims = cfg->max_simulations; a.n_rollouts = cfg->n_rollouts; a.solve = cfg->solve; a.uct_c = cfg->uct_c;
  a.puct = cfg->child_selection_policy == B2S_MCTS_PUCT;
  a.max_nodes = (int)cfg->max_nodes_per_tree; a.max_seconds = cfg->max_wall_clock_time;
  a.seed = cfg->seed; a.tree_offset = cfg->tree_index_offset; a.log_table = B->mcts_log;
  a.pool = B->mcts_pool; a.nodes_per_tree = per_tree; a.nodes_used = B->mcts_top; a.compact = compact;
  { const char* t = getenv("B2S_MCTS_TUNING"); a.tuning = t ? atoi(t) : 0; }
  a.visits_out = visit_counts_d; a.reward_out = total_reward_d; a.outcome_out = outcome_p0_d;
  a.best_out = best_action_d; a.sims_out = sims_run_d; a.gc_out = cfg->gc_runs_d; a.err = B->err;
  const char* e = B->ops->mcts(B->ctx(), work, n_trees, a, st);
  if (e) return fail(e);
  if (int r = post()) return r;
  CU(cudaStreamSynchronize(st));          // the search is a long-running call; results are ready on return
  return 0;
}

int b2s_mcts_nodes_used(void* roots_batch, int64_t* nodes) {
  if (int r = check(roots_batch, 0)) return r;
  Batch* B = (Batch*)roots_batch;
  unsigned long long v = 0;
  if (B->mcts_top) CU(cudaMemcpy(&v, B->mcts_top, sizeof v, cudaMemcpyDeviceToHost));
  if (nodes) *nodes = (int64_t)v;
  return 0;
}

int b2s_host_alloc(void** out, size_t bytes) {
  if (!out) return fail("null out");
  CU(cudaHostAlloc(out, bytes, cudaHostAllocDefault));
  return 0;
}
void b2s_host_free(void* p) { if (p) cudaFreeHost(p); }
int b2s_device_alloc(int device, void** out, size_t bytes) {
  if (!out) return fail("null out");
  CU(cudaSetDevice(device));
  CU(cudaMalloc(out, bytes));
  return 0;
}
void b2s_device_free(int device, void* p) { if (p) { cudaSetDevice(device); cudaFree(p); } }
int b2s_memcpy_h2d(int device, void* dst_d, const void* src_h, size_t bytes, void* stream) {
  CU(cudaSetDevice(device));
  CU(cudaMemcpyAsync(dst_d, src_h, bytes, cudaMemcpyHostToDevice, (cudaStream_t)stream));
  return 0;
}
int b2s_memcpy_d2h(int device, void* dst_h, const void* src_d, size_t bytes, void* stream) {
  CU(cudaSetDevice(device));
  CU(cudaMemcpyAsync(dst_h, src_d, bytes, cudaMemcpyDeviceToHost, (cudaStream_t)stream));
  return 0;
}
int b2s_stream_synchronize(int device, void* stream) {
  CU(cudaSetDevice(device));
  CU(cudaStreamSynchronize((cudaStream_t)stream));
  return 0;
}

}  // extern "C"
