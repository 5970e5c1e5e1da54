// The CFR solver's game tree — expanded level by level through the C ABI, flattened on the host, uploaded — and the solver's
// lifetime, table export / import.  Layout and conventions: cfr.cuh.
#include <string.h>

#include <algorithm>
#include <cmath>
#include <memory>
#include <unordered_map>

#include "cfr.cuh"

namespace b2s {

// The expanded tree on the host: nodes in level order (children of one node consecutive, in action order), and its
// information states in order of first appearance.
struct HostTree {
  std::vector<int> parent, first_child, infoset, level_off;
  std::vector<signed char> kind, actor, nchild, aidx;
  std::vector<double> chance_prob, ret;
  std::vector<int> is_player, is_off, legal_actions, node_counts;    // node_counts = {chance, decision, terminal}
  std::vector<float> keys;                                           // [I][tensor_size] information-state tensors
};

#define TRY(x) do { if (int _r = (x)) return _r; } while (0)

// (a) Level-by-level expansion with the batched device kernels: status, legal actions and information-state tensor of every
// lane of a level, then the next level as a clone of each parent lane with the child's action applied.
static int expand_tree(int game_id, const b2s_params* params, int device, const b2s_game_info& gi, HostTree& t) {
  const int T = gi.information_state_tensor_size, MW = gi.mask_words;
  std::unordered_map<std::string, int> key_to_is;
  std::vector<int> is_nact;
  t.node_counts.assign(3, 0);
  // level 0 = the initial state
  void *level = nullptr, *next = nullptr;
  const ScopeExit destroy_batches{[&] { b2s_batch_destroy(level); b2s_batch_destroy(next); }};
  TRY(b2s_batch_create(game_id, params, 1, device, &level));
  long long n = 1;
  t.parent.push_back(-1); t.aidx.push_back(0); t.chance_prob.push_back(1.0);
  t.level_off.push_back(0);
  long long base = 0;                       // node id of lane 0 of the current level
  for (int depth = 0; n > 0; ++depth) {
    if (depth > 4096 || base + n > 50000000LL) return fail("cfr: game tree too large for the device solver");
    // per-lane facts of this level, computed by the batched kernels
    std::vector<signed char> cur(n); std::vector<unsigned char> term(n); std::vector<float> rets(2 * n), tens((size_t)T * n);
    std::vector<uint32_t> mask((size_t)MW * n);
    {
      signed char* cur_d = nullptr; unsigned char* term_d = nullptr; float* rets_d = nullptr; uint32_t* mask_d = nullptr; float* tens_d = nullptr;
      const ScopeExit free_level{[&] { for (void* p : {(void*)cur_d, (void*)term_d, (void*)rets_d, (void*)mask_d, (void*)tens_d}) b2s_device_free(device, p); }};
      TRY(b2s_device_alloc(device, (void**)&cur_d, n));
      TRY(b2s_device_alloc(device, (void**)&term_d, n));
      TRY(b2s_device_alloc(device, (void**)&rets_d, sizeof(float) * 2 * n));
      TRY(b2s_device_alloc(device, (void**)&mask_d, sizeof(uint32_t) * MW * n));
      TRY(b2s_device_alloc(device, (void**)&tens_d, sizeof(float) * (size_t)T * n));
      TRY(b2s_status(level, (int8_t*)cur_d, term_d, rets_d, n, nullptr));
      TRY(b2s_legal_mask(level, mask_d, n, nullptr));
      TRY(b2s_information_state(level, -1, tens_d, n, nullptr));
      TRY(b2s_memcpy_d2h(device, cur.data(), cur_d, n, nullptr));
      TRY(b2s_memcpy_d2h(device, term.data(), term_d, n, nullptr));
      TRY(b2s_memcpy_d2h(device, rets.data(), rets_d, sizeof(float) * 2 * n, nullptr));
      TRY(b2s_memcpy_d2h(device, mask.data(), mask_d, sizeof(uint32_t) * MW * n, nullptr));
      TRY(b2s_memcpy_d2h(device, tens.data(), tens_d, sizeof(float) * (size_t)T * n, nullptr));
      TRY(b2s_stream_synchronize(device, nullptr));
    }
    // node records + the child list of the next level
    std::vector<long long> src_lanes;
    std::vector<int32_t> actions;
    t.kind.resize(base + n); t.actor.resize(base + n); t.nchild.resize(base + n); t.first_child.resize(base + n);
    t.infoset.resize(base + n, -1); t.ret.resize(2 * (base + n), 0.0);
    long long next_base = base + n;
    for (long long i = 0; i < n; ++i) {
      long long id = base + i;
      t.first_child[id] = (int)(next_base + (long long)src_lanes.size());
      if (term[i]) {
        t.kind[id] = 0; t.actor[id] = 0; t.nchild[id] = 0;
        t.ret[2 * id] = (double)rets[2 * i]; t.ret[2 * id + 1] = (double)rets[2 * i + 1];
        t.node_counts[2]++;
        continue;
      }
      std::vector<int> acts;
      for (int w = 0; w < MW; ++w)
        for (int b = 0; b < 32; ++b) if ((mask[(size_t)i * MW + w] >> b) & 1u) acts.push_back(w * 32 + b);
      if (acts.empty() || acts.size() > 120) return fail("cfr: unexpected legal-action count");
      t.nchild[id] = (signed char)acts.size();
      if (cur[i] == -1) {                                    // chance: uniform over the available outcomes
        t.kind[id] = 1; t.actor[id] = 2; t.node_counts[0]++;        // (kuhn_poker.cc:329-337, leduc_poker.cc:546-571)
      } else {
        t.kind[id] = 2; t.actor[id] = cur[i]; t.node_counts[1]++;
        std::string key((const char*)&tens[(size_t)i * T], sizeof(float) * T);
        auto itk = key_to_is.find(key);
        int is;
        if (itk == key_to_is.end()) {
          is = (int)key_to_is.size();
          key_to_is.emplace(key, is);
          t.is_player.push_back(cur[i]);
          is_nact.push_back((int)acts.size());
          t.keys.insert(t.keys.end(), tens.begin() + (size_t)i * T, tens.begin() + (size_t)(i + 1) * T);
          t.is_off.push_back((int)t.legal_actions.size());
          for (int a : acts) t.legal_actions.push_back(a);
        } else {
          is = itk->second;
          if (is_nact[is] != (int)acts.size()) return fail("cfr: information state with inconsistent legal actions");
        }
        t.infoset[id] = is;
      }
      for (size_t k = 0; k < acts.size(); ++k) {
        src_lanes.push_back(i);
        actions.push_back(acts[k]);
        t.parent.push_back((int)id);
        t.aidx.push_back((signed char)k);
        t.chance_prob.push_back(cur[i] == -1 ? 1.0 / (double)acts.size() : 0.0);
      }
    }
    t.level_off.push_back((int)(base + n));
    long long m = (long long)src_lanes.size();
    if (m == 0) break;
    // next level = clone of each parent lane, then the child action applied
    TRY(b2s_batch_create(game_id, params, m, device, &next));
    {
      long long* lanes_d = nullptr; int32_t* act_d = nullptr;
      const ScopeExit free_lanes{[&] { b2s_device_free(device, lanes_d); b2s_device_free(device, act_d); }};
      TRY(b2s_device_alloc(device, (void**)&lanes_d, sizeof(long long) * m));
      TRY(b2s_device_alloc(device, (void**)&act_d, sizeof(int32_t) * m));
      TRY(b2s_memcpy_h2d(device, lanes_d, src_lanes.data(), sizeof(long long) * m, nullptr));
      TRY(b2s_memcpy_h2d(device, act_d, actions.data(), sizeof(int32_t) * m, nullptr));
      TRY(b2s_gather_states(next, level, (const int64_t*)lanes_d, m, nullptr));
      TRY(b2s_apply_actions(next, act_d, m, nullptr));
      int64_t bad = 0;
      TRY(b2s_error_count(next, &bad, nullptr, nullptr));
      if (bad) return fail("cfr: tree expansion applied an illegal action");
    }
    b2s_batch_destroy(level);
    level = next; next = nullptr;
    base += n; n = m;
  }
  t.is_off.push_back((int)t.legal_actions.size());
  return 0;
}

// The arrays the kernels read besides the node records themselves.
struct FlatTree {
  std::vector<int> hist_off, hist, hist_is, hist_entry_off, policy_index, is_level;
  std::vector<signed char> par_actor, entry_player;
  std::vector<double> chance_reach;
  std::vector<int4> mc_node;
  int cap_es = 0, cap_os = 0;
};

// (b) Pure host derivation of the flattened arrays from the expanded tree.
static int flatten_tree(const HostTree& t, FlatTree& f) {
  const int N = (int)t.kind.size(), I = (int)t.is_player.size();
  // histories of each information state in the reference's DFS order (children in action order)
  std::vector<std::vector<int>> by_is(I);
  {
    std::vector<int> stack = {0};
    while (!stack.empty()) {
      int v = stack.back(); stack.pop_back();
      if (t.kind[v] == 2) by_is[t.infoset[v]].push_back(v);
      for (int c = t.nchild[v] - 1; c >= 0; --c) stack.push_back(t.first_child[v] + c);
    }
  }
  f.hist_off.assign(1, 0);
  for (int i = 0; i < I; ++i) { f.hist.insert(f.hist.end(), by_is[i].begin(), by_is[i].end()); f.hist_off.push_back((int)f.hist.size()); }
  f.hist_is.assign(f.hist.size(), 0);
  f.hist_entry_off.assign(1, 0);
  for (int i = 0; i < I; ++i)
    for (int hh = f.hist_off[i]; hh < f.hist_off[i + 1]; ++hh) {
      f.hist_is[hh] = i;
      f.hist_entry_off.push_back(f.hist_entry_off.back() + (t.is_off[i + 1] - t.is_off[i]));
    }
  f.policy_index.assign(N, -1);
  f.par_actor.assign(N, 2);
  f.chance_reach.assign(N, 1.0);
  for (int v = 1; v < N; ++v) {
    int par = t.parent[v];
    f.par_actor[v] = t.actor[par];
    if (t.kind[par] == 2) f.policy_index[v] = t.is_off[t.infoset[par]] + t.aidx[v];
    f.chance_reach[v] = t.kind[par] == 1 ? f.chance_reach[par] * t.chance_prob[v] : f.chance_reach[par];   // parents precede children
  }
  f.mc_node.resize(N);
  for (int v = 0; v < N; ++v)
    f.mc_node[v] = make_int4(t.first_child[v], t.kind[v] == 2 ? t.is_off[t.infoset[v]] : -1,
                             (int)t.kind[v] | ((int)(t.actor[v] & 0xff) << 8) | ((int)t.nchild[v] << 16), 0);
  // Most delta records one sampled traversal can produce, exactly, from the tree (children follow their parents in the node
  // order, so one backward sweep suffices).  External sampling (UpdateRegrets): the traverser's nodes explore every action and
  // write one regret delta per action; the other player's nodes follow one action and write one average-policy delta per
  // action; chance nodes follow one outcome.  Outcome sampling: one path, two deltas per action at the update player's nodes.
  std::vector<int> es(N), os(N);
  for (int pl = 0; pl < 2; ++pl) {
    for (int v = N - 1; v >= 0; --v) {
      int sum_es = 0, max_es = 0, max_os = 0;
      for (int c = 0; c < t.nchild[v]; ++c) {
        const int w = t.first_child[v] + c;
        sum_es += es[w]; max_es = std::max(max_es, es[w]); max_os = std::max(max_os, os[w]);
      }
      if (t.kind[v] == 2) {
        es[v] = t.nchild[v] + (t.actor[v] == pl ? sum_es : max_es);
        os[v] = (t.actor[v] == pl ? 2 * t.nchild[v] : 0) + max_os;
      } else {
        es[v] = max_es; os[v] = max_os;                 // chance (one outcome followed) or terminal (no children)
      }
    }
    f.cap_es = std::max(f.cap_es, es[0]); f.cap_os = std::max(f.cap_os, os[0]);
  }
  f.cap_es = std::max(f.cap_es, 1); f.cap_os = std::max(f.cap_os, 1);
  f.entry_player.assign(t.legal_actions.size(), 0);
  for (int i = 0; i < I; ++i)
    for (int k = t.is_off[i]; k < t.is_off[i + 1]; ++k) f.entry_player[k] = (signed char)t.is_player[i];
  std::vector<int> node_level(N, 0);
  for (int l = 0; l + 1 < (int)t.level_off.size(); ++l)
    for (int v = t.level_off[l]; v < t.level_off[l + 1]; ++v) node_level[v] = l;
  f.is_level.assign(I, 0);
  for (int i = 0; i < I; ++i) {
    f.is_level[i] = node_level[by_is[i][0]];
    for (int v : by_is[i]) if (node_level[v] != f.is_level[i]) return fail("cfr: information state spans tree levels");
  }
  return 0;
}

template <typename T>
static int upload(CfrSolver* s, const std::vector<T>& v, const T** out) {
  void* p = nullptr;
  B2S_CU(cudaMalloc(&p, sizeof(T) * (v.empty() ? 1 : v.size())));
  s->allocs.push_back(p);
  if (!v.empty()) B2S_CU(cudaMemcpy(p, v.data(), sizeof(T) * v.size(), cudaMemcpyHostToDevice));
  *out = (const T*)p;
  return 0;
}
static int alloc_d(CfrSolver* s, size_t n, double** out) {
  void* p = nullptr;
  B2S_CU(cudaMalloc(&p, sizeof(double) * (n ? n : 1)));
  s->allocs.push_back(p);
  B2S_CU(cudaMemset(p, 0, sizeof(double) * (n ? n : 1)));
  *out = (double*)p;
  return 0;
}

// (c) Upload: the node records and flattened arrays, zeroed scratch and tables, the initial tables.
static int upload_tree(CfrSolver* S, const HostTree& t, const FlatTree& f) {
  const int N = (int)t.kind.size(), I = (int)S->is_player.size(), E = (int)S->legal_actions.size();
  CfrDev& d = S->d;
  memset(&d, 0, sizeof d);
  d.n_nodes = N; d.n_levels = (int)t.level_off.size() - 1; d.n_infosets = I; d.n_entries = E;
  d.n_hist = (int)f.hist.size();
  d.n_contrib = f.hist_entry_off.back();
  TRY(upload(S, t.level_off, &d.level_off)); TRY(upload(S, t.parent, &d.parent)); TRY(upload(S, t.kind, &d.kind));
  TRY(upload(S, t.actor, &d.actor)); TRY(upload(S, t.first_child, &d.first_child)); TRY(upload(S, t.nchild, &d.nchild));
  TRY(upload(S, t.aidx, &d.aidx)); TRY(upload(S, t.chance_prob, &d.chance_prob)); TRY(upload(S, t.ret, &d.ret));
  TRY(upload(S, t.infoset, &d.infoset)); TRY(upload(S, S->is_player, &d.is_player)); TRY(upload(S, S->is_off, &d.is_off));
  TRY(upload(S, f.hist_off, &d.hist_off)); TRY(upload(S, f.hist, &d.hist));
  TRY(upload(S, f.hist_is, &d.hist_is)); TRY(upload(S, f.hist_entry_off, &d.hist_entry_off));
  TRY(upload(S, f.mc_node, &d.mc_node)); TRY(upload(S, f.entry_player, &d.entry_player));
  TRY(upload(S, f.policy_index, &d.policy_index)); TRY(upload(S, f.par_actor, &d.par_actor));
  TRY(upload(S, f.chance_reach, &d.chance_reach)); TRY(upload(S, f.is_level, &d.is_level));
  const size_t traversals = S->best_response_opponents ? 2 : 1;      // CFR-BR runs both players' traversals at once
  TRY(alloc_d(S, 2 * traversals * N, &d.reach)); TRY(alloc_d(S, traversals * N, &d.edge_prob));
  TRY(alloc_d(S, 2 * traversals * N, &d.value));
  if (S->best_response_opponents) {
    TRY(alloc_d(S, (size_t)d.n_hist, &S->br.cf_reach)); TRY(alloc_d(S, 2 * (size_t)N, &S->br.value));
    void* best = nullptr;
    B2S_CU(cudaMalloc(&best, sizeof(int) * (I ? I : 1)));
    S->allocs.push_back(best);
    B2S_CU(cudaMemset(best, 0, sizeof(int) * (I ? I : 1)));
    S->br.best = (int*)best;
  }
  TRY(alloc_d(S, E, &d.regrets)); TRY(alloc_d(S, E, &d.cum_policy)); TRY(alloc_d(S, E, &d.cur_policy));
  TRY(alloc_d(S, 2 * (size_t)d.n_contrib, &d.delta));
  {
    void* it = nullptr;
    B2S_CU(cudaMalloc(&it, sizeof(int)));
    S->allocs.push_back(it);
    B2S_CU(cudaMemset(it, 0, sizeof(int)));
    d.iter_d = (int*)it;
  }
  // CFRInfoStateValues(legal_actions): regrets 0, cumulative policy 0, current policy uniform (cfr.h:42-98)
  std::vector<double> uni(E);
  for (int i = 0; i < I; ++i)
    for (int k = S->is_off[i]; k < S->is_off[i + 1]; ++k) uni[k] = 1.0 / (double)(S->is_off[i + 1] - S->is_off[i]);
  B2S_CU(cudaMemcpy(d.cur_policy, uni.data(), sizeof(double) * E, cudaMemcpyHostToDevice));
  if (S->mccfr_tables) {     // CFRInfoStateValues(legal_actions, kInitialTableValues), external_sampling_mccfr.cc:143
    std::vector<double> init(E, 0.000001);
    B2S_CU(cudaMemcpy(d.regrets, init.data(), sizeof(double) * E, cudaMemcpyHostToDevice));
    B2S_CU(cudaMemcpy(d.cum_policy, init.data(), sizeof(double) * E, cudaMemcpyHostToDevice));
  }
  return 0;
}

}  // namespace b2s

using namespace b2s;

extern "C" {

int b2s_cfr_create(int game_id, const b2s_params* params, int flags, int device, void** out_solver) {
  if (!out_solver) return fail("cfr: null out_solver");
  *out_solver = nullptr;
  if (b2s_device_count() <= 0) return fail("no CUDA device: the b2s device path has no CPU fallback");
  b2s_game_info gi;
  if (int r = b2s_game_info_get(game_id, params, &gi)) return r;
  if (gi.num_players != 2) return fail("cfr: two-player games only");
  if (gi.information_state_tensor_size <= 0)
    return fail("cfr: the game provides no information-state tensor (device CFR keys information states by it)");
  const int br = (flags & B2S_CFR_BEST_RESPONSE_OPPONENTS) ? 1 : 0;
  if (br && (flags & (B2S_CFR_LINEAR_AVERAGING | B2S_CFR_REGRET_MATCHING_PLUS | B2S_CFR_MCCFR_TABLES)))
    return fail("cfr: B2S_CFR_BEST_RESPONSE_OPPONENTS (CFRBRSolver) takes no other flag: it averages plainly, without RM+, "
                "on CFR tables");
  HostTree t;
  FlatTree f;
  TRY(expand_tree(game_id, params, device, gi, t));
  TRY(flatten_tree(t, f));
  std::unique_ptr<CfrSolver> S(new CfrSolver);
  S->device = device; S->game_id = game_id; S->tensor_size = gi.information_state_tensor_size;
  S->linear_averaging = (flags & B2S_CFR_LINEAR_AVERAGING) ? 1 : 0;
  S->rm_plus = (flags & B2S_CFR_REGRET_MATCHING_PLUS) ? 1 : 0;
  S->mccfr_tables = (flags & B2S_CFR_MCCFR_TABLES) ? 1 : 0;
  S->best_response_opponents = br;
  S->is_player = std::move(t.is_player); S->is_off = std::move(t.is_off); S->legal_actions = std::move(t.legal_actions);
  S->node_counts = std::move(t.node_counts); S->keys = std::move(t.keys);
  S->mc_cap_es = f.cap_es; S->mc_cap_os = f.cap_os;
  for (size_t i = 0; i + 1 < S->is_off.size(); ++i) S->max_actions = std::max(S->max_actions, S->is_off[i + 1] - S->is_off[i]);
  // CFR-BR sums children in the device's child order where the reference's best response iterates its btree_map of
  // actions: both are ascending only when every information state lists its legal actions in ascending order.
  if (br)
    for (size_t i = 0; i + 1 < S->is_off.size(); ++i)
      for (int k = S->is_off[i] + 1; k < S->is_off[i + 1]; ++k)
        if (S->legal_actions[k] <= S->legal_actions[k - 1]) return fail("cfr: CFR-BR needs legal actions in ascending order");
  B2S_CU(cudaSetDevice(device));
  TRY(upload_tree(S.get(), t, f));
  *out_solver = S.release();
  return 0;
}

int b2s_dcfr_create(int game_id, const b2s_params* params, double alpha, double beta, double gamma, int device,
                    void** out_solver) {
  if (!out_solver) return fail("dcfr: null out_solver");
  *out_solver = nullptr;
  if (!std::isfinite(alpha) || !std::isfinite(beta) || !std::isfinite(gamma))
    return fail("dcfr: alpha, beta and gamma must be finite");
  TRY(b2s_cfr_create(game_id, params, 0, device, out_solver));
  CfrSolver* S = (CfrSolver*)*out_solver;
  S->dcfr = 1; S->dcfr_alpha = alpha; S->dcfr_beta = beta; S->dcfr_gamma = gamma;
  return 0;
}

void b2s_cfr_destroy(void* solver) {
  if (!solver) return;
  CfrSolver* S = (CfrSolver*)solver;
  cudaSetDevice(S->device);
  delete S;
}

int b2s_cfr_info_get(void* solver, b2s_cfr_info* out) {
  if (!solver || !out) return fail("cfr: null argument");
  CfrSolver* S = (CfrSolver*)solver;
  out->num_nodes = S->d.n_nodes; out->num_levels = S->d.n_levels; out->num_infosets = S->d.n_infosets;
  out->num_entries = S->d.n_entries; out->key_floats = S->tensor_size; out->iteration = S->iteration;
  out->chance_nodes = S->node_counts[0]; out->decision_nodes = S->node_counts[1]; out->terminal_nodes = S->node_counts[2];
  return 0;
}

int b2s_cfr_export(void* solver, double* regrets_h, double* cum_policy_h, double* cur_policy_h, int32_t* offsets_h,
                   int32_t* legal_actions_h, int32_t* players_h, float* keys_h, void* stream) {
  if (!solver) return fail("cfr: null solver");
  CfrSolver* S = (CfrSolver*)solver;
  B2S_CU(cudaSetDevice(S->device));
  cudaStream_t st = (cudaStream_t)stream;
  size_t eb = sizeof(double) * S->d.n_entries;
  if (regrets_h) B2S_CU(cudaMemcpyAsync(regrets_h, S->d.regrets, eb, cudaMemcpyDeviceToHost, st));
  if (cum_policy_h) B2S_CU(cudaMemcpyAsync(cum_policy_h, S->d.cum_policy, eb, cudaMemcpyDeviceToHost, st));
  if (cur_policy_h) B2S_CU(cudaMemcpyAsync(cur_policy_h, S->d.cur_policy, eb, cudaMemcpyDeviceToHost, st));
  B2S_CU(cudaStreamSynchronize(st));
  if (offsets_h) memcpy(offsets_h, S->is_off.data(), sizeof(int) * S->is_off.size());
  if (legal_actions_h) memcpy(legal_actions_h, S->legal_actions.data(), sizeof(int) * S->legal_actions.size());
  if (players_h) memcpy(players_h, S->is_player.data(), sizeof(int) * S->is_player.size());
  if (keys_h) memcpy(keys_h, S->keys.data(), sizeof(float) * S->keys.size());
  return 0;
}

int b2s_cfr_import(void* solver, const double* regrets_h, const double* cum_policy_h, const double* cur_policy_h,
                   int iteration, void* stream) {
  if (!solver) return fail("cfr: null solver");
  CfrSolver* S = (CfrSolver*)solver;
  B2S_CU(cudaSetDevice(S->device));
  cudaStream_t st = (cudaStream_t)stream;
  size_t eb = sizeof(double) * S->d.n_entries;
  if (regrets_h) B2S_CU(cudaMemcpyAsync(S->d.regrets, regrets_h, eb, cudaMemcpyHostToDevice, st));
  if (cum_policy_h) B2S_CU(cudaMemcpyAsync(S->d.cum_policy, cum_policy_h, eb, cudaMemcpyHostToDevice, st));
  if (cur_policy_h) B2S_CU(cudaMemcpyAsync(S->d.cur_policy, cur_policy_h, eb, cudaMemcpyHostToDevice, st));
  B2S_CU(cudaStreamSynchronize(st));
  if (iteration >= 0) S->iteration = iteration;
  return 0;
}

int b2s_cfr_set_iteration(void* solver, int iteration) {
  if (!solver) return fail("cfr: null solver");
  ((CfrSolver*)solver)->iteration = iteration;
  return 0;
}

// Device pointers of the per-action tables (regrets, cumulative policy, current policy; num_entries doubles
// each) so a caller can all-reduce them in place (NCCL) between b2s_cfr_iterate calls.
int b2s_cfr_tables(void* solver, double** regrets_d, double** cum_policy_d, double** cur_policy_d) {
  if (!solver) return fail("cfr: null solver");
  CfrSolver* S = (CfrSolver*)solver;
  if (regrets_d) *regrets_d = S->d.regrets;
  if (cum_policy_d) *cum_policy_d = S->d.cum_policy;
  if (cur_policy_d) *cur_policy_d = S->d.cur_policy;
  return 0;
}

}  // extern "C"
