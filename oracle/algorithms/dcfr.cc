// TEST INFRASTRUCTURE ONLY (see oracle/oracle.h).
// CPU restatement of the reference's Python Discounted CFR, open_spiel/python/algorithms/discounted_cfr.py (_DCFRSolver with
// alternating updates and linear averaging, as DCFRSolver and LCFRSolver construct it) on top of cfr.py's _CFRSolver, for
// two-player games over the oracle's State objects.  The tree is walked once to build the nodes and information states
// (_initialize_info_state_nodes, discounted_cfr.py:65-91); each iteration then recurses over those nodes exactly as
// _compute_counterfactual_regret_for_player does (:93-188), with its pruning of decision nodes no player reaches, so every
// product and sum is the reference's, in its order.  The per-iteration factors come from std::pow in double, which is
// glibc's pow, as CPython's float ** is; integral exponents agree with Python's int arithmetic while t**k + 1 <= 2**53.
#include <cmath>
#include <cstring>
#include <map>
#include <memory>
#include <string>
#include <vector>

#include "../oracle.h"

namespace oracle {
namespace {

struct Values {                        // cfr.py _InfoStateNode (:36-50)
  std::vector<int64_t> legal;
  std::vector<double> regrets, cum_policy, cur_policy;
  int player = 0;
};

struct Node {
  int kind = 0;                        // 0 terminal, 1 chance, 2 decision
  int player = 0;
  double ret[2] = {0, 0};
  std::vector<double> probs;           // chance outcome probabilities
  std::vector<Node> children;          // chance outcomes / legal actions in order
  Values* v = nullptr;
};

struct Dcfr {
  const Game* game;
  double alpha, beta, gamma;
  // kPrune: the reference's pruning.  The other two modes exist to show that a test case depends on each half of it:
  // kPruneUpdates prunes only the table updates and keeps the unpruned values, kPruneNone prunes nothing.
  enum Mode { kPruneNone = 0, kPrune = 1, kPruneUpdates = 2 } prune = kPrune;
  int iteration = 0;
  std::map<std::string, Values> table;
  std::vector<std::string> order;      // first-visit (DFS) order of information states
  Node root;

  void Build(const State& s, Node& node) {   // _initialize_info_state_nodes, discounted_cfr.py:65-91
    if (s.IsTerminal()) {
      auto r = s.Returns();
      node.kind = 0; node.ret[0] = r[0]; node.ret[1] = r[1];
      return;
    }
    std::vector<int64_t> acts;
    if (s.IsChanceNode()) {
      node.kind = 1;
      for (auto& ap : s.ChanceOutcomes()) { acts.push_back(ap.first); node.probs.push_back(ap.second); }
    } else {
      node.kind = 2;
      node.player = s.CurrentPlayer();
      std::string key = s.InformationStateString(node.player);
      acts = s.LegalActions();
      auto it = table.find(key);
      if (it == table.end()) {
        order.push_back(key);
        Values v;
        v.legal = acts; v.player = node.player;
        v.regrets.assign(acts.size(), 0.0); v.cum_policy.assign(acts.size(), 0.0);
        v.cur_policy.assign(acts.size(), 1.0 / acts.size());   // TabularPolicy: uniform over the legal actions
        it = table.emplace(key, v).first;
      }
      node.v = &it->second;
    }
    node.children.resize(acts.size());
    for (size_t i = 0; i < acts.size(); ++i) {
      auto c = s.Clone();
      c->ApplyAction(acts[i]);
      Build(*c, node.children[i]);
    }
  }

  struct V2 { double v[2]; };

  // _compute_counterfactual_regret_for_player (discounted_cfr.py:93-188); reach = [player 0, player 1, chance].
  V2 Regret(const Node& node, int player, const double* reach) {
    if (node.kind == 0) return {{node.ret[0], node.ret[1]}};
    if (node.kind == 1) {              // :114-123: state_value = 0.0; += action_prob * child
      V2 value{{0.0, 0.0}};
      for (size_t i = 0; i < node.children.size(); ++i) {
        double nr[3] = {reach[0], reach[1], reach[2] * node.probs[i]};
        V2 cv = Regret(node.children[i], player, nr);
        for (int k = 0; k < 2; ++k) value.v[k] += node.probs[i] * cv.v[k];
      }
      return value;
    }
    const bool unreached = reach[0] == 0 && reach[1] == 0;
    if (prune == kPrune && unreached) return {{0.0, 0.0}};              // :132-133
    const int cur = node.player;
    Values& v = *node.v;
    const std::vector<double> policy = v.cur_policy;                   // _get_infostate_policy (cfr.py:365-373)
    V2 value{{0.0, 0.0}};
    std::vector<double> child(policy.size());
    for (size_t a = 0; a < policy.size(); ++a) {                       // :148-160
      double nr[3] = {reach[0], reach[1], reach[2]};
      nr[cur] *= policy[a];
      V2 cv = Regret(node.children[a], player, nr);
      for (int k = 0; k < 2; ++k) value.v[k] += policy[a] * cv.v[k];
      child[a] = cv.v[cur];
    }
    if (cur != player || (prune == kPruneUpdates && unreached)) return value;   // :166-168
    const double reach_prob = reach[cur];
    double before = 1.0, after = 1.0;                                  // np.prod(reach[:cur]) * np.prod(reach[cur + 1:])
    for (int i = 0; i < cur; ++i) before *= reach[i];
    for (int i = cur + 1; i < 3; ++i) after *= reach[i];
    const double cf_reach = before * after;
    const double w = std::pow((double)iteration, gamma);              // self._iteration ** self.gamma
    for (size_t a = 0; a < policy.size(); ++a) {                       // :175-186
      v.regrets[a] += cf_reach * (child[a] - value.v[cur]);
      v.cum_policy[a] += reach_prob * policy[a] * w;
    }
    return value;
  }

  void Iterate() {                     // evaluate_and_update_policy, discounted_cfr.py:190-209
    ++iteration;
    const double t = iteration;
    const double ta = std::pow(t, alpha), tb = std::pow(t, beta);
    const double pos = ta / (ta + 1), neg = tb / (tb + 1);
    for (int p = 0; p < 2; ++p) {
      const double reach[3] = {1.0, 1.0, 1.0};
      Regret(root, p, reach);
      for (auto& kv : table) {         // :199-209
        if (kv.second.player != p) continue;
        for (double& r : kv.second.regrets) r *= r >= 0 ? pos : neg;
      }
      for (auto& kv : table) {         // cfr._update_current_policy / _regret_matching, cfr.py:78-98, 375-399
        Values& v = kv.second;
        double sum = 0.0;
        for (double r : v.regrets) if (r > 0) sum += r;
        for (size_t a = 0; a < v.regrets.size(); ++a)
          v.cur_policy[a] = sum > 0 ? (v.regrets[a] > 0 ? v.regrets[a] / sum : 0.0) : 1.0 / v.legal.size();
      }
    }
  }
};

}  // namespace
}  // namespace oracle

extern "C" {

// A DCFR solver over a two-player game (nullptr otherwise); prune: 1 = the reference's zero-reach pruning, 2 = of the
// table updates only, 0 = none (the last two are test contrasts only).
void* orc_dcfr_new(void* game, double alpha, double beta, double gamma, int prune) {
  using namespace oracle;
  const Game* g = (const Game*)game;
  if (g->info.num_players != 2) return nullptr;
  auto* c = new Dcfr;
  c->game = g; c->alpha = alpha; c->beta = beta; c->gamma = gamma; c->prune = (Dcfr::Mode)prune;
  c->Build(*g->NewInitialState(), c->root);
  return c;
}
void orc_dcfr_free(void* c) { delete (oracle::Dcfr*)c; }
void orc_dcfr_iterate(void* c, int iters) { for (int i = 0; i < iters; ++i) ((oracle::Dcfr*)c)->Iterate(); }
int orc_dcfr_iteration(void* c) { return ((oracle::Dcfr*)c)->iteration; }
void orc_dcfr_set_iteration(void* c, int iteration) { ((oracle::Dcfr*)c)->iteration = iteration; }
int orc_dcfr_num_infosets(void* c) { return (int)((oracle::Dcfr*)c)->table.size(); }
// k-th information state in first-visit order: key string + arrays; returns the number of legal actions.
int orc_dcfr_get(void* c, int k, char* key, int key_cap, int64_t* legal, double* regrets, double* cum, double* cur, int cap,
                 int* player) {
  auto* s = (oracle::Dcfr*)c;
  if (k < 0 || k >= (int)s->order.size()) return -1;
  const std::string& ks = s->order[k];
  const auto& v = s->table.at(ks);
  int m = (int)ks.size() < key_cap - 1 ? (int)ks.size() : key_cap - 1;
  memcpy(key, ks.data(), m); key[m] = 0;
  int n = (int)v.legal.size();
  for (int i = 0; i < n && i < cap; ++i) { legal[i] = v.legal[i]; regrets[i] = v.regrets[i]; cum[i] = v.cum_policy[i]; cur[i] = v.cur_policy[i]; }
  if (player) *player = v.player;
  return n;
}
// Overwrite one information state's tables; -1 if the key is unknown or the action count differs.
int orc_dcfr_set(void* c, const char* key, const double* regrets, const double* cum, const double* cur, int n) {
  auto* s = (oracle::Dcfr*)c;
  auto it = s->table.find(key);
  if (it == s->table.end() || (int)it->second.legal.size() != n) return -1;
  it->second.regrets.assign(regrets, regrets + n);
  it->second.cum_policy.assign(cum, cum + n);
  it->second.cur_policy.assign(cur, cur + n);
  return 0;
}

}  // extern "C"
