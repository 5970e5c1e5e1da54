// TEST INFRASTRUCTURE ONLY (see oracle/oracle.h).
// CPU restatement of reference open_spiel/algorithms/cfr_br.{h,cc} (CFRBRSolver::EvaluateAndUpdatePolicy :50-82) and of the
// TabularBestResponse it uses (best_response.cc:79-228, history_tree.cc:160-240; prob_cut_threshold and
// action_value_tolerance at their defaults of -1), over the oracle's State objects: the recursive, string-keyed CFR
// traversal of cfr.cc:331-469 with policy overrides and all-zero-reach pruning; a best response with a memoised node value,
// GetAllInfoSets' counterfactual reach formed from each history upward, and the first strict maximum over ascending actions.
#include <algorithm>
#include <cstring>
#include <limits>
#include <map>
#include <memory>
#include <string>

#include "../oracle.h"

namespace oracle {
namespace {

using PolicyTable = std::map<std::string, std::vector<double>>;   // information state -> probabilities in legal-action order

// The evaluated policy at a decision state: the table's entry, uniform (UniformPolicy) without a table.
std::vector<double> PolicyAt(const State& s, const PolicyTable* table) {
  if (table) {
    auto it = table->find(s.InformationStateString(s.CurrentPlayer()));
    if (it != table->end()) return it->second;
  }
  auto la = s.LegalActions();
  return std::vector<double>(la.size(), 1. / static_cast<double>(la.size()));
}

// TabularBestResponse(game, responder, policy); policy == nullptr is the UniformPolicy.
struct BestResponse {
  struct Node {
    std::unique_ptr<State> s;
    std::vector<int64_t> actions;     // ascending (the history tree's btree_map of children)
    std::vector<double> probs;        // chance probabilities (chance nodes)
    std::vector<std::unique_ptr<Node>> children;
    bool cached = false;
    double value = 0;
  };
  int responder;
  const PolicyTable* policy;
  std::unique_ptr<Node> root;
  std::map<std::string, std::vector<std::pair<Node*, double>>> infosets;
  std::vector<std::string> infoset_order;
  std::map<std::string, int64_t> best;    // information state -> chosen action

  BestResponse(const Game& game, int p, const PolicyTable* pol) : responder(p), policy(pol) {
    root = Build(game.NewInitialState());
    DecisionNodes(root.get());
  }
  std::unique_ptr<Node> Build(std::unique_ptr<State> s) {
    auto n = std::make_unique<Node>();
    if (!s->IsTerminal()) {
      std::vector<std::pair<int64_t, double>> kids;
      if (s->IsChanceNode()) kids = s->ChanceOutcomes();
      else for (auto a : s->LegalActions()) kids.push_back({a, 1.0});
      std::sort(kids.begin(), kids.end(), [](auto& x, auto& y) { return x.first < y.first; });
      for (auto& k : kids) {
        auto c = s->Clone();
        c->ApplyAction(k.first);
        n->actions.push_back(k.first); n->probs.push_back(k.second);
        n->children.push_back(Build(std::move(c)));
      }
    }
    n->s = std::move(s);
    return n;
  }
  Node* Child(Node* n, int64_t a) {
    for (size_t i = 0; i < n->actions.size(); ++i) if (n->actions[i] == a) return n->children[i].get();
    return nullptr;
  }
  // DecisionNodes (history_tree.cc:183-216): the responder's decision nodes in DFS order with policy_prob * prob, the
  // product formed from the node upward.
  std::vector<std::pair<Node*, double>> DecisionNodesOf(Node* n) {
    const State& s = *n->s;
    if (s.IsTerminal()) return {};
    std::vector<std::pair<Node*, double>> out;
    if (!s.IsChanceNode() && s.CurrentPlayer() == responder) out.push_back({n, 1.});
    std::vector<int64_t> la;
    std::vector<double> probs;
    if (s.IsChanceNode()) for (auto& ap : s.ChanceOutcomes()) { la.push_back(ap.first); probs.push_back(ap.second); }
    else {
      la = s.LegalActions();
      if (s.CurrentPlayer() == responder) probs.assign(la.size(), 1.);
      else probs = PolicyAt(s, policy);
    }
    for (size_t i = 0; i < la.size(); ++i) {
      for (auto& sp : DecisionNodesOf(Child(n, la[i]))) out.push_back({sp.first, probs[i] * sp.second});
    }
    return out;
  }
  void DecisionNodes(Node* r) {         // GetAllInfoSets (history_tree.cc:218-238)
    for (auto& sp : DecisionNodesOf(r)) {
      std::string key = sp.first->s->InformationStateString(responder);
      if (!infosets.count(key)) infoset_order.push_back(key);
      infosets[key].push_back(sp);
    }
  }
  int64_t BestAction(const std::string& key) {   // BestResponseAction (best_response.cc:194-228)
    auto it = best.find(key);
    if (it != best.end()) return it->second;
    auto& iset = infosets.at(key);
    int64_t best_action = -1;
    double best_value = std::numeric_limits<double>::lowest();
    for (int64_t a : iset[0].first->actions) {
      double value = 0;
      for (auto& sp : iset) value += sp.second * Value(Child(sp.first, a));
      if (value > best_value) { best_value = value; best_action = a; }
    }
    best[key] = best_action;
    return best_action;
  }
  double Value(Node* n) {               // Value / Handle*Case (best_response.cc:79-192)
    if (n->cached) return n->value;
    const State& s = *n->s;
    double v = 0;
    if (s.IsTerminal()) v = s.Returns()[responder];
    else if (s.IsChanceNode()) {
      for (size_t i = 0; i < n->actions.size(); ++i) v += n->probs[i] * Value(n->children[i].get());
    } else if (s.CurrentPlayer() == responder) {
      int64_t b = BestAction(s.InformationStateString(responder));
      for (size_t i = 0; i < n->actions.size(); ++i) v += Value(n->children[i].get()) * (n->actions[i] == b ? 1.0 : 0.0);
    } else {
      auto la = s.LegalActions();
      auto probs = PolicyAt(s, policy);
      for (size_t i = 0; i < la.size(); ++i) v += probs[i] * Value(Child(n, la[i]));
    }
    n->cached = true; n->value = v;
    return v;
  }
  // GetBestResponsePolicy: 1.0 / 0.0 over each responder information state's actions.
  PolicyTable Policy() {
    PolicyTable out;
    for (auto& key : infoset_order) {
      int64_t b = BestAction(key);
      std::vector<double> p;
      for (int64_t a : infosets[key][0].first->actions) p.push_back(a == b ? 1.0 : 0.0);
      out[key] = p;
    }
    return out;
  }
};

struct Values {                        // CFRInfoStateValues, cfr.h:42-98
  std::vector<int64_t> legal;
  std::vector<double> regrets, cum_policy, cur_policy;
  int player = 0;
};

struct CfrBr {
  const Game* game;
  int iteration = 0;
  int n;
  std::map<std::string, Values> table;
  std::vector<std::string> order;      // first-visit (DFS) order of information states

  void Init(const State& s) {          // InitializeInfostateNodes, cfr.cc:234-261
    if (s.IsTerminal()) return;
    if (s.IsChanceNode()) {
      for (auto& ap : s.ChanceOutcomes()) { auto c = s.Clone(); c->ApplyAction(ap.first); Init(*c); }
      return;
    }
    int p = s.CurrentPlayer();
    std::string key = s.InformationStateString(p);
    auto la = s.LegalActions();
    if (!table.count(key)) order.push_back(key);
    Values v;
    v.legal = la; v.player = p;
    v.regrets.assign(la.size(), 0.0); v.cum_policy.assign(la.size(), 0.0);
    v.cur_policy.assign(la.size(), 1.0 / la.size());
    table[key] = v;
    for (auto a : la) { auto c = s.Clone(); c->ApplyAction(a); Init(*c); }
  }
  PolicyTable Current() const {
    PolicyTable t;
    for (auto& kv : table) t[kv.first] = kv.second.cur_policy;
    return t;
  }
  PolicyTable Average() const {        // CFRAveragePolicy, cfr.cc:104-125
    PolicyTable t;
    for (auto& kv : table) {
      const auto& c = kv.second.cum_policy;
      double sum = 0.0;
      for (double x : c) sum += x;
      std::vector<double> p(c.size());
      for (size_t a = 0; a < c.size(); ++a) p[a] = sum == 0.0 ? 1.0 / c.size() : c[a] / sum;
      t[kv.first] = p;
    }
    return t;
  }
  // ComputeCounterFactualRegret (cfr.cc:331-408) with policy overrides: overrides[q] replaces player q's current policy.
  std::vector<double> Regret(const State& s, int upd, const std::vector<double>& reach, const std::vector<const PolicyTable*>& ov) {
    if (s.IsTerminal()) return s.Returns();
    std::vector<int64_t> acts;
    std::vector<double> probs;
    int cur;
    if (s.IsChanceNode()) {
      for (auto& ap : s.ChanceOutcomes()) { acts.push_back(ap.first); probs.push_back(ap.second); }
      cur = n;
    } else {
      bool all_zero = true;
      for (int i = 0; i < n; ++i) if (reach[i] != 0.0) all_zero = false;
      if (all_zero) return std::vector<double>(n, 0.0);
      cur = s.CurrentPlayer();
      acts = s.LegalActions();
      std::string key = s.InformationStateString(cur);
      probs = ov[cur] ? ov[cur]->at(key) : table[key].cur_policy;
    }
    std::vector<double> value(n), child;
    for (size_t i = 0; i < acts.size(); ++i) {   // ComputeCounterFactualRegretForActionProbs, cfr.cc:443-469
      auto ns = s.Clone();
      ns->ApplyAction(acts[i]);
      std::vector<double> nr(reach);
      nr[cur] *= probs[i];
      auto cv = Regret(*ns, upd, nr, ov);
      for (int k = 0; k < n; ++k) value[k] += probs[i] * cv[k];
      if (cur < n) child.push_back(cv[cur]);
    }
    if (cur == upd) {
      Values& v = table[s.InformationStateString(cur)];
      double self = reach[cur], cfr = 1.0;
      for (size_t i = 0; i < reach.size(); ++i) if ((int)i != cur) cfr *= reach[i];
      for (size_t a = 0; a < acts.size(); ++a) {
        v.regrets[a] += cfr * (child[a] - value[cur]);
        v.cum_policy[a] += self * probs[a];
      }
    }
    return value;
  }
  void Iterate() {                     // CFRBRSolver::EvaluateAndUpdatePolicy, cfr_br.cc:50-82
    ++iteration;
    PolicyTable current = Current();
    const PolicyTable* evaluated = iteration > 1 ? &current : nullptr;   // uniform until SetPolicy runs (iteration_ > 1)
    std::vector<PolicyTable> br;
    for (int p = 0; p < n; ++p) br.push_back(BestResponse(*game, p, evaluated).Policy());
    auto root = game->NewInitialState();
    for (int p = 0; p < n; ++p) {
      std::vector<const PolicyTable*> ov(n, nullptr);
      for (int q = 0; q < n; ++q) if (q != p) ov[q] = &br[q];
      Regret(*root, p, std::vector<double>(n + 1, 1.0), ov);
    }
    for (auto& kv : table) {           // ApplyRegretMatching, cfr.cc:596-615
      Values& v = kv.second;
      double sum = 0.0;
      for (double r : v.regrets) if (r > 0) sum += r;
      for (size_t a = 0; a < v.regrets.size(); ++a)
        v.cur_policy[a] = sum > 0 ? (v.regrets[a] > 0 ? v.regrets[a] / sum : 0) : 1.0 / v.legal.size();
    }
  }
};

// On-policy values of every player (ExpectedReturns with depth_limit -1).
std::vector<double> OnPolicy(const State& s, const PolicyTable& pol, int n) {
  if (s.IsTerminal()) return s.Returns();
  std::vector<int64_t> acts;
  std::vector<double> probs;
  if (s.IsChanceNode()) for (auto& ap : s.ChanceOutcomes()) { acts.push_back(ap.first); probs.push_back(ap.second); }
  else { acts = s.LegalActions(); probs = PolicyAt(s, &pol); }
  std::vector<double> v(n, 0.0);
  for (size_t i = 0; i < acts.size(); ++i) {
    auto c = s.Clone();
    c->ApplyAction(acts[i]);
    auto cv = OnPolicy(*c, pol, n);
    for (int k = 0; k < n; ++k) v[k] += probs[i] * cv[k];
  }
  return v;
}

PolicyTable ReadPolicy(const char* keys, const int* counts, const double* probs, int n_keys, std::vector<std::string>* names) {
  PolicyTable t;
  const char* k = keys;
  for (int i = 0, off = 0; i < n_keys; ++i) {
    const char* e = strchr(k, '\n');
    std::string key(k, e ? e - k : strlen(k));
    k = e ? e + 1 : k + key.size();
    t[key] = std::vector<double>(probs + off, probs + off + counts[i]);
    off += counts[i];
    names->push_back(key);
  }
  return t;
}

}  // namespace
}  // namespace oracle

extern "C" {

void* orc_cfrbr_new(void* game) {
  using namespace oracle;
  auto* c = new CfrBr;
  c->game = (Game*)game;
  c->n = c->game->info.num_players;
  c->Init(*c->game->NewInitialState());
  return c;
}
void orc_cfrbr_free(void* c) { delete (oracle::CfrBr*)c; }
void orc_cfrbr_iterate(void* c, int iters) { for (int i = 0; i < iters; ++i) ((oracle::CfrBr*)c)->Iterate(); }
int orc_cfrbr_iteration(void* c) { return ((oracle::CfrBr*)c)->iteration; }
int orc_cfrbr_num_infosets(void* c) { return (int)((oracle::CfrBr*)c)->table.size(); }
// k-th information state in first-visit order: key string + arrays; returns the number of legal actions.
int orc_cfrbr_get(void* c, int k, char* key, int key_cap, int64_t* legal, double* regrets, double* cum, double* cur, int cap, int* player) {
  auto* s = (oracle::CfrBr*)c;
  if (k < 0 || k >= (int)s->order.size()) return -1;
  const std::string& ks = s->order[k];
  const auto& v = s->table[ks];
  int m = (int)ks.size() < key_cap - 1 ? (int)ks.size() : key_cap - 1;
  memcpy(key, ks.data(), m); key[m] = 0;
  int n = (int)v.legal.size();
  for (int i = 0; i < n && i < cap; ++i) { legal[i] = v.legal[i]; regrets[i] = v.regrets[i]; cum[i] = v.cum_policy[i]; cur[i] = v.cur_policy[i]; }
  if (player) *player = v.player;
  return n;
}
// Overwrite one information state's tables (a deserialized solver, DeserializeCFRInfoStateValuesTable); -1 if unknown.
int orc_cfrbr_set(void* c, const char* key, const double* regrets, const double* cum, const double* cur, int n) {
  auto* s = (oracle::CfrBr*)c;
  auto it = s->table.find(key);
  if (it == s->table.end() || (int)it->second.legal.size() != n) return -1;
  it->second.regrets.assign(regrets, regrets + n);
  it->second.cum_policy.assign(cum, cum + n);
  it->second.cur_policy.assign(cur, cur + n);
  return 0;
}
void orc_cfrbr_set_iteration(void* c, int iteration) { ((oracle::CfrBr*)c)->iteration = iteration; }
// Best-response values of players 0, 1 and on-policy values of players 0, 1 of the average policy (NashConv = sum of the
// differences).
void orc_cfrbr_average_values(void* c, double* out) {
  using namespace oracle;
  auto* s = (CfrBr*)c;
  PolicyTable avg = s->Average();
  for (int p = 0; p < 2; ++p) {
    BestResponse br(*s->game, p, &avg);
    out[p] = br.Value(br.root.get());
  }
  auto v = OnPolicy(*s->game->NewInitialState(), avg, s->n);
  out[2] = v[0]; out[3] = v[1];
}
// TabularBestResponse(game, player, policy) on a policy given as n_keys information states ('\n'-separated keys, counts[i]
// probabilities each in legal-action order, concatenated): actions[i] = the action chosen at key i (-1 where key i is not
// the player's), *value = the best-response value of the initial state.
int orc_tabular_br(void* game, int player, const char* keys, const int* counts, const double* probs, int n_keys,
                   int64_t* actions, double* value) {
  using namespace oracle;
  std::vector<std::string> names;
  PolicyTable pol = ReadPolicy(keys, counts, probs, n_keys, &names);
  BestResponse br(*(Game*)game, player, &pol);
  *value = br.Value(br.root.get());
  for (int i = 0; i < n_keys; ++i) actions[i] = br.infosets.count(names[i]) ? br.BestAction(names[i]) : -1;
  return 0;
}

}  // extern "C"
