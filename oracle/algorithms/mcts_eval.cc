// TEST INFRASTRUCTURE ONLY (see oracle/oracle.h).
// CPU restatement of reference open_spiel/algorithms/mcts.{h,cc} MCTSBot::MCTSearch with a deterministic Evaluator (mcts.h:83-92)
// instead of the RandomRolloutEvaluator: the search the device's caller-evaluated MCTS (b2s_mcts_eval_*, csrc/mcts_eval.cuh)
// is checked against.  Structure follows the reference (ApplyTreePolicy :273-351 with Evaluator::Prior at the expansion and the
// root's Dirichlet mix :284-292, Evaluate at a non-terminal leaf :379, backup + solver :384-434, node budget + GarbageCollect
// :441-482, PUCTValue :103-112 with the child's prior, UCTValue :90-101, BestChild / CompareFinal :114-143).
// Random decisions, two sources (as oracle/algorithms/mcts.cc):
//   rng_mode 0: the position-keyed Philox stream shared with the device kernel — expansion #e shuffles the ascending
//               legal list by Fisher-Yates, j = RngUniform(key, e, i, 1, i + 1) for i = n-1..1; the root's Dirichlet noise is
//               the caller's, by action id (root_noise);
//   rng_mode 1: the reference's own MCTSBot::rng_ = std::mt19937(seed): std::shuffle of the new children (mcts.cc:294) and, when
//               dirichlet_alpha > 0, the reference's dirichlet_noise (mcts.cc:188-203: std::gamma_distribution, drawn before the
//               shuffle), so that results can be compared with the unmodified reference bit for bit.
//   key = seed + tree_index * 0x9E3779B97F4A7C15.
// The test evaluator (TestEvaluate / TestPrior) is defined identically in oracle/ref_glue/ref_mcts_eval.cc (a reference
// Evaluator) and in tests/mcts_eval_lib.py (torch).
#include <algorithm>
#include <cmath>
#include <limits>
#include <random>

#include "../oracle.h"
#include "philox.h"

namespace oracle {
namespace {

struct ENode {                     // SearchNode, mcts.h:114-146
  int64_t action = kInvalidAction;
  double prior = 0;
  int player = 0;                  // the player who chose `action`
  int explore_count = 0;
  double total_reward = 0;
  std::vector<double> outcome;
  std::vector<ENode> children;
};

double UctValue(const ENode& n, int parent_explore_count, double uct_c) {   // mcts.cc:90-101
  if (!n.outcome.empty()) return n.outcome[n.player];
  if (n.explore_count == 0) return std::numeric_limits<double>::infinity();
  return n.total_reward / n.explore_count + uct_c * std::sqrt(std::log(parent_explore_count) / n.explore_count);
}

double PuctValue(const ENode& n, int parent_explore_count, double uct_c) {   // mcts.cc:103-112
  if (!n.outcome.empty()) return n.outcome[n.player];
  return ((n.explore_count != 0 ? n.total_reward / n.explore_count : 0) +
          uct_c * n.prior * std::sqrt(parent_explore_count) / (n.explore_count + 1));
}

bool CompareFinal(const ENode& a, const ENode& b) {                        // mcts.cc:114-125
  double out = (a.player >= 0 && a.player < (int)a.outcome.size()) ? a.outcome[a.player] : 0;
  double out_b = (b.player >= 0 && b.player < (int)b.outcome.size()) ? b.outcome[b.player] : 0;
  if (out != out_b) return out < out_b;
  if (a.explore_count != b.explore_count) return a.explore_count < b.explore_count;
  return a.total_reward < b.total_reward;
}

// The test evaluator.  x = ObservationTensor(CurrentPlayer()), I = its non-zero indices:
//   h1 = sum_{i in I} (7i + 3) mod 11,  h2 = sum_{i in I} i mod 13
//   Evaluate = {v, -v}, v = ((h1 mod 9) - 4) / 7.0
//   Prior(a) = w_a / sum_b w_b over the ascending legal actions, w_a = 1 + (h2 + 13a) mod 5
// Integer sums and one correctly rounded division each, so every implementation gives the same doubles; /7.0 makes
// accumulated rewards non-dyadic, so summation order is tested too.
void TestHashes(const State& s, int obs_size, int64_t* h1, int64_t* h2) {
  std::vector<float> x(obs_size);
  s.ObservationTensor(s.CurrentPlayer(), x.data());
  *h1 = 0; *h2 = 0;
  for (int i = 0; i < obs_size; ++i)
    if (x[i] != 0.f) { *h1 += (7 * i + 3) % 11; *h2 += i % 13; }
}
std::vector<double> TestEvaluate(const State& s, int obs_size) {
  int64_t h1, h2;
  TestHashes(s, obs_size, &h1, &h2);
  const double v = (double)(h1 % 9 - 4) / 7.0;
  return {v, -v};
}
std::vector<double> TestPrior(const State& s, int obs_size, const std::vector<int64_t>& legal) {
  int64_t h1, h2;
  TestHashes(s, obs_size, &h1, &h2);
  int64_t total = 0;
  for (auto a : legal) total += 1 + (h2 + 13 * a) % 5;
  std::vector<double> p;
  for (auto a : legal) p.push_back((double)(1 + (h2 + 13 * a) % 5) / (double)total);
  return p;
}

// dirichlet_noise (mcts.cc:188-203)
std::vector<double> DirichletNoise(int count, double alpha, std::mt19937* rng) {
  std::vector<double> noise;
  std::gamma_distribution<double> gamma(alpha, 1.0);
  for (int i = 0; i < count; ++i) noise.push_back(gamma(*rng));
  double sum = 0.0;
  for (double v : noise) sum += v;
  for (double& v : noise) v /= sum;
  return noise;
}

struct EvalSearch {
  int rng_mode = 0;
  std::mt19937 bot_rng;
  uint64_t key;
  double uct_c, max_utility;
  bool puct = false;
  bool solve;
  int obs_size = 0;
  double dirichlet_alpha = 0, dirichlet_epsilon = 0;
  const double* root_noise = nullptr;
  uint32_t expansions = 0;
  int nodes = 1;                   // MCTSBot::nodes_
  int max_nodes = 1;               // MCTSBot::max_nodes_; <= 1: never collect
  int gc_limit = 5;                // MCTSBot::gc_limit_ (MIN_GC_LIMIT, mcts.cc:37)
  int gc_runs = 0;

  void GarbageCollect(ENode* node) {                                       // mcts.cc:469-482
    if (node->children.empty()) return;
    bool clear_children = node->explore_count < gc_limit;
    for (ENode& child : node->children) GarbageCollect(&child);
    if (clear_children) {
      nodes -= (int)node->children.capacity();
      node->children.clear();
      node->children.shrink_to_fit();
    }
  }

  std::unique_ptr<State> TreePolicy(ENode* root, const State& state, std::vector<ENode*>* path) {   // mcts.cc:273-351
    path->push_back(root);
    auto ws = state.Clone();
    ENode* cur = root;
    while (!ws->IsTerminal() && cur->explore_count > 0) {
      if (cur->children.empty()) {
        auto legal = ws->LegalActions();
        std::vector<double> prior = TestPrior(*ws, obs_size, legal);      // Evaluator::Prior
        const bool mix = cur == root && (rng_mode == 1 ? dirichlet_alpha > 0 : root_noise != nullptr);
        if (mix) {                                                        // mcts.cc:284-292
          std::vector<double> noise;
          if (rng_mode == 1) noise = DirichletNoise((int)legal.size(), dirichlet_alpha, &bot_rng);
          else for (auto a : legal) noise.push_back(root_noise[a]);
          for (size_t i = 0; i < legal.size(); ++i) prior[i] = (1 - dirichlet_epsilon) * prior[i] + dirichlet_epsilon * noise[i];
        }
        std::vector<std::pair<int64_t, double>> children;
        for (size_t i = 0; i < legal.size(); ++i) children.push_back({legal[i], prior[i]});
        uint32_t e = expansions++;
        if (rng_mode == 1) std::shuffle(children.begin(), children.end(), bot_rng);
        else for (int i = (int)children.size() - 1; i >= 1; --i) std::swap(children[i], children[RngUniform(key, e, i, 1, i + 1)]);
        int player = ws->CurrentPlayer();
        cur->children.reserve(children.size());
        for (auto& ap : children) { ENode c; c.action = ap.first; c.prior = ap.second; c.player = player; cur->children.push_back(c); }
        nodes += (int)cur->children.capacity();
      }
      ENode* chosen = nullptr;
      double max_value = -std::numeric_limits<double>::infinity();
      for (ENode& child : cur->children) {
        double val = puct ? PuctValue(child, cur->explore_count, uct_c) : UctValue(child, cur->explore_count, uct_c);
        if (val > max_value) { max_value = val; chosen = &child; }
      }
      cur = chosen;
      ws->ApplyAction(chosen->action);
      path->push_back(cur);
    }
    return ws;
  }

  int Run(ENode* root, const State& state, int max_simulations) {         // mcts.cc:353-467
    std::vector<ENode*> path;
    int i = 0;
    for (; i < max_simulations; ++i) {
      path.clear();
      auto ws = TreePolicy(root, state, &path);
      std::vector<double> returns;
      bool solved;
      if (ws->IsTerminal()) {
        returns = ws->Returns();
        path.back()->outcome = returns;
        solved = solve;
      } else {
        returns = TestEvaluate(*ws, obs_size);                            // Evaluator::Evaluate
        solved = false;
      }
      while (!path.empty()) {
        ENode* node = path.back();
        node->total_reward += returns[node->player];
        node->explore_count += 1;
        path.pop_back();
        if (solved && !node->children.empty()) {
          int player = node->children[0].player;
          const ENode* best = nullptr;
          bool all_solved = true;
          for (const ENode& child : node->children) {
            if (child.outcome.empty()) all_solved = false;
            else if (best == nullptr || child.outcome[player] > best->outcome[player]) best = &child;
          }
          if (best != nullptr && (all_solved || best->outcome[player] == max_utility)) node->outcome = best->outcome;
          else solved = false;
        }
      }
      if (!root->outcome.empty() || root->children.size() == 1) { ++i; break; }
      if (max_nodes > 1 && nodes >= max_nodes) {
        GarbageCollect(root);
        ++gc_runs;
        gc_limit *= (nodes > max_nodes / 2 ? 1.25 : 0.9);                 // int *= double, as the reference's int gc_limit_
        gc_limit = std::max(5, gc_limit);
      }
    }
    return i;
  }
};

}  // namespace
}  // namespace oracle

extern "C" {

// One MCTSearch with the test evaluator from `state` for tree #tree_index.  Root children in child (shuffled) order:
// child_actions/visits/rewards/outcome_p0 (NaN when unproven); returns the number of root children.  max_nodes =
// MCTSBot::max_nodes_ (<= 1: no garbage collection).  root_noise (rng_mode 0, nullable, [num_distinct_actions] by action id)
// or dirichlet_alpha (rng_mode 1), with dirichlet_epsilon: the root's Dirichlet noise.
int orc_mcts_eval_search(void* game, void* state, double uct_c, int max_simulations, int solve, uint64_t seed, uint64_t tree_index,
                         int child_selection_policy, int rng_mode, int max_nodes, const double* root_noise, double dirichlet_alpha,
                         double dirichlet_epsilon, int64_t* child_actions, int* child_visits, double* child_rewards,
                         double* child_outcome_p0, int cap, int64_t* best_action, int* root_visits, int* sims_run, int* gc_runs_out) {
  using namespace oracle;
  Game* g = (Game*)game;
  State* s = (State*)state;
  EvalSearch srch;
  srch.key = seed + tree_index * 0x9E3779B97F4A7C15ull;
  srch.uct_c = uct_c;
  srch.max_utility = g->info.max_utility;
  srch.solve = solve != 0;
  srch.puct = child_selection_policy == 1;
  srch.rng_mode = rng_mode;
  srch.max_nodes = max_nodes;
  srch.obs_size = g->info.observation_tensor_size;
  srch.root_noise = root_noise;
  srch.dirichlet_alpha = dirichlet_alpha;
  srch.dirichlet_epsilon = dirichlet_epsilon;
  if (rng_mode == 1) srch.bot_rng.seed((uint32_t)seed);
  ENode root;
  root.player = s->CurrentPlayer();
  int ran = srch.Run(&root, *s, max_simulations);
  int n = (int)root.children.size();
  for (int i = 0; i < n && i < cap; ++i) {
    child_actions[i] = root.children[i].action;
    child_visits[i] = root.children[i].explore_count;
    child_rewards[i] = root.children[i].total_reward;
    child_outcome_p0[i] = root.children[i].outcome.empty() ? std::nan("") : root.children[i].outcome[0];
  }
  *best_action = kInvalidAction;
  if (n) {
    const ENode* best = &root.children[0];
    for (int i = 1; i < n; ++i) if (CompareFinal(*best, root.children[i])) best = &root.children[i];   // std::max_element
    *best_action = best->action;
  }
  *root_visits = root.explore_count;
  *sims_run = ran;
  *gc_runs_out = srch.gc_runs;
  return n;
}

// The test evaluator on one state: values [num_players] and priors [num_distinct_actions] by action id (0 if illegal).
void orc_mcts_eval_test_evaluator(void* game, void* state, double* values, double* priors) {
  using namespace oracle;
  Game* g = (Game*)game;
  State* s = (State*)state;
  auto v = TestEvaluate(*s, g->info.observation_tensor_size);
  values[0] = v[0]; values[1] = v[1];
  for (int a = 0; a < g->info.num_distinct_actions; ++a) priors[a] = 0.0;
  auto legal = s->LegalActions();
  auto p = TestPrior(*s, g->info.observation_tensor_size, legal);
  for (size_t i = 0; i < legal.size(); ++i) priors[legal[i]] = p[i];
}

}  // extern "C"
