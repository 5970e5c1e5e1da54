// TEST INFRASTRUCTURE ONLY.  The UNMODIFIED reference's MCTSBot (algorithms/mcts.h:149-230) driven by a deterministic
// Evaluator (mcts.h:83-92): the test evaluator of oracle/algorithms/mcts_eval.cc as a reference Evaluator subclass.  Built by
// oracle/ref_eval.mk into oracle/_ref/libspiel_ref_mcts_eval.so, linked against the reference inside
// oracle/_ref/libspiel_ref_c.so (oracle/ref_build.mk).  The entry point loads the game and replays the root's history itself.
#include <memory>
#include <stdexcept>
#include <string>
#include <vector>

#include "open_spiel/algorithms/mcts.h"
#include "open_spiel/spiel.h"
#include "open_spiel/spiel_utils.h"

using open_spiel::Action;
using open_spiel::State;

namespace {
thread_local std::string g_err;
void ThrowingHandler(const std::string& msg) { throw std::runtime_error(msg); }
struct Init { Init() { open_spiel::SetErrorHandler(ThrowingHandler); } } g_init;

// x = ObservationTensor(CurrentPlayer()), I = its non-zero indices: h1 = sum (7i + 3) mod 11, h2 = sum i mod 13;
// Evaluate = {v, -v}, v = ((h1 mod 9) - 4) / 7.0; Prior(a) = w_a / sum_b w_b over the legal actions, w_a = 1 + (h2 + 13a) mod 5
class TestEvaluator : public open_spiel::algorithms::Evaluator {
 public:
  std::vector<double> Evaluate(const State& state) override {
    int64_t h1, h2;
    Hashes(state, &h1, &h2);
    const double v = (double)(h1 % 9 - 4) / 7.0;
    return {v, -v};
  }
  open_spiel::ActionsAndProbs Prior(const State& state) override {
    int64_t h1, h2;
    Hashes(state, &h1, &h2);
    std::vector<Action> legal = state.LegalActions();
    int64_t total = 0;
    for (Action a : legal) total += 1 + (h2 + 13 * a) % 5;
    open_spiel::ActionsAndProbs prior;
    for (Action a : legal) prior.emplace_back(a, (double)(1 + (h2 + 13 * a) % 5) / (double)total);
    return prior;
  }

 private:
  static void Hashes(const State& state, int64_t* h1, int64_t* h2) {
    std::vector<float> x = state.ObservationTensor(state.CurrentPlayer());
    *h1 = 0; *h2 = 0;
    for (int i = 0; i < (int)x.size(); ++i)
      if (x[i] != 0.f) { *h1 += (7 * i + 3) % 11; *h2 += i % 13; }
  }
};
}  // namespace

extern "C" {

const char* refe_last_error() { return g_err.c_str(); }
int refe_sizeof_search_node() { return (int)sizeof(open_spiel::algorithms::SearchNode); }

// MCTSBot::MCTSearch with the test evaluator from the position after `history` of `game_string`: UCT or PUCT, Dirichlet noise at
// the root (dirichlet_alpha / dirichlet_epsilon), the node budget of max_memory_mb.  Reports the root's children in child
// order (action, visits, total reward), BestChild and the root's visit count; returns the number of children, -1 on error.
int refe_mcts_eval_search(const char* game_string, const int64_t* history, int n_history, double uct_c, int max_simulations,
                          int solve, int seed, int child_selection_policy, double dirichlet_alpha, double dirichlet_epsilon,
                          int max_memory_mb, int64_t* child_actions, int* child_visits, double* child_rewards, int cap,
                          int64_t* best_action, int* root_visits) {
  try {
    std::shared_ptr<const open_spiel::Game> game = open_spiel::LoadGame(std::string(game_string));
    std::unique_ptr<State> state = game->NewInitialState();
    for (int i = 0; i < n_history; ++i) state->ApplyAction(history[i]);
    open_spiel::algorithms::MCTSBot bot(*game, std::make_shared<TestEvaluator>(), uct_c, max_simulations, max_memory_mb, solve != 0,
                                        seed, /*verbose=*/false,
                                        child_selection_policy == 1 ? open_spiel::algorithms::ChildSelectionPolicy::PUCT
                                                                    : open_spiel::algorithms::ChildSelectionPolicy::UCT,
                                        dirichlet_alpha, dirichlet_epsilon);
    std::unique_ptr<open_spiel::algorithms::SearchNode> root = bot.MCTSearch(*state);
    int n = (int)root->children.size();
    for (int i = 0; i < n && i < cap; ++i) {
      child_actions[i] = root->children[i].action;
      child_visits[i] = root->children[i].explore_count;
      child_rewards[i] = root->children[i].total_reward;
    }
    *best_action = root->BestChild().action;
    *root_visits = root->explore_count;
    return n;
  } catch (const std::exception& e) { g_err = e.what(); return -1; }
}

}  // extern "C"
