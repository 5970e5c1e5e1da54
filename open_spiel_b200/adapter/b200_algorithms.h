// C++ host adapters for the two search / solving loops, with the reference's own constructor signatures, so existing
// OpenSpiel code switches by changing a type name:
//   B200MCTSBot   : open_spiel::Bot           <- algorithms::MCTSBot (mcts.h:149-230) with a RandomRolloutEvaluator
//   B200CFRSolver                             <- algorithms::CFRSolver / CFRPlusSolver (cfr.h:312-357)
//   B200CFRBRSolver                           <- algorithms::CFRBRSolver (cfr_br.h)
// Every computation is a call into the b2s C ABI (libb2s.so); these classes only translate between the reference's
// host objects (State history, TabularPolicy keyed by information-state strings) and device batches / tables.
#ifndef OPEN_SPIEL_B200_ADAPTER_B200_ALGORITHMS_H_
#define OPEN_SPIEL_B200_ADAPTER_B200_ALGORITHMS_H_

#include <memory>
#include <string>
#include <unordered_map>
#include <vector>

#include "b200_games.h"
#include "open_spiel/algorithms/mcts.h"
#include "open_spiel/algorithms/minimax.h"
#include "open_spiel/policy.h"
#include "open_spiel/spiel.h"
#include "open_spiel/spiel_bots.h"

namespace open_spiel {
namespace b200 {

// b2s game id + parameters for a reference Game object (by short name and GetParameters()).
int GameIdAndParams(const Game& game, b2s_params* params);

class B200MCTSBot : public Bot {
 public:
  // Argument order of MCTSBot's constructor (mcts.h:161-169); the evaluator is RandomRolloutEvaluator(n_rollouts, seed).
  B200MCTSBot(const Game& game, int n_rollouts, double uct_c, int max_simulations, int64_t max_memory_mb, bool solve,
              int seed, bool verbose,
              algorithms::ChildSelectionPolicy child_selection_policy = algorithms::ChildSelectionPolicy::UCT);
  ~B200MCTSBot() override;
  Action Step(const State& state) override;
  // MCTSBot::MCTSearch (mcts.cc:353-467): the root SearchNode with one level of children (action, player,
  // explore_count, total_reward, proven outcome) — the statistics BestChild / ChildrenStr / the callers of
  // pyspiel.MCTSBot.mcts_search read; deeper levels stay on the device.
  std::unique_ptr<algorithms::SearchNode> MCTSearch(const State& state);
  void Restart() override {}
  void RestartAt(const State& state) override {}
  // Root statistics of the last Step: visit count per action id (0 for illegal actions).
  const std::vector<int>& LastVisitCounts() const { return visits_; }

 private:
  b2s_params params_;
  b2s_mcts_config cfg_;
  int gid_ = -1;
  int num_actions_ = 0;
  void RootToDevice(const State& state);
  std::shared_ptr<const Game> b200_game_;   // the packed-state twin of `game` (B200Game), for moving roots to the device
  void* batch_ = nullptr;      // one lane: the search root
  void* dev_ = nullptr;        // device scratch: action, visits, rewards, best
  std::vector<int> visits_;
  uint64_t steps_ = 0;
  Action last_best_ = kInvalidAction;
};

// algorithms::AlphaBetaSearch (minimax.h) with the reference's signature.  With no value function, on a game the device search
// serves (b2s_alpha_beta_search: the deterministic b200 games except go 10..19), the root is copied to a one-lane batch and
// solved on the device; reaching depth 0 at a non-terminal state, or kInvalidPlayer on a terminal root, is SpielFatalError as
// in the reference.  Every other call (a value function, any other game) is the stock algorithms::AlphaBetaSearch.
std::pair<double, Action> AlphaBetaSearch(const Game& game, const State* state, std::function<double(const State&)> value_function,
                                          int depth_limit, Player maximizing_player, bool use_undo = true);

class B200CFRSolver {
 public:
  explicit B200CFRSolver(const Game& game, bool cfr_plus = false);
  // extra_create_flags: b2s_cfr_create flags OR-ed in (the MCCFR solvers below create their tables with B2S_CFR_MCCFR_TABLES)
  B200CFRSolver(const Game& game, bool cfr_plus, int extra_create_flags);
  ~B200CFRSolver();
  void EvaluateAndUpdatePolicy();                       // CFRSolverBase::EvaluateAndUpdatePolicy (cfr.cc:263-282)
  void EvaluateAndUpdatePolicy(int iterations);         // ... `iterations` times inside one kernel launch
  TabularPolicy AveragePolicy() const;                  // CFRAveragePolicy (cfr.cc:104-125) as a TabularPolicy
  TabularPolicy CurrentPolicy() const;
  double NashConv() const;                              // on the device (b2s_cfr_nash_conv)
  // checkpoint: iteration counter + the three per-entry tables in device row order (b2s_cfr_export / b2s_cfr_import)
  struct Tables { int iteration = 0; std::vector<double> regrets, cumulative_policy, current_policy; };
  Tables Export() const;
  void Import(const Tables& t);
  bool cfr_plus() const { return cfr_plus_; }
  const Game& game() const { return *game_; }
  int NumInfoStates() const { return info_.num_infosets; }

 protected:
  void* solver_ = nullptr;

 private:
  TabularPolicy PolicyFrom(const std::vector<double>& per_entry, bool normalise) const;
  std::shared_ptr<const Game> game_;
  bool cfr_plus_ = false;
  b2s_cfr_info info_;
  std::vector<std::string> keys_;                       // information-state string of every device table row
  std::vector<int32_t> offsets_, legal_;
};

// CFRBRSolver (cfr_br.h): each iteration both players' pure best responses to the current policy (the uniform policy on
// iteration 1), each player's traversal against the other's best response, then regret matching; tables match the reference
// bit for bit (B2S_CFR_BEST_RESPONSE_OPPONENTS).
class B200CFRBRSolver : public B200CFRSolver {
 public:
  explicit B200CFRBRSolver(const Game& game);
};

// ExternalSamplingMCCFRSolver (external_sampling_mccfr.h:40-95) / OutcomeSamplingMCCFRSolver (outcome_sampling_mccfr.h:40-66,
// default uniform policy, no baseline) with device-resident tables.  `per_update` independent traversals / episodes run in
// parallel per (iteration, player) phase against frozen tables; 1 = the reference's algorithm.  Randomness is the library's
// position-keyed Philox stream (the reference consumes a std::mt19937 sequentially), so runs are reproducible for a seed but
// not sample-path identical to the stock solvers; the table arithmetic is (DESIGN.md 5a).
class B200MCCFRSolver : public B200CFRSolver {
 public:
  enum class Kind { kExternalSampling, kOutcomeSampling };
  B200MCCFRSolver(const Game& game, Kind kind, uint64_t seed, bool full_average = false, double epsilon = 0.6, int per_update = 1);
  void RunIteration() { RunIterations(1); }             // ...::RunIteration() (external_sampling_mccfr.cc:71-80, outcome_sampling_mccfr.cc:60-67)
  void RunIterations(int iterations);
  Kind kind() const { return kind_; }

 private:
  Kind kind_;
  uint64_t seed_;
  bool full_average_;
  double epsilon_;
  int per_update_;
};

}  // namespace b200
}  // namespace open_spiel
#endif
