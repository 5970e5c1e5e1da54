#include "b200_algorithms.h"

#include <algorithm>
#include <cstring>
#include <functional>

namespace open_spiel {
namespace b200 {
namespace {

void Check(int rc) {
  if (rc != 0) SpielFatalError(std::string("b2s: ") + b2s_last_error());
}

}  // namespace

int GameIdAndParams(const Game& game, b2s_params* p) {
  const std::string name = game.GetType().short_name;
  const GameParameters params = game.GetParameters();
  b2s_params_default(p);
  auto geti = [&](const char* k, int32_t* out) {
    auto it = params.find(k);
    if (it == params.end()) return;
    if (it->second.has_int_value()) *out = it->second.int_value();
    else if (it->second.has_bool_value()) *out = it->second.bool_value() ? 1 : 0;
  };
  auto getd = [&](const char* k, double* out) {
    auto it = params.find(k);
    if (it != params.end() && it->second.has_double_value()) *out = it->second.double_value();
  };
  geti("rows", &p->rows); geti("columns", &p->columns); geti("x_in_row", &p->x_in_row);
  geti("egocentric_obs_tensor", &p->egocentric_obs_tensor);
  geti("board_size", &p->board_size); geti("swap", &p->swap); geti("plain_obs_tensor", &p->plain_obs_tensor);
  geti("num_rows", &p->rows); geti("num_cols", &p->columns);
  geti("handicap", &p->handicap); geti("max_game_length", &p->max_game_length); getd("komi", &p->komi);
  geti("players", &p->players); geti("starting_player", &p->starting_player);
  int gid = b2s_game_id(name.c_str());
  if (gid < 0) SpielFatalError("b200: unsupported game " + name);
  return gid;
}

// ---- AlphaBetaSearch -------------------------------------------------------------------------------------------
std::pair<double, Action> AlphaBetaSearch(const Game& game, const State* state, std::function<double(const State&)> value_function,
                                          int depth_limit, Player maximizing_player, bool use_undo) {
  const int gid = value_function ? -1 : b2s_game_id(game.GetType().short_name.c_str());
  std::shared_ptr<const Game> packed_game = gid >= 0 ? B200Game::Create(game.GetType(), game.GetParameters()) : nullptr;
  // kInvalidPlayer (the root's mover) is the C ABI's -1
  b2s_alpha_beta_config cfg = {depth_limit, maximizing_player == kInvalidPlayer ? -1 : maximizing_player, 0};
  void* batch = nullptr;
  if (packed_game && (maximizing_player == kInvalidPlayer || maximizing_player == 0 || maximizing_player == 1)) {
    // the packed game's own parameters (it reads every game's, e.g. mnk's m, n, k)
    const B200Game& pg = static_cast<const B200Game&>(*packed_game);
    Check(b2s_batch_create(gid, &pg.cparams(), 1, 0, &batch));
    // a search of no roots checks only the game: kuhn_poker, leduc_poker and go 10..19 are not served on the device
    if (b2s_alpha_beta_search(batch, 0, &cfg, nullptr, nullptr, nullptr, nullptr, nullptr) != 0) {
      b2s_batch_destroy(batch);
      batch = nullptr;
    }
  }
  if (!batch) return algorithms::AlphaBetaSearch(game, state, value_function, depth_limit, maximizing_player, use_undo);
  // the root as a packed lane, rebuilt from its history when it is not a B200State (as B200MCTSBot::RootToDevice)
  std::unique_ptr<State> root = packed_game->NewInitialState();
  const B200State* packed = state ? dynamic_cast<const B200State*>(state) : nullptr;
  if (!packed) {
    if (state)
      for (Action a : state->History()) root->ApplyAction(a);
    packed = static_cast<const B200State*>(root.get());
  }
  packed->ToBatchLane(batch, 0);
  void* dev = nullptr;
  Check(b2s_device_alloc(0, &dev, 32));
  char* d = (char*)dev;
  Check(b2s_alpha_beta_search(batch, 1, &cfg, (double*)d, (int32_t*)(d + 16), (int64_t*)(d + 8), (uint8_t*)(d + 20), nullptr));
  char out[32];
  Check(b2s_memcpy_d2h(0, out, dev, sizeof out, nullptr));
  Check(b2s_stream_synchronize(0, nullptr));
  b2s_device_free(0, dev);
  b2s_batch_destroy(batch);
  double value;
  int32_t best;
  memcpy(&value, out, sizeof value);
  memcpy(&best, out + 16, sizeof best);
  switch ((uint8_t)out[20]) {
    case 2: SpielFatalError("We assume we can walk the full depth of the tree. Try increasing depth or provide a value_function.");
    case 3: SpielFatalError("AlphaBetaSearch: maximizing_player is kInvalidPlayer at a terminal state");
  }
  return {value, (Action)best};
}

// ---- MCTS ------------------------------------------------------------------------------------------------------
B200MCTSBot::B200MCTSBot(const Game& game, int n_rollouts, double uct_c, int max_simulations, int64_t max_memory_mb,
                         bool solve, int seed, bool verbose, algorithms::ChildSelectionPolicy policy) {
  gid_ = GameIdAndParams(game, &params_);
  num_actions_ = game.NumDistinctActions();
  memset(&cfg_, 0, sizeof cfg_);
  cfg_.max_simulations = max_simulations;
  cfg_.n_rollouts = n_rollouts;
  cfg_.solve = solve ? 1 : 0;
  cfg_.child_selection_policy = policy == algorithms::ChildSelectionPolicy::PUCT ? B2S_MCTS_PUCT : B2S_MCTS_UCT;
  cfg_.uct_c = uct_c;
  cfg_.seed = (uint64_t)seed;
  // MCTSBot::max_nodes_ (mcts.cc:214): the node budget that triggers the garbage collector
  cfg_.max_nodes_per_tree = max_memory_mb > 0 ? (max_memory_mb << 20) / (int64_t)sizeof(algorithms::SearchNode) + 1 : 0;
  b200_game_ = B200Game::Create(game.GetType(), game.GetParameters());
  if (!b200_game_) SpielFatalError("b200: " + game.ToString() + " does not fit the packed device layouts");
  Check(b2s_batch_create(gid_, &params_, 1, 0, &batch_));
  Check(b2s_device_alloc(0, &dev_, 64 + (2 * sizeof(int32_t) + sizeof(double) + sizeof(float)) * (size_t)(num_actions_ + 2)));
  visits_.assign(num_actions_, 0);
}

B200MCTSBot::~B200MCTSBot() {
  if (batch_) b2s_batch_destroy(batch_);
  if (dev_) b2s_device_free(0, dev_);
}

// The search root: the reference state as a packed lane.  A B200State is copied as it is; any other State of the same
// game (e.g. the stock C++ state) is rebuilt from its action history on the host rule core first.
void B200MCTSBot::RootToDevice(const State& state) {
  const B200State* packed = dynamic_cast<const B200State*>(&state);
  std::unique_ptr<State> rebuilt;
  if (!packed) {
    rebuilt = b200_game_->NewInitialState();
    for (Action a : state.History()) rebuilt->ApplyAction(a);
    packed = static_cast<const B200State*>(rebuilt.get());
  }
  packed->ToBatchLane(batch_, 0);
}

std::unique_ptr<algorithms::SearchNode> B200MCTSBot::MCTSearch(const State& state) {
  if (state.IsTerminal()) SpielFatalError("b200: MCTS called on a terminal state");
  char* d = (char*)dev_;
  int32_t* best_d = (int32_t*)(d + 16);
  int32_t* visits_d = (int32_t*)(d + 64);
  const size_t A = (size_t)num_actions_, A2 = (A + 1) & ~(size_t)1;
  double* reward_d = (double*)(d + 64 + sizeof(int32_t) * A2);
  float* outcome_d = (float*)(d + 64 + sizeof(int32_t) * A2 + sizeof(double) * A);
  RootToDevice(state);
  cfg_.tree_index_offset = (int64_t)steps_++;            // a fresh random stream per move, like the bot's advancing rng_
  Check(b2s_mcts_search(batch_, 1, &cfg_, visits_d, reward_d, outcome_d, best_d, nullptr, nullptr));
  std::vector<double> reward(A);
  std::vector<float> outcome(A);
  int32_t best = -1;
  Check(b2s_memcpy_d2h(0, &best, best_d, sizeof best, nullptr));
  Check(b2s_memcpy_d2h(0, visits_.data(), visits_d, sizeof(int32_t) * A, nullptr));
  Check(b2s_memcpy_d2h(0, reward.data(), reward_d, sizeof(double) * A, nullptr));
  Check(b2s_memcpy_d2h(0, outcome.data(), outcome_d, sizeof(float) * A, nullptr));
  Check(b2s_stream_synchronize(0, nullptr));
  const Player mover = state.CurrentPlayer();
  auto root = std::make_unique<algorithms::SearchNode>(kInvalidAction, mover, 1.0);
  std::vector<Action> legal = state.LegalActions();
  // The device keeps the children in its own (random) expansion order and resolves BestChild ties in that order;
  // its choice goes first here so that SearchNode::BestChild (first maximum) returns the same child.
  for (size_t i = 0; i < legal.size(); ++i)
    if (legal[i] == best) std::rotate(legal.begin(), legal.begin() + i, legal.begin() + i + 1);
  last_best_ = best;
  for (Action a : legal) {
    algorithms::SearchNode child(a, mover, 1.0 / (double)legal.size());     // uniform prior, mcts.cc:74-87
    child.explore_count = visits_[a];
    child.total_reward = reward[a];
    if (outcome[a] == outcome[a]) child.outcome = {(double)outcome[a], -(double)outcome[a]};   // proven (NaN = not)
    root->explore_count += visits_[a];
    root->children.push_back(std::move(child));
  }
  root->explore_count += 1;                               // the root's own first visit
  return root;
}

Action B200MCTSBot::Step(const State& state) {
  MCTSearch(state);
  if (last_best_ < 0) SpielFatalError("b200: MCTS found no action");
  return last_best_;
}

// ---- CFR -------------------------------------------------------------------------------------------------------
B200CFRSolver::B200CFRSolver(const Game& game, bool cfr_plus) : B200CFRSolver(game, cfr_plus, 0) {}

B200CFRSolver::B200CFRSolver(const Game& game, bool cfr_plus, int extra_create_flags) : game_(game.shared_from_this()), cfr_plus_(cfr_plus) {
  b2s_params p;
  int gid = GameIdAndParams(game, &p);
  Check(b2s_cfr_create(gid, &p, (cfr_plus ? (B2S_CFR_LINEAR_AVERAGING | B2S_CFR_REGRET_MATCHING_PLUS) : 0) | extra_create_flags, 0, &solver_));
  Check(b2s_cfr_info_get(solver_, &info_));
  const int I = info_.num_infosets, E = info_.num_entries, T = info_.key_floats;
  offsets_.resize(I + 1); legal_.resize(E);
  std::vector<float> keys((size_t)I * T);
  Check(b2s_cfr_export(solver_, nullptr, nullptr, nullptr, offsets_.data(), legal_.data(), nullptr, keys.data(), nullptr));
  // The device keys its rows by information-state TENSOR, the reference's policies by information-state STRING: walk the
  // stock game tree once on the host and pair the two for every decision node.
  std::unordered_map<std::string, std::string> tensor_to_string;
  std::function<void(const State&)> walk = [&](const State& s) {
    if (s.IsTerminal()) return;
    if (!s.IsChanceNode()) {
      Player pl = s.CurrentPlayer();
      std::vector<float> t = s.InformationStateTensor(pl);
      tensor_to_string.emplace(std::string((const char*)t.data(), sizeof(float) * t.size()), s.InformationStateString(pl));
    }
    for (Action a : s.LegalActions()) walk(*s.Child(a));
  };
  walk(*game.NewInitialState());
  keys_.resize(I);
  for (int i = 0; i < I; ++i) {
    auto it = tensor_to_string.find(std::string((const char*)&keys[(size_t)i * T], sizeof(float) * T));
    if (it == tensor_to_string.end()) SpielFatalError("b200: device information state without a host counterpart");
    keys_[i] = it->second;
  }
}

B200CFRSolver::~B200CFRSolver() { if (solver_) b2s_cfr_destroy(solver_); }

void B200CFRSolver::EvaluateAndUpdatePolicy() { EvaluateAndUpdatePolicy(1); }
void B200CFRSolver::EvaluateAndUpdatePolicy(int iterations) {
  Check(b2s_cfr_iterate(solver_, iterations, nullptr));
  Check(b2s_stream_synchronize(0, nullptr));
}

TabularPolicy B200CFRSolver::PolicyFrom(const std::vector<double>& v, bool normalise) const {
  std::unordered_map<std::string, ActionsAndProbs> table;
  for (int i = 0; i < info_.num_infosets; ++i) {
    const int lo = offsets_[i], hi = offsets_[i + 1];
    double sum = 0.0;
    for (int k = lo; k < hi; ++k) sum += v[k];
    ActionsAndProbs ap;
    for (int k = lo; k < hi; ++k) {
      double p = !normalise ? v[k] : (sum > 0 ? v[k] / sum : 1.0 / (hi - lo));   // GetStatePolicyFromInformationStateValues, cfr.cc:104-125
      ap.push_back({legal_[k], p});
    }
    table.emplace(keys_[i], ap);
  }
  return TabularPolicy(table);
}

TabularPolicy B200CFRSolver::AveragePolicy() const {
  std::vector<double> cum(info_.num_entries);
  Check(b2s_cfr_export(solver_, nullptr, cum.data(), nullptr, nullptr, nullptr, nullptr, nullptr, nullptr));
  return PolicyFrom(cum, true);
}

TabularPolicy B200CFRSolver::CurrentPolicy() const {
  std::vector<double> cur(info_.num_entries);
  Check(b2s_cfr_export(solver_, nullptr, nullptr, cur.data(), nullptr, nullptr, nullptr, nullptr, nullptr));
  return PolicyFrom(cur, false);
}

B200CFRSolver::Tables B200CFRSolver::Export() const {
  Tables t;
  b2s_cfr_info info;
  Check(b2s_cfr_info_get(solver_, &info));
  t.iteration = info.iteration;
  t.regrets.resize(info_.num_entries); t.cumulative_policy.resize(info_.num_entries); t.current_policy.resize(info_.num_entries);
  Check(b2s_cfr_export(solver_, t.regrets.data(), t.cumulative_policy.data(), t.current_policy.data(), nullptr, nullptr, nullptr, nullptr, nullptr));
  return t;
}

void B200CFRSolver::Import(const Tables& t) {
  if ((int)t.regrets.size() != info_.num_entries || (int)t.cumulative_policy.size() != info_.num_entries ||
      (int)t.current_policy.size() != info_.num_entries)
    SpielFatalError("b200: CFR checkpoint does not match this game's table size");
  Check(b2s_cfr_import(solver_, t.regrets.data(), t.cumulative_policy.data(), t.current_policy.data(), t.iteration, nullptr));
  Check(b2s_stream_synchronize(0, nullptr));
}

B200CFRBRSolver::B200CFRBRSolver(const Game& game) : B200CFRSolver(game, false, B2S_CFR_BEST_RESPONSE_OPPONENTS) {}

B200MCCFRSolver::B200MCCFRSolver(const Game& game, Kind kind, uint64_t seed, bool full_average, double epsilon, int per_update)
    : B200CFRSolver(game, false, B2S_CFR_MCCFR_TABLES), kind_(kind), seed_(seed), full_average_(full_average), epsilon_(epsilon),
      per_update_(per_update < 1 ? 1 : per_update) {}

void B200MCCFRSolver::RunIterations(int iterations) {
  if (kind_ == Kind::kExternalSampling)
    Check(b2s_mccfr_external_iterate_ex(solver_, iterations, per_update_, seed_, full_average_ ? B2S_MCCFR_FULL_AVERAGE : 0, nullptr));
  else
    Check(b2s_mccfr_outcome_iterate(solver_, iterations, per_update_, seed_, epsilon_, nullptr));
  Check(b2s_stream_synchronize(0, nullptr));
}

double B200CFRSolver::NashConv() const {
  double nc = 0, vals[4];
  Check(b2s_cfr_nash_conv(solver_, 1, &nc, vals, nullptr));
  return nc;
}

}  // namespace b200
}  // namespace open_spiel
