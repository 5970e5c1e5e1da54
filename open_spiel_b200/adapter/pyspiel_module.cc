// pyspiel-compatible Python module for the b2s path (pybind11): the surface SURVEY §8(b) lists —
// pyspiel.load_game, Game, State, MCTSBot / RandomRolloutEvaluator / SearchNode, CFRSolver / CFRPlusSolver / CFRBRSolver, policies,
// exploitability — over the unmodified reference library plus the B200 drop-ins, which this module registers over the
// stock tic_tac_toe / connect_four / breakthrough / hex / go / kuhn_poker / leduc_poker at import time, so
// `pyspiel.load_game("go(board_size=9)")` returns a B200Game.  Method names and argument orders are those of
// open_spiel/python/pybind11/pyspiel.cc:355-476 (State), :478-560 (Game), :720-735 (load_game), bots.cc:106-149
// (MCTSBot) and policy.cc:224-245 (CFRSolver); bodies are thin calls into the C++ API.
// Scalar State methods run on the host rule cores; MCTSBot and CFRSolver run on the GPU through libb2s.so.
#include <pybind11/numpy.h>
#include <pybind11/pybind11.h>
#include <pybind11/stl.h>

#include <memory>
#include <string>

#include "b200_algorithms.h"
#include "b200_games.h"
#include "open_spiel/algorithms/cfr.h"
#include "open_spiel/algorithms/mcts.h"
#include "open_spiel/algorithms/external_sampling_mccfr.h"
#include "open_spiel/algorithms/outcome_sampling_mccfr.h"
#include "open_spiel/algorithms/tabular_exploitability.h"
#include "open_spiel/observer.h"
#include "open_spiel/policy.h"
#include "open_spiel/spiel.h"

namespace py = pybind11;
using namespace open_spiel;

namespace {

class SpielException : public std::exception {
 public:
  explicit SpielException(std::string msg) : msg_(std::move(msg)) {}
  const char* what() const noexcept override { return msg_.c_str(); }
 private:
  std::string msg_;
};

// GameParameter <-> Python (game_parameters.h:31-120): bool / int / float / str / nested dict
py::object ParamToPy(const GameParameter& p);
py::dict ParamsToPy(const GameParameters& params) {
  py::dict d;
  for (const auto& kv : params) d[py::str(kv.first)] = ParamToPy(kv.second);
  return d;
}
py::object ParamToPy(const GameParameter& p) {
  if (p.has_bool_value()) return py::bool_(p.bool_value());
  if (p.has_int_value()) return py::int_(p.int_value());
  if (p.has_double_value()) return py::float_(p.double_value());
  if (p.has_string_value()) return py::str(p.string_value());
  if (p.has_game_value()) return ParamsToPy(p.game_value());
  return py::none();
}
GameParameters ParamsFromPy(const py::dict& d);
GameParameter ParamFromPy(const py::handle& h) {
  if (py::isinstance<py::bool_>(h)) return GameParameter(h.cast<bool>());
  if (py::isinstance<py::int_>(h)) return GameParameter(h.cast<int>());
  if (py::isinstance<py::float_>(h)) return GameParameter(h.cast<double>());
  if (py::isinstance<py::str>(h)) return GameParameter(h.cast<std::string>());
  if (py::isinstance<py::dict>(h)) return GameParameter(ParamsFromPy(h.cast<py::dict>()));
  throw SpielException("unsupported game parameter type");
}
GameParameters ParamsFromPy(const py::dict& d) {
  GameParameters params;
  for (auto kv : d) params[kv.first.cast<std::string>()] = ParamFromPy(kv.second);
  return params;
}

std::shared_ptr<Game> Mutable(std::shared_ptr<const Game> g) { return std::const_pointer_cast<Game>(g); }

// RandomRolloutEvaluator whose arguments stay readable (the reference keeps them private): MCTSBot moves the search
// to the device when it is given one of these and stays on the stock host MCTSBot for any other Evaluator.
class DeviceRolloutEvaluator : public algorithms::RandomRolloutEvaluator {
 public:
  DeviceRolloutEvaluator(int n_rollouts, int seed) : algorithms::RandomRolloutEvaluator(n_rollouts, seed), n_rollouts(n_rollouts), seed(seed) {}
  const int n_rollouts, seed;
};

class PyMCTSBot {
 public:
  PyMCTSBot(std::shared_ptr<const Game> game, std::shared_ptr<algorithms::Evaluator> evaluator, double uct_c, int max_simulations,
            int64_t max_memory_mb, bool solve, int seed, bool verbose, algorithms::ChildSelectionPolicy policy,
            double dirichlet_alpha, double dirichlet_epsilon, bool dont_return_chance_node, double max_wall_clock_time)
      : game_(game) {
    auto rollout = std::dynamic_pointer_cast<DeviceRolloutEvaluator>(evaluator);
    const bool device_ok = rollout && dirichlet_alpha == 0 && max_wall_clock_time == 0 &&
                           game->GetType().chance_mode == GameType::ChanceMode::kDeterministic &&
                           dynamic_cast<const b200::B200Game*>(game.get()) != nullptr;
    if (device_ok) {
      device_ = std::make_unique<b200::B200MCTSBot>(*game, rollout->n_rollouts, uct_c, max_simulations, max_memory_mb, solve, seed,
                                                     verbose, policy);
    } else {   // the Evaluator plug point (mcts.h:83-92), Dirichlet noise, wall-clock budgets, chance nodes: stock host search
      host_ = std::make_unique<algorithms::MCTSBot>(*game, evaluator, uct_c, max_simulations, max_memory_mb, solve, seed, verbose,
                                                     policy, dirichlet_alpha, dirichlet_epsilon, dont_return_chance_node,
                                                     max_wall_clock_time);
    }
  }
  Action Step(const State& state) { return device_ ? device_->Step(state) : host_->Step(state); }
  std::unique_ptr<algorithms::SearchNode> MCTSearch(const State& state) {
    return device_ ? device_->MCTSearch(state) : host_->MCTSearch(state);
  }
  bool on_device() const { return device_ != nullptr; }

 private:
  std::shared_ptr<const Game> game_;
  std::unique_ptr<b200::B200MCTSBot> device_;
  std::unique_ptr<algorithms::MCTSBot> host_;
};

py::dict PolicyDict(const ActionsAndProbs& ap) {
  py::dict d;
  for (const auto& [a, p] : ap) d[py::int_(a)] = p;
  return d;
}

}  // namespace

PYBIND11_MODULE(pyspiel, m) {
  m.doc() = "pyspiel-compatible module over the B200 (b2s) drop-in games and device search / solving loops";

  // SpielFatalError -> exception -> pyspiel.SpielError (pyspiel.cc:131-160, 831-837)
  SetErrorHandler([](const std::string& msg) { throw SpielException(msg); });
  py::register_exception<SpielException>(m, "SpielError", PyExc_RuntimeError);

  b200::RegisterB200Games();

  py::enum_<PlayerId>(m, "PlayerId")
      .value("DEFAULT_PLAYER_ID", PlayerId::kDefaultPlayerId).value("INVALID", PlayerId::kInvalidPlayer)
      .value("TERMINAL", PlayerId::kTerminalPlayerId).value("CHANCE", PlayerId::kChancePlayerId)
      .value("MEAN_FIELD", PlayerId::kMeanFieldPlayerId).value("SIMULTANEOUS", PlayerId::kSimultaneousPlayerId);
  m.attr("INVALID_ACTION") = py::int_(kInvalidAction);

  py::class_<GameType> game_type(m, "GameType");
  py::enum_<GameType::Dynamics>(game_type, "Dynamics")
      .value("SEQUENTIAL", GameType::Dynamics::kSequential).value("SIMULTANEOUS", GameType::Dynamics::kSimultaneous)
      .value("MEAN_FIELD", GameType::Dynamics::kMeanField);
  py::enum_<GameType::ChanceMode>(game_type, "ChanceMode")
      .value("DETERMINISTIC", GameType::ChanceMode::kDeterministic)
      .value("EXPLICIT_STOCHASTIC", GameType::ChanceMode::kExplicitStochastic)
      .value("SAMPLED_STOCHASTIC", GameType::ChanceMode::kSampledStochastic);
  py::enum_<GameType::Information>(game_type, "Information")
      .value("ONE_SHOT", GameType::Information::kOneShot)
      .value("PERFECT_INFORMATION", GameType::Information::kPerfectInformation)
      .value("IMPERFECT_INFORMATION", GameType::Information::kImperfectInformation);
  py::enum_<GameType::Utility>(game_type, "Utility")
      .value("ZERO_SUM", GameType::Utility::kZeroSum).value("CONSTANT_SUM", GameType::Utility::kConstantSum)
      .value("GENERAL_SUM", GameType::Utility::kGeneralSum).value("IDENTICAL", GameType::Utility::kIdentical);
  py::enum_<GameType::RewardModel>(game_type, "RewardModel")
      .value("REWARDS", GameType::RewardModel::kRewards).value("TERMINAL", GameType::RewardModel::kTerminal);
  game_type.def_readonly("short_name", &GameType::short_name)
      .def_readonly("long_name", &GameType::long_name)
      .def_readonly("dynamics", &GameType::dynamics)
      .def_readonly("chance_mode", &GameType::chance_mode)
      .def_readonly("information", &GameType::information)
      .def_readonly("utility", &GameType::utility)
      .def_readonly("reward_model", &GameType::reward_model)
      .def_readonly("max_num_players", &GameType::max_num_players)
      .def_readonly("min_num_players", &GameType::min_num_players)
      .def_readonly("provides_information_state_string", &GameType::provides_information_state_string)
      .def_readonly("provides_information_state_tensor", &GameType::provides_information_state_tensor)
      .def_readonly("provides_observation_string", &GameType::provides_observation_string)
      .def_readonly("provides_observation_tensor", &GameType::provides_observation_tensor)
      .def_readonly("provides_factored_observation_string", &GameType::provides_factored_observation_string)
      .def_readonly("default_loadable", &GameType::default_loadable)
      .def_property_readonly("parameter_specification", [](const GameType& t) { return ParamsToPy(t.parameter_specification); })
      .def("__repr__", [](const GameType& t) { return "<GameType '" + t.short_name + "'>"; });

  py::enum_<PrivateInfoType>(m, "PrivateInfoType")
      .value("NONE", PrivateInfoType::kNone).value("SINGLE_PLAYER", PrivateInfoType::kSinglePlayer)
      .value("ALL_PLAYERS", PrivateInfoType::kAllPlayers);
  py::class_<IIGObservationType>(m, "IIGObservationType")
      .def(py::init([](bool public_info, bool perfect_recall, PrivateInfoType private_info) {
             return IIGObservationType{public_info, perfect_recall, private_info};
           }),
           py::arg("public_info") = true, py::arg("perfect_recall"), py::arg("private_info") = PrivateInfoType::kSinglePlayer)
      .def_readonly("public_info", &IIGObservationType::public_info)
      .def_readonly("perfect_recall", &IIGObservationType::perfect_recall)
      .def_readonly("private_info", &IIGObservationType::private_info);

  py::class_<Observer, std::shared_ptr<Observer>>(m, "Observer")
      .def("has_string", &Observer::HasString)
      .def("has_tensor", &Observer::HasTensor);
  // open_spiel::Observation (observer.h:350-407): named tensor pieces + string form, as python/observation.py consumes it
  py::class_<Observation>(m, "_Observation")
      .def(py::init([](std::shared_ptr<Game> game, std::shared_ptr<Observer> observer) { return new Observation(*game, observer); }))
      .def("has_string", &Observation::HasString)
      .def("has_tensor", &Observation::HasTensor)
      .def("set_from", &Observation::SetFrom)
      .def("string_from", [](const Observation& o, const State& s, int player) -> py::object {
        if (!o.HasString()) return py::none();
        return py::str(o.StringFrom(s, player));
      })
      .def("tensors_info", [](const Observation& o) {
        std::vector<std::pair<std::string, std::vector<int>>> out;
        for (const SpanTensorInfo& t : o.tensors_info()) out.push_back({t.name(), t.vector_shape<int>()});
        return out;
      })
      .def("tensor", [](Observation& o) {
        absl::Span<float> t = o.Tensor();
        return py::array_t<float>((py::ssize_t)t.size(), t.data());
      });

  py::class_<State> state(m, "State");
  state.def("current_player", &State::CurrentPlayer)
      .def("apply_action", &State::ApplyAction)
      .def("apply_action_with_legality_check", py::overload_cast<Action>(&State::ApplyActionWithLegalityCheck))
      .def("apply_actions", &State::ApplyActions)
      .def("undo_action", &State::UndoAction)
      .def("legal_actions", (std::vector<Action>(State::*)(Player) const) & State::LegalActions)
      .def("legal_actions", (std::vector<Action>(State::*)() const) & State::LegalActions)
      .def("legal_actions_mask", (std::vector<int>(State::*)(Player) const) & State::LegalActionsMask)
      .def("legal_actions_mask", (std::vector<int>(State::*)() const) & State::LegalActionsMask)
      .def("action_to_string", (std::string(State::*)(Player, Action) const) & State::ActionToString)
      .def("action_to_string", (std::string(State::*)(Action) const) & State::ActionToString)
      .def("string_to_action", (Action(State::*)(Player, const std::string&) const) & State::StringToAction)
      .def("string_to_action", (Action(State::*)(const std::string&) const) & State::StringToAction)
      .def("__str__", &State::ToString)
      .def("__repr__", &State::ToString)
      .def("to_string", &State::ToString)
      .def("is_terminal", &State::IsTerminal)
      .def("is_initial_state", &State::IsInitialState)
      .def("move_number", &State::MoveNumber)
      .def("rewards", &State::Rewards)
      .def("returns", &State::Returns)
      .def("player_reward", &State::PlayerReward)
      .def("player_return", &State::PlayerReturn)
      .def("is_chance_node", &State::IsChanceNode)
      .def("is_mean_field_node", &State::IsMeanFieldNode)
      .def("is_simultaneous_node", &State::IsSimultaneousNode)
      .def("is_player_node", &State::IsPlayerNode)
      .def("history", &State::History)
      .def("history_str", &State::HistoryString)
      .def("full_history", [](const State& s) {
        std::vector<std::pair<Player, Action>> out;
        for (const auto& pa : s.FullHistory()) out.push_back({pa.player, pa.action});
        return out;
      })
      .def("information_state_string", (std::string(State::*)(Player) const) & State::InformationStateString)
      .def("information_state_string", (std::string(State::*)() const) & State::InformationStateString)
      .def("information_state_tensor", (std::vector<float>(State::*)(Player) const) & State::InformationStateTensor)
      .def("information_state_tensor", (std::vector<float>(State::*)() const) & State::InformationStateTensor)
      .def("observation_string", (std::string(State::*)(Player) const) & State::ObservationString)
      .def("observation_string", (std::string(State::*)() const) & State::ObservationString)
      .def("observation_tensor", (std::vector<float>(State::*)(Player) const) & State::ObservationTensor)
      .def("observation_tensor", (std::vector<float>(State::*)() const) & State::ObservationTensor)
      .def("clone", &State::Clone)
      .def("child", &State::Child)
      .def("num_distinct_actions", &State::NumDistinctActions)
      .def("num_players", &State::NumPlayers)
      .def("chance_outcomes", &State::ChanceOutcomes)
      .def("get_game", [](const State& s) { return Mutable(s.GetGame()); })
      .def("get_type", &State::GetType)
      .def("serialize", &State::Serialize)
      .def("distribution_support", &State::DistributionSupport)
      .def("update_distribution", &State::UpdateDistribution)
      // b2s bridge: the packed lane (b2s_state_get / b2s_state_set layout) and transfers to / from a device batch whose
      // handle is given as an integer (open_spiel_b200.spiel.BatchedState._h.value)
      .def("packed_state", [](const State& s) {
        const auto* b = dynamic_cast<const b200::B200State*>(&s);
        if (!b) throw SpielException("not a B200 state");
        return py::bytes((const char*)b->blob(), b->blob_bytes());
      })
      .def("to_batch_lane", [](const State& s, uintptr_t batch, int64_t lane) {
        const auto* b = dynamic_cast<const b200::B200State*>(&s);
        if (!b) throw SpielException("not a B200 state");
        b->ToBatchLane((void*)batch, lane);
      })
      .def(py::pickle([](const State& s) { return SerializeGameAndState(*s.GetGame(), s); },
                      [](const std::string& data) { return DeserializeGameAndState(data).second; }));

  py::class_<Game, std::shared_ptr<Game>>(m, "Game")
      .def("num_distinct_actions", &Game::NumDistinctActions)
      .def("policy_tensor_shape", &Game::PolicyTensorShape)
      .def("new_initial_state", [](const Game& g) { return g.NewInitialState(); })
      .def("new_initial_state", [](const Game& g, const std::string& s) { return g.NewInitialState(s); })
      .def("new_initial_states", &Game::NewInitialStates)
      .def("max_chance_outcomes", &Game::MaxChanceOutcomes)
      .def("get_parameters", [](const Game& g) { return ParamsToPy(g.GetParameters()); })
      .def("num_players", &Game::NumPlayers)
      .def("min_utility", &Game::MinUtility)
      .def("max_utility", &Game::MaxUtility)
      .def("get_type", &Game::GetType)
      .def("utility_sum", &Game::UtilitySum)
      .def("information_state_tensor_shape", &Game::InformationStateTensorShape)
      .def("information_state_tensor_layout", [](const Game& g) { return g.InformationStateTensorLayout() == TensorLayout::kCHW ? "TensorLayout.CHW" : "TensorLayout.HWC"; })
      .def("information_state_tensor_size", &Game::InformationStateTensorSize)
      .def("observation_tensor_shape", &Game::ObservationTensorShape)
      .def("observation_tensor_layout", [](const Game& g) { return g.ObservationTensorLayout() == TensorLayout::kCHW ? "TensorLayout.CHW" : "TensorLayout.HWC"; })
      .def("observation_tensor_size", &Game::ObservationTensorSize)
      .def("policy_tensor_shape", &Game::PolicyTensorShape)
      .def("deserialize_state", &Game::DeserializeState)
      .def("max_game_length", &Game::MaxGameLength)
      .def("max_chance_nodes_in_history", &Game::MaxChanceNodesInHistory)
      .def("action_to_string", &Game::ActionToString)
      .def("make_observer", [](std::shared_ptr<Game> g, py::object iig, const py::dict& params) {
             absl::optional<IIGObservationType> t;
             if (!iig.is_none()) t = iig.cast<IIGObservationType>();
             return g->MakeObserver(t, ParamsFromPy(params));
           }, py::arg("imperfect_information_observation_type") = py::none(), py::arg("params") = py::dict())
      .def("is_b200", [](const Game& g) { return dynamic_cast<const b200::B200Game*>(&g) != nullptr; })
      .def("__str__", &Game::ToString)
      .def("__repr__", &Game::ToString)
      .def("__eq__", [](const Game& a, const Game& b) { return a.ToString() == b.ToString(); })
      .def(py::pickle([](std::shared_ptr<Game> g) { return g->ToString(); },
                      [](const std::string& data) { return Mutable(LoadGame(data)); }));

  m.def("load_game", [](const std::string& s) { return Mutable(LoadGame(s)); });
  m.def("load_game", [](const std::string& name, const py::dict& params) { return Mutable(LoadGame(name, ParamsFromPy(params))); });
  m.def("registered_names", &RegisteredGames);
  m.def("registered_games", &RegisteredGameTypes);
  m.def("serialize_game_and_state", &SerializeGameAndState);
  m.def("deserialize_game_and_state", [](const std::string& data) {
    auto gs = DeserializeGameAndState(data);
    return std::make_pair(Mutable(gs.first), std::move(gs.second));
  });
  m.def("game_parameters_from_string", [](const std::string& s) { return ParamsToPy(GameParametersFromString(s)); });
  m.def("game_parameters_to_string", [](const py::dict& d) { return GameParametersToString(ParamsFromPy(d)); });

  // ---- policies --------------------------------------------------------------------------------------------------
  py::class_<Policy, std::shared_ptr<Policy>>(m, "Policy")
      .def("action_probabilities", [](const Policy& p, const State& s) { return PolicyDict(p.GetStatePolicy(s)); })
      .def("action_probabilities", [](const Policy& p, const std::string& key) { return PolicyDict(p.GetStatePolicy(key)); })
      .def("get_state_policy", [](const Policy& p, const State& s) { return p.GetStatePolicy(s); })
      .def("get_state_policy", [](const Policy& p, const std::string& key) { return p.GetStatePolicy(key); })
      .def("get_state_policy_as_parallel_vectors", [](const Policy& p, const State& s) { return p.GetStatePolicyAsParallelVectors(s); });
  py::class_<TabularPolicy, std::shared_ptr<TabularPolicy>, Policy>(m, "TabularPolicy")
      .def(py::init<const std::unordered_map<std::string, ActionsAndProbs>&>())
      .def("policy_table", [](const TabularPolicy& p) { return p.PolicyTable(); })
      .def("__str__", &TabularPolicy::ToString);
  m.def("exploitability", [](std::shared_ptr<Game> g, const Policy& p) { return algorithms::Exploitability(*g, p); });
  m.def("nash_conv", [](std::shared_ptr<Game> g, const Policy& p) { return algorithms::NashConv(*g, p); });
  m.def("get_uniform_policy", [](std::shared_ptr<Game> g) { return std::make_shared<TabularPolicy>(GetUniformPolicy(*g)); });

  // ---- CFR on the device (policy.cc:224-245 names) -----------------------------------------------------------------
  py::class_<b200::B200CFRSolver>(m, "CFRSolver")
      .def(py::init([](std::shared_ptr<Game> g) { return new b200::B200CFRSolver(*g, false); }))
      .def("evaluate_and_update_policy", [](b200::B200CFRSolver& s) { s.EvaluateAndUpdatePolicy(1); })
      .def("iterate", [](b200::B200CFRSolver& s, int n) { s.EvaluateAndUpdatePolicy(n); }, py::arg("iterations"))
      .def("current_policy", [](const b200::B200CFRSolver& s) { return std::make_shared<TabularPolicy>(s.CurrentPolicy()); })
      .def("average_policy", [](const b200::B200CFRSolver& s) { return std::make_shared<TabularPolicy>(s.AveragePolicy()); })
      .def("tabular_average_policy", [](const b200::B200CFRSolver& s) { return std::make_shared<TabularPolicy>(s.AveragePolicy()); })
      .def("nash_conv", &b200::B200CFRSolver::NashConv)
      .def("num_info_states", &b200::B200CFRSolver::NumInfoStates)
      .def(py::pickle(
          [](const b200::B200CFRSolver& s) {
            b200::B200CFRSolver::Tables t = s.Export();
            return py::make_tuple(s.game().ToString(), s.cfr_plus(), t.iteration, t.regrets, t.cumulative_policy, t.current_policy);
          },
          [](py::tuple st) {
            auto solver = std::make_unique<b200::B200CFRSolver>(*LoadGame(st[0].cast<std::string>()), st[1].cast<bool>());
            b200::B200CFRSolver::Tables t;
            t.iteration = st[2].cast<int>();
            t.regrets = st[3].cast<std::vector<double>>();
            t.cumulative_policy = st[4].cast<std::vector<double>>();
            t.current_policy = st[5].cast<std::vector<double>>();
            solver->Import(t);
            return solver;
          }));
  m.def("CFRPlusSolver", [](std::shared_ptr<Game> g) { return new b200::B200CFRSolver(*g, true); });
  py::class_<b200::B200CFRBRSolver, b200::B200CFRSolver>(m, "CFRBRSolver")   // policy.cc:264-280
      .def(py::init([](std::shared_ptr<Game> g) { return new b200::B200CFRBRSolver(*g); }))
      .def(py::pickle(
          [](const b200::B200CFRBRSolver& s) {
            b200::B200CFRSolver::Tables t = s.Export();
            return py::make_tuple(s.game().ToString(), t.iteration, t.regrets, t.cumulative_policy, t.current_policy);
          },
          [](py::tuple st) {
            auto solver = std::make_unique<b200::B200CFRBRSolver>(*LoadGame(st[0].cast<std::string>()));
            b200::B200CFRSolver::Tables t;
            t.iteration = st[1].cast<int>();
            t.regrets = st[2].cast<std::vector<double>>();
            t.cumulative_policy = st[3].cast<std::vector<double>>();
            t.current_policy = st[4].cast<std::vector<double>>();
            solver->Import(t);
            return solver;
          }));

  // ---- MCCFR (python/pybind11/policy.cc:282-335 names; extra keyword: traversals / trajectories per update) ------------
  py::enum_<algorithms::AverageType>(m, "MCCFRAverageType")
      .value("SIMPLE", algorithms::AverageType::kSimple).value("FULL", algorithms::AverageType::kFull);
  py::class_<b200::B200MCCFRSolver>(m, "_B200MCCFRSolver")
      .def("run_iteration", [](b200::B200MCCFRSolver& s) { s.RunIteration(); })
      .def("run_iterations", &b200::B200MCCFRSolver::RunIterations, py::arg("iterations"))
      .def("average_policy", [](const b200::B200MCCFRSolver& s) { return std::make_shared<TabularPolicy>(s.AveragePolicy()); })
      .def("nash_conv", [](const b200::B200MCCFRSolver& s) { return s.NashConv(); })
      .def("num_info_states", [](const b200::B200MCCFRSolver& s) { return s.NumInfoStates(); });
  m.def("ExternalSamplingMCCFRSolver", [](std::shared_ptr<Game> g, int seed, algorithms::AverageType avg, int traversals_per_update) {
          return new b200::B200MCCFRSolver(*g, b200::B200MCCFRSolver::Kind::kExternalSampling, (uint64_t)(int64_t)seed,
                                           avg == algorithms::AverageType::kFull, 0.6, traversals_per_update);
        }, py::arg("game"), py::arg("seed") = 0, py::arg("avg_type") = algorithms::AverageType::kSimple, py::arg("traversals_per_update") = 1);
  m.def("OutcomeSamplingMCCFRSolver", [](std::shared_ptr<Game> g, double epsilon, int seed, int trajectories_per_update) {
          return new b200::B200MCCFRSolver(*g, b200::B200MCCFRSolver::Kind::kOutcomeSampling, (uint64_t)(int64_t)seed, false, epsilon,
                                           trajectories_per_update);
        }, py::arg("game"), py::arg("epsilon") = algorithms::OutcomeSamplingMCCFRSolver::kDefaultEpsilon, py::arg("seed") = -1,
        py::arg("trajectories_per_update") = 1);

  // ---- MCTS (bots.cc:106-149 names) --------------------------------------------------------------------------------
  py::enum_<algorithms::ChildSelectionPolicy>(m, "ChildSelectionPolicy")
      .value("UCT", algorithms::ChildSelectionPolicy::UCT).value("PUCT", algorithms::ChildSelectionPolicy::PUCT);
  py::class_<algorithms::Evaluator, std::shared_ptr<algorithms::Evaluator>>(m, "Evaluator")
      .def("evaluate", &algorithms::Evaluator::Evaluate)
      .def("prior", &algorithms::Evaluator::Prior);
  py::class_<DeviceRolloutEvaluator, std::shared_ptr<DeviceRolloutEvaluator>, algorithms::Evaluator>(m, "RandomRolloutEvaluator")
      .def(py::init<int, int>(), py::arg("n_rollouts"), py::arg("seed"))
      .def_readonly("n_rollouts", &DeviceRolloutEvaluator::n_rollouts)
      .def_readonly("seed", &DeviceRolloutEvaluator::seed);
  py::class_<algorithms::SearchNode>(m, "SearchNode")
      .def_readonly("action", &algorithms::SearchNode::action)
      .def_readonly("prior", &algorithms::SearchNode::prior)
      .def_readonly("player", &algorithms::SearchNode::player)
      .def_readonly("explore_count", &algorithms::SearchNode::explore_count)
      .def_readonly("total_reward", &algorithms::SearchNode::total_reward)
      .def_readonly("outcome", &algorithms::SearchNode::outcome)
      .def_readonly("children", &algorithms::SearchNode::children)
      .def("best_child", &algorithms::SearchNode::BestChild)
      .def("to_string", &algorithms::SearchNode::ToString)
      .def("children_str", &algorithms::SearchNode::ChildrenStr);
  py::class_<PyMCTSBot>(m, "MCTSBot")
      .def(py::init([](std::shared_ptr<Game> game, std::shared_ptr<algorithms::Evaluator> evaluator, double uct_c, int max_simulations,
                       int64_t max_memory_mb, bool solve, int seed, bool verbose, algorithms::ChildSelectionPolicy policy,
                       double dirichlet_alpha, double dirichlet_epsilon, bool dont_return_chance_node, double max_wall_clock_time) {
             return new PyMCTSBot(game, evaluator, uct_c, max_simulations, max_memory_mb, solve, seed, verbose, policy, dirichlet_alpha,
                                  dirichlet_epsilon, dont_return_chance_node, max_wall_clock_time);
           }),
           py::arg("game"), py::arg("evaluator"), py::arg("uct_c"), py::arg("max_simulations"), py::arg("max_memory_mb"),
           py::arg("solve"), py::arg("seed"), py::arg("verbose"),
           py::arg("child_selection_policy") = algorithms::ChildSelectionPolicy::UCT, py::arg("dirichlet_alpha") = 0.0,
           py::arg("dirichlet_epsilon") = 0.0, py::arg("dont_return_chance_node") = false, py::arg("max_wall_clock_time") = 0.0)
      .def("step", &PyMCTSBot::Step, py::call_guard<py::gil_scoped_release>())
      .def("mcts_search", &PyMCTSBot::MCTSearch, py::call_guard<py::gil_scoped_release>())
      .def("on_device", &PyMCTSBot::on_device);

  m.attr("B200") = py::bool_(true);
}
