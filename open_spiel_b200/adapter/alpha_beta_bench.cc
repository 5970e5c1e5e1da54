// CPU baseline of scripts/bench_alpha_beta.py: the reference's stock algorithms::AlphaBetaSearch on the roots given on stdin, first
// on one thread, then on every hardware thread (each takes the next root).  argv[1]: use_undo, 1 (the reference's default) or 0
// (Child per move: connect_four, hex, othello, y and havannah do not implement UndoAction).
// argv[2] (optional, the CPU baseline of scripts/bench_alpha_beta_eval.py): a depth limit >= 0, searched with the test value
// function "hash" of tests/alpha_beta_eval_lib.py: with I the non-zero indices of ObservationTensor(CurrentPlayer()),
// k = (sum_{i in I} (7i + 3) mod 11) mod 9 and v = (k - 4) / 7, the value of the maximizing player is v for player 0, -v for 1.
// stdin: the game string on the first line, then one root per line as its comma-separated action history.
// stdout: one JSON line {"roots", "one_core_seconds", "threads", "all_cores_seconds", "value_sum"}.
#include <atomic>
#include <chrono>
#include <iostream>
#include <sstream>
#include <string>
#include <thread>
#include <vector>

#include "open_spiel/algorithms/minimax.h"
#include "open_spiel/spiel.h"

using namespace open_spiel;

int main(int argc, char** argv) {
  const bool use_undo = argc < 2 || std::string(argv[1]) != "0";
  const int depth_limit = argc < 3 ? -1 : std::stoi(argv[2]);
  std::string line;
  std::getline(std::cin, line);
  std::shared_ptr<const Game> game = LoadGame(line);
  std::vector<std::unique_ptr<State>> roots;
  while (std::getline(std::cin, line)) {
    std::unique_ptr<State> s = game->NewInitialState();
    std::stringstream ss(line);
    std::string a;
    while (std::getline(ss, a, ','))
      if (!a.empty()) s->ApplyAction(std::stol(a));
    roots.push_back(std::move(s));
  }
  const int n = (int)roots.size();
  std::vector<double> value(n);
  auto run = [&](int threads) {
    std::atomic<int> next{0};
    auto work = [&] {
      for (int i; (i = next++) < n;) {
        if (depth_limit < 0) {
          value[i] = algorithms::AlphaBetaSearch(*game, roots[i].get(), {}, -1, kInvalidPlayer, use_undo).first;
          continue;
        }
        const Player maxp = roots[i]->CurrentPlayer();
        auto hash = [maxp](const State& s) {
          const std::vector<float> obs = s.ObservationTensor(s.CurrentPlayer());
          long long h1 = 0;
          for (size_t e = 0; e < obs.size(); ++e)
            if (obs[e] != 0) h1 += (7 * (long long)e + 3) % 11;
          const double v = (double)(h1 % 9 - 4) / 7.0;
          return maxp == 0 ? v : -v;
        };
        value[i] = algorithms::AlphaBetaSearch(*game, roots[i].get(), hash, depth_limit, kInvalidPlayer, use_undo).first;
      }
    };
    const auto t0 = std::chrono::steady_clock::now();
    std::vector<std::thread> pool;
    for (int t = 1; t < threads; ++t) pool.emplace_back(work);
    work();
    for (auto& t : pool) t.join();
    return std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
  };
  const double one = run(1);
  double sum = 0;
  for (double v : value) sum += v;
  const int threads = (int)std::thread::hardware_concurrency();
  const double all = run(threads);
  std::cout << "{\"roots\": " << n << ", \"use_undo\": " << (use_undo ? "true" : "false") << ", \"one_core_seconds\": " << one << ", \"threads\": " << threads
            << ", \"all_cores_seconds\": " << all << ", \"value_sum\": " << sum << "}" << std::endl;
  return 0;
}
