// GPU test of the AlphaBetaSearch drop-in (b200::AlphaBetaSearch) against the reference's stock algorithms::AlphaBetaSearch,
// compiled unmodified from algorithms/minimax.cc: the three cases of minimax_test.cc, seeded random positions of every served
// game (every maximizing player; on the stock side use_undo true and false where the game implements UndoAction), and the
// routing of a call with a value function to the stock search.
#include <iostream>
#include <random>

#include "b200_algorithms.h"
#include "open_spiel/algorithms/minimax.h"
#include "open_spiel/spiel.h"

using namespace open_spiel;

int main() {
  std::shared_ptr<const Game> ttt = LoadGame("tic_tac_toe");
  const long long launches0 = b2s_launch_count();
  SPIEL_CHECK_EQ(b200::AlphaBetaSearch(*ttt, nullptr, {}, -1, kInvalidPlayer).first, 0.0);
  SPIEL_CHECK_EQ(b2s_launch_count(), launches0 + 3);   // solved on the device: batch reset, root copy, search
  std::unique_ptr<State> s = ttt->NewInitialState();
  s->ApplyAction(4);
  s->ApplyAction(1);
  SPIEL_CHECK_EQ(b200::AlphaBetaSearch(*ttt, s.get(), {}, -1, kInvalidPlayer).first, 1.0);
  s = ttt->NewInitialState();
  for (Action a : {5, 4, 3, 8}) s->ApplyAction(a);
  SPIEL_CHECK_EQ(b200::AlphaBetaSearch(*ttt, s.get(), {}, -1, kInvalidPlayer).first, -1.0);

  // (game, root plies lo..hi, roots): the sizes of tests/alpha_beta_lib.py's VARIANTS, whose searches stay small
  // undo: the reference's state implements UndoAction (connect_four, hex, othello, y and havannah do not)
  struct Variant { const char* game; int lo, hi, count; bool undo; };
  const Variant variants[] = {
      {"tic_tac_toe", 0, 9, 12, true}, {"connect_four", 28, 34, 8, false}, {"connect_four(rows=4,columns=4,x_in_row=3)", 4, 16, 8, false},
      {"breakthrough(rows=4,columns=4)", 6, 14, 8, true}, {"hex(board_size=3)", 0, 9, 8, false}, {"hex(board_size=4)", 6, 16, 6, false},
      {"othello", 48, 60, 4, false}, {"mnk(m=4,n=4,k=3)", 4, 16, 8, true}, {"y(board_size=4)", 3, 10, 8, false},
      {"havannah(board_size=3)", 10, 19, 8, false}, {"go(board_size=2)", 0, 6, 8, true}, {"go(board_size=3)", 4, 18, 6, true},
      {"go(board_size=5)", 36, 46, 4, true}};
  std::mt19937 rng(7);
  int compared = 0;
  for (const Variant& v : variants) {
    std::shared_ptr<const Game> g = LoadGame(v.game);
    for (int k = 0; k < v.count; ++k) {
      std::unique_ptr<State> root = g->NewInitialState();
      const int plies = v.lo + (int)(rng() % (unsigned)(v.hi - v.lo + 1));
      for (int t = 0; t < plies && !root->IsTerminal(); ++t) {
        std::vector<Action> legal = root->LegalActions();
        root->ApplyAction(legal[rng() % legal.size()]);
      }
      for (Player maxp : {kInvalidPlayer, Player{0}, Player{1}}) {
        if (root->IsTerminal() && maxp == kInvalidPlayer) continue;   // the reference indexes the returns with player -4
        const long long launches = b2s_launch_count();
        auto want = algorithms::AlphaBetaSearch(*g, root.get(), {}, -1, maxp, /*use_undo=*/v.undo && (k & 1) == 0);
        auto got = b200::AlphaBetaSearch(*g, root.get(), {}, -1, maxp);
        SPIEL_CHECK_EQ(b2s_launch_count(), launches + 3);   // solved on the device: batch reset, root copy, search
        if (got != want) {
          std::cerr << v.game << " " << root->HistoryString() << " player " << maxp << ": device (" << got.first << ", " << got.second
                    << "), stock (" << want.first << ", " << want.second << ")" << std::endl;
          return 1;
        }
        ++compared;
      }
    }
  }

  // a value function routes to the stock search: same result, the function called as often, no device launch
  std::shared_ptr<const Game> c4 = LoadGame("connect_four");
  int calls = 0;
  auto value_function = [&calls](const State& st) { ++calls; return (double)((int)st.History().size() % 3) - 1.0; };
  auto want = algorithms::AlphaBetaSearch(*c4, nullptr, value_function, 2, kInvalidPlayer, /*use_undo=*/false);
  const int want_calls = calls;
  calls = 0;
  const long long launches = b2s_launch_count();
  auto got = b200::AlphaBetaSearch(*c4, nullptr, value_function, 2, kInvalidPlayer, /*use_undo=*/false);
  SPIEL_CHECK_TRUE(got == want);
  SPIEL_CHECK_EQ(calls, want_calls);
  SPIEL_CHECK_GT(calls, 0);
  SPIEL_CHECK_EQ(b2s_launch_count(), launches);
  std::cout << "alpha_beta_test ok: " << compared << " positions equal to the stock search" << std::endl;
  return 0;
}
