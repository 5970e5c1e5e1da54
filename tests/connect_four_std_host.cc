// Host build of connect_four's two rule-core instantiations (rules_connect_four.cuh), driven by
// tests/test_connect_four_std_host.py: on the default board (6x7, four in a row) ConnectFourCore<true>, whose sizes are
// compile-time constants, must compute exactly what ConnectFourCore<false> computes from the configuration — every key,
// terminal flag, outcome, legal mask, observation (both perspectives) and accepted / rejected action along random games —
// and it must refuse to configure any other board.  Exit code 0 and an "ok" line when every check passes.
#include "open_spiel_b200/csrc/host_compat.h"
#include "open_spiel_b200/csrc/common.cuh"
#include "open_spiel_b200/csrc/rules_connect_four.cuh"

#include <cstdio>
#include <random>

using namespace b2s;
typedef ConnectFourRules G;      // sizes from the configuration
typedef ConnectFourStdRules D;   // sizes known at compile time

#define CHECK(c, ...) do { if (!(c)) { printf("FAIL %s:%d: ", __FILE__, __LINE__); printf(__VA_ARGS__); printf("\n"); return 1; } } while (0)

static b2s_params params(int rows, int cols, int k, int ego) {
  b2s_params p;
  memset(&p, 0xff, sizeof p);
  p.rows = rows; p.columns = cols; p.x_in_row = k; p.egocentric_obs_tensor = ego;
  return p;
}

int main() {
  b2s_game_info gi;
  {
    D::Cfg c;
    CHECK(D::make_cfg(params(-1, -1, -1, -1), c, gi) == nullptr, "default board refused");
    CHECK(D::make_cfg(params(6, 7, 4, -1), c, gi) == nullptr, "6x7 refused");
    CHECK(D::make_cfg(params(7, 7, -1, -1), c, gi) != nullptr && D::make_cfg(params(-1, 6, -1, -1), c, gi) != nullptr &&
          D::make_cfg(params(-1, -1, 3, -1), c, gi) != nullptr, "another board accepted");
  }
  std::mt19937_64 rng(3);
  long checks = 0;
  for (int ego = 0; ego <= 1; ++ego) {
    G::Cfg gc;
    D::Cfg dc;
    CHECK(G::make_cfg(params(-1, -1, -1, ego), gc, gi) == nullptr && D::make_cfg(params(-1, -1, -1, ego), dc, gi) == nullptr, "config");
    Ctx ctx = {};
    for (int game = 0; game < 3000; ++game) {
      G::S g;
      D::S d;
      G::init(g, gc, ctx, 0);
      D::init(d, dc, ctx, 0);
      for (int ply = 0;; ++ply) {
        const u64 key = G::pack(g, gc);
        CHECK(D::pack(d, dc) == key && d.x == g.x && d.o == g.o, "game %d ply %d: state", game, ply);
        D::S u;
        D::unpack(u, key, dc);
        CHECK(u.x == g.x && u.o == g.o, "game %d ply %d: unpack", game, ply);
        CHECK(D::terminal(d, dc) == G::terminal(g, gc) && D::outcome(d, dc) == G::outcome(g, gc) &&
              D::cur_player(d, dc) == G::cur_player(g, gc), "game %d ply %d: status", game, ply);
        float rg[2], rd[2];
        G::returns(g, gc, rg);
        D::returns(d, dc, rd);
        CHECK(rg[0] == rd[0] && rg[1] == rd[1], "game %d ply %d: returns", game, ply);
        u32 mg, md;
        G::legal(g, gc, &mg);
        D::legal(d, dc, &md);
        CHECK(mg == md, "game %d ply %d: legal %x vs %x", game, ply, mg, md);
        for (int pl = 0; pl < 2; ++pl) {
          G::ObsPack og;
          D::ObsPack od;
          G::obs_pack(g, gc, pl, 0, og);
          D::obs_pack(d, dc, pl, 0, od);
          CHECK(memcmp(&og, &od, sizeof og) == 0, "game %d ply %d: observation of player %d", game, ply, pl);
        }
        ++checks;
        if (G::terminal(g, gc)) break;
        // every action, legal or not, is accepted / rejected alike and leaves the same state
        for (int a = -1; a <= 7; ++a) {
          G::S g2 = g;
          D::S d2 = d;
          const bool okg = G::apply(g2, a, gc, ctx, 0), okd = D::apply(d2, a, dc, ctx, 0);
          CHECK(okg == okd && g2.x == d2.x && g2.o == d2.o, "game %d ply %d: action %d", game, ply, a);
        }
        int k = (int)(rng() % (u64)__builtin_popcount(mg)), a = 0;
        while (!((mg >> a) & 1u) || k-- > 0) ++a;
        G::apply(g, a, gc, ctx, 0);
        D::apply(d, a, dc, ctx, 0);
      }
    }
  }
  printf("ok: %ld positions\n", checks);
  return 0;
}
