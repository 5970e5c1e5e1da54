"""CPU: connect_four's 8-byte batch key (rules_connect_four.cuh pack / unpack) on every board shape the device path accepts
((rows+1)*columns <= 64, columns <= 32), compiled for the host from the product header.  Along random games, unpack(pack(s))
gives s back, every position of a game has its own key, and the start position is the bottom row's marker bits."""
import os
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CUDA_INC = "/usr/local/cuda/include"

SRC = r"""
#include "open_spiel_b200/csrc/host_compat.h"
#include "open_spiel_b200/csrc/common.cuh"
#include "open_spiel_b200/csrc/rules_connect_four.cuh"
#include <cstdio>
#include <random>
#include <set>
using namespace b2s;
typedef ConnectFourRules R;
int main() {
  std::mt19937_64 rng(1);
  long checks = 0, shapes = 0;
  for (int rows = 1; rows <= 63; ++rows)
    for (int cols = 1; cols <= 32; ++cols) {
      if ((rows + 1) * cols > 64) continue;
      b2s_params p;
      memset(&p, 0xff, sizeof p);
      p.rows = rows; p.columns = cols; p.x_in_row = 4;
      R::Cfg c;
      b2s_game_info gi;
      if (R::make_cfg(p, c, gi)) { printf("rejected %dx%d\n", rows, cols); return 1; }
      ++shapes;
      Ctx ctx = {};
      for (int game = 0; game < 200; ++game) {
        R::S s;
        R::init(s, c, ctx, 0);
        if (R::pack(s, c) != c.bottom) { printf("start key %dx%d\n", rows, cols); return 1; }
        std::set<u64> keys;
        for (int ply = 0;; ++ply) {
          const u64 key = R::pack(s, c);
          R::S t;
          R::unpack(t, key, c);
          if (t.x != s.x || t.o != s.o || !keys.insert(key).second) {
            printf("%dx%d ply %d: x %llx o %llx key %llx -> x %llx o %llx\n", rows, cols, ply, s.x, s.o, key, t.x, t.o);
            return 1;
          }
          ++checks;
          if (R::terminal(s, c)) break;
          u32 m;
          R::legal_nonterminal(s, c, &m);
          int k = (int)(rng() % (u64)__builtin_popcount(m)), a = 0;
          while (!((m >> a) & 1u) || k-- > 0) ++a;
          if (!R::apply(s, a, c, ctx, 0)) { printf("%dx%d: legal drop %d rejected\n", rows, cols, a); return 1; }
        }
      }
    }
  printf("%ld positions on %ld shapes\n", checks, shapes);
  return shapes == 216 ? 0 : 1;
}
"""


@pytest.mark.skipif(shutil.which("g++") is None or not os.path.isdir(CUDA_INC), reason="needs g++ and the CUDA headers")
def test_key_round_trips_on_every_accepted_board_shape(tmp_path):
    src = tmp_path / "key.cc"
    src.write_text(SRC)
    exe = tmp_path / "key"
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-I", ROOT, "-I", CUDA_INC, "-o", str(exe), str(src)])
    r = subprocess.run([str(exe)], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
