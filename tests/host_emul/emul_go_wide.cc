// TEST INFRASTRUCTURE ONLY — never part of the product (libb2s.so has no CPU path and fails without a GPU).
//
// emul.cc (the host build of the rule cores and of the k_mcts kernel body) with go on boards 10..19 added: emu_create
// builds the 384-bit core GoWideRules for go with board_size unset (19) or above 9, as api.cu's make_ops does, and leaves
// every other game to emul.cc's own emu_create.  The CPU tests of go 10..19 (tests/test_go_large_*.py) load this library in
// place of libemul.so through tests/go_wide_emul.py.
#define emu_create emu_create_up_to_9x9
#include "emul.cc"
#undef emu_create

extern "C" void* emu_create(int game_id, const b2s_params* p, long long cap) {
  if (game_id == B2S_GO && (p->board_size < 0 || p->board_size > 9)) return make<GoWideRules>(*p, cap);
  return emu_create_up_to_9x9(game_id, p, cap);
}
