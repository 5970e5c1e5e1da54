// TEST INFRASTRUCTURE ONLY — never part of the product (libb2s.so has no CPU path and fails without a GPU).
//
// emul_eval.cc (the host build of the k_mcts_eval_step / k_mcts_eval_report kernel bodies) with go on boards 10..19 added:
// emv_create builds the 384-bit core GoWideRules for go with board_size unset (19) or above 9, as api.cu's make_ops does,
// and leaves every other game to emul_eval.cc's own emv_create.  Loaded in place of libemul_eval.so by tests/go_wide_emul.py.
#define emv_create emv_create_up_to_9x9
#include "emul_eval.cc"
#undef emv_create

extern "C" void* emv_create(int game_id, const b2s_params* p, long long cap) {
  if (game_id == B2S_GO && (p->board_size < 0 || p->board_size > 9)) return make<GoWideRules>(*p, cap);
  return emv_create_up_to_9x9(game_id, p, cap);
}
