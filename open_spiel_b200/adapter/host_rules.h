// Scalar (one State) execution of the b2s rule cores on the host, for the open_spiel::State adapter.
//
// SURVEY §8(b)(i): "scalar State methods run the same __host__ __device__ rule core on the CPU and keep history_ via
// the base class".  host_rules.cc compiles open_spiel_b200/csrc/rules_*.cuh — the exact source the sm_90a kernels are
// instantiated from — with the host compiler, so a single open_spiel::State never pays a kernel launch + PCIe round
// trip per method call.  This is NOT a CPU fallback of the batched path: there is no batched entry point here, and
// every batched call (b2s_apply_actions, b2s_step_fused, b2s_mcts_search, b2s_cfr_iterate, ...) exists only in
// libb2s.so and fails without a CUDA device.  A scalar state and a device lane share one packed format: the blob below
// is byte-for-byte what b2s_state_get / b2s_state_set move (state chunks in plane order, then go's hash-history column),
// so states cross between the two worlds without conversion (B200State::ToBatchLane / FromBatchLane).
//
// This header has no CUDA and no OpenSpiel dependency.
#ifndef OPEN_SPIEL_B200_ADAPTER_HOST_RULES_H_
#define OPEN_SPIEL_B200_ADAPTER_HOST_RULES_H_

#include <stddef.h>
#include <stdint.h>

#include <memory>
#include <string>
#include <vector>

extern "C" {
#include "b2s.h"
}

namespace b2s_host {

// Game-independent decode of a packed state, enough to print the reference's strings.
struct Decoded {
  // board games: one code per cell in the game's natural order
  //   tic_tac_toe   [r*3+c]                0 empty, 1 player 0 ("x"), 2 player 1 ("o")
  //   connect_four  [r*cols+c], r = 0 bottom, same codes
  //   breakthrough  [r*cols+c]             0 empty, 1 black (player 0), 2 white
  //   hex           [cell]                 0 empty, 1 black, 2 black-north, 3 black-south, 4 black-win,
  //                                        5 white, 6 white-west, 7 white-east, 8 white-win   (hex.h:68-78)
  //   go            [row*n+col], row 0 = "1"  0 empty, 1 black, 2 white
  //   mnk, othello  [r*cols+c]             0 empty, 1 player 0 ("x"), 2 player 1 ("o")
  //   y             [x + y*board_size]     0 empty (or off the triangle), 1 player 0 ("O"), 2 player 1 ("@")
  //   havannah      [x + y*diameter]       0 empty (or off the hexagon), 1 player 0 ("O"), 2 player 1 ("@")
  std::vector<int8_t> cells;
  int to_play = 0;          // go: colour to move even at terminal states; others: mover
  int last_move = -1;       // y, havannah: the cell of the last stone (-1: none), which ToString brackets
  // leduc_poker (kInvalidCard = -10000 in the reference, reported here as -1)
  int num_players = 2;
  int round = 0, cur_player = 0, public_card = -1, private_card[5] = {-1, -1, -1, -1, -1};
  int ante[4] = {0, 0, 0, 0}, folded[4] = {0, 0, 0, 0};
  std::vector<int> round1, round2;     // 0 fold, 1 call, 2 raise
  // kuhn_poker: num_players, private_card[p] (-1 = not dealt yet) and round1 = the betting actions (0 pass, 1 bet) in order
};

class Rules {
 public:
  // nullptr + *error when the parameters do not fit the packed layouts (the caller falls back to the stock game).
  static std::unique_ptr<Rules> Create(int game_id, const b2s_params& params, std::string* error);
  virtual ~Rules() = default;
  const b2s_game_info& info() const { return info_; }
  size_t state_bytes() const { return (size_t)info_.state_bytes; }
  size_t blob_bytes() const { return (size_t)info_.state_bytes + (size_t)info_.history_bytes; }

  // blob = blob_bytes() bytes, 16-byte aligned
  virtual void Init(void* blob) const = 0;                        // Game::NewInitialState
  virtual bool Apply(void* blob, int action) const = 0;           // false: illegal / terminal (blob untouched)
  virtual int CurrentPlayer(const void* blob) const = 0;          // >= 0, -1 chance, -4 terminal
  virtual void Returns(const void* blob, float* out) const = 0;   // [num_players]
  virtual void LegalMask(const void* blob, uint32_t* words) const = 0;   // [mask_words]; chance outcomes at chance nodes
  // which = 0 ObservationTensor, 1 InformationStateTensor; false when the game has no such tensor
  virtual bool Tensor(const void* blob, int player, int which, float* out) const = 0;
  virtual void Decode(const void* blob, Decoded* out) const = 0;

 protected:
  b2s_game_info info_;
};

}  // namespace b2s_host
#endif
