// Kernel instantiations for go: the 128-bit core (board_size 2..9) and the 384-bit core (10..19, handicap stones).
#include "batch_kernels.cuh"
#include "rules_go.cuh"
namespace b2s {
GameOps* make_ops_go() { return new GameOpsT<GoRules>(); }
GameOps* make_ops_go_wide() { return new GameOpsT<GoWideRules>(); }
}  // namespace b2s
