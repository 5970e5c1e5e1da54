// Kernel instantiations for connect_four: the default board (6x7, four in a row, sizes known at compile time) and every
// other board.
#include "batch_kernels.cuh"
#include "rules_connect_four.cuh"
namespace b2s {
GameOps* make_ops_connect_four() { return new GameOpsT<ConnectFourRules>(); }
GameOps* make_ops_connect_four_std() { return new GameOpsT<ConnectFourStdRules>(); }
}  // namespace b2s
